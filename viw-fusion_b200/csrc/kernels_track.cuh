// kernels_track.cuh -- the bookkeeping of FeatureTracker::trackImage() (featureTracker/feature_tracker.cpp:99-331) that sits between
// the calcOpticalFlowPyrLK / setMask / goodFeaturesToTrack calls, so that a camera tick of every stream runs on the device from the
// uploaded images to the featureFrame table without a host round trip (SURVEY 8 f-1):
//   reduceVector(prev_pts / cur_pts / ids / track_cnt, status) + track_cnt++                      :163-171
//   rebuild of cur_pts / ids / track_cnt in setMask's visiting order + the new corners (ids n_id++) :72-88, :199-204
//   undistortedPts + ptsVelocity through the id -> point maps of the previous tick                 :207-208, :606-657
//   the stereo half: ids_right = ids, reduceVector by the stereo status, right undistort / velocity  :254-268
//   prev_* = cur_* (:296-300) and the featureFrame rows (:307-350)
// hasPrediction (:122-137): forward flow seeded with predict_pts at maxLevel 1, repeated at maxLevel 3 when fewer than 10 succeed.
// Between two ticks, the estimator's way back into the session (estimator.cpp:841-843): removeOutliers (:739-755) and setPrediction (:715-736).
//
// One block per camera stream (these are 150-point lists); `tid` / `nt` = thread index / count, the emulation build runs nt = 1.
#pragma once
#include <stdint.h>
#include "vmath.cuh"
#include "kernels_feat.cuh"

namespace viwb {

typedef CamModel TrkCam;                 // m_camera[0] / m_camera[1]: PINHOLE, MEI or KANNALA_BRANDT (kernels_feat.cuh)

struct TrkArgs {                         // one camera stream; every array holds `maxn` entries
    // --- tracker buffers (viwb_lk_batch): prev_pts = points of the previous image, lk_cur = temporal LK result, stereo_in / right = stereo LK in / out
    float *prev_pts; const float *lk_cur; const uint8_t *lk_status; int *n_temporal;
    float *stereo_in; const float *right_pts; const uint8_t *st_right; int *n_stereo;
    // --- detector buffers (viwb_detector): setMask input, survivors in visiting order, new corners
    float *det_pts; int *det_cnt; int *det_n; const int *keep; const int *n_keep; const float *corners; const int *n_corners;
    // --- session state
    int *ids, *track_cnt, *tmp_ids;      // aligned with prev_pts; tmp_ids aligned with det_pts
    int *n_id;                           // next feature id of this stream (feature_tracker.h: n_id)
    int *mapL_ids; float *mapL_un; int *mapL_n;      // prev_un_pts_map
    int *mapR_ids; float *mapR_un; int *mapR_n;      // prev_un_right_pts_map
    // --- prediction
    uint8_t *has_pred; int *pred_n, *redo_n;
    // --- featureFrame rows: {x, y, u, v, vx, vy} (z = 1), left rows in cur_pts order, right rows in ids_right order
    int *out_n; int *out_ids, *out_cnt; float *out_feat;
    int *out_nr; int *out_ids_r; float *out_feat_r;
    int *flags;                          // bit 0: goodFeaturesToTrack candidate list overflowed in this tick
};
struct TrkRun { const TrkArgs *tasks; TrkCam cam[2]; double dt; int maxn; };

// warp-cooperative order-preserving position of an element with `flag` among the flagged ones of a group of nt consecutive indices
VIWB_D int trk_rank(bool flag, int tid, int &total) {
#ifdef VIWB_HOST_EMU
    (void)tid; total = flag ? 1 : 0; return 0;
#else
    const unsigned m = __ballot_sync(0xffffffffu, flag);
    total = __popc(m);
    return __popc(m & ((1u << tid) - 1u));
#endif
}

// PinholeCamera::liftProjective (camera_models/src/camera_models/PinholeCamera.cc:450-517), CataCamera::liftProjective (CataCamera.cc:556-626)
// or EquidistantCamera::liftProjective (EquidistantCamera.cc:428-442)
// narrowed to cv::Point2f (feature_tracker.cpp:614)
VIWB_D void trk_lift(const TrkCam &c, float u, float v, float &x, float &y) {
    UndistArgs a; a.n = 1; a.pts = nullptr; a.prev_un = nullptr; a.has_prev = nullptr; a.vel = nullptr;
    a.fx = c.fx; a.fy = c.fy; a.cx = c.cx; a.cy = c.cy; a.k1 = c.k1; a.k2 = c.k2; a.p1 = c.p1; a.p2 = c.p2; a.dt = 1.0; a.model = c.model; a.xi = c.xi;
    const float p[2] = {u, v}; float un[2];
    a.pts = p; a.un = un;
    undistort_item(a, 0);
    x = un[0]; y = un[1];
}

// ptsVelocity (:619-657): (cur - prev) / dt for ids found in the previous tick's map, float difference and double division, else 0
VIWB_D void trk_velocity(const int *map_ids, const float *map_un, int map_n, int id, float ux, float uy, double dt, float &vx, float &vy) {
    vx = 0.f; vy = 0.f;
    for (int k = 0; k < map_n; k++) if (map_ids[k] == id) {
        vx = (float)((double)(ux - map_un[2 * k]) / dt);
        vy = (float)((double)(uy - map_un[2 * k + 1]) / dt);
        return;
    }
}

// ---- stage 0 (only when a prediction was set): point counts of the seeded maxLevel-1 pass
VIWB_D void trk_pred_setup(const TrkArgs &a, int tid) {
    if (tid != 0) return;
    const int n = *a.n_temporal;
    const bool hp = a.has_pred && *a.has_pred;
    *a.pred_n = hp ? n : 0;
    *a.redo_n = hp ? 0 : n;
}
// succ_num < 10 -> the stream repeats the forward flow over the full pyramid (:130-137)
VIWB_D void trk_pred_check(const TrkArgs &a, int tid, int nt) {
    const int n = *a.pred_n;
    if (n == 0) return;                                       // stream without a prediction: redo_n already holds its count
    int succ = 0;
    for (int base = 0; base < n; base += nt) {
        const int i = base + tid; int tot;
        trk_rank(i < n && a.lk_status[i] != 0, tid, tot);
        succ += tot;
    }
    if (tid == 0) *a.redo_n = succ < 10 ? n : 0;
}

// ---- between two ticks: FeatureTracker::removeOutliers then FeatureTracker::setPrediction, one warp per stream.
// The id lists arrive sorted and free of duplicates (the host orders them as the reference's std::set / std::map do), stream f's slice is
// [off[f], off[f + 1]).
struct TrkFeedback { const int *rm_off, *rm_ids, *pr_off, *pr_ids; const double *pr_pts; const uint8_t *pr_flag; float *pred_pts; };

VIWB_D int trk_find_id(const int *ids, int n, int id) {          // position of id in the ascending list, -1 when absent
    int lo = 0, hi = n;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (ids[mid] < id) lo = mid + 1; else hi = mid; }
    return (lo < n && ids[lo] == id) ? lo : -1;
}
// PinholeCamera::spaceToPlane (PinholeCamera.cc:520-542, distortion :646-662) narrowed to cv::Point2f (feature_tracker.cpp:730).  Every
// product and sum is rounded on its own (no fused multiply-add), so that the pixel is the float the reference's build (-ffp-contract=off
// here, SSE2 there) hands to calcOpticalFlowPyrLK, bit for bit.  An MEI camera projects through CataCamera::spaceToPlane instead,
// a Kannala-Brandt one through EquidistantCamera::spaceToPlane (kb_space_to_plane).
VIWB_D void trk_space_to_plane(const TrkCam &c, const double *P, float &u, float &v) {
    if (c.model == CAM_MEI) { mei_space_to_plane(c, P, u, v); return; }
    if (c.model == CAM_KB) { kb_space_to_plane(c, P, u, v); return; }
    const double x = P[0] / P[2], y = P[1] / P[2];
    double xd = x, yd = y;
    if (!(c.k1 == 0.0 && c.k2 == 0.0 && c.p1 == 0.0 && c.p2 == 0.0)) {       // m_noDistortion
        const double mx2 = trk_mul(x, x), my2 = trk_mul(y, y), mxy = trk_mul(x, y), rho2 = trk_add(mx2, my2);
        const double rad = trk_add(trk_mul(c.k1, rho2), trk_mul(trk_mul(c.k2, rho2), rho2));
        const double dx = trk_add(trk_add(trk_mul(x, rad), trk_mul(trk_mul(2.0, c.p1), mxy)), trk_mul(c.p2, trk_add(rho2, trk_mul(2.0, mx2))));
        const double dy = trk_add(trk_add(trk_mul(y, rad), trk_mul(trk_mul(2.0, c.p2), mxy)), trk_mul(c.p1, trk_add(rho2, trk_mul(2.0, my2))));
        xd = trk_add(x, dx); yd = trk_add(y, dy);
    }
    u = (float)trk_add(trk_mul(c.fx, xd), c.cx); v = (float)trk_add(trk_mul(c.fy, yd), c.cy);
}
VIWB_D void trk_feedback(const TrkArgs &a, const TrkRun &r, const TrkFeedback &fb, int f, int tid, int nt) {
    const int n = *a.n_temporal;
    int m = n;
    if (fb.rm_off) {
        // reduceVector(prev_pts / ids / track_cnt, status) in place: a row moves to a lower or equal index, so every thread of a group reads
        // its row before any thread of the group writes
        const int *rm = fb.rm_ids + fb.rm_off[f]; const int nrm = fb.rm_off[f + 1] - fb.rm_off[f];
        m = 0;
        for (int base = 0; base < n; base += nt) {
            const int i = base + tid; int tot;
            float u = 0.f, v = 0.f; int id = 0, cnt = 0;
            if (i < n) { u = a.prev_pts[2 * i]; v = a.prev_pts[2 * i + 1]; id = a.ids[i]; cnt = a.track_cnt[i]; }
            const bool keep = i < n && trk_find_id(rm, nrm, id) < 0;
            const int j = m + trk_rank(keep, tid, tot);
            VIWB_SYNCWARP();
            if (keep) { a.prev_pts[2 * j] = u; a.prev_pts[2 * j + 1] = v; a.ids[j] = id; a.track_cnt[j] = cnt; }
            m += tot;
        }
        VIWB_SYNCWARP();
    }
    const bool hp = fb.pr_off && fb.pr_flag[f] != 0;
    if (hp) {
        const int *pid = fb.pr_ids + fb.pr_off[f]; const int np = fb.pr_off[f + 1] - fb.pr_off[f];
        float *out = fb.pred_pts + (size_t)f * r.maxn * 2;
        for (int j = tid; j < m; j += nt) {
            const int k = trk_find_id(pid, np, a.ids[j]);
            float u = a.prev_pts[2 * j], v = a.prev_pts[2 * j + 1];                // no prediction for this id: predict_pts[i] = prev_pts[i]
            if (k >= 0) trk_space_to_plane(r.cam[0], fb.pr_pts + 3 * ((size_t)fb.pr_off[f] + k), u, v);
            out[2 * j] = u; out[2 * j + 1] = v;
        }
    }
    if (tid == 0) { *a.n_temporal = m; *a.n_stereo = m; *a.has_pred = hp ? 1 : 0; }
}

// ---- stage 1, after the temporal flow: reduceVector by status and track_cnt++ straight into the detector's setMask input
VIWB_D void trk_advance(const TrkArgs &a, int tid, int nt) {
    const int n = *a.n_temporal;
    int m = 0;
    for (int base = 0; base < n; base += nt) {
        const int i = base + tid; int tot;
        const bool ok = i < n && a.lk_status[i] != 0;
        const int j = m + trk_rank(ok, tid, tot);
        if (ok) {
            a.det_pts[2 * j] = a.lk_cur[2 * i]; a.det_pts[2 * j + 1] = a.lk_cur[2 * i + 1];
            a.det_cnt[j] = a.track_cnt[i] + 1;
            a.tmp_ids[j] = a.ids[i];
        }
        m += tot;
    }
    if (tid == 0) { *a.det_n = m; *a.flags = 0; }
}

// ---- stage 2, after setMask + goodFeaturesToTrack: the tick's cur_pts / ids / track_cnt, undistortedPts, ptsVelocity, left featureFrame
// rows, the stereo flow's input and next tick's prev_pts.  Needs a block barrier between the map lookups and the map replacement.
VIWB_D void trk_merge(const TrkArgs &a, const TrkRun &r, int tid, int nt) {
    const int nk = *a.n_keep;
    int nc = *a.n_corners;
    if (nc < 0) { nc = 0; if (tid == 0) *a.flags |= 1; }
    int total = nk + nc;
    if (total > r.maxn) { total = r.maxn; nc = total - nk; }
    const int id0 = *a.n_id, map_n = *a.mapL_n;
    for (int j = tid; j < total; j += nt) {
        float u, v; int id, cnt;
        if (j < nk) { const int s = a.keep[j]; u = a.det_pts[2 * s]; v = a.det_pts[2 * s + 1]; id = a.tmp_ids[s]; cnt = a.det_cnt[s]; }
        else { u = a.corners[2 * (j - nk)]; v = a.corners[2 * (j - nk) + 1]; id = id0 + (j - nk); cnt = 1; }
        a.prev_pts[2 * j] = u; a.prev_pts[2 * j + 1] = v;
        a.stereo_in[2 * j] = u; a.stereo_in[2 * j + 1] = v;
        a.ids[j] = id; a.track_cnt[j] = cnt;
        float ux, uy, vx = 0.f, vy = 0.f;
        trk_lift(r.cam[0], u, v, ux, uy);
        if (j < nk) trk_velocity(a.mapL_ids, a.mapL_un, map_n, id, ux, uy, r.dt, vx, vy);     // a new corner's id is in no map
        a.out_ids[j] = id; a.out_cnt[j] = cnt;
        float *o = a.out_feat + 6 * j;
        o[0] = ux; o[1] = uy; o[2] = u; o[3] = v; o[4] = vx; o[5] = vy;
    }
    VIWB_SYNC();
    for (int j = tid; j < total; j += nt) { a.mapL_ids[j] = a.out_ids[j]; a.mapL_un[2 * j] = a.out_feat[6 * j]; a.mapL_un[2 * j + 1] = a.out_feat[6 * j + 1]; }
    if (tid == 0) { *a.n_id = id0 + nc; *a.mapL_n = total; *a.out_n = total; *a.n_temporal = total; *a.n_stereo = total; *a.out_nr = 0; }
}

// ---- stage 3, after the stereo flow: ids_right / cur_right_pts by status, right undistort + velocity, right featureFrame rows
VIWB_D void trk_stereo(const TrkArgs &a, const TrkRun &r, int tid, int nt) {
    const int n = *a.n_stereo, map_n = *a.mapR_n;
    int m = 0;
    for (int base = 0; base < n; base += nt) {
        const int i = base + tid; int tot;
        const bool ok = i < n && a.st_right[i] != 0;
        const int j = m + trk_rank(ok, tid, tot);
        if (ok) {
            const float u = a.right_pts[2 * i], v = a.right_pts[2 * i + 1];
            const int id = a.ids[i];
            float ux, uy, vx, vy;
            trk_lift(r.cam[1], u, v, ux, uy);
            trk_velocity(a.mapR_ids, a.mapR_un, map_n, id, ux, uy, r.dt, vx, vy);
            a.out_ids_r[j] = id;
            float *o = a.out_feat_r + 6 * j;
            o[0] = ux; o[1] = uy; o[2] = u; o[3] = v; o[4] = vx; o[5] = vy;
        }
        m += tot;
    }
    VIWB_SYNC();
    for (int j = tid; j < m; j += nt) { a.mapR_ids[j] = a.out_ids_r[j]; a.mapR_un[2 * j] = a.out_feat_r[6 * j]; a.mapR_un[2 * j + 1] = a.out_feat_r[6 * j + 1]; }
    if (tid == 0) { *a.mapR_n = m; *a.out_nr = m; }
}

#ifndef VIWB_HOST_EMU
// one warp per stream for the compactions (ballot ranks), one 128-thread block per stream for the merge
__global__ void trk_pred_setup_kernel(TrkRun r) { trk_pred_setup(r.tasks[blockIdx.x], threadIdx.x); }
__global__ void trk_pred_check_kernel(TrkRun r) { trk_pred_check(r.tasks[blockIdx.x], threadIdx.x, 32); }
__global__ void trk_advance_kernel(TrkRun r) { trk_advance(r.tasks[blockIdx.x], threadIdx.x, 32); }
__global__ void trk_merge_kernel(TrkRun r) { trk_merge(r.tasks[blockIdx.x], r, threadIdx.x, blockDim.x); }
__global__ void trk_stereo_kernel(TrkRun r) { trk_stereo(r.tasks[blockIdx.x], r, threadIdx.x, 32); }
__global__ void trk_feedback_kernel(TrkRun r, TrkFeedback fb) { trk_feedback(r.tasks[blockIdx.x], r, fb, blockIdx.x, threadIdx.x, 32); }
#endif

}  // namespace viwb
