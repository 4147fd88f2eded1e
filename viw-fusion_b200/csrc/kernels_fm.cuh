// kernels_fm.cuh -- FeatureManager (estimator/feature_manager.{h,cpp}) resident in HBM for `F` independent streams, one block per stream:
//   addFeatureCheckParallax + compensatedParallax2   feature_manager.cpp:52-119, 538-571
//   triangulate (the two live branches)              feature_manager.cpp:309-389 (triangulate_item of kernels_feat.cuh)
//   the visual-table loop of optimization()          estimator.cpp:1585-1638, getDepthVector feature_manager.cpp:179-195
//   setDepth / removeOutlier / removeFailures        feature_manager.cpp:142-171, 440-455
//   predictPtsInNextFrame                            estimator.cpp:2080-2113 (predict_pts_item)
//   removeBackShiftDepth / removeBack / removeFront  feature_manager.cpp:457-536 (shift_depth_item)
// A stream's list is a dense structure of arrays in list order (the std::list's order: insertion order, erasures stable), capacity M:
// id, start_frame, num_obs, solve_flag, estimated_depth, and per feature FM_SLOTS observation slots of 12 floats {x, y, p_u, p_v, v_x, v_y}
// of the left and then the right camera (z = 1 in every featureFrame the reference produces, and every value there comes from a float), the
// slot's cur_td and its is_stereo flag.  Erasing features is a stable compaction from one buffer into the other (the host flips them).
#pragma once
#include "kernels_feat.cuh"
#include "layout.cuh"

namespace viwb {

enum { FM_SLOTS = 11, FM_OBS = 12, FM_NT = 256, FM_MAX_ROWS = 1024 };
enum { FM_ERR_DUP = 1, FM_ERR_RIGHT = 2, FM_ERR_ROWS = 4, FM_ERR_CAP = 8, FM_ERR_OBS = 16, FM_ERR_TRACKER = 32 };
enum { FM_COMPACT_OUTLIERS = 0, FM_COMPACT_SLIDE = 1, FM_COMPACT_FAILURES = 2 };
// dec [F][FM_DEC_N]: the decision and statistics of the last applied add, then the statistics the pending add's check counted
enum { FM_DEC_FLAG = 0, FM_DEC_LAST_TRACK, FM_DEC_LONG_TRACK, FM_DEC_NEW, FM_DEC_PENDING, FM_DEC_N = 8 };

struct FmList { int *id, *start, *nobs, *flag; double *depth; float *obs; double *td; unsigned char *ster; };
// featureFrame rows of one tick: stream s holds n[s] left rows (ids, feat [6]) and nr[s] right rows at s * stride
struct FmRows { const int *n, *nr, *ids, *ids_r; const float *feat, *feat_r; int stride; const int *trk_flags; };
struct FmRun {
    int F, M, R, stereo, mode;
    double min_parallax, focal, init_depth;
    FmList src, dst;                        // dst: compactions only
    int *n, *err, *any_err, *dec;           // n [F]; err [F] / any_err [1]: error bits of the adds since the host last read them (sticky); dec [F][FM_DEC_N]
    double *avg;                            // [F] last_average_parallax
    long long *keys; int *rmatch, *rright, *newpos;      // [F][R] add scratch: sorted (id, row) keys, matched feature, right row, new position
    int *iscr; double *dscr;                // [F][M] scratch
    FmRows rows; const int *fc; const double *td;         // add: rows, frame_count [F], td [F]
    const double *state;                    // [F][207] triangulate / predict
    const int *off; const double *xin; const unsigned char *verdict;      // set_depth / outliers: landmark k of stream s at off[s] + k
    const int *verdict_i;                   // outliers from a batch: its int verdicts (lm_outlier) in place of `verdict`
    const int *st_off;                      // predict from a batch: stream s's fixed state at state + st_off[s] (NULL: s * 207)
    const unsigned char *shift; const double *mats;       // slide: [F] flags, [F][24] = marg_R 9, marg_P 3, new_R 9, new_P 3
    int *o_cnt, *o_ids; double *o_pts;      // [F], [F][M], [F][M][3]: removed ids / predictions
    const int *w_off;                       // window: [F][2] packed row / landmark offsets
    int *w_type, *w_lm, *w_fi, *w_fj, *w_id; double *w_obs, *w_inv;
    unsigned *w_dig;                        // window digest: one word per landmark at w_off[s] (fm_digest_word)
    const WinMeta *b_meta; const int *b_oi; double *b_obs_i, *b_obs_j, *b_x; const double *b_xfix;      // batch fill: window s of a batch slab
};

VIWB_HD int fm_imin(int a, int b) { return a < b ? a : b; }

// Stable block-wide compaction helper: items [0, n) are split into contiguous chunks, one per thread; weight(i) >= 0 is summed in item order
// and write(i, offset) is called for every item with its exclusive prefix.  sc: nt + 1 ints of shared memory.  Returns the total.
template <typename Wt, typename Wr>
VIWB_D int fm_scan(int n, int tid, int nt, int *sc, Wt weight, Wr write) {
    const int c = (n + nt - 1) / nt, lo = fm_imin(n, tid * c), hi = fm_imin(n, lo + c);
    int cnt = 0;
    for (int i = lo; i < hi; i++) cnt += weight(i);
    sc[tid] = cnt;
    VIWB_SYNC();
    if (tid == 0) { int s = 0; for (int t = 0; t < nt; t++) { const int v = sc[t]; sc[t] = s; s += v; } sc[nt] = s; }
    VIWB_SYNC();
    int r = sc[tid];
    for (int i = lo; i < hi; i++) { const int w = weight(i); if (w) { write(i, r); r += w; } }
    const int tot = sc[nt];
    VIWB_SYNC();
    return tot;
}

VIWB_D int fm_cas(int *p, int cmp, int val) {
#ifdef VIWB_HOST_EMU
    const int old = *p; if (old == cmp) *p = val; return old;
#else
    return atomicCAS(p, cmp, val);
#endif
}
VIWB_D void fm_or(int *p, int v) {
#ifdef VIWB_HOST_EMU
    *p |= v;
#else
    atomicOr(p, v);
#endif
}

// (id, row) keys: ascending id, the row breaks no tie (ids are unique once the duplicate check passed)
VIWB_HD long long fm_key(int id, int row) { return (long long)id * 4294967296LL + row; }
VIWB_HD int fm_key_row(long long k) { long long r = k % 4294967296LL; if (r < 0) r += 4294967296LL; return (int)r; }
VIWB_HD int fm_key_id(long long k) { return (int)((k - (long long)fm_key_row(k)) / 4294967296LL); }
VIWB_D int fm_find(const long long *keys, int n, int id) {          // row of `id` among n sorted keys, -1 if absent
    int lo = 0, hi = n;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (fm_key_id(keys[mid]) < id) lo = mid + 1; else hi = mid; }
    return (lo < n && fm_key_id(keys[lo]) == id) ? fm_key_row(keys[lo]) : -1;
}

// ---- addFeatureCheckParallax, launch 1 of 2: sort the left rows by id, match the list against them, and check everything that could make the
// call fail.  Nothing of the list is written: an error in any stream leaves every list as it was (launch 2 returns at once).
VIWB_D void fm_add_check(const FmRun &r, int s, int tid, int nt, int *sc, long long *keys) {
    const FmRows &w = r.rows;
    long long *gk = r.keys + (size_t)s * r.R;
    int *rmatch = r.rmatch + (size_t)s * r.R, *rright = r.rright + (size_t)s * r.R, *newpos = r.newpos + (size_t)s * r.R;
    const int n = r.n[s];
    const int nl = w.n[s], nr = r.stereo && w.nr ? w.nr[s] : 0;
    if (w.trk_flags && (w.trk_flags[s] & 1)) { if (tid == 0) r.err[s] |= FM_ERR_TRACKER; return; }       // not consumed, reported later
    if (nl < 0 || nl > r.R || nr < 0 || nr > r.R) { if (tid == 0) { r.err[s] |= FM_ERR_ROWS; fm_or(r.any_err, 1); } return; }
    const int *ids = w.ids + (size_t)s * w.stride, *ids_r = w.ids_r ? w.ids_r + (size_t)s * w.stride : nullptr;
    int n2 = 1; while (n2 < nl) n2 <<= 1;
    for (int i = tid; i < n2; i += nt) keys[i] = i < nl ? fm_key(ids[i], i) : 0x7fffffffffffffffLL;
    VIWB_SYNC();
    for (int k = 2; k <= n2; k <<= 1)                                    // bitonic sort
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < n2; i += nt) {
                const int p = i ^ j;
                if (p > i) {
                    const long long a = keys[i], b = keys[p];
                    if (((i & k) == 0) == (a > b)) { keys[i] = b; keys[p] = a; }
                }
            }
            VIWB_SYNC();
        }
    for (int i = tid; i < nl; i += nt) { gk[i] = keys[i]; rmatch[i] = -1; rright[i] = -1; }
    if (tid == 0) sc[nt + 1] = 0;
    VIWB_SYNC();
    int e = 0;
    for (int i = tid + 1; i < nl; i += nt) if (fm_key_id(keys[i]) == fm_key_id(keys[i - 1])) e |= FM_ERR_DUP;
    for (int k = tid; k < n; k += nt) { const int row = fm_find(keys, nl, r.src.id[(size_t)s * r.M + k]); if (row >= 0) rmatch[row] = k; }
    for (int q = tid; q < nr; q += nt) {
        const int row = fm_find(keys, nl, ids_r[q]);
        if (row < 0) e |= FM_ERR_RIGHT;
        else if (fm_cas(rright + row, -1, q) != -1) e |= FM_ERR_DUP;
    }
    if (e) fm_or(sc + nt + 1, e);
    VIWB_SYNC();
    // new features in ascending id order (the order the image map iterates in), the statistics of :58-91
    const int *nobs = r.src.nobs + (size_t)s * r.M;
    const int n_new = fm_scan(nl, tid, nt, sc, [&](int i) { return rmatch[fm_key_row(keys[i])] < 0 ? 1 : 0; }, [&](int i, int o) { newpos[i] = o; });
    const int n_long = fm_scan(nl, tid, nt, sc, [&](int i) { const int k = rmatch[fm_key_row(keys[i])]; return k >= 0 && nobs[k] + 1 >= 4 ? 1 : 0; }, [&](int, int) {});
    const int n_full = fm_scan(nl, tid, nt, sc, [&](int i) { const int k = rmatch[fm_key_row(keys[i])]; return k >= 0 && nobs[k] >= FM_SLOTS ? 1 : 0; }, [&](int, int) {});
    if (tid == 0) {
        int err = sc[nt + 1];
        if (n + n_new > r.M) err |= FM_ERR_CAP;
        if (n_full) err |= FM_ERR_OBS;
        if (err) { r.err[s] |= err; fm_or(r.any_err, 1); }
        int *d = r.dec + (size_t)s * FM_DEC_N + FM_DEC_PENDING;
        d[FM_DEC_LAST_TRACK] = nl - n_new; d[FM_DEC_LONG_TRACK] = n_long; d[FM_DEC_NEW] = n_new;
    }
}

// compensatedParallax2 (:538-571) with p_i(2) = p_j(2) = 1: the compensated and plain distances coincide
VIWB_D double fm_parallax(const float *oi, const float *oj) {
    const double u_j = (double)oj[0], v_j = (double)oj[1];
    const double u_i = trk_div((double)oi[0], 1.0), v_i = trk_div((double)oi[1], 1.0);
    const double du = trk_sub(u_i, u_j), dv = trk_sub(v_i, v_j);
    const double s = trk_sqrt(trk_add(trk_mul(du, du), trk_mul(dv, dv)));
    return 0.0 < s ? s : 0.0;                                          // max(ans = 0, sqrt(min(a, a)))
}

// ---- launch 2 of 2: append the observations, then the keyframe decision of :95-118.  Nothing happens while an error of this add or of an
// earlier one is unread (any stream's for the list rules, this stream's for a tracker overflow): the lists and decisions stay as they were.
VIWB_D void fm_add_apply(const FmRun &r, int s, int tid, int nt, int *sc) {
    if (*r.any_err || r.err[s]) return;
    const FmRows &w = r.rows;
    const long long *keys = r.keys + (size_t)s * r.R;
    const int *rmatch = r.rmatch + (size_t)s * r.R, *rright = r.rright + (size_t)s * r.R, *newpos = r.newpos + (size_t)s * r.R;
    const size_t base = (size_t)s * r.M;
    const int n = r.n[s], nl = w.n[s], fc = r.fc[s];
    const double td = r.td[s];
    const float *feat = w.feat + (size_t)s * w.stride * 6, *feat_r = w.feat_r ? w.feat_r + (size_t)s * w.stride * 6 : nullptr;
    const FmList &L = r.src;
    for (int i = tid; i < nl; i += nt) {
        const int row = fm_key_row(keys[i]);
        int k = rmatch[row], slot;
        if (k >= 0) { slot = L.nobs[base + k]; L.nobs[base + k] = slot + 1; }
        else {
            k = n + newpos[i]; slot = 0;
            L.id[base + k] = fm_key_id(keys[i]); L.start[base + k] = fc; L.nobs[base + k] = 1; L.flag[base + k] = 0; L.depth[base + k] = -1.0;
        }
        const size_t o = (base + k) * FM_SLOTS + slot;
        float *ob = L.obs + o * FM_OBS;
        for (int c = 0; c < 6; c++) ob[c] = feat[6 * row + c];
        const int q = rright[row];
        for (int c = 0; c < 6; c++) ob[6 + c] = q >= 0 ? feat_r[6 * q + c] : 0.f;
        L.td[o] = td; L.ster[o] = q >= 0 ? 1 : 0;
    }
    int *d = r.dec + (size_t)s * FM_DEC_N;
    const int m = n + d[FM_DEC_PENDING + FM_DEC_NEW];
    const int last = d[FM_DEC_PENDING + FM_DEC_LAST_TRACK], lng = d[FM_DEC_PENDING + FM_DEC_LONG_TRACK], nw = d[FM_DEC_PENDING + FM_DEC_NEW];
    VIWB_SYNC();
    if (tid == 0) { r.n[s] = m; d[FM_DEC_LAST_TRACK] = last; d[FM_DEC_LONG_TRACK] = lng; d[FM_DEC_NEW] = nw; }
    if (fc < 2 || last < 20 || lng < 40 || (double)nw > 0.5 * (double)last) {
        if (tid == 0) { d[FM_DEC_FLAG] = 0; r.avg[s] = 0.0; }
        return;
    }
    double *par = r.dscr + base;
    for (int k = tid; k < m; k += nt) {
        const int st = L.start[base + k], no = L.nobs[base + k];
        double p = -1.0;
        if (st <= fc - 2 && st + no - 1 >= fc - 1) {
            const float *o = L.obs + (base + k) * FM_SLOTS * FM_OBS;
            p = fm_parallax(o + (size_t)(fc - 2 - st) * FM_OBS, o + (size_t)(fc - 1 - st) * FM_OBS);
        }
        par[k] = p;
    }
    VIWB_SYNC();
    if (tid == 0) {                                                     // the sum in list order, as the reference adds it
        double sum = 0.0; int num = 0;
        for (int k = 0; k < m; k++) if (par[k] >= 0.0) { sum = trk_add(sum, par[k]); num++; }
        if (num == 0) { d[FM_DEC_FLAG] = 0; r.avg[s] = 0.0; }
        else {
            const double mean = trk_div(sum, (double)num);
            r.avg[s] = trk_mul(mean, r.focal);
            d[FM_DEC_FLAG] = mean >= r.min_parallax ? 0 : 1;
        }
    }
}

// ---- FeatureManager::triangulate: every feature without a positive depth, stereo pair of its first frame or its first two frames
VIWB_D void fm_triangulate(const FmRun &r, int s, int tid, int nt) {
    const size_t base = (size_t)s * r.M;
    const FmList &L = r.src;
    for (int k = tid; k < r.n[s]; k += nt) {
        if (L.depth[base + k] > 0) continue;
        const float *o = L.obs + (base + k) * FM_SLOTS * FM_OBS;
        const int stereo = r.stereo && L.ster[(base + k) * FM_SLOTS] ? 1 : 0;
        if (!stereo && L.nobs[base + k] < 2) continue;                   // the multi-view branch needs >= 4 observations: unreachable
        int fr = L.start[base + k];
        double p0[2] = {(double)o[0], (double)o[1]}, p1[2], out;
        if (stereo) { p1[0] = (double)o[6]; p1[1] = (double)o[7]; } else { p1[0] = (double)o[FM_OBS]; p1[1] = (double)o[FM_OBS + 1]; }
        TriArgs a; a.n = 1; a.state = r.state + (size_t)s * 207; a.stereo = &stereo; a.frame = &fr; a.pt0 = p0; a.pt1 = p1; a.init_depth = r.init_depth; a.depth = &out;
        triangulate_item(a, 0);
        L.depth[base + k] = out;
    }
}

// ---- the landmark numbering of optimization() / setDepth / getDepthVector: list order, features with >= 4 observations
VIWB_D int fm_number(const FmRun &r, int s, int tid, int nt, int *sc) {
    const int *nobs = r.src.nobs + (size_t)s * r.M;
    int *lm = r.iscr + (size_t)s * r.M;
    const int n = r.n[s];
    for (int k = tid; k < n; k += nt) lm[k] = -1;
    VIWB_SYNC();
    return fm_scan(n, tid, nt, sc, [&](int k) { return nobs[k] >= 4 ? 1 : 0; }, [&](int k, int o) { lm[k] = o; });
}

VIWB_D int fm_rows_of(const FmRun &r, size_t f) {
    const int no = r.src.nobs[f];
    if (no < 4) return 0;
    int c = no - 1;
    if (r.stereo) for (int j = 0; j < no; j++) c += r.src.ster[f * FM_SLOTS + j];
    return c;
}

// The visual factors of one landmark in the order of estimator.cpp:1585-1638: per observation slot j, the left camera (2F1C, from slot 1 on), then on
// a stereo slot the right one (2F2C, or 1F2C on slot 0).  ster: bit j = slot j is stereo (and the configuration is).
// visit(slot, camera, VIWB_F_PROJ_2F1C / 2F2C / 1F2C, imu_i, imu_j).  The export, the batch fill and the host lowering of a digest all enumerate here.
#ifdef __CUDACC__
#pragma nv_exec_check_disable      // the host lowering's visitor is a host lambda; the kernels' are device lambdas
#endif
template <typename V>
VIWB_HD void fm_factors(int start, int nobs, unsigned ster, V visit) {
    for (int j = 0; j < nobs; j++)
        for (int cam = 0; cam < 2; cam++) {
            if (cam == 0 ? j == 0 : !((ster >> j) & 1u)) continue;
            visit(j, cam, cam == 0 ? 0 : (j != 0 ? 1 : 2), start, start + j);
        }
}
VIWB_D unsigned fm_ster_mask(const FmRun &r, size_t f) {
    unsigned m = 0;
    if (r.stereo) for (int j = 0; j < r.src.nobs[f]; j++) m |= (unsigned)r.src.ster[f * FM_SLOTS + j] << j;
    return m;
}
// digest word of a landmark: start frame (4 bits), observation count (4 bits), stereo mask (FM_SLOTS bits)
VIWB_HD unsigned fm_digest_word(int start, int nobs, unsigned ster) { return (unsigned)start | (unsigned)nobs << 4 | ster << 8; }
VIWB_HD int fm_digest_start(unsigned d) { return (int)(d & 15u); }
VIWB_HD int fm_digest_nobs(unsigned d) { return (int)((d >> 4) & 15u); }
VIWB_HD unsigned fm_digest_ster(unsigned d) { return d >> 8; }

// ---- window, launch 1 of 2: landmarks and visual rows per stream
VIWB_D void fm_window_count(const FmRun &r, int s, int tid, int nt, int *sc) {
    const size_t base = (size_t)s * r.M;
    const int nlm = fm_scan(r.n[s], tid, nt, sc, [&](int k) { return r.src.nobs[base + k] >= 4 ? 1 : 0; }, [&](int, int) {});
    const int nrow = fm_scan(r.n[s], tid, nt, sc, [&](int k) { return fm_rows_of(r, base + k); }, [&](int, int) {});
    if (tid == 0) { r.o_cnt[2 * s] = nlm; r.o_cnt[2 * s + 1] = nrow; }
}

// ---- window, launch 2 of 2: the rows of estimator.cpp:1585-1638 at the packed offsets the host computed from launch 1
VIWB_D void fm_window_write(const FmRun &r, int s, int tid, int nt, int *sc) {
    const size_t base = (size_t)s * r.M;
    const FmList &L = r.src;
    const int *lm = r.iscr + base;
    const int row0 = r.w_off[2 * s], lm0 = r.w_off[2 * s + 1];
    fm_number(r, s, tid, nt, sc);
    fm_scan(r.n[s], tid, nt, sc, [&](int k) { return fm_rows_of(r, base + k); }, [&](int k, int o) {
        const size_t f = base + k;
        const int l = lm[k];
        r.w_inv[lm0 + l] = trk_div(1.0, L.depth[f]); r.w_id[lm0 + l] = L.id[f];
        const float *o0 = L.obs + f * FM_SLOTS * FM_OBS;
        int q = row0 + o;
        fm_factors(L.start[f], L.nobs[f], fm_ster_mask(r, f), [&](int j, int cam, int type, int imu_i, int imu_j) {
            const float *pj = o0 + (size_t)j * FM_OBS + 6 * cam;
            double *ob = r.w_obs + (size_t)q * 12;
            ob[0] = (double)o0[0]; ob[1] = (double)o0[1]; ob[2] = 1.0;
            ob[3] = (double)pj[0]; ob[4] = (double)pj[1]; ob[5] = 1.0;
            ob[6] = (double)o0[4]; ob[7] = (double)o0[5]; ob[8] = (double)pj[4]; ob[9] = (double)pj[5];
            ob[10] = L.td[f * FM_SLOTS]; ob[11] = L.td[f * FM_SLOTS + j];
            r.w_type[q] = type; r.w_lm[q] = l; r.w_fi[q] = imu_i; r.w_fj[q] = imu_j;
            q++;
        });
    });
}

// ---- window digest (viwb_features_batch_create, after fm_window_count): one word per landmark, in the export's numbering, at w_off[s]
VIWB_D void fm_window_digest(const FmRun &r, int s, int tid, int nt, int *sc) {
    const size_t base = (size_t)s * r.M;
    const FmList &L = r.src;
    const int l0 = r.w_off[s];
    fm_scan(r.n[s], tid, nt, sc, [&](int k) { return L.nobs[base + k] >= 4 ? 1 : 0; }, [&](int k, int l) {
        const size_t f = base + k;
        r.w_dig[l0 + l] = fm_digest_word(L.start[f], L.nobs[f], fm_ster_mask(r, f));
    });
}

// ---- batch fill: the observations and inverse depths of window s of a batch built from the digest, straight into its slab in the wire format
// (kernels_lin.cuh vis_expand reads them next): the host side once per landmark from its first observation, at the index the lowering gave the
// landmark's first factor, the observer side per factor, x_init's landmark part as fm_window_write's 1 / estimated_depth beside the uploaded
// fixed state
VIWB_D void fm_batch_fill(const FmRun &r, int s, int tid, int nt, int *sc) {
    const size_t base = (size_t)s * r.M;
    const FmList &L = r.src;
    const WinMeta &m = r.b_meta[s];
    const int *lm = r.iscr + base;
    for (int k = tid; k < SFIX; k += nt) r.b_x[m.state_off + k] = r.b_xfix[(size_t)s * SFIX + k];
    fm_number(r, s, tid, nt, sc);
    fm_scan(r.n[s], tid, nt, sc, [&](int k) { return fm_rows_of(r, base + k); }, [&](int k, int o) {
        const size_t f = base + k;
        r.b_x[m.state_off + SFIX + lm[k]] = trk_div(1.0, L.depth[f]);
        const float *o0 = L.obs + f * FM_SLOTS * FM_OBS;
        int q = m.vis_off + o;
        double *hi = r.b_obs_i + (size_t)r.b_oi[q] * 6;
        hi[0] = (double)o0[0]; hi[1] = (double)o0[1]; hi[2] = 1.0; hi[3] = (double)o0[4]; hi[4] = (double)o0[5]; hi[5] = L.td[f * FM_SLOTS];
        fm_factors(L.start[f], L.nobs[f], fm_ster_mask(r, f), [&](int j, int cam, int, int, int) {
            const float *pj = o0 + (size_t)j * FM_OBS + 6 * cam;
            double *hj = r.b_obs_j + (size_t)q * 6;
            hj[0] = (double)pj[0]; hj[1] = (double)pj[1]; hj[2] = 1.0; hj[3] = (double)pj[4]; hj[4] = (double)pj[5]; hj[5] = L.td[f * FM_SLOTS + j];
            q++;
        });
    });
}

// ---- setDepth (:142-160): estimated_depth = 1 / x of landmark k, solve_flag 2 if negative else 1
VIWB_D void fm_set_depth(const FmRun &r, int s, int tid, int nt, int *sc) {
    const size_t base = (size_t)s * r.M;
    fm_number(r, s, tid, nt, sc);
    const int *lm = r.iscr + base;
    for (int k = tid; k < r.n[s]; k += nt) {
        if (lm[k] < 0) continue;
        const double d = trk_div(1.0, r.xin[r.off[s] + lm[k]]);
        r.src.depth[base + k] = d; r.src.flag[base + k] = d < 0 ? 2 : 1;
    }
}

// ---- predictPtsInNextFrame, compacted to the features it inserts into predictPts, in list order
VIWB_D void fm_predict(const FmRun &r, int s, int tid, int nt, int *sc) {
    const size_t base = (size_t)s * r.M;
    const FmList &L = r.src;
    int *ok = r.iscr + base;
    const int n = r.n[s];
    double *pts = r.dscr + base * 3;
    for (int k = tid; k < n; k += nt) {
        const float *o = L.obs + (base + k) * FM_SLOTS * FM_OBS;
        double p0[3] = {(double)o[0], (double)o[1], 1.0};
        unsigned char v;
        PredictArgs a; a.n = 1; a.frame_count = r.fc[s]; a.state = r.state + (r.st_off ? (size_t)r.st_off[s] : (size_t)s * 207); a.start_frame = L.start + base + k; a.num_obs = L.nobs + base + k;
        a.pt0 = p0; a.depth = L.depth + base + k; a.pts_cam = pts + 3 * k; a.valid = &v;
        predict_pts_item(a, 0);
        ok[k] = v;
    }
    VIWB_SYNC();
    const int cnt = fm_scan(n, tid, nt, sc, [&](int k) { return ok[k] ? 1 : 0; }, [&](int k, int o) {
        r.o_ids[base + o] = L.id[base + k];
        for (int c = 0; c < 3; c++) r.o_pts[(base + o) * 3 + c] = pts[3 * k + c];
    });
    if (tid == 0) r.o_cnt[s] = cnt;
}

// ---- the erasures, as stable compactions src -> dst of every stream (a stream with nothing to erase is copied):
//   FM_COMPACT_OUTLIERS  removeOutlier (:440-455) of the landmarks flagged in `verdict` (numbering of the last export); their ids -> o_ids
//   FM_COMPACT_SLIDE     frame_count == WINDOW_SIZE only: MARGIN_OLD -> removeBackShiftDepth (:457-495) if shift[s] else removeBack (:497-513);
//                        MARGIN_SECOND_NEW -> removeFront(frame_count) (:515-536), keeping its TODO: no depth shift when slot 0 is dropped
//   FM_COMPACT_FAILURES  removeFailures (:162-171): solve_flag == 2
VIWB_D void fm_compact(const FmRun &r, int s, int tid, int nt, int *sc) {
    const size_t base = (size_t)s * r.M;
    const FmList &A = r.src, &B = r.dst;
    const int n = r.n[s];
    int *plan = r.iscr + base;                   // 0 = erase, 1 = keep, 2 + j = keep without observation slot j
    if (r.mode == FM_COMPACT_OUTLIERS) fm_number(r, s, tid, nt, sc);      // plan[k] holds the landmark index until overwritten below
    const int fc = r.fc ? r.fc[s] : 0, flag = r.dec[(size_t)s * FM_DEC_N + FM_DEC_FLAG];
    const bool shift = r.shift && r.shift[s];
    for (int k = tid; k < n; k += nt) {
        const size_t f = base + k;
        const int st = A.start[f], no = A.nobs[f];
        int p = 1, st2 = st;
        double dep = A.depth[f];
        if (r.mode == FM_COMPACT_OUTLIERS) {
            const int l = plan[k];
            p = (l >= 0 && (r.verdict ? r.verdict[r.off[s] + l] != 0 : r.verdict_i[r.off[s] + l] != 0)) ? 0 : 1;
        } else if (r.mode == FM_COMPACT_FAILURES) {
            p = A.flag[f] == 2 ? 0 : 1;
        } else if (fc == VIWB_WINDOW_SIZE) {
            if (flag == 0) {
                if (st != 0) st2 = st - 1;
                else if (shift) {
                    if (no - 1 < 2) p = 0;
                    else {
                        const float *o = A.obs + f * FM_SLOTS * FM_OBS;
                        double uv[3] = {(double)o[0], (double)o[1], 1.0}, out;
                        ShiftArgs a; a.n = 1; a.uv = uv; a.depth_in = &dep; a.init_depth = r.init_depth; a.depth_out = &out;
                        const double *m = r.mats + (size_t)s * 24;
                        for (int c = 0; c < 9; c++) { a.margR[c] = m[c]; a.newR[c] = m[12 + c]; }
                        for (int c = 0; c < 3; c++) { a.margP[c] = m[9 + c]; a.newP[c] = m[21 + c]; }
                        shift_depth_item(a, 0);
                        dep = out; p = 2;
                    }
                } else p = no - 1 == 0 ? 0 : 2;
            } else {
                if (st == fc) st2 = st - 1;
                else if (st + no - 1 >= fc - 1) {
                    const int j = VIWB_WINDOW_SIZE - 1 - st;
                    p = no - 1 == 0 ? 0 : 2 + j;
                }
            }
        }
        if (r.mode == FM_COMPACT_SLIDE) { A.start[f] = st2; A.depth[f] = dep; }   // copied to dst after the barrier
        plan[k] = p;
    }
    VIWB_SYNC();
    const int m = fm_scan(n, tid, nt, sc, [&](int k) { return plan[k] ? 1 : 0; }, [&](int k, int o) {
        const size_t f = base + k, g = base + o;
        const int drop = plan[k] >= 2 ? plan[k] - 2 : -1, no = A.nobs[f];
        B.id[g] = A.id[f]; B.start[g] = A.start[f]; B.flag[g] = A.flag[f]; B.depth[g] = A.depth[f];
        B.nobs[g] = drop >= 0 ? no - 1 : no;
        for (int j = 0, t = 0; j < no; j++) {
            if (j == drop) continue;
            const size_t a = f * FM_SLOTS + j, b = g * FM_SLOTS + t;
            for (int c = 0; c < FM_OBS; c++) B.obs[b * FM_OBS + c] = A.obs[a * FM_OBS + c];
            B.td[b] = A.td[a]; B.ster[b] = A.ster[a];
            t++;
        }
    });
    if (r.mode == FM_COMPACT_OUTLIERS)
        fm_scan(n, tid, nt, sc, [&](int k) { return plan[k] ? 0 : 1; }, [&](int k, int o) { r.o_ids[base + o] = A.id[base + k]; });
    if (tid == 0) { if (r.mode == FM_COMPACT_OUTLIERS) r.o_cnt[s] = n - m; r.n[s] = m; }
}

#ifndef VIWB_HOST_EMU
// one FM_NT-thread block per stream
__global__ void __launch_bounds__(FM_NT) fm_add_check_kernel(FmRun r) { __shared__ int sc[FM_NT + 2]; __shared__ long long keys[FM_MAX_ROWS]; fm_add_check(r, blockIdx.x, threadIdx.x, blockDim.x, sc, keys); }
__global__ void __launch_bounds__(FM_NT) fm_add_apply_kernel(FmRun r) { __shared__ int sc[FM_NT + 2]; fm_add_apply(r, blockIdx.x, threadIdx.x, blockDim.x, sc); }
__global__ void __launch_bounds__(FM_NT) fm_triangulate_kernel(FmRun r) { fm_triangulate(r, blockIdx.x, threadIdx.x, blockDim.x); }
__global__ void __launch_bounds__(FM_NT) fm_window_count_kernel(FmRun r) { __shared__ int sc[FM_NT + 2]; fm_window_count(r, blockIdx.x, threadIdx.x, blockDim.x, sc); }
__global__ void __launch_bounds__(FM_NT) fm_window_write_kernel(FmRun r) { __shared__ int sc[FM_NT + 2]; fm_window_write(r, blockIdx.x, threadIdx.x, blockDim.x, sc); }
__global__ void __launch_bounds__(FM_NT) fm_window_digest_kernel(FmRun r) { __shared__ int sc[FM_NT + 2]; fm_window_digest(r, blockIdx.x, threadIdx.x, blockDim.x, sc); }
__global__ void __launch_bounds__(FM_NT) fm_batch_fill_kernel(FmRun r) { __shared__ int sc[FM_NT + 2]; fm_batch_fill(r, blockIdx.x, threadIdx.x, blockDim.x, sc); }
__global__ void __launch_bounds__(FM_NT) fm_set_depth_kernel(FmRun r) { __shared__ int sc[FM_NT + 2]; fm_set_depth(r, blockIdx.x, threadIdx.x, blockDim.x, sc); }
__global__ void __launch_bounds__(FM_NT) fm_predict_kernel(FmRun r) { __shared__ int sc[FM_NT + 2]; fm_predict(r, blockIdx.x, threadIdx.x, blockDim.x, sc); }
__global__ void __launch_bounds__(FM_NT) fm_compact_kernel(FmRun r) { __shared__ int sc[FM_NT + 2]; fm_compact(r, blockIdx.x, threadIdx.x, blockDim.x, sc); }
#endif

}  // namespace viwb
