// kernels_feat.cuh -- per-landmark geometry around the window solve (SURVEY 8 f-3):
//   FeatureManager::triangulate / triangulatePoint   estimator/feature_manager.cpp:198-213, 309-380
//   FeatureManager::removeBackShiftDepth             estimator/feature_manager.cpp:457-493
//   Estimator::predictPtsInNextFrame                 estimator/estimator.cpp:2080-2113
// One thread per feature; everything is a handful of 3x3 / 4x4 operations.
#pragma once
#include "vmath.cuh"

namespace viwb {

// Right singular vector of the smallest singular value of a 4x4 matrix (what triangulatePoint takes from
// jacobiSvd(ComputeFullV).matrixV().rightCols<1>()), by one-sided (Hestenes) Jacobi on the columns: no squaring of the
// condition number.  D is row-major and is overwritten; v receives the unit vector (sign as produced by the rotations).
VIWB_HD void smallest_right_singular_4x4(double *D, double *v) {
    double V[16];
    for (int i = 0; i < 16; i++) V[i] = (i / 4 == i % 4) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 30; sweep++) {
        double off = 0.0;
        for (int p = 0; p < 3; p++) for (int q = p + 1; q < 4; q++) {
            double a = 0.0, b = 0.0, c = 0.0;
            for (int r = 0; r < 4; r++) { a += D[r * 4 + p] * D[r * 4 + p]; b += D[r * 4 + q] * D[r * 4 + q]; c += D[r * 4 + p] * D[r * 4 + q]; }
            if (c == 0.0 || fabs(c) <= 1e-300 + 2.220446049250313e-16 * sqrt(a * b)) continue;
            off += fabs(c);
            const double zeta = (b - a) / (2.0 * c);
            const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
            const double cs = 1.0 / sqrt(1.0 + t * t), sn = cs * t;
            for (int r = 0; r < 4; r++) {
                const double dp = D[r * 4 + p], dq = D[r * 4 + q];
                D[r * 4 + p] = cs * dp - sn * dq; D[r * 4 + q] = sn * dp + cs * dq;
                const double vp = V[r * 4 + p], vq = V[r * 4 + q];
                V[r * 4 + p] = cs * vp - sn * vq; V[r * 4 + q] = sn * vp + cs * vq;
            }
        }
        if (off == 0.0) break;
    }
    int best = 0; double nb = 0.0;
    for (int c = 0; c < 4; c++) { double n2 = 0.0; for (int r = 0; r < 4; r++) n2 += D[r * 4 + c] * D[r * 4 + c]; if (c == 0 || n2 < nb) { nb = n2; best = c; } }
    for (int r = 0; r < 4; r++) v[r] = V[r * 4 + best];
}

// camera pose [R^T | -R^T t] (3x4, row-major) of camera `cam` at the frame whose pose block starts at `pose`
VIWB_HD void camera_pose34(const double *pose, const double *ex, double *P) {
    const Q4 Qi = ldq(pose + 3), qic = ldq(ex + 3);
    const V3 t = ld3(pose) + qrot(Qi, ld3(ex));                 // w_t_c = Ps + Rs tic
    const M3 R = qR(Qi) * qR(qic);                               // w_R_c = Rs ric
    const M3 Rt = transpose(R);
    const V3 mt = -(Rt * t);
    for (int r = 0; r < 3; r++) { for (int c = 0; c < 3; c++) P[r * 4 + c] = Rt.m[r * 3 + c]; P[r * 4 + 3] = comp(mt, r); }
}

struct TriArgs { int n; const double *state; const int *stereo, *frame; const double *pt0, *pt1; double init_depth; double *depth; };
// stereo[k] = 1: left / right camera of frame[k] (feature_manager.cpp:316-352); 0: left camera of frame[k] and frame[k]+1 (:353-385)
VIWB_D void triangulate_item(const TriArgs &a, int k) {
    if (k >= a.n) return;
    const double *x = a.state;
    const int i = a.frame[k], st = a.stereo[k];
    double P0[12], P1[12];
    camera_pose34(x + 7 * i, x + 176, P0);
    if (st) camera_pose34(x + 7 * i, x + 183, P1); else camera_pose34(x + 7 * (i + 1), x + 176, P1);
    const double u0 = a.pt0[2 * k], v0 = a.pt0[2 * k + 1], u1 = a.pt1[2 * k], v1 = a.pt1[2 * k + 1];
    double D[16], tp[4];
    for (int c = 0; c < 4; c++) {
        D[0 * 4 + c] = u0 * P0[2 * 4 + c] - P0[0 * 4 + c];
        D[1 * 4 + c] = v0 * P0[2 * 4 + c] - P0[1 * 4 + c];
        D[2 * 4 + c] = u1 * P1[2 * 4 + c] - P1[0 * 4 + c];
        D[3 * 4 + c] = v1 * P1[2 * 4 + c] - P1[1 * 4 + c];
    }
    smallest_right_singular_4x4(D, tp);
    const double px = tp[0] / tp[3], py = tp[1] / tp[3], pz = tp[2] / tp[3];
    const double depth = P0[2 * 4 + 0] * px + P0[2 * 4 + 1] * py + P0[2 * 4 + 2] * pz + P0[2 * 4 + 3];      // (leftPose * point).z
    a.depth[k] = depth > 0 ? depth : a.init_depth;
}

struct ShiftArgs { int n; const double *uv, *depth_in; double margR[9], margP[3], newR[9], newP[3]; double init_depth; double *depth_out; };
VIWB_D void shift_depth_item(const ShiftArgs &a, int k) {
    if (k >= a.n) return;
    const V3 pts_i = ld3(a.uv + 3 * k) * a.depth_in[k];
    const V3 w = m3_ld(a.margR) * pts_i + ld3(a.margP);
    const V3 pts_j = tmul(m3_ld(a.newR), w - ld3(a.newP));
    a.depth_out[k] = pts_j.z > 0 ? pts_j.z : a.init_depth;
}

// Estimator::predictPtsInNextFrame (estimator.cpp:2080-2113).  nextT = curT * (prevT^-1 * curT) with prevT^-1 taken as the rigid inverse
// [R^T | -R^T p] instead of the reference's general Matrix4d inverse: the two agree to rounding for a rotation block, and the parity tests
// hold the result to 1e-9 against the reference's compiled code.
struct PredictArgs { int n, frame_count; const double *state; const int *start_frame, *num_obs; const double *pt0, *depth; double *pts_cam; unsigned char *valid; };
VIWB_D void predict_pts_item(const PredictArgs &a, int k) {
    if (k >= a.n) return;
    const double *x = a.state;
    const int fc = a.frame_count, first = a.start_frame[k], nobs = a.num_obs[k];
    const double depth = a.depth[k];
    const bool ok = fc >= 2 && depth > 0 && nobs >= 2 && first + nobs - 1 == fc;             // :2083, :2094, :2099
    a.valid[k] = ok ? 1 : 0;
    V3 pts_cam = v3(0.0, 0.0, 0.0);
    if (ok) {
        const M3 Rc = qR(ldq(x + 7 * fc + 3)), Rp = qR(ldq(x + 7 * (fc - 1) + 3)), ric = qR(ldq(x + 176 + 3));
        const V3 Pc = ld3(x + 7 * fc), Pp = ld3(x + 7 * (fc - 1)), tic = ld3(x + 176);
        const M3 nextR = Rc * (transpose(Rp) * Rc);
        const V3 nextP = Rc * tmul(Rp, Pc - Pp) + Pc;
        const V3 pts_j = ric * (depth * ld3(a.pt0 + 3 * k)) + tic;
        const V3 pts_w = qR(ldq(x + 7 * first + 3)) * pts_j + ld3(x + 7 * first);
        const V3 pts_local = tmul(nextR, pts_w - nextP);
        pts_cam = tmul(ric, pts_local - tic);
    }
    st3(a.pts_cam + 3 * k, pts_cam);
}

// FP64 operations rounded one by one (no fused multiply-add, IEEE division and square root), so that a result is the double the
// reference's build (-ffp-contract=off here, SSE2 there) computes, and its float narrowing the same float, bit for bit
#ifdef VIWB_HOST_EMU
static inline double trk_mul(double a, double b) { return a * b; }
static inline double trk_add(double a, double b) { return a + b; }
static inline double trk_sub(double a, double b) { return a - b; }
static inline double trk_div(double a, double b) { return a / b; }
static inline double trk_sqrt(double a) { return sqrt(a); }
#else
VIWB_D double trk_mul(double a, double b) { return __dmul_rn(a, b); }
VIWB_D double trk_add(double a, double b) { return __dadd_rn(a, b); }
VIWB_D double trk_sub(double a, double b) { return __dsub_rn(a, b); }
VIWB_D double trk_div(double a, double b) { return __ddiv_rn(a, b); }
VIWB_D double trk_sqrt(double a) { return __dsqrt_rn(a); }
#endif

// Camera models of viwb_camera (include/viwb.h).  One record holds either: PINHOLE's fx, fy, cx, cy or MEI's gamma1, gamma2, u0, v0 in
// the same four slots (both are the K of a lift mx = (u - cx) / fx), the radtan coefficients k1, k2, p1, p2 shared by both, and MEI's xi.
enum { CAM_PINHOLE = 0, CAM_MEI = 1 };
struct CamModel { int model; double fx, fy, cx, cy, k1, k2, p1, p2, xi; };

// CataCamera::distortion (camera_models/src/camera_models/CataCamera.cc:766-782)
VIWB_D void mei_distortion(const CamModel &c, double x, double y, double &dx, double &dy) {
    const double mx2 = trk_mul(x, x), my2 = trk_mul(y, y), mxy = trk_mul(x, y), rho2 = trk_add(mx2, my2);
    const double rad = trk_add(trk_mul(c.k1, rho2), trk_mul(trk_mul(c.k2, rho2), rho2));
    dx = trk_add(trk_add(trk_mul(x, rad), trk_mul(trk_mul(2.0, c.p1), mxy)), trk_mul(c.p2, trk_add(rho2, trk_mul(2.0, mx2))));
    dy = trk_add(trk_add(trk_mul(y, rad), trk_mul(trk_mul(2.0, c.p2), mxy)), trk_mul(c.p1, trk_add(rho2, trk_mul(2.0, my2))));
}
// CataCamera::liftProjective (CataCamera.cc:556-626; m_inv_K* of :319-323, m_noDistortion of :307-317, recursive model n = 8) followed by
// FeatureTracker::undistortedPts' b.x() / b.z(), b.y() / b.z() narrowed to cv::Point2f (featureTracker/feature_tracker.cpp:606-617).
// A ray with 1 + (1 - xi^2) rho^2 < 0 gives NaN, one with b.z() == 0 gives inf, as in the reference.
VIWB_D void mei_lift(const CamModel &c, float u, float v, float &x, float &y) {
    const double inv_K11 = trk_div(1.0, c.fx), inv_K13 = trk_div(-c.cx, c.fx), inv_K22 = trk_div(1.0, c.fy), inv_K23 = trk_div(-c.cy, c.fy);
    const double mx_d = trk_add(trk_mul(inv_K11, (double)u), inv_K13), my_d = trk_add(trk_mul(inv_K22, (double)v), inv_K23);
    double mx_u = mx_d, my_u = my_d;
    if (!(c.k1 == 0.0 && c.k2 == 0.0 && c.p1 == 0.0 && c.p2 == 0.0)) {
        for (int it = 0; it < 8; it++) {
            double dx, dy;
            mei_distortion(c, mx_u, my_u, dx, dy);                             // it == 0: (mx_u, my_u) == (mx_d, my_d)
            mx_u = trk_sub(mx_d, dx); my_u = trk_sub(my_d, dy);
        }
    }
    double z;
    if (c.xi == 1.0) z = trk_div(trk_sub(trk_sub(1.0, trk_mul(mx_u, mx_u)), trk_mul(my_u, my_u)), 2.0);
    else {
        const double rho2 = trk_add(trk_mul(mx_u, mx_u), trk_mul(my_u, my_u));
        z = trk_sub(1.0, trk_div(trk_mul(c.xi, trk_add(rho2, 1.0)), trk_add(c.xi, trk_sqrt(trk_add(1.0, trk_mul(trk_sub(1.0, trk_mul(c.xi, c.xi)), rho2))))));
    }
    x = (float)trk_div(mx_u, z); y = (float)trk_div(my_u, z);
}
// CataCamera::spaceToPlane (CataCamera.cc:636-659) narrowed to cv::Point2f (feature_tracker.cpp:730).  |P| = sqrt((x^2 + y^2) + z^2).
VIWB_D void mei_space_to_plane(const CamModel &c, const double *P, float &u, float &v) {
    const double norm = trk_sqrt(trk_add(trk_add(trk_mul(P[0], P[0]), trk_mul(P[1], P[1])), trk_mul(P[2], P[2])));
    const double z = trk_add(P[2], trk_mul(c.xi, norm));
    double xd = trk_div(P[0], z), yd = trk_div(P[1], z);
    if (!(c.k1 == 0.0 && c.k2 == 0.0 && c.p1 == 0.0 && c.p2 == 0.0)) {
        double dx, dy;
        mei_distortion(c, xd, yd, dx, dy);
        xd = trk_add(xd, dx); yd = trk_add(yd, dy);
    }
    u = (float)trk_add(trk_mul(c.fx, xd), c.cx); v = (float)trk_add(trk_mul(c.fy, yd), c.cy);
}

// FeatureTracker::undistortedPts (featureTracker/feature_tracker.cpp:606-617) -> PinholeCamera::liftProjective with the recursive
// distortion model, n = 8 (camera_models/src/camera_models/PinholeCamera.cc:450-517, distortion :646-662), results narrowed to
// cv::Point2f, or mei_lift when model == CAM_MEI; and FeatureTracker::ptsVelocity (:619-657) for points paired index-wise with the
// previous tick (SURVEY 8 f-1).
struct UndistArgs { int n; const float *pts, *prev_un; const unsigned char *has_prev; double fx, fy, cx, cy, k1, k2, p1, p2, dt; float *un, *vel; int model; double xi; };
VIWB_D void undistort_item(const UndistArgs &a, int i) {
    if (i >= a.n) return;
    float ux, uy;
    if (a.model == CAM_MEI) {
        const CamModel c = {a.model, a.fx, a.fy, a.cx, a.cy, a.k1, a.k2, a.p1, a.p2, a.xi};
        mei_lift(c, a.pts[2 * i], a.pts[2 * i + 1], ux, uy);
    } else {                                                                // the pinhole lift keeps its contracted arithmetic (2e-7 bar)
        const double inv_K11 = 1.0 / a.fx, inv_K13 = -a.cx / a.fx, inv_K22 = 1.0 / a.fy, inv_K23 = -a.cy / a.fy;     // PinholeCamera.cc:105-108
        const double mx_d = inv_K11 * (double)a.pts[2 * i] + inv_K13, my_d = inv_K22 * (double)a.pts[2 * i + 1] + inv_K23;
        double mx_u = mx_d, my_u = my_d;
        if (!(a.k1 == 0.0 && a.k2 == 0.0 && a.p1 == 0.0 && a.p2 == 0.0)) {       // m_noDistortion
            for (int it = 0; it < 8; it++) {
                const double x = (it == 0) ? mx_d : mx_u, y = (it == 0) ? my_d : my_u;
                const double mx2 = x * x, my2 = y * y, mxy = x * y, rho2 = mx2 + my2, rad = a.k1 * rho2 + a.k2 * rho2 * rho2;
                const double dx = x * rad + 2.0 * a.p1 * mxy + a.p2 * (rho2 + 2.0 * mx2), dy = y * rad + 2.0 * a.p2 * mxy + a.p1 * (rho2 + 2.0 * my2);
                mx_u = mx_d - dx; my_u = my_d - dy;
            }
        }
        ux = (float)(mx_u / 1.0); uy = (float)(my_u / 1.0);                     // b.x() / b.z() with b.z() = 1
    }
    a.un[2 * i] = ux; a.un[2 * i + 1] = uy;
    if (a.vel) {
        float vx = 0.f, vy = 0.f;
        if (a.prev_un && (!a.has_prev || a.has_prev[i])) {
            vx = (float)((double)(ux - a.prev_un[2 * i]) / a.dt);               // float difference, double division (:640-641)
            vy = (float)((double)(uy - a.prev_un[2 * i + 1]) / a.dt);
        }
        a.vel[2 * i] = vx; a.vel[2 * i + 1] = vy;
    }
}

#ifndef VIWB_HOST_EMU
__global__ void undistort_kernel(UndistArgs a) { undistort_item(a, blockIdx.x * blockDim.x + threadIdx.x); }
__global__ void triangulate_kernel(TriArgs a) { triangulate_item(a, blockIdx.x * blockDim.x + threadIdx.x); }
__global__ void shift_depth_kernel(ShiftArgs a) { shift_depth_item(a, blockIdx.x * blockDim.x + threadIdx.x); }
__global__ void predict_pts_kernel(PredictArgs a) { predict_pts_item(a, blockIdx.x * blockDim.x + threadIdx.x); }
#endif

}  // namespace viwb
