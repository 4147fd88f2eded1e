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

// FeatureTracker::undistortedPts (featureTracker/feature_tracker.cpp:606-617) -> PinholeCamera::liftProjective with the recursive
// distortion model, n = 8 (camera_models/src/camera_models/PinholeCamera.cc:450-517, distortion :646-662), results narrowed to
// cv::Point2f; and FeatureTracker::ptsVelocity (:619-657) for points paired index-wise with the previous tick (SURVEY 8 f-1).
struct UndistArgs { int n; const float *pts, *prev_un; const unsigned char *has_prev; double fx, fy, cx, cy, k1, k2, p1, p2, dt; float *un, *vel; };
VIWB_D void undistort_item(const UndistArgs &a, int i) {
    if (i >= a.n) return;
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
    const float ux = (float)(mx_u / 1.0), uy = (float)(my_u / 1.0);          // b.x() / b.z() with b.z() = 1
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
