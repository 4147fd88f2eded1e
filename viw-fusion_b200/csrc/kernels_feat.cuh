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
// KANNALA_BRANDT puts mu, mv, u0, v0 in fx, fy, cx, cy and its odd-polynomial coefficients k2, k3, k4, k5 in k1, k2, p1, p2 (xi unused).
enum { CAM_PINHOLE = 0, CAM_MEI = 1, CAM_KB = 2 };
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

// ---- Kannala-Brandt (camodocal EquidistantCamera).  The trigonometric calls are the only operations not rounded like the reference's:
// CUDA's sin / cos / acos / atan2 are within 2 ulp of the exact result, glibc's within 1, so a double may differ in its last bits, and a
// float narrowed from it by one ulp where that moves it across a rounding boundary.  Everything else is rounded operation by operation.
#ifdef VIWB_HOST_EMU
static inline double kb_sin(double a) { return sin(a); }
static inline double kb_cos(double a) { return cos(a); }
static inline double kb_acos(double a) { return acos(a); }
static inline double kb_atan2(double y, double x) { return atan2(y, x); }
#else
VIWB_D double kb_sin(double a) { return sin(a); }
VIWB_D double kb_cos(double a) { return cos(a); }
VIWB_D double kb_acos(double a) { return acos(a); }
VIWB_D double kb_atan2(double y, double x) { return atan2(y, x); }
#endif
VIWB_D double kb_maxi(double a, double b) { return a < b ? b : a; }             // numext::maxi = std::max

// The degree of the polynomial backprojectSymmetric solves (EquidistantCamera.cc:731-747): 9, less 2 for every zero coefficient wherever it
// sits -- so k2 == 0 drops the degree to 7 and with it k5, the reference's own quirk.
VIWB_HD int kb_npow(const CamModel &c) {
    int npow = 9;
    if (c.p2 == 0.0) npow -= 2;                                                  // k5
    if (c.p1 == 0.0) npow -= 2;                                                  // k4
    if (c.k2 == 0.0) npow -= 2;                                                  // k3
    if (c.k1 == 0.0) npow -= 2;                                                  // k2
    return npow;
}

// Eigen 3.3's MatrixBase::makeHouseholder of the m-vector x (m = 2 or 3): essential part ess[m - 1], tau, beta
VIWB_D void kb_householder(const double *x, int m, double *ess, double &tau, double &beta) {
    const double tail = m == 3 ? trk_add(trk_mul(x[1], x[1]), trk_mul(x[2], x[2])) : trk_mul(x[1], x[1]);
    const double c0 = x[0];
    if (tail <= 2.2250738585072014e-308) { tau = 0.0; beta = c0; ess[0] = 0.0; ess[1] = 0.0; return; }
    beta = trk_sqrt(trk_add(trk_mul(c0, c0), tail));
    if (c0 >= 0.0) beta = -beta;
    const double d = trk_sub(c0, beta);
    ess[0] = trk_div(x[1], d); ess[1] = m == 3 ? trk_div(x[2], d) : 0.0;
    tau = trk_div(trk_sub(beta, c0), beta);
}

// The eigenvalues of the n x n companion matrix in T (column-major, leading dimension 9, overwritten), as Eigen 3.3's
// EigenSolver<MatrixXd>(A) returns them: RealSchur::compute (A scaled by max |a_ij|, then computeFromHessenberg: the deflation test with
// considerAsZero, Wilkinson's exceptional shift at iteration 10 and MATLAB's at 30, at most 40 n iterations, the Francis double-shift step,
// splitOffTwoRows) and EigenSolver::compute's extraction (the scaled 2 x 2 formula).  A companion matrix is already upper Hessenberg: its
// HessenbergDecomposition finds every Householder tail zero, so tau = 0, H = T and Q = I, and it is skipped.  Only the leading (iu + 1) x (iu + 1)
// block is updated: the columns right of iu hold converged blocks whose entries the later steps and the extraction never read (Eigen updates
// them for the Schur vectors, which the eigenvalues do not need).  Without convergence EigenSolver extracts nothing and the eigenvalues stay
// 0; extraction stops at the first non-finite value, the later ones staying 0.  wr / wi: real and imaginary parts, in Eigen's order.
// The solver is called, not inlined, and its loops stay rolled: its 81-entry matrix lives in its own stack frame, and it adds as few registers
// as it can to the kernels that reach it (trk_merge, trk_stereo, undistort_kernel), whose pinhole and MEI paths run with the same allocation.
#ifdef VIWB_HOST_EMU
#define KB_NOINLINE static
#define UNROLL1
#else
#define KB_NOINLINE __device__ __noinline__
#define UNROLL1 _Pragma("unroll 1")
#endif
#define KB_T(i, j) T[(j) * 9 + (i)]
KB_NOINLINE void kb_eigenvalues(double *T, int n, double *wr, double *wi) {
    const double eps = 2.220446049250313e-16, tiny = 2.2250738585072014e-308;
    UNROLL1 for (int i = 0; i < n; i++) { wr[i] = 0.0; wi[i] = 0.0; }
    double scale = 0.0;                                                          // RealSchur::compute: cwiseAbs().maxCoeff()
    UNROLL1 for (int j = 0; j < n; j++) for (int i = 0; i < n; i++) scale = kb_maxi(scale, fabs(KB_T(i, j)));
    if (scale < tiny) return;                                                    // T = 0: every eigenvalue 0
    UNROLL1 for (int j = 0; j < n; j++) for (int i = 0; i < n; i++) KB_T(i, j) = trk_div(KB_T(i, j), scale);
    double norm = 0.0;                                                           // computeNormOfT, column by column
    UNROLL1 for (int j = 0; j < n; j++) {
        double s = 0.0;
        UNROLL1 for (int i = 0; i < n && i <= j + 1; i++) s = trk_add(s, fabs(KB_T(i, j)));
        norm = trk_add(norm, s);
    }
    const double zero = kb_maxi(trk_mul(norm, eps * eps), tiny);                 // considerAsZero
    int iu = n - 1, iter = 0, total = 0;
    const int max_iters = 40 * n;
    double exshift = 0.0;
    if (norm != 0.0) {
        while (iu >= 0) {
            int il = iu;                                                         // findSmallSubdiagEntry
            while (il > 0) {
                const double s = kb_maxi(trk_mul(trk_add(fabs(KB_T(il - 1, il - 1)), fabs(KB_T(il, il))), eps), zero);
                if (fabs(KB_T(il, il - 1)) <= s) break;
                il--;
            }
            if (il == iu) {                                                      // one root
                KB_T(iu, iu) = trk_add(KB_T(iu, iu), exshift);
                if (iu > 0) KB_T(iu, iu - 1) = 0.0;
                iu--; iter = 0;
            } else if (il == iu - 1) {                                           // two roots: splitOffTwoRows
                const double p = trk_mul(0.5, trk_sub(KB_T(iu - 1, iu - 1), KB_T(iu, iu)));
                const double q = trk_add(trk_mul(p, p), trk_mul(KB_T(iu, iu - 1), KB_T(iu - 1, iu)));
                KB_T(iu, iu) = trk_add(KB_T(iu, iu), exshift);
                KB_T(iu - 1, iu - 1) = trk_add(KB_T(iu - 1, iu - 1), exshift);
                if (q >= 0.0) {
                    const double z = trk_sqrt(fabs(q));
                    const double gp = p >= 0.0 ? trk_add(p, z) : trk_sub(p, z), gq = KB_T(iu, iu - 1);
                    double c, s;                                                 // JacobiRotation::makeGivens(gp, gq)
                    if (gq == 0.0) { c = gp < 0.0 ? -1.0 : 1.0; s = 0.0; }
                    else if (gp == 0.0) { c = 0.0; s = gq < 0.0 ? 1.0 : -1.0; }
                    else if (fabs(gp) > fabs(gq)) {
                        const double t = trk_div(gq, gp);
                        double u = trk_sqrt(trk_add(1.0, trk_mul(t, t)));
                        if (gp < 0.0) u = -u;
                        c = trk_div(1.0, u); s = trk_mul(-t, c);
                    } else {
                        const double t = trk_div(gp, gq);
                        double u = trk_sqrt(trk_add(1.0, trk_mul(t, t)));
                        if (gq < 0.0) u = -u;
                        s = trk_div(-1.0, u); c = trk_mul(-t, s);
                    }
                    // rows iu-1, iu by rot.adjoint() on the left, then columns iu-1, iu by rot on the right: x' = c x - s y, y' = s x + c y
                    // (apply_rotation_in_the_plane), over the 2 x 2 block only -- its other rows and columns lie right of the next iu
                    UNROLL1 for (int j = iu - 1; j <= iu; j++) {
                        const double x = KB_T(iu - 1, j), y = KB_T(iu, j);
                        KB_T(iu - 1, j) = trk_add(trk_mul(c, x), trk_mul(-s, y));
                        KB_T(iu, j) = trk_add(trk_mul(s, x), trk_mul(c, y));
                    }
                    UNROLL1 for (int i = iu - 1; i <= iu; i++) {
                        const double x = KB_T(i, iu - 1), y = KB_T(i, iu);
                        KB_T(i, iu - 1) = trk_add(trk_mul(c, x), trk_mul(-s, y));
                        KB_T(i, iu) = trk_add(trk_mul(s, x), trk_mul(c, y));
                    }
                    KB_T(iu, iu - 1) = 0.0;
                }
                if (iu > 1) KB_T(iu - 1, iu - 2) = 0.0;
                iu -= 2; iter = 0;
            } else {                                                             // no convergence yet: computeShift
                double sx = KB_T(iu, iu), sy = KB_T(iu - 1, iu - 1), sw = trk_mul(KB_T(iu, iu - 1), KB_T(iu - 1, iu));
                if (iter == 10) {                                                // Wilkinson's ad hoc shift
                    exshift = trk_add(exshift, sx);
                    UNROLL1 for (int i = 0; i <= iu; i++) KB_T(i, i) = trk_sub(KB_T(i, i), sx);
                    const double s = trk_add(fabs(KB_T(iu, iu - 1)), fabs(KB_T(iu - 1, iu - 2)));
                    sx = trk_mul(0.75, s); sy = trk_mul(0.75, s); sw = trk_mul(trk_mul(-0.4375, s), s);
                }
                if (iter == 30) {                                                // MATLAB's ad hoc shift
                    double s = trk_div(trk_sub(sy, sx), 2.0);
                    s = trk_add(trk_mul(s, s), sw);
                    if (s > 0.0) {
                        s = trk_sqrt(s);
                        if (sy < sx) s = -s;
                        s = trk_add(s, trk_div(trk_sub(sy, sx), 2.0));
                        s = trk_sub(sx, trk_div(sw, s));
                        exshift = trk_add(exshift, s);
                        UNROLL1 for (int i = 0; i <= iu; i++) KB_T(i, i) = trk_sub(KB_T(i, i), s);
                        sx = sy = sw = 0.964;
                    }
                }
                iter++; total++;
                if (total > max_iters) break;
                double v[3] = {0.0, 0.0, 0.0};                                   // initFrancisQRStep
                int im;
                UNROLL1 for (im = iu - 2; im >= il; --im) {
                    const double tmm = KB_T(im, im), r = trk_sub(sx, tmm), s = trk_sub(sy, tmm);
                    v[0] = trk_add(trk_div(trk_sub(trk_mul(r, s), sw), KB_T(im + 1, im)), KB_T(im, im + 1));
                    v[1] = trk_sub(trk_sub(trk_sub(KB_T(im + 1, im + 1), tmm), r), s);
                    v[2] = KB_T(im + 2, im + 1);
                    if (im == il) break;
                    const double lhs = trk_mul(KB_T(im, im - 1), trk_add(fabs(v[1]), fabs(v[2])));
                    const double rhs = trk_mul(v[0], trk_add(trk_add(fabs(KB_T(im - 1, im - 1)), fabs(tmm)), fabs(KB_T(im + 1, im + 1))));
                    if (fabs(lhs) < trk_mul(eps, rhs)) break;
                }
                UNROLL1 for (int k = im; k <= iu - 2; ++k) {                             // performFrancisQRStep
                    const bool first = k == im;
                    double x[3], ess[2], tau, beta;
                    if (first) { x[0] = v[0]; x[1] = v[1]; x[2] = v[2]; }
                    else { x[0] = KB_T(k, k - 1); x[1] = KB_T(k + 1, k - 1); x[2] = KB_T(k + 2, k - 1); }
                    kb_householder(x, 3, ess, tau, beta);
                    if (beta != 0.0) {
                        if (first && k > il) KB_T(k, k - 1) = -KB_T(k, k - 1);
                        else if (!first) KB_T(k, k - 1) = beta;
                        if (tau != 0.0) {
                            const double te0 = trk_mul(tau, ess[0]), te1 = trk_mul(tau, ess[1]);
                            UNROLL1 for (int j = k; j <= iu; j++) {                      // applyHouseholderOnTheLeft, columns k..iu
                                const double tmp = trk_add(trk_add(trk_mul(ess[0], KB_T(k + 1, j)), trk_mul(ess[1], KB_T(k + 2, j))), KB_T(k, j));
                                KB_T(k, j) = trk_sub(KB_T(k, j), trk_mul(tau, tmp));
                                KB_T(k + 1, j) = trk_sub(KB_T(k + 1, j), trk_mul(tmp, te0));
                                KB_T(k + 2, j) = trk_sub(KB_T(k + 2, j), trk_mul(tmp, te1));
                            }
                            const int ie = iu < k + 3 ? iu : k + 3;
                            UNROLL1 for (int i = 0; i <= ie; i++) {                      // applyHouseholderOnTheRight, rows 0..min(iu, k + 3)
                                const double tmp = trk_add(trk_add(trk_mul(KB_T(i, k + 1), ess[0]), trk_mul(KB_T(i, k + 2), ess[1])), KB_T(i, k));
                                const double tt = trk_mul(tau, tmp);
                                KB_T(i, k) = trk_sub(KB_T(i, k), tt);
                                KB_T(i, k + 1) = trk_sub(KB_T(i, k + 1), trk_mul(tt, ess[0]));
                                KB_T(i, k + 2) = trk_sub(KB_T(i, k + 2), trk_mul(tt, ess[1]));
                            }
                        }
                    }
                }
                {
                    double x[2] = {KB_T(iu - 1, iu - 2), KB_T(iu, iu - 2)}, ess[2], tau, beta;
                    kb_householder(x, 2, ess, tau, beta);
                    if (beta != 0.0) {
                        KB_T(iu - 1, iu - 2) = beta;
                        if (tau != 0.0) {
                            const double te0 = trk_mul(tau, ess[0]);
                            UNROLL1 for (int j = iu - 1; j <= iu; j++) {
                                const double tmp = trk_add(trk_mul(ess[0], KB_T(iu, j)), KB_T(iu - 1, j));
                                KB_T(iu - 1, j) = trk_sub(KB_T(iu - 1, j), trk_mul(tau, tmp));
                                KB_T(iu, j) = trk_sub(KB_T(iu, j), trk_mul(tmp, te0));
                            }
                            UNROLL1 for (int i = 0; i <= iu; i++) {
                                const double tmp = trk_add(trk_mul(KB_T(i, iu), ess[0]), KB_T(i, iu - 1));
                                const double tt = trk_mul(tau, tmp);
                                KB_T(i, iu - 1) = trk_sub(KB_T(i, iu - 1), tt);
                                KB_T(i, iu) = trk_sub(KB_T(i, iu), trk_mul(tt, ess[0]));
                            }
                        }
                    }
                }
                UNROLL1 for (int i = im + 2; i <= iu; ++i) {                             // round-off pollution
                    KB_T(i, i - 2) = 0.0;
                    if (i > im + 2) KB_T(i, i - 3) = 0.0;
                }
            }
        }
    }
    if (total > max_iters) return;                                               // NoConvergence
    UNROLL1 for (int i = 0; i < n;) {                                                    // EigenSolver::compute, on T * scale
        const double sub = i == n - 1 ? 0.0 : trk_mul(KB_T(i + 1, i), scale);
        if (i == n - 1 || sub == 0.0) {
            wr[i] = trk_mul(KB_T(i, i), scale);
            if (!isfinite(wr[i])) return;
            i++;
        } else {
            const double a = trk_mul(KB_T(i, i), scale), d = trk_mul(KB_T(i + 1, i + 1), scale);
            const double p = trk_mul(0.5, trk_sub(a, d));
            double t0 = sub, t1 = trk_mul(KB_T(i, i + 1), scale);
            const double maxval = kb_maxi(fabs(p), kb_maxi(fabs(t0), fabs(t1)));
            t0 = trk_div(t0, maxval); t1 = trk_div(t1, maxval);
            const double p0 = trk_div(p, maxval);
            const double z = trk_mul(maxval, trk_sqrt(fabs(trk_add(trk_mul(p0, p0), trk_mul(t0, t1)))));
            wr[i] = trk_add(d, p); wi[i] = z; wr[i + 1] = wr[i]; wi[i + 1] = -z;
            if (!(isfinite(wr[i]) && isfinite(z))) return;
            i += 2;
        }
    }
}
#undef KB_T

// EquidistantCamera::backprojectSymmetric (EquidistantCamera.cc:716-818) of the normalised point (mx, my): theta is the smallest
// non-negative real root of theta + k2 theta^3 + k3 theta^5 + k4 theta^7 + k5 theta^9 = |p_u| (up to degree npow), taken from the
// eigenvalues of the companion matrix; |p_u| itself when none survives or npow == 1.  npow > 1 needs a non-zero coefficient at npow, which
// camera_model() (track_host.inl) guarantees.
VIWB_D void kb_backproject(const CamModel &c, double mx, double my, double &theta, double &phi) {
    const double norm = trk_sqrt(trk_add(trk_mul(mx, mx), trk_mul(my, my)));
    phi = norm < 1e-10 ? 0.0 : kb_atan2(my, mx);
    const int npow = kb_npow(c);
    if (npow == 1) { theta = norm; return; }
    double coeffs[10] = {-norm, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    if (npow >= 3) coeffs[3] = c.k1;
    if (npow >= 5) coeffs[5] = c.k2;
    if (npow >= 7) coeffs[7] = c.p1;
    if (npow >= 9) coeffs[9] = c.p2;
    double T[81], wr[9], wi[9];
    for (int j = 0; j < npow; j++) for (int i = 0; i < npow; i++) T[j * 9 + i] = (i == j + 1) ? 1.0 : 0.0;
    for (int i = 0; i < npow; i++) T[(npow - 1) * 9 + i] = trk_div(-coeffs[i], coeffs[npow]);     // A.col(npow-1) = -coeffs / coeffs(npow)
    kb_eigenvalues(T, npow, wr, wi);
    bool any = false;
    double best = 0.0;
    for (int i = 0; i < npow; i++) {                                             // std::min_element over the surviving roots, in order
        if (fabs(wi[i]) > 1e-10) continue;
        double t = wr[i];
        if (t < -1e-10) continue;
        else if (t < 0.0) t = 0.0;
        if (!any || t < best) best = t;
        any = true;
    }
    theta = any ? best : norm;
}
// EquidistantCamera::liftProjective (EquidistantCamera.cc:428-442; m_inv_K* of :271-274) followed by FeatureTracker::undistortedPts'
// b.x() / b.z(), b.y() / b.z() narrowed to cv::Point2f (feature_tracker.cpp:606-617).  A ray past 90 degrees (b.z() < 0) lifts to the
// mirrored point, as in the reference.
VIWB_D void kb_lift(const CamModel &c, float u, float v, float &x, float &y) {
    const double inv_K11 = trk_div(1.0, c.fx), inv_K13 = trk_div(-c.cx, c.fx), inv_K22 = trk_div(1.0, c.fy), inv_K23 = trk_div(-c.cy, c.fy);
    const double mx = trk_add(trk_mul(inv_K11, (double)u), inv_K13), my = trk_add(trk_mul(inv_K22, (double)v), inv_K23);
    double theta, phi;
    kb_backproject(c, mx, my, theta, phi);
    const double st = kb_sin(theta);
    const double px = trk_mul(st, kb_cos(phi)), py = trk_mul(st, kb_sin(phi)), pz = kb_cos(theta);
    x = (float)trk_div(px, pz); y = (float)trk_div(py, pz);
}
// EquidistantCamera::spaceToPlane (EquidistantCamera.cc:451-461, r() of EquidistantCamera.h:158-168 with its literal product order) narrowed
// to cv::Point2f (feature_tracker.cpp:730).  |P| = sqrt((x^2 + y^2) + z^2).
VIWB_D void kb_space_to_plane(const CamModel &c, const double *P, float &u, float &v) {
    const double norm = trk_sqrt(trk_add(trk_add(trk_mul(P[0], P[0]), trk_mul(P[1], P[1])), trk_mul(P[2], P[2])));
    const double theta = kb_acos(trk_div(P[2], norm)), phi = kb_atan2(P[1], P[0]);
    // r = theta + k2 theta theta theta + k3 theta^5 + ..., each product taken left to right
    const double k[4] = {c.k1, c.k2, c.p1, c.p2};
    double r = theta;
    for (int t = 0; t < 4; t++) {
        double m = k[t];
        for (int i = 0; i < 2 * t + 3; i++) m = trk_mul(m, theta);
        r = trk_add(r, m);
    }
    u = (float)trk_add(trk_mul(c.fx, trk_mul(r, kb_cos(phi))), c.cx); v = (float)trk_add(trk_mul(c.fy, trk_mul(r, kb_sin(phi))), c.cy);
}

// FeatureTracker::undistortedPts (featureTracker/feature_tracker.cpp:606-617) -> PinholeCamera::liftProjective with the recursive
// distortion model, n = 8 (camera_models/src/camera_models/PinholeCamera.cc:450-517, distortion :646-662), results narrowed to
// cv::Point2f, or mei_lift when model == CAM_MEI, kb_lift when model == CAM_KB; and FeatureTracker::ptsVelocity (:619-657) for points paired index-wise with the
// previous tick (SURVEY 8 f-1).
struct UndistArgs { int n; const float *pts, *prev_un; const unsigned char *has_prev; double fx, fy, cx, cy, k1, k2, p1, p2, dt; float *un, *vel; int model; double xi; };
VIWB_D void undistort_item(const UndistArgs &a, int i) {
    if (i >= a.n) return;
    float ux, uy;
    if (a.model == CAM_MEI) {
        const CamModel c = {a.model, a.fx, a.fy, a.cx, a.cy, a.k1, a.k2, a.p1, a.p2, a.xi};
        mei_lift(c, a.pts[2 * i], a.pts[2 * i + 1], ux, uy);
    } else if (a.model == CAM_KB) {
        const CamModel c = {a.model, a.fx, a.fy, a.cx, a.cy, a.k1, a.k2, a.p1, a.p2, a.xi};
        kb_lift(c, a.pts[2 * i], a.pts[2 * i + 1], ux, uy);
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
