/* vo_kb.c -- TEST INFRASTRUCTURE ONLY.  CPU restatement of camodocal's Kannala-Brandt camera (camodocal::EquidistantCamera) where
 * FeatureTracker calls a camera, for the checks of the library's Kannala-Brandt lift and projection:
 *
 *   EquidistantCamera::liftProjective      camera_models/src/camera_models/EquidistantCamera.cc:428-442, m_inv_K* :271-274
 *   EquidistantCamera::backprojectSymmetric                                                  :716-818
 *   EquidistantCamera::spaceToPlane                                                          :451-461, r() EquidistantCamera.h:158-168
 *
 * and of the eigen-solver backprojectSymmetric calls, Eigen 3.3's EigenSolver<MatrixXd>: RealSchur::compute (the matrix scaled by its largest
 * |a_ij|; HessenbergDecomposition, the identity on a matrix that is already upper Hessenberg as a companion matrix is; computeFromHessenberg
 * with findSmallSubdiagEntry's considerAsZero, computeShift's exceptional shifts at iterations 10 and 30, at most 40 n iterations,
 * initFrancisQRStep, performFrancisQRStep and splitOffTwoRows) and EigenSolver::compute's extraction of the eigenvalues from the real Schur
 * form (the 2 x 2 formula scaled by max(|p|, |t0|, |t1|)).  Only the leading (iu + 1) x (iu + 1) block is transformed: the columns right of
 * iu hold converged blocks that no later step and no extraction reads (Eigen transforms them for the Schur vectors).  Where Eigen leaves the
 * eigenvalues unset (no convergence; after the first non-finite one) they are 0 here.  Operation by operation as the library's kb_* device
 * functions (viw-fusion_b200/csrc/kernels_feat.cuh) run them; built with -ffp-contract=off (oracle/kb.mk) so no product is fused, and the
 * trigonometric functions are glibc's.  The same eigen-solver stands in for Eigen's in oracle/refshim/kb_shim.h, where the reference's
 * own EquidistantCamera.cc is compiled.
 *
 * A camera is double cam[8] = k2 k3 k4 k5 mu mv u0 v0 (EquidistantCamera::Parameters' order). */
#include <math.h>
#include <float.h>
#include <stdint.h>

#define T_(i, j) T[(j) * 9 + (i)]

static double maxi(double a, double b) { return a < b ? b : a; }

static void householder(const double *x, int m, double *ess, double *tau, double *beta) {
    const double tail = m == 3 ? x[1] * x[1] + x[2] * x[2] : x[1] * x[1];
    const double c0 = x[0];
    if (tail <= DBL_MIN) { *tau = 0.0; *beta = c0; ess[0] = 0.0; ess[1] = 0.0; return; }
    *beta = sqrt(c0 * c0 + tail);
    if (c0 >= 0.0) *beta = -*beta;
    const double d = c0 - *beta;
    ess[0] = x[1] / d; ess[1] = m == 3 ? x[2] / d : 0.0;
    *tau = (*beta - c0) / *beta;
}

/* eigenvalues of the n x n matrix A (column-major, leading dimension n, upper Hessenberg, n <= 9) as EigenSolver<MatrixXd>(A).eigenvalues();
 * returns 0 on convergence, 1 where RealSchur gives up (eigenvalues 0), 2 where a non-finite eigenvalue stopped the extraction */
int vo_kb_eigenvalues(const double *A, int n, double *wr, double *wi) {
    const double eps = DBL_EPSILON;
    double T[81];
    for (int i = 0; i < n; i++) { wr[i] = 0.0; wi[i] = 0.0; }
    if (n < 1 || n > 9) return 1;
    double scale = 0.0;
    for (int j = 0; j < n; j++) for (int i = 0; i < n; i++) scale = maxi(scale, fabs(A[j * n + i]));
    if (scale < DBL_MIN) return 0;
    for (int j = 0; j < n; j++) for (int i = 0; i < n; i++) T_(i, j) = A[j * n + i] / scale;
    double norm = 0.0;
    for (int j = 0; j < n; j++) {
        double s = 0.0;
        for (int i = 0; i < n && i <= j + 1; i++) s = s + fabs(T_(i, j));
        norm = norm + s;
    }
    const double zero = maxi(norm * (eps * eps), DBL_MIN);
    int iu = n - 1, iter = 0, total = 0;
    const int max_iters = 40 * n;
    double exshift = 0.0;
    if (norm != 0.0) {
        while (iu >= 0) {
            int il = iu;
            while (il > 0) {
                const double s = maxi((fabs(T_(il - 1, il - 1)) + fabs(T_(il, il))) * eps, zero);
                if (fabs(T_(il, il - 1)) <= s) break;
                il--;
            }
            if (il == iu) {
                T_(iu, iu) = T_(iu, iu) + exshift;
                if (iu > 0) T_(iu, iu - 1) = 0.0;
                iu--; iter = 0;
            } else if (il == iu - 1) {
                const double p = 0.5 * (T_(iu - 1, iu - 1) - T_(iu, iu));
                const double q = p * p + T_(iu, iu - 1) * T_(iu - 1, iu);
                T_(iu, iu) = T_(iu, iu) + exshift;
                T_(iu - 1, iu - 1) = T_(iu - 1, iu - 1) + exshift;
                if (q >= 0.0) {
                    const double z = sqrt(fabs(q));
                    const double gp = p >= 0.0 ? p + z : p - z, gq = T_(iu, iu - 1);
                    double c, s;
                    if (gq == 0.0) { c = gp < 0.0 ? -1.0 : 1.0; s = 0.0; }
                    else if (gp == 0.0) { c = 0.0; s = gq < 0.0 ? 1.0 : -1.0; }
                    else if (fabs(gp) > fabs(gq)) {
                        const double t = gq / gp;
                        double u = sqrt(1.0 + t * t);
                        if (gp < 0.0) u = -u;
                        c = 1.0 / u; s = -t * c;
                    } else {
                        const double t = gp / gq;
                        double u = sqrt(1.0 + t * t);
                        if (gq < 0.0) u = -u;
                        s = -1.0 / u; c = -t * s;
                    }
                    for (int j = iu - 1; j <= iu; j++) {
                        const double x = T_(iu - 1, j), y = T_(iu, j);
                        T_(iu - 1, j) = c * x + (-s) * y;
                        T_(iu, j) = s * x + c * y;
                    }
                    for (int i = iu - 1; i <= iu; i++) {
                        const double x = T_(i, iu - 1), y = T_(i, iu);
                        T_(i, iu - 1) = c * x + (-s) * y;
                        T_(i, iu) = s * x + c * y;
                    }
                    T_(iu, iu - 1) = 0.0;
                }
                if (iu > 1) T_(iu - 1, iu - 2) = 0.0;
                iu -= 2; iter = 0;
            } else {
                double sx = T_(iu, iu), sy = T_(iu - 1, iu - 1), sw = T_(iu, iu - 1) * T_(iu - 1, iu);
                if (iter == 10) {
                    exshift = exshift + sx;
                    for (int i = 0; i <= iu; i++) T_(i, i) = T_(i, i) - sx;
                    const double s = fabs(T_(iu, iu - 1)) + fabs(T_(iu - 1, iu - 2));
                    sx = 0.75 * s; sy = 0.75 * s; sw = (-0.4375 * s) * s;
                }
                if (iter == 30) {
                    double s = (sy - sx) / 2.0;
                    s = s * s + sw;
                    if (s > 0.0) {
                        s = sqrt(s);
                        if (sy < sx) s = -s;
                        s = s + (sy - sx) / 2.0;
                        s = sx - sw / s;
                        exshift = exshift + s;
                        for (int i = 0; i <= iu; i++) T_(i, i) = T_(i, i) - s;
                        sx = sy = sw = 0.964;
                    }
                }
                iter++; total++;
                if (total > max_iters) break;
                double v[3] = {0.0, 0.0, 0.0};
                int im;
                for (im = iu - 2; im >= il; --im) {
                    const double tmm = T_(im, im), r = sx - tmm, s = sy - tmm;
                    v[0] = (r * s - sw) / T_(im + 1, im) + T_(im, im + 1);
                    v[1] = ((T_(im + 1, im + 1) - tmm) - r) - s;
                    v[2] = T_(im + 2, im + 1);
                    if (im == il) break;
                    const double lhs = T_(im, im - 1) * (fabs(v[1]) + fabs(v[2]));
                    const double rhs = v[0] * ((fabs(T_(im - 1, im - 1)) + fabs(tmm)) + fabs(T_(im + 1, im + 1)));
                    if (fabs(lhs) < eps * rhs) break;
                }
                for (int k = im; k <= iu - 2; ++k) {
                    const int first = k == im;
                    double x[3], ess[2], tau, beta;
                    if (first) { x[0] = v[0]; x[1] = v[1]; x[2] = v[2]; }
                    else { x[0] = T_(k, k - 1); x[1] = T_(k + 1, k - 1); x[2] = T_(k + 2, k - 1); }
                    householder(x, 3, ess, &tau, &beta);
                    if (beta != 0.0) {
                        if (first && k > il) T_(k, k - 1) = -T_(k, k - 1);
                        else if (!first) T_(k, k - 1) = beta;
                        if (tau != 0.0) {
                            const double te0 = tau * ess[0], te1 = tau * ess[1];
                            for (int j = k; j <= iu; j++) {
                                const double tmp = (ess[0] * T_(k + 1, j) + ess[1] * T_(k + 2, j)) + T_(k, j);
                                T_(k, j) = T_(k, j) - tau * tmp;
                                T_(k + 1, j) = T_(k + 1, j) - tmp * te0;
                                T_(k + 2, j) = T_(k + 2, j) - tmp * te1;
                            }
                            const int ie = iu < k + 3 ? iu : k + 3;
                            for (int i = 0; i <= ie; i++) {
                                const double tmp = (T_(i, k + 1) * ess[0] + T_(i, k + 2) * ess[1]) + T_(i, k);
                                const double tt = tau * tmp;
                                T_(i, k) = T_(i, k) - tt;
                                T_(i, k + 1) = T_(i, k + 1) - tt * ess[0];
                                T_(i, k + 2) = T_(i, k + 2) - tt * ess[1];
                            }
                        }
                    }
                }
                {
                    double x[2] = {T_(iu - 1, iu - 2), T_(iu, iu - 2)}, ess[2], tau, beta;
                    householder(x, 2, ess, &tau, &beta);
                    if (beta != 0.0) {
                        T_(iu - 1, iu - 2) = beta;
                        if (tau != 0.0) {
                            const double te0 = tau * ess[0];
                            for (int j = iu - 1; j <= iu; j++) {
                                const double tmp = ess[0] * T_(iu, j) + T_(iu - 1, j);
                                T_(iu - 1, j) = T_(iu - 1, j) - tau * tmp;
                                T_(iu, j) = T_(iu, j) - tmp * te0;
                            }
                            for (int i = 0; i <= iu; i++) {
                                const double tmp = T_(i, iu) * ess[0] + T_(i, iu - 1);
                                const double tt = tau * tmp;
                                T_(i, iu - 1) = T_(i, iu - 1) - tt;
                                T_(i, iu) = T_(i, iu) - tt * ess[0];
                            }
                        }
                    }
                }
                for (int i = im + 2; i <= iu; ++i) {
                    T_(i, i - 2) = 0.0;
                    if (i > im + 2) T_(i, i - 3) = 0.0;
                }
            }
        }
    }
    if (total > max_iters) return 1;
    for (int i = 0; i < n;) {
        const double sub = i == n - 1 ? 0.0 : T_(i + 1, i) * scale;
        if (i == n - 1 || sub == 0.0) {
            wr[i] = T_(i, i) * scale;
            if (!isfinite(wr[i])) return 2;
            i++;
        } else {
            const double a = T_(i, i) * scale, d = T_(i + 1, i + 1) * scale;
            const double p = 0.5 * (a - d);
            double t0 = sub, t1 = T_(i, i + 1) * scale;
            const double maxval = maxi(fabs(p), maxi(fabs(t0), fabs(t1)));
            t0 = t0 / maxval; t1 = t1 / maxval;
            const double p0 = p / maxval;
            const double z = maxval * sqrt(fabs(p0 * p0 + t0 * t1));
            wr[i] = d + p; wi[i] = z; wr[i + 1] = wr[i]; wi[i + 1] = -z;
            if (!(isfinite(wr[i]) && isfinite(z))) return 2;
            i += 2;
        }
    }
    return 0;
}

/* npow of backprojectSymmetric (:731-747): 9, less 2 for every zero k_i wherever it sits */
int vo_kb_npow(const double *cam) {
    int npow = 9;
    if (cam[3] == 0.0) npow -= 2;
    if (cam[2] == 0.0) npow -= 2;
    if (cam[1] == 0.0) npow -= 2;
    if (cam[0] == 0.0) npow -= 2;
    return npow;
}

/* the companion matrix backprojectSymmetric builds for |p_u| = norm (:749-782), column-major n x n into A; returns n = npow (no matrix
 * when npow == 1) */
int vo_kb_companion(const double *cam, double norm, double *A) {
    const int npow = vo_kb_npow(cam);
    double coeffs[10] = {-norm, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    if (npow >= 3) coeffs[3] = cam[0];
    if (npow >= 5) coeffs[5] = cam[1];
    if (npow >= 7) coeffs[7] = cam[2];
    if (npow >= 9) coeffs[9] = cam[3];
    if (npow == 1) return 1;
    for (int j = 0; j < npow; j++) for (int i = 0; i < npow; i++) A[j * npow + i] = (i == j + 1) ? 1.0 : 0.0;
    for (int i = 0; i < npow; i++) A[(npow - 1) * npow + i] = -coeffs[i] / coeffs[npow];
    return npow;
}

/* backprojectSymmetric of the normalised point (mx, my) */
static void backproject(const double *cam, double mx, double my, double *theta, double *phi) {
    const double norm = sqrt(mx * mx + my * my);
    *phi = norm < 1e-10 ? 0.0 : atan2(my, mx);
    double A[81], wr[9], wi[9];
    const int npow = vo_kb_companion(cam, norm, A);
    if (npow == 1) { *theta = norm; return; }
    vo_kb_eigenvalues(A, npow, wr, wi);
    int any = 0;
    double best = 0.0;
    for (int i = 0; i < npow; i++) {
        if (fabs(wi[i]) > 1e-10) continue;
        double t = wr[i];
        if (t < -1e-10) continue;
        else if (t < 0.0) t = 0.0;
        if (!any || t < best) best = t;
        any = 1;
    }
    *theta = any ? best : norm;
}

/* FeatureTracker::undistortedPts with an EquidistantCamera: pixels pts[n][2] -> un[n][2] = (b.x() / b.z(), b.y() / b.z()) narrowed to
 * float; theta[n] (optional): backprojectSymmetric's theta */
void vo_kb_lift(const double *cam, int n, const float *pts, float *un, double *theta_out) {
    const double inv_K11 = 1.0 / cam[4], inv_K13 = -cam[6] / cam[4], inv_K22 = 1.0 / cam[5], inv_K23 = -cam[7] / cam[5];
    for (int k = 0; k < n; k++) {
        const double mx = inv_K11 * (double)pts[2 * k] + inv_K13, my = inv_K22 * (double)pts[2 * k + 1] + inv_K23;
        double theta, phi;
        backproject(cam, mx, my, &theta, &phi);
        const double st = sin(theta);
        const double px = st * cos(phi), py = st * sin(phi), pz = cos(theta);
        un[2 * k] = (float)(px / pz); un[2 * k + 1] = (float)(py / pz);
        if (theta_out) theta_out[k] = theta;
    }
}

/* EquidistantCamera::spaceToPlane: P[n][3] -> uv[n][2] in double (|P| = sqrt((x^2 + y^2) + z^2)) */
void vo_kb_space_to_plane(const double *cam, int n, const double *P, double *uv) {
    for (int k = 0; k < n; k++) {
        const double *p = P + 3 * k;
        const double norm = sqrt((p[0] * p[0] + p[1] * p[1]) + p[2] * p[2]);
        const double theta = acos(p[2] / norm), phi = atan2(p[1], p[0]);
        double r = theta;
        for (int t = 0; t < 4; t++) {
            double m = cam[t];
            for (int i = 0; i < 2 * t + 3; i++) m = m * theta;
            r = r + m;
        }
        uv[2 * k] = cam[4] * (r * cos(phi)) + cam[6];
        uv[2 * k + 1] = cam[5] * (r * sin(phi)) + cam[7];
    }
}
