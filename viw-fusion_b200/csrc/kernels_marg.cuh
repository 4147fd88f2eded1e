// kernels_marg.cuh -- gauge re-anchoring and marginalisation, one block per window.
//
//   reanchor : Estimator::double2vector + vector2double (estimator.cpp:1224-1332, 1155-1222)
//   marg     : MarginalizationInfo::marginalize + getParameterBlocks (marginalization_factor.cpp:183-334) on the
//              dense system assembled by assemble_block(MODE_MARG) from the same Jacobian kernels the solver uses.
// The dropped landmark block is diagonal, so it is eliminated exactly (Schur sum T0 = sum w w^T / a); the remaining
// dropped block (pose 0 + speed-bias 0, or pose 9) goes through the reference's eigen pseudo-inverse (eps 1e-8),
// and the kept n x n system through tred2 / tql2 in shared memory (stands in for Eigen::SelfAdjointEigenSolver) to produce
// J_lin = sqrt(S) V^T, r_lin = sqrt(S^-1) V^T b.  Two kernels: marg_prep (assembly over the compact kept | dropped dimensions in shared
// memory, all block-parallel) and marg_eig (the eigen-decomposition, three windows per SM).
#pragma once
#include "kernels_lin.cuh"
#include "kernels_solve.cuh"

namespace viwb {

VIWB_D void reanchor_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by; (void)smem; (void)mode; (void)nt;
    if (tid != 0) return;
    const WinMeta &m = bd.meta[bx];
    double *st = bd.x_cur + m.state_off;
    const double *before = bd.x_before + m.state_off;
    const bool use_imu = (m.flags[BLK_SB0] & 1u) != 0;
    const int nfr = m.frame_count + 1;
    if (use_imu) {
        const M3 Rs0 = qR(ldq(before + 3)), R00 = qR(ldq(st + 3));
        const V3 o0 = R_to_ypr(Rs0), o00 = R_to_ypr(R00), P0 = ld3(before), p00 = ld3(st);
        M3 rot = yaw_to_R(o0.x - o00.x);
        if (fabs(fabs(o0.y) - 90) < 1.0 || fabs(fabs(o00.y) - 90) < 1.0) rot = Rs0 * transpose(R00);
        for (int i = 0; i < nfr; i++) {
            double *p = st + 7 * i;
            const M3 Ri = rot * qR(qnormalized(ldq(p + 3)));
            const V3 Pi = rot * (ld3(p) - p00) + P0;
            st3(p, Pi); stq(p + 3, q_from_R(Ri));
            st3(st + 77 + 9 * i, rot * ld3(st + 77 + 9 * i));
        }
        for (int c = 0; c < 2; c++) if (m.flags[BLK_EX0 + c] & 1u) { double *e = st + blk_off(BLK_EX0 + c); stq(e + 3, q_from_R(qR(qnormalized(ldq(e + 3))))); }
    } else {
        for (int i = 0; i < nfr; i++) { double *p = st + 7 * i; stq(p + 3, q_from_R(qR(qnormalized(ldq(p + 3))))); }
    }
    if (m.flags[BLK_EXW] & 1u) {
        double *e = st + blk_off(BLK_EXW);
        stq(e + 3, q_from_R(qR(qnormalized(ldq(e + 3)))));
        if (m.flags[BLK_PR] & 1u) for (int k = 0; k < 4; k++) st[blk_off(BLK_PR) + k] = e[3 + k];   // quirk 1 (estimator.cpp:1209-1213)
    }
    for (int k = 0; k < m.nlm; k++) st[SFIX + k] = 1.0 / (1.0 / st[SFIX + k]);   // setDepth(1/x), getDepthVector(1/depth)
}

// The implicit QL iteration (EISPACK tql2) with eigenvector accumulation, in shared memory: the second half of the eigen-decomposition that stands
// in for Eigen::SelfAdjointEigenSolver, after tridiag_block.  The O(n) scalar recurrence runs on thread 0, the rotation of V's rows is spread over
// the block.  In: V = Q of the tridiagonalisation (n x n, leading dimension ld), d (n) its diagonal, e (n) its sub-diagonal (e[n-1] = 0).
// Out: V = eigenvectors in columns, d = eigenvalues (unsorted).  cs (2n), sc (8): scratch.
VIWB_D void tql2_block(double *V, double *d, double *e, double *cs, double *sc, int n, int ld, int tid, int nt) {
#define VV(i, j) V[(i) * ld + (j)]
    if (tid == 0) { sc[1] = 0.0 /* f */; sc[2] = 0.0 /* tst1 */; }
    VIWB_SYNC();
    const double eps = 2.220446049250313e-16;
    for (int l = 0; l < n; l++) {
        if (tid == 0) {
            const double t = fabs(d[l]) + fabs(e[l]); if (t > sc[2]) sc[2] = t;
            int m = l; while (m < n) { if (fabs(e[m]) <= eps * sc[2]) break; m++; }
            sc[3] = (double)m;
        }
        VIWB_SYNC();
        const int m = (int)sc[3];
        if (m > l) {
            for (int iter = 0; iter < 200; iter++) {
                if (tid == 0) {
                    double g = d[l], p = (d[l + 1] - g) / (2.0 * e[l]), r = sqrt(p * p + 1.0);
                    if (p < 0) r = -r;
                    d[l] = e[l] / (p + r); d[l + 1] = e[l] * (p + r);
                    const double dl1 = d[l + 1]; double h = g - d[l];
                    for (int i = l + 2; i < n; i++) d[i] -= h;
                    sc[1] += h;
                    p = d[m];
                    double c = 1.0, c2 = c, c3 = c, s = 0.0, s2 = 0.0; const double el1 = e[l + 1];
                    // the rotation chain is the serial critical path of the whole decomposition: operands of the next link are
                    // fetched before the current link's sqrt / reciprocal, and one reciprocal replaces two divisions
                    double ei = e[m - 1], di = d[m - 1];
                    for (int i = m - 1; i >= l; i--) {
                        const double ein = i > l ? e[i - 1] : 0.0, din = i > l ? d[i - 1] : 0.0;
                        c3 = c2; c2 = c; s2 = s;
                        g = c * ei; h = c * p;
                        const double q2 = p * p + ei * ei, rinv = q2 > 0.0 ? rsqrt(q2) : 0.0;      // r = q2 * rsqrt(q2): one special-function chain, no division
                        r = q2 * rinv;
                        e[i + 1] = s * r; s = ei * rinv; c = p * rinv;
                        p = c * di - s * g; d[i + 1] = h + s * (c * g + s * di);
                        cs[2 * i] = c; cs[2 * i + 1] = s;
                        ei = ein; di = din;
                    }
                    p = -s * s2 * c3 * el1 * e[l] / dl1;
                    e[l] = s * p; d[l] = c * p;
                    sc[4] = (fabs(e[l]) > eps * sc[2]) ? 1.0 : 0.0;
                }
                VIWB_SYNC();
                for (int k = tid; k < n; k += nt)
                    for (int i = m - 1; i >= l; i--) { const double c = cs[2 * i], s = cs[2 * i + 1], h = VV(k, i + 1); VV(k, i + 1) = s * VV(k, i) + c * h; VV(k, i) = c * VV(k, i) - s * h; }
                VIWB_SYNC();
                if (sc[4] == 0.0) break;
                VIWB_SYNC();
            }
        }
        if (tid == 0) { d[l] = d[l] + sc[1]; e[l] = 0.0; }
        VIWB_SYNC();
    }
#undef VV
}

// Householder tridiagonalisation + accumulation of the transformations (EISPACK tred2, the first half before tql2_block; outputs: V = Q, d = diagonal,
// e[0 .. n-2] = sub-diagonal, e[n-1] = 0), organised for the block instead of statement by statement.  The first version spent 59 % of its warp samples at
// barriers (profiles/r02m_marg_tri_kernel.ncu.txt): 15 barriers per column with one thread per row walking up to n elements while the others waited.  Here
//   * the scale, the squared norm and d[i-1] come out of ONE three-way reduction (h = sum d^2 / scale^2 instead of a second pass over d / scale),
//   * the product A d, the dot product e . d and the rank-2 update use T lanes per row (T = 1, 2, 4, 8 as the shrinking column count frees threads;
//     partial sums over interleaved columns, combined by shuffles), the scratch vector e is formed on the fly in the update,
//   * the accumulation runs T lanes per column and merges its zeroing / scaling phases: 7 + 2 barriers per column instead of 11 + 4.
// Summation orders differ from EISPACK's at rounding level; red: 3 * 32 doubles.
VIWB_D void tridiag_block(double *V, double *d, double *e, double *cs, double *red, int n, int ld, int tid, int nt) {
#define VV(i, j) V[(i) * ld + (j)]
    for (int j = tid; j < n; j += nt) d[j] = VV(n - 1, j);
    VIWB_SYNC();
    for (int i = n - 1; i > 0; i--) {
        int T = 1;
#ifndef VIWB_HOST_EMU
        while (T < 8 && 2 * T * i <= nt) T *= 2;
#endif
        const int rpp = nt / T > 0 ? nt / T : 1, row0 = tid / T, p = tid % T;       // rows per pass, this thread's row within a pass and its lane in the row
        double v3[3] = {0.0, 0.0, 0.0};
        for (int k = tid; k < i; k += nt) { const double x = d[k]; v3[0] += fabs(x); v3[1] += x * x; if (k == i - 1) v3[2] = x; }
        block_sum_n<3>(v3, tid, nt, red);
        const double scale = v3[0];
        if (scale == 0.0) {
            if (tid == 0) e[i] = d[i - 1];
            VIWB_SYNC();
            for (int j = tid; j < i; j += nt) { d[j] = VV(i - 1, j); VV(i, j) = 0.0; VV(j, i) = 0.0; }
            if (tid == 0) d[i] = 0.0;
            VIWB_SYNC();
            continue;
        }
        const double f = v3[2] / scale;
        double g = sqrt(v3[1] / (scale * scale)); if (f > 0) g = -g;
        const double h = v3[1] / (scale * scale) - f * g;
        for (int k = tid; k < i; k += nt) d[k] = (k == i - 1) ? f - g : d[k] / scale;
        if (tid == 0) e[i] = scale * g;
        VIWB_SYNC();
        // cs[j] = (A d)[j] / h over the leading i x i block (lower triangle storage); column i keeps the Householder vector
        double part = 0.0;
        for (int j0 = 0; j0 < i; j0 += rpp) {
            const int j = j0 + row0;
            double a = 0.0;
            if (j < i) {
                int k = p;
                for (; k <= j; k += T) a += VV(j, k) * d[k];
                for (; k < i; k += T) a += VV(k, j) * d[k];
            }
#ifndef VIWB_HOST_EMU
            for (int o = 1; o < T; o <<= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
#endif
            if (j < i && p == 0) { const double c = a / h; cs[j] = c; VV(j, i) = d[j]; part += c * d[j]; }
        }
        const double f2 = block_sum(part, tid, nt, red);
        const double hh = f2 / (h + h);
        // rank-2 update of the lower triangle with e[j] = cs[j] - hh d[j] formed on the fly: V[k][j] -= d[j] e[k] + e[j] d[k],  j <= k < i
        for (int k0 = 0; k0 < i; k0 += rpp) {
            const int k = k0 + row0;
            if (k < i) {
                // batches of four: all loads of a batch are issued before its stores (the compiler cannot move a load of d / cs across a store to V on its own)
                const double dk = d[k], ek = cs[k] - hh * dk;
                double *row = &VV(k, 0);
                int j = p;
                for (; j + 3 * T <= k; j += 4 * T) {
                    const double v0 = row[j], v1 = row[j + T], v2 = row[j + 2 * T], v3 = row[j + 3 * T];
                    const double d0 = d[j], d1 = d[j + T], d2 = d[j + 2 * T], d3 = d[j + 3 * T];
                    const double c0 = cs[j], c1 = cs[j + T], c2 = cs[j + 2 * T], c3 = cs[j + 3 * T];
                    row[j] = v0 - (d0 * ek + (c0 - hh * d0) * dk); row[j + T] = v1 - (d1 * ek + (c1 - hh * d1) * dk);
                    row[j + 2 * T] = v2 - (d2 * ek + (c2 - hh * d2) * dk); row[j + 3 * T] = v3 - (d3 * ek + (c3 - hh * d3) * dk);
                }
                for (; j <= k; j += T) row[j] -= d[j] * ek + (cs[j] - hh * d[j]) * dk;
            }
        }
        VIWB_SYNC();
        for (int j = tid; j < i; j += nt) { d[j] = VV(i - 1, j); VV(i, j) = 0.0; }
        if (tid == 0) d[i] = h;
        VIWB_SYNC();
    }
    // ---- accumulate the transformations
    for (int i = 0; i < n - 1; i++) {
        int T = 1;
#ifndef VIWB_HOST_EMU
        while (T < 8 && 2 * T * (i + 1) <= nt) T *= 2;
#endif
        const int cpp = nt / T > 0 ? nt / T : 1, col0 = tid / T, p = tid % T;
        const double h = d[i + 1];
        if (i > 0) for (int k = tid; k < i; k += nt) VV(k, i) = 0.0;          // the previous column's Householder vector has done its work
        if (tid == 0) { VV(n - 1, i) = VV(i, i); VV(i, i) = 1.0; }
        if (h != 0.0) for (int k = tid; k <= i; k += nt) d[k] = VV(k, i + 1) / h;
        VIWB_SYNC();
        if (h != 0.0) {
            for (int j0 = 0; j0 <= i; j0 += cpp) {
                const int j = j0 + col0;
                double a = 0.0;
                if (j <= i) for (int k = p; k <= i; k += T) a += VV(k, i + 1) * VV(k, j);
#ifndef VIWB_HOST_EMU
                for (int o = 1; o < T; o <<= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
#endif
                if (j <= i) {
                    int k = p;
                    for (; k + 3 * T <= i; k += 4 * T) {
                        const double v0 = VV(k, j), v1 = VV(k + T, j), v2 = VV(k + 2 * T, j), v3 = VV(k + 3 * T, j);
                        const double d0 = d[k], d1 = d[k + T], d2 = d[k + 2 * T], d3 = d[k + 3 * T];
                        VV(k, j) = v0 - a * d0; VV(k + T, j) = v1 - a * d1; VV(k + 2 * T, j) = v2 - a * d2; VV(k + 3 * T, j) = v3 - a * d3;
                    }
                    for (; k <= i; k += T) VV(k, j) -= a * d[k];
                }
            }
        }
        VIWB_SYNC();
    }
    for (int k = tid; k < n - 1; k += nt) VV(k, n - 1) = 0.0;
    VIWB_SYNC();
    for (int j = tid; j < n; j += nt) { d[j] = VV(n - 1, j); VV(n - 1, j) = 0.0; }
    VIWB_SYNC();
    if (tid == 0) VV(n - 1, n - 1) = 1.0;
    // sub-diagonal: e[i] <- e[i + 1], e[n - 1] = 0
    for (int i = 1 + tid; i < n; i += nt) cs[i - 1] = e[i];
    VIWB_SYNC();
    for (int i = tid; i < n - 1; i += nt) e[i] = cs[i];
    if (tid == 0) e[n - 1] = 0.0;
    VIWB_SYNC();
#undef VV
}

// Symmetric eigen-decomposition in shared memory by the parallel cyclic Jacobi method (stands in for Eigen::SelfAdjointEigenSolver,
// marginalization_factor.cpp:282,294): every round rotates n/2 disjoint index pairs (round-robin tournament order, n - 1 rounds per
// sweep), so the whole block works on every round -- no serial QL rotation chain.  Per round: (1) one thread per pair computes its
// rotation from a_pp, a_qq, a_pq; (2) every 2x2 block (pair P x pair Q, P <= Q) of A' = J^T A J is computed by ONE thread from the same
// 2x2 block of A (rows and columns rotate together, so the update is in place without an intermediate copy) and mirrored, and every
// (row, pair) item of V' = V J likewise.  Two barriers per round; fixed order, deterministic.  Sweeps stop when the off-diagonal
// Frobenius norm is below 1e-14 of the diagonal's (or after 16 sweeps).
// A (n x n, leading dimension lda): in = symmetric matrix (both triangles), out = diagonal holds the eigenvalues.  V (n x n, ldv): out =
// eigenvectors in columns.  d (n): eigenvalues (unsorted).  rot: 4 * ((n + 1) / 2) doubles of scratch; red: 32 doubles.
VIWB_HD void jacobi_pair(int m, int r, int k, int &p, int &q) {      // pair k of round r among m (even) players
    if (k == 0) { p = m - 1; q = r; }
    else { p = (r + k) % (m - 1); q = (r - k + (m - 1)) % (m - 1); }
}
// WARP = true: called by ONE warp (tid < 32, nt = 32) while the rest of the block waits at the caller's barrier, the 2 x 14 synchronisations of a sweep being
// warp-level then.  Measured slower for the 15 x 15 block of marg_prep (156 items per round on 32 lanes instead of 256 threads); kept as the measured alternative.
template <bool WARP>
VIWB_D void sym_eig_jacobi(double *A, int lda, double *V, int ldv, double *d, double *rot, double *red, int n, int tid, int nt) {
#define JSYNC() do { if (WARP) VIWB_SYNCWARP(); else VIWB_SYNC(); } while (0)
    for (int e = tid; e < n * n; e += nt) { const int i = e / n, j = e - i * n; V[i * ldv + j] = (i == j) ? 1.0 : 0.0; }
    JSYNC();
    if (n == 1) { if (tid == 0) d[0] = A[0]; JSYNC(); return; }
    const int m = n + (n & 1), np = m / 2;      // an odd n gets a bye: pairs with the phantom index m - 1 do not rotate
    for (int sweep = 0; sweep < 16; sweep++) {
        // convergence test: off(A)^2 <= (1e-15)^2 * diag(A)^2
        double off = 0.0, dg = 0.0;
        for (int e = tid; e < n * n; e += nt) { const int i = e / n, j = e - i * n; const double v = A[i * lda + j]; if (i == j) dg += v * v; else off += v * v; }
        if (WARP) {
#ifndef VIWB_HOST_EMU
            for (int o = 16; o > 0; o >>= 1) { off += __shfl_xor_sync(0xffffffffu, off, o); dg += __shfl_xor_sync(0xffffffffu, dg, o); }
#endif
        } else { double v2[2] = {off, dg}; block_sum_n<2>(v2, tid, nt, red); off = v2[0]; dg = v2[1]; }
        if (off <= 1e-28 * dg || off == 0.0) break;
        for (int r = 0; r < m - 1; r++) {
            for (int k = tid; k < np; k += nt) {
                int p, q; jacobi_pair(m, r, k, p, q);
                double c = 1.0, sn = 0.0;
                if (p < n && q < n) {
                    const double apq = A[p * lda + q];
                    if (apq != 0.0) {
                        const double app = A[p * lda + p], aqq = A[q * lda + q];
                        const double tau = (aqq - app) / (2.0 * apq);
                        const double t = (tau >= 0.0 ? 1.0 : -1.0) / (fabs(tau) + sqrt(1.0 + tau * tau));
                        if (isfinite(t)) { c = 1.0 / sqrt(1.0 + t * t); sn = t * c; }      // |tau| overflowing: the element is negligible, no rotation
                    }
                }
                rot[4 * k] = c; rot[4 * k + 1] = sn; rot[4 * k + 2] = (double)p; rot[4 * k + 3] = (double)q;
            }
            JSYNC();
            const int nblk = np * (np + 1) / 2, nv = n * np;
            for (int e = tid; e < nblk + nv; e += nt) {
                if (e < nblk) {
                    int P, Q; sym_unrank(e, Q, P);          // P <= Q
                    const int p0 = (int)rot[4 * P + 2], p1 = (int)rot[4 * P + 3], q0 = (int)rot[4 * Q + 2], q1 = (int)rot[4 * Q + 3];
                    if (p0 >= n || p1 >= n || q0 >= n || q1 >= n) {
                        // a pair with the phantom index: its real member keeps its row / column, which still rotates with the other pair
                        const int pr = p0 < n ? p0 : p1, qr = q0 < n ? q0 : q1;
                        if (P == Q) continue;
                        if (pr >= n || qr >= n) continue;
                        if (p0 < n && p1 < n) {            // P rotates, Q is the bye: column qr, rows p0 / p1
                            const double c = rot[4 * P], s = rot[4 * P + 1], b0 = A[p0 * lda + qr], b1 = A[p1 * lda + qr];
                            const double n0 = c * b0 - s * b1, n1 = s * b0 + c * b1;
                            A[p0 * lda + qr] = n0; A[qr * lda + p0] = n0; A[p1 * lda + qr] = n1; A[qr * lda + p1] = n1;
                        } else if (q0 < n && q1 < n) {     // Q rotates, P is the bye: row pr, columns q0 / q1
                            const double c = rot[4 * Q], s = rot[4 * Q + 1], b0 = A[pr * lda + q0], b1 = A[pr * lda + q1];
                            const double n0 = c * b0 - s * b1, n1 = s * b0 + c * b1;
                            A[pr * lda + q0] = n0; A[q0 * lda + pr] = n0; A[pr * lda + q1] = n1; A[q1 * lda + pr] = n1;
                        }
                        continue;
                    }
                    const double cP = rot[4 * P], sP = rot[4 * P + 1], cQ = rot[4 * Q], sQ = rot[4 * Q + 1];
                    if (P == Q) {
                        const double app = A[p0 * lda + p0], aqq = A[p1 * lda + p1], apq = A[p0 * lda + p1];
                        // J^T [app apq; apq aqq] J with the rotation that annihilates apq
                        const double t00 = cP * app - sP * apq, t01 = cP * apq - sP * aqq, t10 = sP * app + cP * apq, t11 = sP * apq + cP * aqq;
                        A[p0 * lda + p0] = cP * t00 - sP * t01; A[p1 * lda + p1] = sP * t10 + cP * t11;
                        A[p0 * lda + p1] = 0.0; A[p1 * lda + p0] = 0.0;
                    } else {
                        const double b00 = A[p0 * lda + q0], b01 = A[p0 * lda + q1], b10 = A[p1 * lda + q0], b11 = A[p1 * lda + q1];
                        const double t00 = cP * b00 - sP * b10, t01 = cP * b01 - sP * b11, t10 = sP * b00 + cP * b10, t11 = sP * b01 + cP * b11;
                        const double n00 = cQ * t00 - sQ * t01, n01 = sQ * t00 + cQ * t01, n10 = cQ * t10 - sQ * t11, n11 = sQ * t10 + cQ * t11;
                        A[p0 * lda + q0] = n00; A[p0 * lda + q1] = n01; A[p1 * lda + q0] = n10; A[p1 * lda + q1] = n11;
                        A[q0 * lda + p0] = n00; A[q1 * lda + p0] = n01; A[q0 * lda + p1] = n10; A[q1 * lda + p1] = n11;
                    }
                } else {
                    const int it = e - nblk, i = it / np, Q = it - i * np;
                    const int q0 = (int)rot[4 * Q + 2], q1 = (int)rot[4 * Q + 3];
                    if (q0 >= n || q1 >= n) continue;
                    const double c = rot[4 * Q], s = rot[4 * Q + 1], v0 = V[i * ldv + q0], v1 = V[i * ldv + q1];
                    V[i * ldv + q0] = c * v0 - s * v1; V[i * ldv + q1] = s * v0 + c * v1;
                }
            }
            JSYNC();
        }
    }
    for (int i = tid; i < n; i += nt) d[i] = A[i * lda + i];
    JSYNC();
#undef JSYNC
}

VIWB_HD int vsub_to_mlay(int p) { return p < 66 ? p : p < 72 ? 165 + (p - 66) : p < 78 ? 171 + (p - 72) : 191; }   // td -> blk_moff(BLK_TD) = 191
VIWB_HD int marg_cap(int nmax) { return nmax < 16 ? 16 : (nmax > 100 ? 100 : nmax); }
enum { MARG_MD = 15 };      // dimension of the dropped fixed block: pose 0 + speed-bias 0 (MARGIN_OLD) or pose 9 (6, MARGIN_SECOND_NEW)
struct CompactTarget {     // marginalisation: dense symmetric matrix over the compact (kept | dropped) dimensions, in shared memory
    double *M, *g; int ld; const unsigned char *flags; const int *cmap;
    VIWB_DM int col(int blk, int k) const { return ((flags[blk] & 1u) && k < blk_msize(blk)) ? cmap[blk_moff(blk) + k] : -1; }
    VIWB_DM void add(int i, int j, double v) const { M[i * ld + j] += v; if (i != j) M[j * ld + i] += v; }
    VIWB_DM void addg(int i, double v) const { g[i] += v; }
};

// marg_prep: dense system of the marginalisation factors over the compact (kept | dropped) dimensions in shared memory, landmark elimination,
// pseudo-inverse of the dropped fixed block, Schur complement -> A (n x n) and b (n) of the kept block to HBM (the head of the window's
// marg_J slot and marg_r), header and linearisation point.  All phases are block-parallel; nothing serial.
VIWB_HD size_t marg_prep_smem_doubles(int nt, int nmax) {
    (void)nt; const int c = marg_cap(nmax), N = c + MARG_MD;
    return (size_t)N * N + (size_t)c * MARG_MD + 3 * 256 + (size_t)N + (size_t)c + 2 * (size_t)(c + 2) + 3 * 32 + 16 + (MLAY + 1) / 2 + 2;
}
VIWB_D void marg_prep_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by; (void)mode;
    const int w = bx;
    const WinMeta &m = bd.meta[w];
    WinWork &ww = bd.work[w];
    if (m.margin_flag < 0) return;
    const double *T = bd.Tvis + (size_t)w * VSUB * VSUB, *tv = bd.tvec + (size_t)w * VSUB;
    int *hdr = bd.marg_hdr + (size_t)w * (3 + 2 * NB);
    const double eps = 1e-8;   // marginalization_factor.h:81
    const int cap = marg_cap(bd.marg_nmax), NC = cap + MARG_MD;
    double *Mc = smem, *Tm = Mc + (size_t)NC * NC, *Amm = Tm + (size_t)cap * MARG_MD, *Vmm = Amm + 256, *Ainv = Vmm + 256;
    double *bc_ = Ainv + 256, *ev = bc_ + NC, *rot = ev + cap, *red = rot + 2 * (cap + 2), *bc = red + 3 * 32;
    int *cmap = (int *)(bc + 16);
    // ---- dropped / kept dimension lists (marginalisation layout -> compact index: kept dims 0..n-1, dropped n..n+md-1)
    if (tid == 0) {
        int md = 0, n = 0, nb = 0;
        unsigned dropped = 0;
        for (int k = 0; k < MLAY; k++) cmap[k] = -1;
        for (int k = 0; k < SFIX; k++) bd.marg_x0[(size_t)w * SFIX + k] = 0.0;
        if (m.margin_flag == 0) dropped = (1u << 0) | (1u << BLK_SB0); else dropped = (1u << 9);
        for (int bq = 0; bq < NB; bq++) {
            if (!(m.flags[bq] & 4u) || ((dropped >> bq) & 1u)) continue;      // bit 2 of flags = seen by a marginalisation factor
            int nid = bq;
            if (m.margin_flag == 0) { if ((bq >= 1 && bq <= 10) || (bq >= 12 && bq <= 21)) nid = bq - 1; }
            else { if (bq == 10 || bq == 21) nid = bq - 1; }
            hdr[3 + nb] = nid; hdr[3 + NB + nb] = n; nb++;
            for (int k = 0; k < blk_msize(bq); k++) { if (n < cap) cmap[blk_moff(bq) + k] = n; n++; }
            // linearisation point of the kept block, stored under its new id (keep_block_data + addr_shift)
            const double *src = bd.x_cur + m.state_off + blk_off(bq);
            double *dst = bd.marg_x0 + (size_t)w * SFIX + blk_off(nid);
            for (int k = 0; k < blk_size(bq); k++) dst[k] = src[k];
        }
        // a dropped block that no factor references contributes nothing (its rows stay zero, its eigenvalues fall under eps); md as the reference counts it
        if (n <= cap) {
            if (m.margin_flag == 0) { for (int k = 0; k < 6; k++) { cmap[k] = n + md; md++; } for (int k = 0; k < 9; k++) { cmap[66 + k] = n + md; md++; } }
            else { for (int k = 0; k < 6; k++) { cmap[54 + k] = n + md; md++; } }
        }
        hdr[0] = 1; hdr[1] = n; hdr[2] = nb;
        bc[2] = (double)md; bc[3] = (double)n;
    }
    VIWB_SYNC();
    const int md = (int)bc[2], n = (int)bc[3];
    if (n > cap) { if (tid == 0) { ww.marg_status = -1; hdr[0] = 0; } return; }
    const int N = n + md;
    for (int e = tid; e < N * N; e += nt) Mc[e] = 0.0;
    for (int i = tid; i < N; i += nt) bc_[i] = 0.0;
    VIWB_SYNC();
    { CompactTarget t; t.M = Mc; t.g = bc_; t.ld = N; t.flags = m.flags; t.cmap = cmap; assemble_into(t, bd, w, MODE_MARG, tid, nt, (int *)Tm); }      // Tm: scratch until the Schur complement
    VIWB_SYNC();
    // ---- eliminate the dropped landmarks: M -= scatter(T0), b -= scatter(tvec0)   (MARGIN_OLD only)
    if (m.margin_flag == 0) {
        for (int e = tid; e < 79 * 79; e += nt) { const int p = e / 79, q = e % 79, ci = cmap[vsub_to_mlay(p)], cj = cmap[vsub_to_mlay(q)]; if (ci >= 0 && cj >= 0) Mc[ci * N + cj] -= T[p * VSUB + q]; }
        for (int p = tid; p < 79; p += nt) { const int ci = cmap[vsub_to_mlay(p)]; if (ci >= 0) bc_[ci] -= tv[p]; }
    }
    VIWB_SYNC();
    // ---- pseudo-inverse of the dropped fixed block (marginalization_factor.cpp:282-287): 15 x 15 (or 6 x 6) parallel Jacobi
    for (int e = tid; e < md * md; e += nt) { const int i = e / md, j = e % md; Amm[e] = 0.5 * (Mc[(n + i) * N + n + j] + Mc[(n + j) * N + n + i]); }
    VIWB_SYNC();
    sym_eig_jacobi<false>(Amm, md, Vmm, md, ev, rot, red, md, tid, nt);      // eigenvalues -> ev, eigenvectors -> columns of Vmm (the whole block: one warp with warp-level synchronisation measured slower, 1.30 vs 0.90 ms per launch, r02v)
    for (int e = tid; e < md * md; e += nt) {
        const int i = e / md, j = e % md;
        double sacc = 0.0;
        for (int k = 0; k < md; k++) { const double l = ev[k]; if (l > eps) sacc += Vmm[i * md + k] * Vmm[j * md + k] / l; }
        Ainv[e] = sacc;
    }
    VIWB_SYNC();
    // Tm = Arm * Ainv (n x md)
    for (int e = tid; e < n * md; e += nt) {
        const int i = e / md, j = e % md;
        double sacc = 0.0;
        for (int k = 0; k < md; k++) sacc += Mc[i * N + n + k] * Ainv[k * md + j];
        Tm[e] = sacc;
    }
    VIWB_SYNC();
    // A = Arr - Arm Amm^-1 Amr ; b = brr - Arm Amm^-1 bmm -> HBM.  SelfAdjointEigenSolver reads the lower triangle: both (i, j) and (j, i)
    // receive the lower-triangle value
    double *Aout = bd.marg_J + (size_t)w * bd.marg_nmax * bd.marg_nmax, *bout = bd.marg_r + (size_t)w * MAXPRI;
    for (int e = tid; e < n * (n + 1) / 2; e += nt) {
        int i, j; sym_unrank(e, i, j);          // j <= i
        double sacc = Mc[i * N + j];
        for (int k = 0; k < md; k++) sacc -= Tm[i * md + k] * Mc[(n + k) * N + j];
        Aout[(size_t)i * n + j] = sacc; Aout[(size_t)j * n + i] = sacc;
    }
    for (int i = tid; i < n; i += nt) {
        double sacc = bc_[i];
        for (int k = 0; k < md; k++) sacc -= Tm[i * md + k] * bc_[n + k];
        bout[i] = sacc;
    }
}

// marg_eig: eigen-decomposition of the kept n x n block in shared memory (tridiag_block + tql2_block, the algorithm family of
// Eigen::SelfAdjointEigenSolver), J_lin = sqrt(S) V^T, r_lin = sqrt(S^-1) V^T b (marginalization_factor.cpp:289-306), in place over A / b in HBM.
// The three-kernel pipeline below runs the same statements in the same order (bit-identical priors in the emulation build; on the device the
// two kernels' code differs at rounding level).
// (A parallel cyclic Jacobi was measured here: 10 sweeps x 81 rounds of 2x2 block updates cost ten times the QL chain, profiles/r02c_*.)
VIWB_HD size_t marg_eig_smem_doubles(int nt, int nmax) { (void)nt; const int c = marg_cap(nmax); return (size_t)c * (c | 1) + (size_t)6 * c + 96 + 16 + 8; }      // V | b | cs (2) | d | e | red (3 x 32: three-way block reductions) | bc
VIWB_D void marg_eig_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by; (void)mode;
    const int w = bx;
    const WinMeta &m = bd.meta[w];
    WinWork &ww = bd.work[w];
    if (m.margin_flag < 0) return;
    const int *hdr = bd.marg_hdr + (size_t)w * (3 + 2 * NB);
    if (hdr[0] == 0) return;                                  // marg_prep gave up (kept dimension beyond the solver's capacity)
    const int n = hdr[1], cap = marg_cap(bd.marg_nmax), ld = n | 1;
    const double eps = 1e-8;
    double *Vn = smem, *bn = Vn + (size_t)cap * (cap | 1), *cs = bn + cap, *ev = cs + 2 * cap, *ee = ev + cap, *red = ee + cap, *bc = red + 96;
    double *Jout = bd.marg_J + (size_t)w * bd.marg_nmax * bd.marg_nmax, *rout = bd.marg_r + (size_t)w * MAXPRI;
    for (int e = tid; e < n * n; e += nt) { const int i = e / n, j = e - i * n; Vn[i * ld + j] = Jout[e]; }
    for (int i = tid; i < n; i += nt) bn[i] = rout[i];
    VIWB_SYNC();
    tridiag_block(Vn, ev, ee, cs, red, n, ld, tid, nt);
    tql2_block(Vn, ev, ee, cs, bc, n, ld, tid, nt);
    VIWB_SYNC();
    for (int e = tid; e < n * n; e += nt) {
        const int i = e / n, k = e - i * n;
        const double l = ev[i];
        Jout[e] = (l > eps ? sqrt(l) : 0.0) * Vn[k * ld + i];
    }
    for (int i = tid; i < n; i += nt) {
        const double l = ev[i], si = l > eps ? sqrt(1.0 / l) : 0.0;
        double vb = 0.0;
        for (int k = 0; k < n; k++) vb += Vn[k * ld + i] * bn[k];
        rout[i] = si * vb;
    }
    if (tid == 0) ww.marg_status = 0;
}

// The eigen-decomposition as a three-kernel pipeline.  The implicit QL iteration (tql2) is a strictly serial chain of plane rotations
// (~n^2 of them, ~120 cycles each): inside a block-per-window kernel it idles 255 threads for 40 % of the run time and only three windows
// fit an SM.  Splitting it off lets EVERY window's chain run at the same time (one warp each, all resident), while the parallel parts keep
// whole blocks busy:
//   marg_tri    block per window : A -> tridiagonal (d, e) + Q (tred2 and the accumulation), Q back to the window's marg_J slot
//   marg_ql     warp per window  : lane 0 runs tql2 on (d, e) alone and LOGS the rotations (c, s) sweep by sweep; eigenvalues to d
//   marg_apply  block per window : thread per row of Q applies the logged rotations (the eigenvector half of tql2), then J_lin, r_lin
// Same arithmetic in the same order as marg_eig: the same tridiag_block, then tql2_block's scalar recurrence statement for statement on lane 0, and
// its rotations applied to each row in the order tql2_block applies them.
enum { MARG_ROT_PER_N2 = 3, MARG_SWEEP_PER_N = 12 };      // rotation-log capacity 3 n^2 (a typical run needs ~n^2), sweep-log capacity 12 n
VIWB_HD size_t marg_rot_cap(int nmax) { const int c = marg_cap(nmax); return (size_t)MARG_ROT_PER_N2 * c * c; }
VIWB_HD size_t marg_sweep_cap(int nmax) { return (size_t)MARG_SWEEP_PER_N * marg_cap(nmax); }
VIWB_D void marg_tri_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by; (void)mode;
    const int w = bx;
    const WinMeta &m = bd.meta[w];
    if (m.margin_flag < 0) return;
    const int *hdr = bd.marg_hdr + (size_t)w * (3 + 2 * NB);
    if (hdr[0] == 0) return;
    const int n = hdr[1], cap = marg_cap(bd.marg_nmax), ld = n | 1;
    double *Vn = smem, *bn = Vn + (size_t)cap * (cap | 1), *cs = bn + cap, *ev = cs + 2 * cap, *ee = ev + cap, *red = ee + cap;
    double *Q = bd.marg_J + (size_t)w * bd.marg_nmax * bd.marg_nmax, *de = bd.marg_de + (size_t)w * 2 * MAXPRI;
    for (int e = tid; e < n * n; e += nt) { const int i = e / n, j = e - i * n; Vn[i * ld + j] = Q[e]; }
    VIWB_SYNC();
    tridiag_block(Vn, ev, ee, cs, red, n, ld, tid, nt);
    VIWB_SYNC();
    for (int e = tid; e < n * n; e += nt) { const int i = e / n, j = e - i * n; Q[e] = Vn[i * ld + j]; }
    for (int i = tid; i < n; i += nt) { de[i] = ev[i]; de[MAXPRI + i] = ee[i]; }
}
// lane 0 of a warp: tql2 on the tridiagonal matrix (the scalar half of tql2_block, statement for statement), rotations logged
VIWB_D void marg_ql_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by; (void)mode; (void)nt;
    const int w = bx;
    const WinMeta &m = bd.meta[w];
    if (m.margin_flag < 0 || tid != 0) return;
    int *hdr = bd.marg_hdr + (size_t)w * (3 + 2 * NB);
    if (hdr[0] == 0) return;
    const int n = hdr[1];
    double *d = smem, *e = smem + MAXPRI;
    double *de = bd.marg_de + (size_t)w * 2 * MAXPRI;
    const size_t rcap = marg_rot_cap(bd.marg_nmax), scap = marg_sweep_cap(bd.marg_nmax);
    double *rot = bd.marg_rot + (size_t)w * 2 * rcap;
    int *swp = bd.marg_sweep + (size_t)w * (2 * scap + 2);
    for (int i = 0; i < n; i++) { d[i] = de[i]; e[i] = de[MAXPRI + i]; }
    const double eps = 2.220446049250313e-16;
    double f = 0.0, tst1 = 0.0;
    size_t nrot = 0; int nsw = 0; bool overflow = false;
    for (int l = 0; l < n; l++) {
        const double t = fabs(d[l]) + fabs(e[l]); if (t > tst1) tst1 = t;
        int mm = l; while (mm < n) { if (fabs(e[mm]) <= eps * tst1) break; mm++; }
        if (mm > l) {
            for (int iter = 0; iter < 200; iter++) {
                double g = d[l], p = (d[l + 1] - g) / (2.0 * e[l]), r = sqrt(p * p + 1.0);
                if (p < 0) r = -r;
                d[l] = e[l] / (p + r); d[l + 1] = e[l] * (p + r);
                const double dl1 = d[l + 1]; double h = g - d[l];
                for (int i = l + 2; i < n; i++) d[i] -= h;
                f += h;
                p = d[mm];
                double c = 1.0, c2 = c, c3 = c, s = 0.0, s2 = 0.0; const double el1 = e[l + 1];
                if (nrot + (size_t)(mm - l) > rcap || nsw >= (int)scap) { overflow = true; break; }
                swp[2 + 2 * nsw] = l | (mm << 16); swp[3 + 2 * nsw] = (int)nrot; nsw++;
                double ei = e[mm - 1], di = d[mm - 1];
                for (int i = mm - 1; i >= l; i--) {
                    const double ein = i > l ? e[i - 1] : 0.0, din = i > l ? d[i - 1] : 0.0;
                    c3 = c2; c2 = c; s2 = s;
                    g = c * ei; h = c * p;
                    const double q2 = p * p + ei * ei, rinv = q2 > 0.0 ? rsqrt(q2) : 0.0;
                    r = q2 * rinv;
                    e[i + 1] = s * r; s = ei * rinv; c = p * rinv;
                    p = c * di - s * g; d[i + 1] = h + s * (c * g + s * di);
                    rot[2 * nrot] = c; rot[2 * nrot + 1] = s; nrot++;
                    ei = ein; di = din;
                }
                p = -s * s2 * c3 * el1 * e[l] / dl1;
                e[l] = s * p; d[l] = c * p;
                if (!(fabs(e[l]) > eps * tst1)) break;
            }
            if (overflow) break;
        }
        d[l] = d[l] + f; e[l] = 0.0;
    }
    swp[0] = overflow ? -1 : nsw; swp[1] = (int)nrot;
    for (int i = 0; i < n; i++) de[i] = d[i];
    if (overflow) { hdr[0] = 0; bd.work[w].marg_status = -2; }
}
VIWB_HD size_t marg_apply_smem_doubles(int nt, int nmax) { (void)nt; const int c = marg_cap(nmax); return (size_t)c * (c | 1) + (size_t)4 * c + 8; }
VIWB_D void marg_apply_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by; (void)mode;
    const int w = bx;
    const WinMeta &m = bd.meta[w];
    WinWork &ww = bd.work[w];
    if (m.margin_flag < 0) return;
    const int *hdr = bd.marg_hdr + (size_t)w * (3 + 2 * NB);
    if (hdr[0] == 0) return;
    const int n = hdr[1], cap = marg_cap(bd.marg_nmax), ld = n | 1;
    const double eps = 1e-8;
    double *Vn = smem, *bn = Vn + (size_t)cap * (cap | 1), *ev = bn + cap, *rs = ev + cap;      // rs: the current sweep's rotations (2 x n)
    double *Jout = bd.marg_J + (size_t)w * bd.marg_nmax * bd.marg_nmax, *rout = bd.marg_r + (size_t)w * MAXPRI;
    const double *de = bd.marg_de + (size_t)w * 2 * MAXPRI;
    const size_t rcap = marg_rot_cap(bd.marg_nmax), scap = marg_sweep_cap(bd.marg_nmax);
    const double *rot = bd.marg_rot + (size_t)w * 2 * rcap;
    const int *swp = bd.marg_sweep + (size_t)w * (2 * scap + 2);
    for (int e = tid; e < n * n; e += nt) { const int i = e / n, j = e - i * n; Vn[i * ld + j] = Jout[e]; }
    for (int i = tid; i < n; i += nt) { bn[i] = rout[i]; ev[i] = de[i]; }
    const int nsw = swp[0];
    VIWB_SYNC();
    for (int sw = 0; sw < nsw; sw++) {
        const int lm = swp[2 + 2 * sw], l = lm & 0xffff, mm = lm >> 16, cnt = mm - l;
        const double *r0 = rot + 2 * (size_t)swp[3 + 2 * sw];
        for (int q = tid; q < 2 * cnt; q += nt) rs[q] = r0[q];
        VIWB_SYNC();
        for (int k = tid; k < n; k += nt) {          // row k: columns mm .. l, the value of column i carried in a register to the next rotation
            double *row = Vn + k * ld;
            double hi = row[mm];                      // V(k, i + 1) for the first rotation (i = mm - 1)
            int q = 0;
            // four rotations per batch: their (c, s) and the four untouched columns they read are fetched before the first store of the batch (a load of rs
            // cannot be moved across a store to the row by the compiler), so one shared-memory latency is paid per batch instead of per rotation
            for (; q + 3 < cnt; q += 4) {
                const int i = mm - 1 - q;
                const double c0 = rs[2 * q], s0 = rs[2 * q + 1], c1 = rs[2 * q + 2], s1 = rs[2 * q + 3], c2 = rs[2 * q + 4], s2 = rs[2 * q + 5], c3 = rs[2 * q + 6], s3 = rs[2 * q + 7];
                const double l0 = row[i], l1 = row[i - 1], l2 = row[i - 2], l3 = row[i - 3];
                const double n0 = s0 * l0 + c0 * hi; hi = c0 * l0 - s0 * hi;
                const double n1 = s1 * l1 + c1 * hi; hi = c1 * l1 - s1 * hi;
                const double n2 = s2 * l2 + c2 * hi; hi = c2 * l2 - s2 * hi;
                const double n3 = s3 * l3 + c3 * hi; hi = c3 * l3 - s3 * hi;
                row[i + 1] = n0; row[i] = n1; row[i - 1] = n2; row[i - 2] = n3;
            }
            for (; q < cnt; q++) {
                const int i = mm - 1 - q;
                const double c = rs[2 * q], s = rs[2 * q + 1], lo = row[i];
                row[i + 1] = s * lo + c * hi;
                hi = c * lo - s * hi;                 // the new V(k, i) is V(k, (i - 1) + 1) of the next rotation
            }
            row[l] = hi;
        }
        VIWB_SYNC();
    }
    // J_lin = sqrt(S) V^T, r_lin = sqrt(S^-1) V^T b   (marginalization_factor.cpp:298-306)
    for (int e = tid; e < n * n; e += nt) {
        const int i = e / n, k = e - i * n;
        const double l = ev[i];
        Jout[e] = (l > eps ? sqrt(l) : 0.0) * Vn[k * ld + i];
    }
    for (int i = tid; i < n; i += nt) {
        const double l = ev[i], si = l > eps ? sqrt(1.0 / l) : 0.0;
        double vb = 0.0;
        for (int k = 0; k < n; k++) vb += Vn[k * ld + i] * bn[k];
        rout[i] = si * vb;
    }
    if (tid == 0) ww.marg_status = 0;
}

// ---------------------------------------------------------------------------------------------------- outlier rejection
// Estimator::outliersRejection (estimator.cpp:2127-2185) on the solved window (SURVEY 8 f-3): per landmark the mean of
// reprojectionError (:2115-2125) over its observations -- left camera of another frame, right camera of another frame, right
// camera of the host frame; the raw normalised points, no td compensation -- times FOCAL_LENGTH against 3 px.
// One thread per landmark (its factors are consecutive in the table).
VIWB_D void outlier_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by; (void)smem; (void)mode;
    const int k = bx * nt + tid;
    if (k >= bd.nlm_total) return;
    const int w = bd.lm_win[k];
    const WinMeta &m = bd.meta[w];
    const double *x = bd.x_cur + m.state_off;
    const int f0 = bd.lm_fptr[k], f1 = bd.lm_fptr[k + 1];
    if (f0 == f1) { bd.lm_outlier[k] = 0; return; }
    const double depth = 1.0 / x[SFIX + (k - m.lm_off)];
    const int ex_off[2] = {blk_off(BLK_EX0), blk_off(BLK_EX1)};
    double err = 0.0; int cnt = 0;
    for (int f = f0; f < f1; f++) {
        const int type = bd.vis_type[f], i = bd.vis_fi[f], j = (type == 2) ? i : bd.vis_fj[f], cam = (type == 0) ? 0 : 1;
        const double *o = bd.vis_obs + (size_t)f * 12;
        const V3 uvi = ld3(o), uvj = ld3(o + 3);
        const V3 Pi = ld3(x + 7 * i), Pj = ld3(x + 7 * j), tici = ld3(x + ex_off[0]), ticj = ld3(x + ex_off[cam]);
        const Q4 Qi = ldq(x + 7 * i + 3), Qj = ldq(x + 7 * j + 3), qici = ldq(x + ex_off[0] + 3), qicj = ldq(x + ex_off[cam] + 3);
        const V3 pts_w = qrot(Qi, qrot(qici, depth * uvi) + tici) + Pi;
        const V3 pts_cj = tmul(qR(qicj), tmul(qR(Qj), pts_w - Pj) - ticj);
        const double rx = pts_cj.x / pts_cj.z - uvj.x, ry = pts_cj.y / pts_cj.z - uvj.y;
        err += sqrt(rx * rx + ry * ry); cnt++;
    }
    bd.lm_outlier[k] = ((err / cnt) * bd.out_focal > bd.out_thresh) ? 1 : 0;
}

}  // namespace viwb
