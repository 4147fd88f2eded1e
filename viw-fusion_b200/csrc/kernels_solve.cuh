// kernels_solve.cuh -- one block per window: the Ceres trust-region recurrence (DENSE_SCHUR + DOGLEG) on the
// assembled normal equations.  Restates ceres-solver 1.14 semantics (SURVEY Appendix B; call site
// estimator.cpp:1643-1658): Jacobi scaling fixed at the first linearisation, D = sqrt(clamp(diag)), Cauchy
// length, mu-regularised Gauss-Newton step through the Schur complement on the inverse depths + dense Cholesky
// (mu x10 on failure), traditional dogleg interpolation, model decrease, candidate = x (+) step; and, one call
// later, the accept/reject decision with the radius / mu updates and all termination tests.
//
// The reduced system (<= 192 active tangent columns) lives in shared memory as a SKYLINE: row i of the lower triangle is stored
// from its first structurally non-zero column efirst[i] (host symbolic analysis, csrc/viwb.cu lower_count).  With the speed-bias
// blocks eliminated first, newest frame first, the stereo+IMU window needs 7.2-7.6 K instead of 13.7 K doubles; with the carve below
// (9.5 K doubles at 256 threads) three such windows share an SM.  All quadratic forms are evaluated on the *unscaled* matrices with unscaled directions
// u = c o (v / D), which equals Ceres' J_scaled products exactly.
#pragma once
#include <vector>
#include "layout.cuh"
#include "factors.cuh"
#include "kernels_asm.cuh"

namespace viwb {

VIWB_HD int pidx(int i, int j) { return i >= j ? i * (i + 1) / 2 + j : j * (j + 1) / 2 + i; }

// block-wide sum / max; red has >= 32 doubles.  Every thread gets the result (fixed reduction order: deterministic).
#ifdef VIWB_HOST_EMU
VIWB_D double block_sum(double v, int, int, double *) { return v; }
VIWB_D double block_max(double v, int, int, double *) { return v; }
#else
VIWB_D double block_sum(double v, int tid, int nt, double *red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if ((tid & 31) == 0) red[tid >> 5] = v;
    __syncthreads();
    const int nw = nt >> 5;
    double r = 0.0;
    for (int k = 0; k < nw; k++) r += red[k];
    __syncthreads();
    return r;
}
VIWB_D double block_max(double v, int tid, int nt, double *red) {
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_down_sync(0xffffffffu, v, o));
    if ((tid & 31) == 0) red[tid >> 5] = v;
    __syncthreads();
    const int nw = nt >> 5;
    double r = red[0];
    for (int k = 1; k < nw; k++) r = fmax(r, red[k]);
    __syncthreads();
    return r;
}
#endif

// several sums in one pass: one barrier pair for all of them (red needs N * 32 doubles)
template <int N>
VIWB_D void block_sum_n(double (&v)[N], int tid, int nt, double *red) {
#ifdef VIWB_HOST_EMU
    (void)v; (void)tid; (void)nt; (void)red;
#else
    for (int q = 0; q < N; q++) for (int o = 16; o > 0; o >>= 1) v[q] += __shfl_down_sync(0xffffffffu, v[q], o);
    const int nw = nt >> 5;
    if ((tid & 31) == 0) for (int q = 0; q < N; q++) red[q * 32 + (tid >> 5)] = v[q];
    __syncthreads();
    for (int q = 0; q < N; q++) { double r = 0.0; for (int k = 0; k < nw; k++) r += red[q * 32 + k]; v[q] = r; }
    __syncthreads();
#endif
}

// The solve kernel's sums are stated over a fixed VIRTUAL layout of SOLVE_VNT threads (12 warps), whatever the block's real size: real thread t
// owns the virtual threads t, t + nt, ... below SOLVE_VNT (SOLVE_VPT of them at most), keeps one partial sum per virtual thread, strides its loops
// by SOLVE_VNT and reduces each virtual warp with the same shuffle tree; the virtual warps' slots are then added in order.  So every sum is the
// same double at any block size that is a multiple of 32, and the block size only changes the occupancy.  (Maxima need no such care: fmax does
// not depend on the order.)  The emulation runs one thread per block, and its virtual layout is that thread.
#ifndef SOLVE_NT
#define SOLVE_NT 256
#endif
#ifdef VIWB_HOST_EMU
enum { SOLVE_VNT = 1, SOLVE_VW = 1, SOLVE_VPT = 1 };
#define VIWB_VT_LOOP(j, vt) for (int j = 0, vt = tid; j < SOLVE_VPT; j++, vt += nt)
#define VIWB_VLM_LOOP(k, vt, N) for (int k = (vt), lane = 0; k < (N); k++)
#else
enum { SOLVE_VNT = 384, SOLVE_VW = SOLVE_VNT / 32, SOLVE_VPT = (SOLVE_VNT + SOLVE_NT - 1) / SOLVE_NT };
#define VIWB_VT_LOOP(j, vt) _Pragma("unroll") for (int j = 0, vt = tid; j < SOLVE_VPT; j++, vt += nt) if (vt < SOLVE_VNT)
// one virtual warp per landmark (vt >> 5 is warp-uniform): lane 0 carries the scalar work and the virtual thread's partial sums
#define VIWB_VLM_LOOP(k, vt, N) for (int k = (vt) >> 5, lane = tid & 31; k < (N); k += SOLVE_VW)
#endif
// v[j][q]: partial sum q of this thread's virtual thread j (0 where it owns none); on return every thread has the block's sums in v[0][q].
// red needs N * SOLVE_RED doubles.
enum { SOLVE_RED = 16 };      // slots per sum: >= the virtual warps and the real ones (block_max)
template <int N>
VIWB_D void vblock_sum_n(double (&v)[SOLVE_VPT][N], int tid, int nt, double *red) {
#ifdef VIWB_HOST_EMU
    (void)v; (void)tid; (void)nt; (void)red;
#else
#pragma unroll
    for (int j = 0; j < SOLVE_VPT; j++) {
        const int vt = tid + j * nt;
        if (vt < SOLVE_VNT) {
#pragma unroll
            for (int q = 0; q < N; q++) for (int o = 16; o > 0; o >>= 1) v[j][q] += __shfl_down_sync(0xffffffffu, v[j][q], o);
            if ((tid & 31) == 0) for (int q = 0; q < N; q++) red[q * SOLVE_RED + (vt >> 5)] = v[j][q];
        }
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < N; q++) { double r = 0.0; for (int k = 0; k < SOLVE_VW; k++) r += red[q * SOLVE_RED + k]; v[0][q] = r; }
    __syncthreads();
#endif
}

// Shared memory of one window, in doubles.  P = solve_nfp(nf_max): the batch's largest nf in whole 4-double groups; R = solve_panel_rows(nf_max):
// the most trailing rows (rhs included, whole 4-row tiles) a panel has, the first panel's; F = solve_fac_warps(nt, nf_max): the warps that hold
// such rows and factor the diagonal block.
//   L     skyline lower triangle, env_max entries (even).  The factor's diagonal holds the inverse pivots 1 / L_kk, which is all the
//         back-substitution reads there.
//   U     union region, max(8 R + CHOL_SCR F, 2 P + 2 VSUB); its parts are live at different times of a step:
//           U[0, P)               g (assembly) | ug (Cauchy point) | u (back-substituted step -> quadratic forms)
//           U[P, 2 P)             imap (assembly, ints) | Hu (Cauchy point, quadratic forms) | xo (back-substitution)
//           U[2 P, 2 P + 2 VSUB)  uvis (Cauchy point, landmark back-substitution)
//           U[0, 8 R)             Pt (Cholesky; 16-byte aligned), then chol: CHOL_SCR per factoring warp (Cholesky)
//         The assembled gradient is read from its copy in HBM (gpk) after the assembly, and the Jacobi scales, D and the scaled gradient from
//         the window's v_* slices, where they are written once per linearisation; the forms recompute ug from those.
//   y     P: right-hand side, then solution of the reduced system (the Cholesky's row n, addressed from L)
//   red   5 * SOLVE_RED: reductions
//   then shorts: vmap (P), fst (P), rp (P + 1)
struct SolveSmem {
    double *L;            // skyline lower triangle: row i holds columns fst[i]..i at L[rp[i] .. rp[i+1])
    short *rp, *fst;      // row pointers (nf + 1) and first columns (nf)
    short *vmap;          // compact column -> visual subspace (-1: not visual)
    double *g, *ug, *u, *Hu, *xo, *Pt, *uvis, *chol, *y, *red;
    int ldp;              // row stride of Pt (R)
};
enum { CHOL_NB = 8, CHOL_SCR = 48 };      // the Cholesky's panel width and per-warp scratch (doubles)
VIWB_HD int solve_nfp(int nf_max) { const int p = (nf_max + 3) & ~3; return p > 4 ? p : 4; }
VIWB_HD int solve_panel_rows(int nf_max) { const int r = nf_max > CHOL_NB ? (nf_max + 1 - CHOL_NB + 3) & ~3 : 4; return r; }
VIWB_HD int solve_fac_warps(int nt, int nf_max) { const int a = (nt + 31) / 32, b = (solve_panel_rows(nf_max) + 31) / 32; return a < b ? a : b; }
VIWB_HD size_t solve_union_doubles(int nt, int nf_max) {
    const size_t a = (size_t)8 * solve_panel_rows(nf_max) + (size_t)CHOL_SCR * solve_fac_warps(nt, nf_max), b = (size_t)2 * solve_nfp(nf_max) + 2 * VSUB;
    return a > b ? a : b;
}
VIWB_HD size_t solve_smem_doubles(int nt, int esize, int nf_max) {
    const int P = solve_nfp(nf_max);
    return (size_t)((esize + 1) & ~1) + solve_union_doubles(nt, nf_max) + P + 5 * SOLVE_RED + (size_t)(3 * P + 1 + 3) / 4;
}
VIWB_HD void carve(SolveSmem &s, double *smem, int nt, int esize, int nf_max) {
    const int P = solve_nfp(nf_max), R = solve_panel_rows(nf_max);
    double *p = smem;
    s.L = p; p += (size_t)((esize + 1) & ~1);
    double *U = p; p += solve_union_doubles(nt, nf_max);
    s.g = s.ug = s.u = U;
    s.Hu = s.xo = U + P;
    s.uvis = U + 2 * P;
    s.Pt = U; s.ldp = R;
    s.chol = U + 8 * R;
    s.y = p; p += P;
    s.red = p; p += 5 * SOLVE_RED;
    s.vmap = (short *)p; s.fst = s.vmap + P; s.rp = s.fst + P;
}
// entry (i, j), j <= i, of the skyline; must lie inside the envelope
#define SKY(s, i, j) ((s).L[(s).rp[i] - (s).fst[i] + (j)])

// assemble the active part of H (unscaled) and g into the skyline / s.g, and keep a copy in HBM
VIWB_D void assemble_H(const BatchDev &bd, int w, const SolveSmem &s, int nf, double *Hpk, double *gpk, int tid, int nt) {
    const int ne = s.rp[nf];
    for (int e = tid; e < ne; e += nt) s.L[e] = 0.0;
    for (int i = tid; i < nf; i += nt) s.g[i] = 0.0;
    VIWB_SYNC();
    PackedTarget t; t.L = s.L; t.g = s.g; t.tcol = bd.meta[w].tcol; t.rp = s.rp; t.fst = s.fst;
    assemble_into(t, bd, w, MODE_SOLVE, tid, nt, (int *)s.Hu);      // Hu is free until the Cauchy point
    for (int e = tid; e < ne; e += nt) Hpk[e] = s.L[e];
    for (int i = tid; i < nf; i += nt) gpk[i] = s.g[i];
    VIWB_SYNC();
}
// reload the copy (after the Cholesky factor overwrote it)
VIWB_D void load_H(const double *Hpk, const SolveSmem &s, int nf, int tid, int nt) {
    const int ne = s.rp[nf];
    for (int e = tid; e < ne; e += nt) s.L[e] = Hpk[e];
    VIWB_SYNC();
}
// Hu = H u over the skyline (u, Hu of length nf): the stored part of row i, then column i of the rows below that reach it
VIWB_D void symv(const SolveSmem &s, int nf, const double *u, double *Hu, int tid, int nt) {
    for (int i = tid; i < nf; i += nt) {
        double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;            // four partial sums (a dependent FMA chain of up to nf otherwise)
        const double *ri = s.L + s.rp[i] - s.fst[i];
        int j = s.fst[i];
        for (; j + 3 <= i; j += 4) { a0 += ri[j] * u[j]; a1 += ri[j + 1] * u[j + 1]; a2 += ri[j + 2] * u[j + 2]; a3 += ri[j + 3] * u[j + 3]; }
        for (; j <= i; j++) a0 += ri[j] * u[j];
        int k = i + 1;
        for (; k + 1 < nf; k += 2) {
            if (s.fst[k] <= i) a1 += s.L[s.rp[k] - s.fst[k] + i] * u[k];
            if (s.fst[k + 1] <= i) a2 += s.L[s.rp[k + 1] - s.fst[k + 1] + i] * u[k + 1];
        }
        for (; k < nf; k++) if (s.fst[k] <= i) a3 += s.L[s.rp[k] - s.fst[k] + i] * u[k];
        Hu[i] = (a0 + a1) + (a2 + a3);
    }
    VIWB_SYNC();
}
// uvis[p] = u mapped to the visual subspace (0 where the column is inactive)
VIWB_D void to_vis(const SolveSmem &s, int nf, const double *u, double *uvis, int tid, int nt) {
    for (int p = tid; p < VSUB; p += nt) uvis[p] = 0.0;
    VIWB_SYNC();
    for (int i = tid; i < nf; i += nt) if (s.vmap[i] >= 0) uvis[s.vmap[i]] = u[i];
    VIWB_SYNC();
}
VIWB_D double dot80(const double *W, const double *v) { double a = 0.0; for (int p = 0; p < 79; p++) a += W[p] * v[p]; return a; }
// the same product by one warp: coalesced reads of the landmark's W row, every lane gets the sum (fixed order: deterministic)
VIWB_D double warp_dot80(const double *W, const double *v, int lane) {
#ifdef VIWB_HOST_EMU
    (void)lane; return dot80(W, v);
#else
    double a = W[lane] * v[lane] + W[lane + 32] * v[lane + 32];
    if (lane < 15) a += W[lane + 64] * v[lane + 64];
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    return a;
#endif
}
// landmark loops that feed no sum run one real warp per landmark (lane 0 carries the scalar work)
#ifdef VIWB_HOST_EMU
#define VIWB_LM_LOOP(k, N) for (int k = 0, lane = 0; k < (N); k++)
#else
#define VIWB_LM_LOOP(k, N) for (int k = tid >> 5, lane = tid & 31; k < (N); k += nt >> 5)
#endif

// Blocked (panel width 8) in-place Cholesky of the packed lower triangle with the right-hand side carried as an extra
// row n, so that on exit y = L^-1 b (forward substitution for free).  Returns false on a non-positive pivot
// (Eigen LLT semantics: schur_complement_solver.cc -> LINEAR_SOLVER_FAILURE).  2 barriers per panel:
//   every warp that holds panel rows factors the 8x8 diagonal block redundantly (8 lanes, one row each, in registers; pivots through rsqrt so
//   that the panel rows multiply instead of divide) into its own scratch, so no barrier separates it from the panel solve;
//   one thread per panel row, which also drops its 8 results into a column-major panel buffer Pt[8][rows]; the trailing
//   update then runs 4x4 register tiles whose operands are 32-byte vector loads from Pt (conflict-free), not strided
//   reads of the packed triangle.
// scratch: CHOL_SCR doubles per warp that holds panel rows (36 packed block entries + 8 inverse pivots + flag); on exit the diagonal of L holds the
// inverse pivots 1 / L_kk instead of L_kk (the back-substitution multiplies by them, and nothing else reads the factor's diagonal);
// Pt: 8 rows of ldp >= the panel rows rounded up to 4 (a multiple of 4) doubles, 16-byte aligned.
VIWB_D void load4(const double *p, double *o) {
#ifdef VIWB_HOST_EMU
    o[0] = p[0]; o[1] = p[1]; o[2] = p[2]; o[3] = p[3];
#else
    const double2 a = reinterpret_cast<const double2 *>(p)[0], b = reinterpret_cast<const double2 *>(p)[1];
    o[0] = a.x; o[1] = a.y; o[2] = b.x; o[3] = b.y;
#endif
}
// Phase probe (measurement build only, `make phases` -> libviwb_phases.so): thread 0 reads clock64() at the barrier-delimited phase
// boundaries of a launch that computes a step and adds the cycles since the previous boundary to its window's slot of the phase.
// The sub-phases of the Cholesky and the back-substitution are summed in registers and written once per factorisation (SOLVE_FLUSH).
// Launches that only decide the pending candidate and stop are not counted.  The product library compiles none of this.
enum { SPH_PRO, SPH_ASM, SPH_DSC, SPH_CAUCHY, SPH_SCHUR, SPH_CHOL_DIAG, SPH_CHOL_PANEL, SPH_CHOL_TRAIL, SPH_BACK_SOLVE, SPH_BACK_UPD,
       SPH_LM2, SPH_FORMS, SPH_DOGLEG, SPH_N, SPH_STEPS = SPH_N, SPH_FACT, SPH_SLOTS, SPH_MAXW = 8192,
       SPH_SUB0 = SPH_CHOL_DIAG, SPH_NSUB = SPH_BACK_UPD + 1 - SPH_CHOL_DIAG };
#if defined(VIWB_SOLVE_PROBE) && !defined(VIWB_HOST_EMU)
__device__ unsigned long long g_solve_phase[SPH_MAXW * SPH_SLOTS];
struct SolveClock { int w; long long t, sub[SPH_NSUB]; };
#define SOLVE_PROBE_START() SolveClock sph; sph.w = w; sph.t = clock64(); for (int q_ = 0; q_ < SPH_NSUB; q_++) sph.sub[q_] = 0
#define SOLVE_MARK(p) do { if (tid == 0 && w < SPH_MAXW) { const long long t_ = clock64(); g_solve_phase[w * SPH_SLOTS + (p)] += t_ - sph.t; sph.t = t_; } } while (0)
#define SOLVE_COUNT(p) do { if (tid == 0 && w < SPH_MAXW) g_solve_phase[w * SPH_SLOTS + (p)]++; } while (0)
#define SOLVE_LAP(p) do { if (tid == 0) { const long long t_ = clock64(); sph.sub[(p) - SPH_SUB0] += t_ - sph.t; sph.t = t_; } } while (0)
#define SOLVE_FLUSH() do { if (tid == 0 && sph.w < SPH_MAXW) for (int q_ = 0; q_ < SPH_NSUB; q_++) { g_solve_phase[sph.w * SPH_SLOTS + SPH_SUB0 + q_] += sph.sub[q_]; sph.sub[q_] = 0; } } while (0)
#else
struct SolveClock {};
#define SOLVE_PROBE_START() SolveClock sph; (void)sph
#define SOLVE_MARK(p) ((void)0)
#define SOLVE_COUNT(p) ((void)0)
#define SOLVE_LAP(p) ((void)0)
#define SOLVE_FLUSH() ((void)0)
#endif

// The factorisation plan of one envelope, built once by the host lowering (viwb.cu chol_plan_build) and shared by the windows with that
// envelope: ints  rp[0..n]  (skyline row pointers),  toff[0..np]  (panel p's trailing-update tiles are tiles[toff[p] .. toff[p+1])),  tiles.
// A tile is the 4x4 block of rows r0 + 4 ti.., columns r0 + 4 tk.. (r0: the panel's first trailing row, tk <= ti) that receives at least one
// entry; its word is ti | tk << 8 | on << 16, bit 4 a + b of `on` set when entry (r0 + 4 ti + a, r0 + 4 tk + b) receives the panel's update:
// the row reaches the panel (first stored column < r0; row n, the right-hand side, always does), so does the column (< n), and it lies on or
// below the diagonal.  Every receiving entry is in exactly one tile.
VIWB_HD int chol_panels(int n) { return (n + CHOL_NB - 1) / CHOL_NB; }
VIWB_HD int chol_plan_head(int n) { return n + 1 + chol_panels(n) + 1; }
inline void chol_plan_build(const short *efirst, int n, std::vector<int> &plan) {
    const int np = chol_panels(n), head = chol_plan_head(n);
    plan.assign((size_t)head, 0);
    for (int i = 0; i < n; i++) plan[i + 1] = plan[i] + i - efirst[i] + 1;
    std::vector<unsigned> rows, cols;      // per 4-row group of the panel's trailing rows: which rows / columns reach the panel
    for (int p = 0; p < np; p++) {
        plan[n + 1 + p] = (int)plan.size() - head;
        const int r0 = (p + 1) * CHOL_NB < n ? (p + 1) * CHOL_NB : n, mt = (n + 1 - r0 + 3) / 4;
        rows.assign(mt, 0u); cols.assign(mt, 0u);
        for (int i = r0; i <= n; i++) {
            const unsigned bit = 1u << ((i - r0) & 3);
            if (i == n) rows[(i - r0) >> 2] |= bit;
            else if (efirst[i] < r0) { rows[(i - r0) >> 2] |= bit; cols[(i - r0) >> 2] |= bit; }
        }
        for (int ti = 0; ti < mt; ti++)
            for (int tk = 0; tk <= ti; tk++) {
                unsigned on = 0;
                for (int a = 0; a < 4; a++) if ((rows[ti] >> a) & 1u) on |= cols[tk] << (4 * a);
                if (tk == ti) on &= 0xf731u;          // on or below the diagonal: column b <= row a
                if (on) plan.push_back((int)((unsigned)ti | (unsigned)tk << 8 | on << 16));
            }
    }
    plan[n + 1 + np] = (int)plan.size() - head;
}
VIWB_D bool cholesky_packed_rhs(double *L, const short *rp, const short *fst, double *y, int n, int tid, int nt, double *scratch, double *Pt, int ldp,
                                const int *__restrict__ plan, SolveClock &sph) {
    (void)sph;
    const int yoff = (int)(y - L);
    const int *toff = plan + n + 1;
    const unsigned *tiles = reinterpret_cast<const unsigned *>(plan + chol_plan_head(n));
    // skyline rows: ROW(i)[j] is entry (i, j) for fst[i] <= j <= i; row n is the right-hand side (dense).  FST(i) = first stored column.
#define ROW(i) ((i) < n ? L + rp[i] - fst[i] : y)
#define FST(i) ((i) < n ? fst[i] : 0)
    const int lane = tid & 31;
    double *my = scratch + (size_t)(tid >> 5) * CHOL_SCR;      // this warp's copy of the factored diagonal block
    for (int c0 = 0; c0 < n; c0 += CHOL_NB) {
        const int nb = (n - c0) < CHOL_NB ? (n - c0) : CHOL_NB;
        const int r0 = c0 + nb;
        const int nr = n + 1 - r0, mt = (nr + 3) / 4;       // panel rows r0..n (row n = rhs), padded to whole 4-row tiles
        // only the warps that hold panel rows factor the diagonal block (warp 0 always: row n and the block's write-back); the others
        // would only take issue slots from them
        const bool fac = (tid & ~31) < 4 * mt;
#ifdef VIWB_HOST_EMU
        if (fac) {   // single-thread statement of the same arithmetic
            (void)lane;
            my[44] = 1.0;
            double a[8][8];
            for (int i = 0; i < nb; i++) for (int j = 0; j <= i; j++) a[i][j] = (c0 + j >= FST(c0 + i)) ? ROW(c0 + i)[c0 + j] : 0.0;
            for (int k = 0; k < nb; k++) {
                const double d = a[k][k];
                if (!(d > 0.0)) { my[44] = 0.0; break; }
                const double inv = 1.0 / sqrt(d);
                a[k][k] = d * inv; my[36 + k] = inv;
                for (int i = k + 1; i < nb; i++) a[i][k] *= inv;
                for (int i = k + 1; i < nb; i++) for (int j = k + 1; j <= i; j++) a[i][j] -= a[i][k] * a[j][k];
            }
            for (int i = 0; i < nb; i++) for (int j = 0; j <= i; j++) my[i * (i + 1) / 2 + j] = a[i][j];
        }
#else
        if (fac) {
            double a[8];
            const bool act = lane < nb;
            const int rr = c0 + (act ? lane : 0), fr = fst[rr];
            const double *src = ROW(rr) + c0;
#pragma unroll
            for (int j = 0; j < 8; j++) a[j] = (act && j <= lane && c0 + j >= fr) ? src[j] : 0.0;
            bool okp = true;
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const double d = __shfl_sync(0xffffffffu, a[k], k);
                if (k < nb && !(d > 0.0)) okp = false;
                const double inv = (k < nb && d > 0.0) ? rsqrt(d) : 0.0;
                if (lane == k) { a[k] = d * inv; if (k < nb) my[36 + k] = inv; }
                else if (lane > k) a[k] *= inv;
#pragma unroll
                for (int j = k + 1; j < 8; j++) {
                    const double ljk = __shfl_sync(0xffffffffu, a[k], j);      // L[j][k]
                    if (lane >= j) a[j] -= a[k] * ljk;
                }
            }
            if (act) {
#pragma unroll
                for (int j = 0; j < 8; j++) if (j <= lane) my[lane * (lane + 1) / 2 + j] = a[j];
            }
            if (lane == 0) my[44] = okp ? 1.0 : 0.0;
            __syncwarp();
        }
#endif
        SOLVE_LAP(SPH_CHOL_DIAG);
        // this panel's tiles; the first word is fetched before the panel solve (the plan does not depend on the matrix)
        const unsigned *tp = tiles + toff[c0 / CHOL_NB];
        const int ntp = toff[c0 / CHOL_NB + 1] - toff[c0 / CHOL_NB];
        unsigned wd = tid < ntp ? tp[tid] : 0u;
        // panel rows (a failed pivot leaves inverse pivots of 0 here; the verdict is read after the barrier and the factor discarded):
        // x_k = (a_ik - sum_m x_m L_km) / L_kk; columns left of a row's envelope are (and stay) structural zeros
        for (int i = r0 + tid; i < r0 + 4 * mt; i += nt) {
            double x[8];
#pragma unroll
            for (int k = 0; k < 8; k++) x[k] = 0.0;
            if (i <= n && FST(i) < r0) {
                double *ri = ROW(i) + c0;
                const int fi = FST(i);
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    if (k < nb && c0 + k >= fi) {
                        double v = ri[k];
#pragma unroll
                        for (int m = 0; m < 8; m++) if (m < k) v -= x[m] * my[k * (k + 1) / 2 + m];
                        x[k] = v * my[36 + k];
                    }
                }
                // (stored after the chain: a store to the row in between would pin every later load of the diagonal block behind it)
#pragma unroll
                for (int k = 0; k < 8; k++) if (k < nb && c0 + k >= fi) ri[k] = x[k];
            }
#pragma unroll
            for (int k = 0; k < 8; k++) Pt[k * ldp + (i - r0)] = x[k];
        }
        VIWB_SYNC();
        SOLVE_LAP(SPH_CHOL_PANEL);
        if (scratch[44] == 0.0) return false;               // warp 0's verdict, the same as every factoring warp's: every thread returns here
        // factored diagonal block back into the matrix (only now: the other warps have finished reading the unfactored one), inverse pivots on
        // the diagonal
        for (int r = tid; r < nb; r += nt) { double *rk = ROW(c0 + r) + c0; const int fr = FST(c0 + r); for (int j = 0; j <= r; j++) if (c0 + j >= fr) rk[j] = j == r ? my[36 + r] : my[r * (r + 1) / 2 + j]; }
        // trailing update with 4x4 register tiles over the plan's tiles of this panel: each receiving entry a_ik -= sum_m L_im L_km once
        for (int t = tid; t < ntp; t += nt) {
            const unsigned cur = wd;
            if (t + nt < ntp) wd = tp[t + nt];
            const int ti = (int)(cur & 0xffu), tk = (int)((cur >> 8) & 0xffu);
            const unsigned on = cur >> 16;
            const int ib = r0 + 4 * ti, kb = r0 + 4 * tk;
            double acc[16];
#pragma unroll
            for (int q = 0; q < 16; q++) acc[q] = 0.0;
#pragma unroll
            for (int m = 0; m < 8; m++) {
                double li[4], lk[4];
                load4(Pt + m * ldp + 4 * ti, li); load4(Pt + m * ldp + 4 * tk, lk);
#pragma unroll
                for (int a = 0; a < 4; a++)
#pragma unroll
                    for (int b2 = 0; b2 < 4; b2++) acc[a * 4 + b2] += li[a] * lk[b2];
            }
            // all sixteen current values are fetched before the first store (four different row pointers: the compiler has to assume they alias)
            int ro[4];      // the rows as offsets from L (row n, the right-hand side y, is carved from the same shared block)
#pragma unroll
            for (int a = 0; a < 4; a++) ro[a] = ((on >> (4 * a)) & 0xfu) ? (ib + a < n ? rp[ib + a] - fst[ib + a] : yoff) : 0;
#pragma unroll
            for (int a = 0; a < 4; a++)
#pragma unroll
                for (int b2 = 0; b2 < 4; b2++) acc[a * 4 + b2] = ((on >> (a * 4 + b2)) & 1u) ? L[ro[a] + kb + b2] - acc[a * 4 + b2] : 0.0;
#pragma unroll
            for (int a = 0; a < 4; a++)
#pragma unroll
                for (int b2 = 0; b2 < 4; b2++) if ((on >> (a * 4 + b2)) & 1u) L[ro[a] + kb + b2] = acc[a * 4 + b2];
        }
        VIWB_SYNC();
        SOLVE_LAP(SPH_CHOL_TRAIL);
    }
#undef ROW
#undef FST
    return true;
}
// back substitution L^T x = y (blocks of 8 from the bottom): every thread that needs it solves the 8x8 triangular block redundantly from
// broadcast reads (no barrier between the block solve and the update), then the rows above that the block's columns reach (from the
// block's first stored column on) are updated.  One barrier per block.  Result in y; xo is scratch of n doubles.
VIWB_D void chol_backsolve_blocked(const double *L, const short *rp, const short *fst, double *y, double *xo, int n, int tid, int nt,
                                   SolveClock &sph) {
    (void)sph;
    const int nblk = chol_panels(n);
    for (int bi = nblk - 1; bi >= 0; bi--) {
        const int c0 = bi * CHOL_NB, nb = (n - c0) < CHOL_NB ? (n - c0) : CHOL_NB;
        double x[8];
        const double *rw[8]; int fr[8];              // the block's skyline rows and their first columns
#pragma unroll
        for (int m = 0; m < 8; m++) { const int r = (m < nb) ? c0 + m : c0; rw[m] = L + rp[r] - fst[r]; fr[m] = fst[r]; }
        int lo = fr[0];
#pragma unroll
        for (int k = 1; k < 8; k++) lo = fr[k] < lo ? fr[k] : lo;
        // only the threads that store the block's solution or update a row above solve the block
        const bool act = tid < CHOL_NB || lo + tid < c0;
#pragma unroll
        for (int k = 7; k >= 0; k--) {
            x[k] = 0.0;
            if (act && k < nb) {
                double v = y[c0 + k];
#pragma unroll
                for (int m = 7; m > k; m--) if (m < nb && c0 + k >= fr[m]) v -= rw[m][c0 + k] * x[m];
                x[k] = v * rw[k][c0 + k];          // the inverse pivot
            }
        }
#pragma unroll
        for (int k = 0; k < 8; k++) if (k < nb && tid == (k < nt ? k : 0)) xo[c0 + k] = x[k];
        SOLVE_LAP(SPH_BACK_SOLVE);
        for (int i = lo + tid; i < c0; i += nt) {
            double v = y[i];
#pragma unroll
            for (int k = 0; k < 8; k++) if (k < nb && i >= fr[k]) v -= rw[k][i] * x[k];
            y[i] = v;
        }
        VIWB_SYNC();
        SOLVE_LAP(SPH_BACK_UPD);
    }
    for (int i = tid; i < n; i += nt) y[i] = xo[i];
    VIWB_SYNC();
    SOLVE_LAP(SPH_BACK_UPD);
}

VIWB_D void terminate(WinWork &ww, int term) { ww.status = ST_DONE; ww.term = term; }

enum { SCHUR_U = 4 };      // envelope entries per thread and trip of the Schur subtraction

// max |x - Plus(x, -g)| over one fixed block (ambient infinity norm of the projected gradient step)
VIWB_D double block_grad_inf(int b, unsigned mask, const double *x, const double *gneg) {
    const int gs = blk_size(b);
    double out[9], m = 0.0;          // the largest fixed block is a speed-bias (9)
    if (gs == 7) pose_plus(x, gneg, mask, out);
    else if (gs == 4) quat_plus(x, gneg, mask, out);
    else for (int i = 0; i < gs; i++) out[i] = x[i] + gneg[i];
    for (int i = 0; i < gs; i++) m = fmax(m, fabs(x[i] - out[i]));
    return m;
}

VIWB_D void solve_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by;
    const int w = bx;
    const WinMeta &m = bd.meta[w];
    WinWork &ww = bd.work[w];
    if (ww.status != ST_RUNNING) return;
    const Opts &op = bd.opt;
    SolveSmem s; carve(s, smem, nt, bd.env_max, bd.nf_max);
    const int nf = m.nf, N = m.nlm, vo = vec_off(bd, w);
    for (int i = tid; i < nf; i += nt) s.fst[i] = m.efirst[i];
    for (int i = tid; i <= nf; i += nt) s.rp[i] = bd.chol_plan[m.plan_off + i];
    double *x = bd.x_cur + m.state_off, *xc = bd.x_cand + m.state_off;
    double *g_scale = bd.v_scale + vo, *g_D = bd.v_D + vo, *g_sg = bd.v_sgrad + vo, *g_gn = bd.v_gn + vo;
    double *wug = bd.v_wug + m.lm_off, *wun = bd.v_wun + m.lm_off;      // per landmark: w_k . u_g (Cauchy direction) and w_k . (C y) (Gauss-Newton step), reused by the quadratic forms
    const double *lm_a = bd.lm_a + m.lm_off, *lm_g = bd.lm_g + m.lm_off, *lm_gamma = bd.lm_gamma + m.lm_off, *lm_sc = bd.lm_scale + m.lm_off;
    const double *W = bd.lm_W + (size_t)m.lm_off * VSUB;
    double *Hpk = bd.Hpk + (size_t)w * (TFIX * (TFIX + 1) / 2), *gpk = bd.gpk + (size_t)w * TFIX;
    const double *Tvis = bd.Tvis + (size_t)w * VSUB * VSUB, *tvec = bd.tvec + (size_t)w * VSUB;
    const double min_mu = 1e-8, max_mu = 1.0, mu_inc = 10.0;
    SOLVE_PROBE_START();

    // compact -> visual index map
    for (int b = tid; b < NB; b += nt) if (m.tcol[b] >= 0) for (int k = 0; k < blk_tsize(b); k++) s.vmap[m.tcol[b] + k] = blk_voff(b) >= 0 ? blk_voff(b) + k : -1;
    VIWB_SYNC();

    if (mode == 2) { assemble_H(bd, w, s, nf, Hpk, gpk, tid, nt); return; }     // debug hook: normal equations only
    bool assembled = false;

    // ================= phase A: decision on the pending candidate ==================================
    double c_part[SOLVE_VPT][1] = {};
    VIWB_VT_LOOP(j, vt) for (int k = vt; k < N; k += SOLVE_VNT) c_part[j][0] += bd.lm_cost[m.lm_off + k];
    vblock_sum_n<1>(c_part, tid, nt, s.red);
    const double cand_cost = c_part[0][0] + ww.small_cost;
    bool new_lin = false;
    if (ww.phase == PH_INIT) {
        if (tid == 0) { ww.x_cost = cand_cost; ww.initial_cost = cand_cost; ww.num_iterations = 1; }
        new_lin = true;
        for (int i = tid; i < SFIX + N; i += nt) x[i] = xc[i];
    } else {
        // ParameterToleranceReached / FunctionToleranceReached / IsStepSuccessful (trust_region_minimizer.cc)
        int verdict = 0;   // 0 rejected, 1 accepted, 2 converged
        const double cost_change = ww.x_cost - cand_cost;
        if (ww.step_norm <= op.parameter_tolerance * (ww.x_norm + op.parameter_tolerance)) verdict = 2;
        else if (fabs(cost_change) <= op.function_tolerance * ww.x_cost) verdict = 2;
        else if (cost_change / ww.model_cost_change > op.min_relative_decrease) verdict = 1;
        if (verdict == 2) { VIWB_SYNC(); if (tid == 0) terminate(ww, 0); return; }
        if (verdict == 1) {
            for (int i = tid; i < SFIX + N; i += nt) x[i] = xc[i];
            new_lin = true;
        }
        VIWB_SYNC();
        if (tid == 0) {
            const double rd = cost_change / ww.model_cost_change;
            if (verdict == 1) {
                ww.x_cost = cand_cost; ww.successful++;
                if (rd < 0.25) ww.radius *= 0.5;                                 // DoglegStrategy::StepAccepted
                if (rd > 0.75) ww.radius = fmax(ww.radius, 3.0 * ww.dogleg_step_norm);
                ww.mu = fmax(min_mu, 2.0 * ww.mu / mu_inc);
                ww.reuse = 0;
            } else { ww.radius *= 0.5; ww.reuse = 1; }                           // StepRejected
            ww.num_iterations++;
        }
        VIWB_SYNC();
        // FinalizeIterationAndCheckIfMinimizerCanContinue (gradient tolerance is tested in phase B)
        if (ww.iteration >= op.max_num_iterations || mode == 3) { VIWB_SYNC(); if (tid == 0) terminate(ww, 1); return; }   // mode 3: max_solver_time reached
        if (ww.radius <= op.min_radius) { VIWB_SYNC(); if (tid == 0) terminate(ww, 0); return; }
    }
    VIWB_SYNC();
    if (new_lin) {   // x_norm over the active blocks
        double a[SOLVE_VPT][1] = {};
        VIWB_VT_LOOP(j, vt) {
            for (int b = vt; b < NB; b += SOLVE_VNT) if (m.tcol[b] >= 0) for (int k = 0; k < blk_size(b); k++) a[j][0] += x[blk_off(b) + k] * x[blk_off(b) + k];
            for (int k = vt; k < N; k += SOLVE_VNT) a[j][0] += x[SFIX + k] * x[SFIX + k];
        }
        vblock_sum_n<1>(a, tid, nt, s.red);
        if (tid == 0) ww.x_norm = sqrt(a[0][0]);
    }
    if (ww.phase == PH_INIT && op.max_num_iterations <= 0) { VIWB_SYNC(); if (tid == 0) terminate(ww, 1); return; }
    VIWB_SYNC();

    // ================= phase B: compute a trust-region step (loops while the step is invalid) =========
    for (;;) {
        if (tid == 0) ww.iteration++;
        VIWB_SYNC();
        SOLVE_MARK(SPH_PRO);
        bool ls_failure = false;
        if (!ww.reuse) {
            VIWB_SYNC();
            if (tid == 0) ww.reuse = 1;
            if (!assembled) { assemble_H(bd, w, s, nf, Hpk, gpk, tid, nt); assembled = true; }
            else load_H(Hpk, s, nf, tid, nt);
            SOLVE_MARK(SPH_ASM);
            if (ww.first) {
                for (int i = tid; i < nf; i += nt) g_scale[i] = op.jacobi_scaling ? 1.0 / (1.0 + sqrt(SKY(s, i, i))) : 1.0;
            }
            VIWB_SYNC();
            if (new_lin) {
                // gradient_max_norm = |x - Plus(x, -g)|_inf  (unscaled gradient)
                double gm = 0.0;
                for (int b = tid; b < NB; b += nt) if (m.tcol[b] >= 0) {
                    double gneg[9];
                    for (int k = 0; k < blk_tsize(b); k++) gneg[k] = -gpk[m.tcol[b] + k];
                    gm = fmax(gm, block_grad_inf(b, m.mask[b], x + blk_off(b), gneg));
                }
                for (int k = tid; k < N; k += nt) gm = fmax(gm, fabs(lm_g[k]));
                gm = block_max(gm, tid, nt, s.red);
                if (tid == 0) ww.gradient_max_norm = gm;
                if (gm <= op.gradient_tolerance) { VIWB_SYNC(); if (tid == 0) terminate(ww, 0); return; }
            }
            // D = sqrt(clamp(diag(J_s^T J_s))), scaled gradient, Cauchy direction u_g = c o (sgrad / D)
            double n2[SOLVE_VPT][1] = {};
            VIWB_VT_LOOP(j, vt) {
                for (int i = vt; i < nf; i += SOLVE_VNT) {
                    const double sc = g_scale[i];
                    double d2 = sc * sc * SKY(s, i, i);
                    d2 = fmin(fmax(d2, op.min_lm_diagonal), op.max_lm_diagonal);
                    const double D = sqrt(d2); g_D[i] = D;
                    const double sg = sc * gpk[i] / D; g_sg[i] = sg; n2[j][0] += sg * sg;
                    s.ug[i] = sc * sg / D;
                }
                for (int k = vt; k < N; k += SOLVE_VNT) {
                    const double c = lm_sc[k];
                    double d2 = c * c * lm_a[k]; d2 = fmin(fmax(d2, op.min_lm_diagonal), op.max_lm_diagonal);
                    const double D = sqrt(d2); g_D[TFIX + k] = D;
                    const double sg = c * lm_g[k] / D; g_sg[TFIX + k] = sg; n2[j][0] += sg * sg;
                }
            }
            vblock_sum_n<1>(n2, tid, nt, s.red);
            SOLVE_MARK(SPH_DSC);
            // q_gg = |J u_g|^2, l_g = g . u_g
            symv(s, nf, s.ug, s.Hu, tid, nt);
            to_vis(s, nf, s.ug, s.uvis, tid, nt);
            double ql[SOLVE_VPT][2] = {};      // q, l
            VIWB_VT_LOOP(j, vt) {
                for (int i = vt; i < nf; i += SOLVE_VNT) { ql[j][0] += s.ug[i] * s.Hu[i]; ql[j][1] += gpk[i] * s.ug[i]; }
                VIWB_VLM_LOOP(k, vt, N) {
                    // the landmark's scalars are fetched (warp-uniform loads) before the dot product so that both latencies overlap
                    const double lsc = lm_sc[k], lsg = g_sg[TFIX + k], lD = g_D[TFIX + k], la = lm_a[k], lg = lm_g[k];
                    const double dw = warp_dot80(W + (size_t)k * VSUB, s.uvis, lane);
                    if (lane == 0) {
                        wug[k] = dw;
                        const double ul = lsc * lsg / lD;
                        ql[j][0] += 2.0 * ul * dw + la * ul * ul;
                        ql[j][1] += lg * ul;
                    }
                }
            }
            vblock_sum_n<2>(ql, tid, nt, s.red);
            if (tid == 0) { const double q = ql[0][0], n2s = n2[0][0]; ww.sgrad_norm = sqrt(n2s); ww.q_gg = q; ww.l_g = ql[0][1]; ww.alpha = n2s / q; }
            VIWB_SYNC();
            SOLVE_MARK(SPH_CAUCHY);
            // ---- Gauss-Newton step: (J^T J + mu D^2) y = J^T r through the Schur complement
            ls_failure = true;
            bool h_dirty = false;
            while (ww.mu < max_mu) {
                if (h_dirty) load_H(Hpk, s, nf, tid, nt);
                const double mu = ww.mu;
                const bool t_ok = (mu == ww.mu_lin);          // gamma / T / tvec were built for mu_lin
                // S = C (H - T) C + mu D^2 ; rhs = C (g - tvec)     (entry-parallel over the envelope: a thread takes SCHUR_U entries
                // per trip, finds their rows by bisection of rp and issues all their T loads before it updates the first one)
                {
                    for (int i = tid; i < nf; i += nt) {
                        const int vi = s.vmap[i];
                        double r = gpk[i];
                        if (vi >= 0) {
                            if (t_ok) r -= tvec[vi];
                            else { double t = 0.0; for (int k = 0; k < N; k++) { const double c = lm_sc[k], sk = c * c * lm_a[k], Dk = g_D[TFIX + k]; t += (c * c / (sk + mu * Dk * Dk)) * W[(size_t)k * VSUB + vi] * lm_g[k]; } r -= t; }
                        }
                        s.y[i] = g_scale[i] * r;
                    }
                    const int ne = s.rp[nf];
                    for (int e0 = tid; e0 < ne; e0 += SCHUR_U * nt) {
                        int ii[SCHUR_U], jj[SCHUR_U];
                        double tv[SCHUR_U];
#pragma unroll
                        for (int u = 0; u < SCHUR_U; u++) {
                            const int e = e0 + u * nt;
                            int lo = 0, hi = nf;                    // row: the last i with rp[i] <= e
                            if (e < ne) while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (s.rp[mid] <= e) lo = mid; else hi = mid; }
                            ii[u] = lo; jj[u] = s.fst[lo] + e - s.rp[lo];
                            const int vi = s.vmap[lo], vj = e < ne ? s.vmap[jj[u]] : -1;
                            tv[u] = (t_ok && vi >= 0 && vj >= 0) ? Tvis[vi * VSUB + vj] : 0.0;
                        }
#pragma unroll
                        for (int u = 0; u < SCHUR_U; u++) {
                            const int e = e0 + u * nt, i = ii[u], j = jj[u];
                            if (e >= ne) break;
                            const int vi = s.vmap[i], vj = s.vmap[j];
                            double hij = s.L[e];
                            if (vi >= 0 && vj >= 0) {
                                if (t_ok) hij -= tv[u];
                                else {
                                    double t = 0.0;
                                    for (int k = 0; k < N; k++) {
                                        const double c = lm_sc[k], sk = c * c * lm_a[k], Dk = g_D[TFIX + k];
                                        t += (c * c / (sk + mu * Dk * Dk)) * W[(size_t)k * VSUB + vi] * W[(size_t)k * VSUB + vj];
                                    }
                                    hij -= t;
                                }
                            }
                            hij *= g_scale[i] * g_scale[j];
                            if (i == j) hij += mu * g_D[i] * g_D[i];
                            s.L[e] = hij;
                        }
                    }
                }
                VIWB_SYNC();
                SOLVE_MARK(SPH_SCHUR);
                SOLVE_COUNT(SPH_FACT);
                h_dirty = true;
                if (tid == 0) ww.num_linear++;
                bool ok = cholesky_packed_rhs(s.L, s.rp, s.fst, s.y, nf, tid, nt, s.chol, s.Pt, s.ldp, bd.chol_plan + m.plan_off, sph);
                if (ok) chol_backsolve_blocked(s.L, s.rp, s.fst, s.y, s.xo, nf, tid, nt, sph);
                SOLVE_FLUSH();
                if (ok) {
                    // back-substitute the inverse depths (scaled): y_k = (c g_k - c w_k . (C y_f)) / h_k
                    for (int i = tid; i < nf; i += nt) s.u[i] = g_scale[i] * s.y[i];
                    VIWB_SYNC();
                    to_vis(s, nf, s.u, s.uvis, tid, nt);
                    double bad = 0.0;
                    for (int i = tid; i < nf; i += nt) { if (!isfinite(s.y[i])) bad = 1.0; g_gn[i] = -g_D[i] * s.y[i]; }
                    VIWB_LM_LOOP(k, N) {
                        const double c = lm_sc[k], Dk = g_D[TFIX + k], la = lm_a[k], lg = lm_g[k];
                        const double dw = warp_dot80(W + (size_t)k * VSUB, s.uvis, lane);
                        if (lane == 0) {
                            wun[k] = dw;
                            const double hk = c * c * la + mu * Dk * Dk;
                            const double yk = c * (lg - dw) / hk;
                            if (!isfinite(yk)) bad = 1.0;
                            g_gn[TFIX + k] = -Dk * yk;
                        }
                    }
                    bad = block_sum(bad, tid, nt, s.red);      // a count of non-finite values: exact in any order
                    ok = (bad == 0.0);
                    SOLVE_MARK(SPH_LM2);
                }
                if (!ok) { VIWB_SYNC(); if (tid == 0) ww.mu *= mu_inc; VIWB_SYNC(); continue; }
                ls_failure = false;
                break;
            }
            VIWB_SYNC();
            if (!ls_failure) {
                // q_gn, q_nn, l_n with u_n = c o (gn / D) = -c o y: s.u still holds c o y from the back-substitution, and the landmark
                // rows' products with it (wun) and with u_g (wug) are on file -- no third pass over W
                load_H(Hpk, s, nf, tid, nt);
                for (int i = tid; i < nf; i += nt) s.u[i] = -s.u[i];
                VIWB_SYNC();
                symv(s, nf, s.u, s.Hu, tid, nt);
                double f[SOLVE_VPT][5] = {};      // q_nn, q_gn, l_n, |gn|^2, sgrad . gn
                VIWB_VT_LOOP(j, vt) {
                    for (int i = vt; i < nf; i += SOLVE_VNT) {
                        const double sg = g_sg[i], ug = g_scale[i] * sg / g_D[i];      // the Cauchy direction, as the Cauchy point computed it
                        f[j][0] += s.u[i] * s.Hu[i]; f[j][1] += ug * s.Hu[i]; f[j][2] += gpk[i] * s.u[i];
                        f[j][3] += g_gn[i] * g_gn[i]; f[j][4] += sg * g_gn[i];
                    }
                    for (int k = vt; k < N; k += SOLVE_VNT) {
                        const double c = lm_sc[k], Dk = g_D[TFIX + k], ggn = g_gn[TFIX + k], gsg = g_sg[TFIX + k], la = lm_a[k], lg = lm_g[k];
                        const double dn = -wun[k], dg = wug[k];
                        const double un = c * ggn / Dk, ug = c * gsg / Dk;
                        f[j][0] += 2.0 * un * dn + la * un * un;
                        f[j][1] += ug * dn + un * dg + la * ug * un;
                        f[j][2] += lg * un;
                        f[j][3] += ggn * ggn; f[j][4] += gsg * ggn;
                    }
                }
                vblock_sum_n<5>(f, tid, nt, s.red);
                if (tid == 0) { ww.q_nn = f[0][0]; ww.q_gn = f[0][1]; ww.l_n = f[0][2]; ww.gn_norm = sqrt(f[0][3]); ww.sgrad_dot_gn = f[0][4]; }
            }
            VIWB_SYNC();
            SOLVE_MARK(SPH_FORMS);
            if (tid == 0) ww.first = 0;
            VIWB_SYNC();
        }
        // ---- ComputeTraditionalDoglegStep: step = ca * sgrad + cb * gn (scaled space), then / D
        double ca = 0.0, cb = 0.0, mcc = 0.0, dsn = 0.0;
        bool valid = false;
        if (!ls_failure) {
            const double gnorm = ww.sgrad_norm, gnn = ww.gn_norm, radius = ww.radius, alpha = ww.alpha;
            if (gnn <= radius) { ca = 0.0; cb = 1.0; dsn = gnn; }
            else if (gnorm * alpha >= radius) { ca = -(radius / gnorm); cb = 0.0; dsn = radius; }
            else {
                const double b_dot_a = -alpha * ww.sgrad_dot_gn, a_sq = (alpha * gnorm) * (alpha * gnorm);
                const double bma = a_sq - 2.0 * b_dot_a + gnn * gnn, c = b_dot_a - a_sq;
                const double d = sqrt(c * c + bma * (radius * radius - a_sq));
                const double beta = (c <= 0) ? (d - c) / bma : (radius * radius - a_sq) / (d + c);
                ca = -alpha * (1.0 - beta); cb = beta;
                dsn = sqrt(ca * ca * gnorm * gnorm + 2.0 * ca * cb * ww.sgrad_dot_gn + cb * cb * gnn * gnn);
            }
            // model_cost_change = -(J t)^T (r + J t / 2) = -(ca l_g + cb l_n) - (ca^2 q_gg + 2 ca cb q_gn + cb^2 q_nn) / 2
            mcc = -(ca * ww.l_g + cb * ww.l_n) - 0.5 * (ca * ca * ww.q_gg + 2.0 * ca * cb * ww.q_gn + cb * cb * ww.q_nn);
            valid = mcc > 0.0;
        }
        VIWB_SYNC();
        if (!valid) {
            // HandleInvalidStep + DoglegStrategy::StepIsInvalid
            bool stop = false;
            if (tid == 0) {
                ww.num_invalid++;
                if (ww.num_invalid >= op.max_invalid) { terminate(ww, 2); }
                else {
                    ww.mu *= mu_inc; ww.reuse = 0; ww.num_iterations++;
                    if (ww.iteration >= op.max_num_iterations) terminate(ww, 1);
                    else if (ww.radius <= op.min_radius) terminate(ww, 0);
                }
            }
            VIWB_SYNC();
            stop = (ww.status != ST_RUNNING);
            if (stop) return;
            new_lin = false;
            continue;
        }
        // ---- candidate: x (+) (step o scale)
        double sn[SOLVE_VPT][1] = {};
        VIWB_VT_LOOP(j, vt) {
        for (int b = vt; b < NB; b += SOLVE_VNT) {
            const int o = blk_off(b), gs = blk_size(b);
            if (m.tcol[b] >= 0) {
                double d[9], out[9];
                for (int k = 0; k < blk_tsize(b); k++) { const int i = m.tcol[b] + k; d[k] = (ca * g_sg[i] + cb * g_gn[i]) / g_D[i] * g_scale[i]; }
                if (gs == 7) pose_plus(x + o, d, m.mask[b], out);
                else if (gs == 4) quat_plus(x + o, d, m.mask[b], out);
                else for (int k = 0; k < gs; k++) out[k] = x[o + k] + d[k];
                for (int k = 0; k < gs; k++) { xc[o + k] = out[k]; const double e = x[o + k] - out[k]; sn[j][0] += e * e; }
            } else for (int k = 0; k < gs; k++) xc[o + k] = x[o + k];
        }
        for (int k = vt; k < N; k += SOLVE_VNT) {
            const double d = (ca * g_sg[TFIX + k] + cb * g_gn[TFIX + k]) / g_D[TFIX + k] * lm_sc[k];
            xc[SFIX + k] = x[SFIX + k] + d; sn[j][0] += d * d;
        }
        }
        vblock_sum_n<1>(sn, tid, nt, s.red);
        if (tid == 0) {
            ww.num_invalid = 0; ww.step_norm = sqrt(sn[0][0]); ww.model_cost_change = mcc; ww.dogleg_step_norm = dsn;
            ww.phase = PH_CAND;
            ww.mu_lin = fmax(min_mu, 2.0 * ww.mu / mu_inc);      // the candidate's linearisation is solved with the post-accept mu
        }
        SOLVE_MARK(SPH_DOGLEG);
        SOLVE_COUNT(SPH_STEPS);
        return;
    }
}

}  // namespace viwb
