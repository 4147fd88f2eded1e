// kernels_fused.cuh -- the solver linearisation of windows whose camera extrinsics and td are constant (C1 / C2 / C6 shapes), and the
// FP64 tensor-core (DMMA, mma.sync.m8n8k4.f64) products of the normal equations.
//
//   lin_vis_lm  (compact windows) one block per HOST RUN: the landmarks hosted in one frame, in landmark order, as tiles of whole landmarks
//               (<= LMB_FACTORS factors).  Per tile, thread per factor evaluates residual, Huber, tangent Jacobians (the three projection
//               factors, factor/projection*Factor.cpp) into a shared-memory tile; the block then
//                 - reduces the per-landmark quantities straight from the tile: a = |J_l|^2, g_l, the cost, the Schur weight gamma and the
//                   row W = J_p^T J_l -- the per-factor records of lin_vis never exist, lm_reduce does not run, and
//                 - forms G = sum_f X_f^T X_f of every (host, observer) pair from the tile, X = [A | B | r] (2 x 13; G: A^T A | A^T B | A^T r /
//                   B^T B | B^T r), per chunk of PAIR_CHUNK records, as a true GEMM on the FP64 tensor pipe (three 8 x 8 accumulator tiles, K = 2
//                   rows per factor): the X records never leave the SM.
//   lin_vis_lm_wide  (wide windows, marginalisation) the same per group of whole landmarks, storing each X record (2 x 26) in FRAME-PAIR order;
//   asm_pairs_wide   one warp per chunk of one frame pair's records turns them into G.  Both replace the three gather walks of asm_items (two
//               frame lists + one pair list per factor).
//   syrk_mma    T = sum_k gamma_k w_k w_k^T (80 x 80) and tvec = sum_k gamma_k g_k w_k as one [80 x K] x [K x 81] DMMA product per window
//               (the dense Schur block of north_star), operands staged by cp.async into a conflict-free shared-memory layout.
// The emulation build (VIWB_HOST_EMU) states the same sums in scalar code.
#pragma once
#include "kernels_asm.cuh"

namespace viwb {

// D (8x8) += A (8x4, row) * B (4x8, col): lane l holds A[l/4][l%4], B[l%4][l/4], D[l/4][2*(l%4) + {0,1}]
#ifndef VIWB_HOST_EMU
VIWB_D void dmma884(double (&c)[2], double a, double b) {
    asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
}
#endif

// ------------------------------------------------------------------------------------------------ record layouts
// X row of a factor (one per residual row): COMPACT  A(6) | B(6) | r | 0            (14 doubles, 13 used): windows whose ex0 / ex1 / td are constant
//                                           WIDE     A(6) | B(6) | E0(6) | E1(6) | td | r | 0 0   (28 doubles, 26 used): extrinsics / td estimated, and
//                                                    every marginalisation (the prior keeps those blocks whatever the solver does with them)
// G = sum X^T X lives in a frame of NTC x NTC tiles of 8 x 8; the NTILE upper-triangular tiles are stored in mma.m8n8k4 accumulator order.
template <bool WIDE> struct XL {
    enum { ROW = WIDE ? 28 : 14, REC = 2 * ROW, USED = WIDE ? 26 : 13, RCOL = WIDE ? 25 : 12, NTC = WIDE ? 4 : 2, NTILE = NTC * (NTC + 1) / 2, OUT = 64 * NTILE,
           TS = REC + 3, U = REC, C = REC + 2,                      // shared-memory tile row: X record | J_lambda (2) | rho / 2 ; odd stride
           NLM = WIDE ? 22 : 9,                                     // per-landmark outputs: host block of W (6), a, g, cost (+ E0 (6), E1 (6), td columns of W)
           FR = WIDE ? 27 + 78 : 27,                                // per-frame reduce outputs: diagonal block (21) + gradient (6) (+ pose x common 6 x 13)
           RED = NFR * FR + NPAIR * 36 + (WIDE ? 91 + 13 : 0) };    // pair_reduce outputs per window
};
// entry (i, j) of a chunk's G as pair_chunk stores it (G is symmetric: tile (tr > tc) is read through its transpose)
template <bool WIDE> VIWB_HD double pair_G(const double *out, int i, int j) {
    if ((i >> 3) > (j >> 3)) { const int t = i; i = j; j = t; }
    const int tr = i >> 3, tc = j >> 3, tl = tr * XL<WIDE>::NTC - tr * (tr - 1) / 2 + (tc - tr);
    return out[64 * tl + 2 * (((i & 7) << 2) + ((j & 7) >> 1)) + (j & 1)];
}

// ------------------------------------------------------------------------------------------------ lin_vis_lm
// The steps of one tile of whole landmarks, shared by the host runs (compact) and the landmark blocks (wide, marginalisation).
// Shared-memory tile row of a factor: X record (2 x ROW) | J_lambda (2) | rho / 2; meta word: landmark (window-local) << 12 | fi << 8 | fj << 4 | type << 2 | dup
VIWB_HD size_t lin_vis_lm_smem_doubles(bool wide) { return (size_t)LMB_FACTORS * (wide ? (int)XL<true>::TS : (int)XL<false>::TS) + LMB_FACTORS / 2 + 2; }      // tile + per-factor meta ints
// step 1: one thread per factor evaluates residual, Huber, tangent Jacobians into its tile row
template <bool WIDE>
VIWB_D void lin_factor_row(const BatchDev &bd, const WinMeta &m, const double *x, int f, int type, int fi, int fj, double *row) {
    typedef XL<WIDE> L;
    double obs[12];
    for (int k = 0; k < 12; k++) obs[k] = bd.vis_obs[(size_t)f * 12 + k];
    VisOut o;
    vis_eval_t<WIDE>(type, obs, x + 7 * fi, x + 7 * fj, x + blk_off(BLK_EX0), x + blk_off(BLK_EX1), x[SFIX + bd.vis_lm[f]], x[blk_off(BLK_TD)], m.S_vis, true, o);
    double half_rho;
    const double sc = huber_scale(o.r[0] * o.r[0] + o.r[1] * o.r[1], m.huber, half_rho);
    for (int h = 0; h < 2; h++) {      // row h of X
        double *xr = row + h * L::ROW;
        for (int q = 0; q < 6; q++) { xr[q] = o.JA[6 * h + q] * sc; xr[6 + q] = o.JB[6 * h + q] * sc; }
        if (WIDE) { for (int q = 0; q < 6; q++) { xr[12 + q] = o.JE0[6 * h + q] * sc; xr[18 + q] = o.JE1[6 * h + q] * sc; } xr[24] = o.Jtd[h] * sc; xr[25] = o.r[h] * sc; xr[26] = 0.0; xr[27] = 0.0; }
        else { xr[12] = o.r[h] * sc; xr[13] = 0.0; }
    }
    row[L::U] = o.Jl[0] * sc; row[L::U + 1] = o.Jl[1] * sc; row[L::C] = half_rho;
}
// rho / 2 of one factor without Jacobians (cost_only)
template <bool WIDE>
VIWB_D double lin_factor_cost(const BatchDev &bd, const WinMeta &m, const double *x, int f) {
    double obs[12];
    for (int k = 0; k < 12; k++) obs[k] = bd.vis_obs[(size_t)f * 12 + k];
    VisOut o;
    vis_eval_t<WIDE>(bd.vis_type[f], obs, x + 7 * bd.vis_fi[f], x + 7 * bd.vis_fj[f], x + blk_off(BLK_EX0), x + blk_off(BLK_EX1), x[SFIX + bd.vis_lm[f]], x[blk_off(BLK_TD)], m.S_vis, false, o);
    double half_rho;
    huber_scale(o.r[0] * o.r[0] + o.r[1] * o.r[1], m.huber, half_rho);
    return half_rho;
}
// step 2b: observing-frame block of W of the factor in tile row t (its six components: three 16-byte stores); two factors of one landmark seen
//          from the same frame (left and right camera) are consecutive in the table: the first one writes the sum
template <bool WIDE, bool MARG>
VIWB_D void lin_w_observer(const BatchDev &bd, const WinMeta &m, const double *tile, const int *meta, int t) {
    typedef XL<WIDE> L;
    const int mt = meta[t], dup = mt & 3;
    if (((mt >> 2) & 3) == 2 || dup == 2) return;
    if (MARG && ((mt >> 8) & 15) != 0) return;
    const double *row = tile + (size_t)t * L::TS;
    const double u0 = row[L::U], u1 = row[L::U + 1];
    double v[6];
#pragma unroll
    for (int q = 0; q < 6; q++) v[q] = row[6 + q] * u0 + row[L::ROW + 6 + q] * u1;
    if (dup == 1) {
        const double *r2 = row + L::TS; const double w0 = r2[L::U], w1 = r2[L::U + 1];
#pragma unroll
        for (int q = 0; q < 6; q++) v[q] += r2[6 + q] * w0 + r2[L::ROW + 6 + q] * w1;
    }
    double *dst = bd.lm_W + (size_t)(m.lm_off + (mt >> 12)) * VSUB + 6 * ((mt >> 4) & 15);      // even offset: 16-byte aligned
#ifdef VIWB_HOST_EMU
    for (int q = 0; q < 6; q++) dst[q] = v[q];
#else
    double2 *d2 = reinterpret_cast<double2 *>(dst);
    d2[0] = make_double2(v[0], v[1]); d2[1] = make_double2(v[2], v[3]); d2[2] = make_double2(v[4], v[5]);
#endif
}
// step 2c: item (landmark k, output q) with the landmark's factors in tile rows [a0, a1): host-frame block of W (6), a, g, cost (+ Jacobi scale and
//          Schur weight) (+ common columns of W).  Every output is sum_t row_t[ca] * p_t + row_t[cb] * q_t with (ca, cb) fixed per output and
//          (p, q) = (u0, u1) or, for the cost, (1, 0): no branch inside the factor loop
template <bool WIDE, bool MARG>
VIWB_D void lin_lm_output(const BatchDev &bd, const WinWork &ww, const double *tile, const int *meta, int k, int q, int a0, int a1) {
    typedef XL<WIDE> L;
    const bool part = a1 > a0 && (!MARG || ((meta[a0] >> 8) & 15) == 0);      // the landmark takes part (marginalisation: hosted in frame 0)
    // q < 6: A column q (one-frame factors carry A = 0); 6: u.u; 7: u.r; 8: cost; > 8 (WIDE): E0 (6) | E1 (6) | td = X columns 12 .. 24
    const int ca = q < 6 ? q : q == 6 ? (int)L::U : q == 7 ? (int)L::RCOL : q == 8 ? (int)L::C : 12 + (q - 9);
    const int cb = q < 6 ? (int)L::ROW + q : q == 6 ? (int)L::U + 1 : q == 7 ? (int)L::ROW + (int)L::RCOL : q == 8 ? (int)L::C : (int)L::ROW + 12 + (q - 9);
    const bool is_cost = q == 8;
    double s = 0.0;
    if (part) {
        const double *row = tile + (size_t)a0 * L::TS;
#pragma unroll 4
        for (int t = a0; t < a1; t++, row += L::TS) {
            const double u0 = is_cost ? 1.0 : row[L::U], u1 = is_cost ? 0.0 : row[L::U + 1];
            s += row[ca] * u0 + row[cb] * u1;
        }
    }
    if (q < 6) { if (part) bd.lm_W[(size_t)k * VSUB + 6 * ((meta[a0] >> 8) & 15) + q] = s; }
    else if (q == 7) bd.lm_g[k] = s;
    else if (q == 8) bd.lm_cost[k] = s;
    else if (q > 8) { if (part) bd.lm_W[(size_t)k * VSUB + 66 + (q - 9)] = s; }
    else {
        bd.lm_a[k] = s;
        if (MARG) bd.lm_gamma[k] = s;                                    // marginalisation keeps the pivot itself (0: the landmark is skipped)
        else if (!part) { bd.lm_gamma[k] = 0.0; if (ww.first) bd.lm_scale[k] = 1.0; }
        else {
            // Jacobi scale (first linearisation only) and the Schur weight for the mu this linearisation will be solved with:
            // scaled pivot h = c^2 a + mu * clamp(c^2 a); gamma = c^2 / h  (SURVEY Appendix B)
            double sc = bd.lm_scale[k];
            if (ww.first) { sc = bd.opt.jacobi_scaling ? 1.0 / (1.0 + sqrt(s)) : 1.0; bd.lm_scale[k] = sc; }
            const double s2 = sc * sc * s;
            double d2 = s2; if (d2 < bd.opt.min_lm_diagonal) d2 = bd.opt.min_lm_diagonal; if (d2 > bd.opt.max_lm_diagonal) d2 = bd.opt.max_lm_diagonal;
            bd.lm_gamma[k] = sc * sc / (s2 + ww.mu_lin * d2);
        }
    }
}

// ---- compact solver windows: one block per host run
// Every factor of a landmark has the landmark's host frame as fi (lower_count), so all records of pair (host, j) belong to one run, and the run meets
// them in landmark order, which is their frame-pair slot order.  The block runs the chunked product of asm_pairs_wide's pair_chunk from the tile:
// the accumulator restarts every PAIR_CHUNK records of a pair, a k-step takes records (chunk start + 2m, + 2m + 1) with the same lane mapping, and
// an odd chunk ends with a zero record.  Between tiles a pair's accumulator is parked in shared memory, and the first record of an open k-step (the
// partner is in the next tile) waits in the pair's carry slot.  A finished chunk goes to its pair_out slot, the last one when the run ends.
VIWB_HD size_t lin_vis_run_smem_doubles() {
    return lin_vis_lm_smem_doubles(false) + (size_t)NFR * (XL<false>::OUT + XL<false>::REC) + (NFR + 1) / 2;      // + parked accumulators, carry slots, record counts
}
VIWB_D void run_pairs(const BatchDev &bd, const RunDesc &rd, const double *tile, const int *meta, int nf, bool last, double *pacc, double *pcarry, int *pcount, int tid, int nt) {
    typedef XL<false> L;
#ifdef VIWB_HOST_EMU
    // the same per-chunk sums, record by record in slot order (the scalar statement of pair_chunk)
    (void)pcarry; (void)tid; (void)nt;
    for (int j = 0; j < NFR; j++) {
        if (rd.pfirst[j] < 0) continue;
        double *acc = pacc + (size_t)j * L::OUT;
        int n = pcount[j];
        auto flush = [&](int chunk) { double *out = bd.pair_out + (size_t)(rd.pfirst[j] + chunk) * bd.pout_stride; for (int e = 0; e < L::OUT; e++) { out[e] = acc[e]; acc[e] = 0.0; } };
        for (int t = 0; t < nf; t++) {
            const int mt = meta[t];
            if (((mt >> 2) & 3) == 2 || ((mt >> 4) & 15) != j) continue;
            for (int rr = 0; rr < 2; rr++) {
                const double *xr = tile + (size_t)t * L::TS + rr * L::ROW;
                int tt = 0;
                for (int tr = 0; tr < L::NTC; tr++) for (int tc = tr; tc < L::NTC; tc++, tt++)
                    for (int l = 0; l < 32; l++) for (int r = 0; r < 2; r++) {
                        const int a = 8 * tr + l / 4, b = 8 * tc + 2 * (l % 4) + r;
                        if (a < L::ROW && b < L::ROW) acc[64 * tt + 2 * l + r] += xr[a] * xr[b];
                    }
            }
            if (++n % PAIR_CHUNK == 0) flush(n / PAIR_CHUNK - 1);
        }
        if (last && n % PAIR_CHUNK) flush(n / PAIR_CHUNK);
        pcount[j] = n;
    }
#else
    const int lane = tid & 31, kk = lane & 3, fo = kk >> 1, rr = kk & 1, c0 = lane >> 2;
    for (int j = tid >> 5; j < NFR; j += nt >> 5) {      // warp-uniform: a pair belongs to one warp for the whole run
        if (rd.pfirst[j] < 0) continue;
        double2 *pa = reinterpret_cast<double2 *>(pacc + (size_t)j * L::OUT);
        double *carry = pcarry + (size_t)j * L::REC;
        double acc[L::NTILE][2];
#pragma unroll
        for (int t = 0; t < L::NTILE; t++) { const double2 v = pa[32 * t + lane]; acc[t][0] = v.x; acc[t][1] = v.y; }
        int n = pcount[j];                   // records of the pair so far; odd: the first record of the open k-step waits in `carry`
        const double *pend = carry;
        auto kstep = [&](const double *p0, const double *p1) {      // records p0, p1 (nullptr: the zero record that ends an odd chunk)
            const double *p = fo ? p1 : p0;
            double a[L::NTC];
#pragma unroll
            for (int t = 0; t < L::NTC; t++) a[t] = (p && c0 + 8 * t < L::ROW) ? p[rr * L::ROW + c0 + 8 * t] : 0.0;
            int t = 0;
#pragma unroll
            for (int tr = 0; tr < L::NTC; tr++)
#pragma unroll
                for (int tc = tr; tc < L::NTC; tc++, t++) dmma884(acc[t], a[tr], a[tc]);
        };
        auto flush = [&](int chunk) {
            double2 *out = reinterpret_cast<double2 *>(bd.pair_out + (size_t)(rd.pfirst[j] + chunk) * bd.pout_stride);
#pragma unroll
            for (int t = 0; t < L::NTILE; t++) { out[32 * t + lane] = make_double2(acc[t][0], acc[t][1]); acc[t][0] = 0.0; acc[t][1] = 0.0; }
        };
        for (int base = 0; base < nf; base += 32) {
            const int t = base + lane, mt = t < nf ? meta[t] : 0;
            unsigned msk = __ballot_sync(0xffffffffu, t < nf && ((mt >> 2) & 3) != 2 && ((mt >> 4) & 15) == j);
            while (msk) {
                const double *rec = tile + (size_t)(base + __ffs(msk) - 1) * L::TS;
                msk &= msk - 1;
                if (!(n & 1)) { pend = rec; n++; continue; }
                kstep(pend, rec);
                if (!(++n & (PAIR_CHUNK - 1))) flush(n / PAIR_CHUNK - 1);
            }
        }
        if (last) {
            if (n & (PAIR_CHUNK - 1)) { if (n & 1) kstep(pend, nullptr); flush(n / PAIR_CHUNK); }
        } else {
            if ((n & 1) && pend != carry) { __syncwarp(); if (lane < L::REC) carry[lane] = pend[lane]; }
#pragma unroll
            for (int t = 0; t < L::NTILE; t++) pa[32 * t + lane] = make_double2(acc[t][0], acc[t][1]);
        }
        if (lane == 0) pcount[j] = n;
    }
#endif
}
// cost_only (the round after the last allowed iteration): only the landmark costs are read afterwards (the decision on the pending candidate),
// so the residuals are evaluated without Jacobians and nothing else is written
VIWB_D void lin_vis_run_cost(const BatchDev &bd, int bx, int tid, int nt, double *smem) {
    const RunDesc &rd = bd.run_desc[bx];
    if (bd.work[rd.win].status != ST_RUNNING) return;
    const WinMeta &m = bd.meta[rd.win];
    const double *x = bd.x_cand + m.state_off;
    for (int ti = 0; ti < rd.ntile; ti++) {
        const RunTile tl = bd.run_tile[rd.t0 + ti];
        const int *fl = bd.run_f + tl.f0, *lm = bd.run_lm + 2 * (size_t)tl.l0;
        for (int t = tid; t < tl.nf; t += nt) smem[t] = lin_factor_cost<false>(bd, m, x, fl[t]);
        VIWB_SYNC();
        for (int kl = tid; kl < tl.nl; kl += nt) {
            const int k = lm[2 * kl], a0 = lm[2 * kl + 1], a1 = a0 + bd.lm_fptr[k + 1] - bd.lm_fptr[k];
            double s = 0.0;
            for (int t = a0; t < a1; t++) s += smem[t];
            bd.lm_cost[k] = s;
        }
        VIWB_SYNC();
    }
}
VIWB_D void lin_vis_run_body(const BatchDev &bd, int bx, int tid, int nt, double *smem) {
    typedef XL<false> L;
    const RunDesc &rd = bd.run_desc[bx];
    const WinWork &ww = bd.work[rd.win];
    if (ww.status != ST_RUNNING) return;
    const WinMeta &m = bd.meta[rd.win];
    const double *x = bd.x_cand + m.state_off;
    double *tile = smem;
    int *meta = (int *)(smem + (size_t)LMB_FACTORS * L::TS);
    double *pacc = smem + lin_vis_lm_smem_doubles(false), *pcarry = pacc + (size_t)NFR * L::OUT;
    int *pcount = (int *)(pcarry + (size_t)NFR * L::REC);
    for (int e = tid; e < NFR * L::OUT; e += nt) pacc[e] = 0.0;
    for (int e = tid; e < NFR; e += nt) pcount[e] = 0;
    for (int ti = 0; ti < rd.ntile; ti++) {
        const RunTile tl = bd.run_tile[rd.t0 + ti];
        const int *fl = bd.run_f + tl.f0, *lm = bd.run_lm + 2 * (size_t)tl.l0;      // the tile's factors; its landmarks (global index, first tile row)
        // ---- 0: the W rows of these landmarks start from zero (frames that do not observe a landmark keep zero blocks)
        for (int e = tid; e < tl.nl * VSUB; e += nt) { const int kl = e / VSUB; bd.lm_W[(size_t)lm[2 * kl] * VSUB + (e - kl * VSUB)] = 0.0; }
        // ---- 1: one thread per factor (the launch has LMB_FACTORS threads: at most one factor each, no loop to hoist the window's constants out of)
#ifdef VIWB_HOST_EMU
        for (int t = tid; t < tl.nf; t += nt) {
#else
        if (const int t = tid; t < tl.nf) {
#endif
            const int f = fl[t];
            const int code = bd.vis_code[f], type = code & 3, fi = (code >> 2) & 15, fj = (code >> 6) & 15;      // the wire format's code word: one load instead of four
            meta[t] = (bd.vis_lm[f] << 12) | (fi << 8) | (fj << 4) | (type << 2) | ((code >> 10) & 3);
            lin_factor_row<false>(bd, m, x, f, type, fi, fj, tile + (size_t)t * L::TS);
        }
        VIWB_SYNC();
        // ---- 2b, 2c and the pair products: all read the tile
        for (int t = tid; t < tl.nf; t += nt) lin_w_observer<false, false>(bd, m, tile, meta, t);
        for (int e = tid; e < tl.nl * L::NLM; e += nt) {
            const int kl = e / L::NLM, k = lm[2 * kl], a0 = lm[2 * kl + 1];
            lin_lm_output<false, false>(bd, ww, tile, meta, k, e - L::NLM * kl, a0, a0 + bd.lm_fptr[k + 1] - bd.lm_fptr[k]);
        }
        run_pairs(bd, rd, tile, meta, tl.nf, ti + 1 == rd.ntile, pacc, pcarry, pcount, tid, nt);
        VIWB_SYNC();      // the next tile overwrites the tile
    }
}

// ---- wide solver windows and marginalisation: one block per group of WHOLE landmarks (<= LMB_FACTORS factors); each X record also goes to its
//      frame-pair slot in xrec for asm_pairs_wide.
// MARG = false: solver linearisation at x_cand of the wide fused windows.
// MARG = true: marginalisation linearisation at x_cur of the windows that drop frame 0: only the factors hosted there take part; every other
//              landmark of the window gets gamma = 0 and a zero row of W (syrk multiplies its row by that weight).
template <bool MARG>
VIWB_D void lin_vis_lm_body(const BatchDev &bd, int bx, int tid, int nt, double *smem, bool cost_only = false) {
    typedef XL<true> L;
    const LmbDesc &ds = bd.lmb_desc[bx];
    const int w = ds.win, k0 = ds.k0, k1 = ds.k1, f0 = ds.f0, nf = ds.nf;      // window; global landmark range; its factors (consecutive, <= LMB_FACTORS)
    const WinWork &ww = bd.work[w];
    const WinMeta &m = bd.meta[w];
    if (MARG) { if (!m.mfused) return; }
    else { if (ww.status != ST_RUNNING || !m.fused || !m.has_common) return; }
    double *tile = smem;
    int *meta = (int *)(smem + (size_t)LMB_FACTORS * L::TS);
    const double *x = (MARG ? bd.x_cur : bd.x_cand) + m.state_off;
    const int *vpos = MARG ? bd.mvis_pos : bd.vis_pos;
    double *xbase = bd.xrec + (size_t)(MARG ? m.mxrec_off : m.xrec_off);
    if (MARG) {      // a block without a landmark hosted in frame 0 takes no part: its landmarks get weight 0 and nothing is evaluated
        if (tid == 0) meta[LMB_FACTORS] = 0;
        VIWB_SYNC();
        bool mine = false;
        for (int t = tid; t < nf; t += nt) if (bd.vis_fi[f0 + t] == 0) mine = true;
        if (mine) meta[LMB_FACTORS] = 1;
        VIWB_SYNC();
        if (!meta[LMB_FACTORS]) {
            for (int k = k0 + tid; k < k1; k += nt) { bd.lm_a[k] = 0.0; bd.lm_g[k] = 0.0; bd.lm_cost[k] = 0.0; bd.lm_gamma[k] = 0.0; }
            return;
        }
    }
    // ---- 0: the W rows of these landmarks start from zero (frames that do not observe a landmark keep zero blocks).  Marginalisation: only the
    //         rows of the landmarks hosted in frame 0 (below, once the hosts are known); the other rows keep their finite solver values and are
    //         multiplied by the weight gamma = 0
    if (!MARG && cost_only) {
        for (int t = tid; t < nf; t += nt) tile[t] = lin_factor_cost<true>(bd, m, x, f0 + t);
        VIWB_SYNC();
        for (int k = k0 + tid; k < k1; k += nt) {
            double s = 0.0;
            for (int t = bd.lm_fptr[k] - f0; t < bd.lm_fptr[k + 1] - f0; t++) s += tile[t];
            bd.lm_cost[k] = s;
        }
        return;
    }
    if (!MARG) { double *Wb = bd.lm_W + (size_t)k0 * VSUB; for (int e = tid; e < (k1 - k0) * VSUB; e += nt) Wb[e] = 0.0; }
    // ---- 1: one thread per factor
    for (int t = tid; t < nf; t += nt) {
        const int f = f0 + t;
        const int code = bd.vis_code[f], type = code & 3, fi = (code >> 2) & 15, fj = (code >> 6) & 15;      // the wire format's code word: one load instead of four
        meta[t] = (bd.vis_lm[f] << 12) | (fi << 8) | (fj << 4) | (type << 2) | ((code >> 10) & 3);
        double *row = tile + (size_t)t * L::TS;
        if (MARG && fi != 0) { row[L::U] = 0.0; row[L::U + 1] = 0.0; row[L::C] = 0.0; continue; }      // not hosted in the dropped frame: takes no part
        lin_factor_row<true>(bd, m, x, f, type, fi, fj, row);
        // the X record goes straight to its frame-pair slot: aligned 16-byte stores (the thread re-reads its own tile row: values it has just written)
        const int pos = vpos[f];
        if (pos >= 0) {
            double *xr = xbase + (size_t)pos * L::REC;
#ifdef VIWB_HOST_EMU
            for (int q = 0; q < L::REC; q++) xr[q] = row[q];
#else
            double2 *d2 = reinterpret_cast<double2 *>(xr);
#pragma unroll
            for (int q = 0; q < L::REC / 2; q++) d2[q] = make_double2(row[2 * q], row[2 * q + 1]);
#endif
        }
    }
    VIWB_SYNC();
    if (MARG) {
        for (int e = tid; e < (k1 - k0) * VSUB; e += nt) {
            const int kl = e / VSUB, a0 = bd.lm_fptr[k0 + kl] - f0, a1 = bd.lm_fptr[k0 + kl + 1] - f0;
            if (a1 > a0 && ((meta[a0] >> 8) & 15) == 0) bd.lm_W[(size_t)k0 * VSUB + e] = 0.0;
        }
        VIWB_SYNC();
    }
    for (int t = tid; t < nf; t += nt) lin_w_observer<true, MARG>(bd, m, tile, meta, t);
    for (int e = tid; e < (k1 - k0) * L::NLM; e += nt) {
        const int kl = e / L::NLM, k = k0 + kl;
        lin_lm_output<true, MARG>(bd, ww, tile, meta, k, e - L::NLM * kl, bd.lm_fptr[k] - f0, bd.lm_fptr[k + 1] - f0);
    }
}
VIWB_D void lin_vis_lm_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by;
    if (mode == MODE_COST) lin_vis_run_cost(bd, bx, tid, nt, smem); else lin_vis_run_body(bd, bx, tid, nt, smem);
}
VIWB_D void lin_vis_lm_wide_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by;
    if (mode == MODE_MARG) lin_vis_lm_body<true>(bd, bx, tid, nt, smem); else lin_vis_lm_body<false>(bd, bx, tid, nt, smem, mode == MODE_COST);
}

// ------------------------------------------------------------------------------------------------ asm_pairs_wide
// One warp per chunk of one frame pair's records: G = sum_f X_f^T X_f on the FP64 tensor pipe.  K index of the product = (factor, residual row): a
// k-step of 4 = two records; lane l feeds X[k = l%4][column l/4 + 8 t] as the A and the B operand of the tiles in tile row / column t.
// the product of ONE chunk, written to `out` in accumulator order
template <bool WIDE>
VIWB_D void pair_chunk(const BatchDev &bd, const AsmItem &item, double *out, int lane) {
    typedef XL<WIDE> L;
    const double *recs = bd.xrec;                      // item.base: the window's record region (offset in doubles); item.lo / item.hi: records inside it
#ifdef VIWB_HOST_EMU
    (void)lane;
    double G[32][32];
    for (int a = 0; a < 32; a++) for (int b = 0; b < 32; b++) G[a][b] = 0.0;
    for (int f = item.lo; f < item.hi; f++) for (int rr = 0; rr < 2; rr++) {
        const double *xrow = recs + (size_t)item.base + (size_t)f * L::REC + rr * L::ROW;
        for (int a = 0; a < L::ROW; a++) for (int b = 0; b < L::ROW; b++) G[a][b] += xrow[a] * xrow[b];
    }
    int t = 0;
    for (int tr = 0; tr < L::NTC; tr++) for (int tc = tr; tc < L::NTC; tc++, t++)
        for (int l = 0; l < 32; l++) for (int r = 0; r < 2; r++) out[64 * t + 2 * l + r] = G[8 * tr + l / 4][8 * tc + 2 * (l % 4) + r];
#else
    const double *base = recs + (size_t)item.base;
    const int kk = lane & 3, fo = kk >> 1, rr = kk & 1, c0 = lane >> 2;
    double acc[L::NTILE][2];
#pragma unroll
    for (int t = 0; t < L::NTILE; t++) { acc[t][0] = 0.0; acc[t][1] = 0.0; }
    for (int f = item.lo; f < item.hi; f += 2) {
        const int ff = f + fo;
        const bool ok = ff < item.hi;
        const double *p = base + (size_t)ff * L::REC + rr * L::ROW;
        double a[L::NTC];
#pragma unroll
        for (int t = 0; t < L::NTC; t++) a[t] = (ok && c0 + 8 * t < L::ROW) ? p[c0 + 8 * t] : 0.0;
        int t = 0;
#pragma unroll
        for (int tr = 0; tr < L::NTC; tr++)
#pragma unroll
            for (int tc = tr; tc < L::NTC; tc++, t++) dmma884(acc[t], a[tr], a[tc]);
    }
#pragma unroll
    for (int t = 0; t < L::NTILE; t++) { double2 v; v.x = acc[t][0]; v.y = acc[t][1]; reinterpret_cast<double2 *>(out + 64 * t)[lane] = v; }
#endif
}
VIWB_D void asm_pairs_wide_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by; (void)smem;
    const int Wd = nt < 32 ? nt : 32, wpb = nt / Wd, lane = tid % Wd;
    const int it = bx * wpb + tid / Wd;
    const bool marg = mode == MODE_MARG;
    if (it >= (marg ? bd.nmpitems_total : bd.npitems_total)) return;
    const AsmItem item = (marg ? bd.mpitems : bd.pitems)[it];
    if (!marg && (bd.work[item.win].status != ST_RUNNING || !item.has_common)) return;      // (compact windows: lin_vis_lm forms their chunks)
    double *out = marg ? bd.mpair_out + (size_t)it * XL<true>::OUT : bd.pair_out + (size_t)it * bd.pout_stride;
    pair_chunk<true>(bd, item, out, lane);
}

// ------------------------------------------------------------------------------------------------ pair_reduce
// Folds the pair chunks of a window into what the consumer (solve / marg_prep through assemble_into) adds to the normal equations: per frame f the
// diagonal block and gradient (every chunk of every pair that contains f, in item order) (+ WIDE: its 6 x 13 block against the common columns),
// per pair (a < b) the 6 x 6 off-diagonal block, (+ WIDE: the 13 x 13 common block and gradient over all chunks).  One block per window, one owner per
// output, fixed order.  Keeps the ~100 dependent L2 reads per entry out of the (latency-bound) consumer kernels.
VIWB_HD int pair_index(int a, int b) { return a * (2 * NFR - a - 1) / 2 + (b - a - 1); }      // a < b
template <bool WIDE>
VIWB_D void pair_reduce_body(const BatchDev &bd, int w, int tid, int nt, int mode, int *ab) {
    typedef XL<WIDE> L;
    const WinMeta &m = bd.meta[w];
    const bool marg = mode == MODE_MARG;
    double *red = bd.pair_red + (size_t)w * PAIR_RED;
    const AsmItem *items = marg ? bd.mpitems + m.mpitem_off : bd.pitems + m.pitem_off;
    const int npi = marg ? m.nmpitems : m.npitems;
    // the chunk products of lin_vis_lm / asm_pairs_wide
    const size_t PS = marg ? (size_t)XL<true>::OUT : (size_t)bd.pout_stride;
    const double *outs = marg ? bd.mpair_out + (size_t)m.mpitem_off * PS : bd.pair_out + (size_t)m.pitem_off * PS;
    // the items' frame pair and chunk phase, staged once: every output below walks the whole list (a | b << 4 | phase << 8)
    for (int ii = tid; ii < npi; ii += nt) { const AsmItem &it = items[ii]; ab[ii] = it.a | (it.b << 4) | (it.phase << 8); }
    VIWB_SYNC();
    for (int e = tid; e < NFR * L::FR; e += nt) {
        const int f = e / L::FR, o = e - L::FR * f;
        int p = 0, q = 0;              // G row offset within the frame's slot, G column (absolute unless it is a pose column)
        bool qpose = false;
        if (o < 21) { sym_unrank(o, p, q); qpose = true; } else if (o < 27) { p = o - 21; q = L::RCOL; } else { p = (o - 27) / 13; q = 12 + (o - 27) % 13; }
        double v = 0.0;
        for (int ii = 0; ii < npi; ii++) {
            const int ia = ab[ii] & 15, ib = (ab[ii] >> 4) & 15;
            int base;
            if (ia == f && ib != f) base = 0; else if (ib == f && ia != f) base = 6; else continue;      // (a == b: the one-frame factors of WIDE records, no pose columns)
            v += pair_G<WIDE>(outs + (size_t)ii * PS, base + p, qpose ? base + q : q);
        }
        red[e] = v;
    }
    for (int e = tid; e < NPAIR * 36; e += nt) red[NFR * L::FR + e] = 0.0;
    VIWB_SYNC();
    for (int e = tid; e < npi * 36; e += nt) {
        const int ii = e / 36, o = e - 36 * ii;
        const int ia = ab[ii] & 15, ib = (ab[ii] >> 4) & 15;
        if ((ab[ii] >> 8) != 0 || ia == ib) continue;
        double v = pair_G<WIDE>(outs + (size_t)ii * PS, o / 6, 6 + o % 6);
        for (int c = 1; ii + c < npi && (ab[ii + c] >> 8) == c; c++) v += pair_G<WIDE>(outs + (size_t)(ii + c) * PS, o / 6, 6 + o % 6);
        red[NFR * L::FR + pair_index(ia, ib) * 36 + o] = v;
    }
    if (WIDE) for (int e = tid; e < 91 + 13; e += nt) {
        int p = 0, q = 0;
        if (e < 91) { sym_unrank(e, p, q); q += 12; } else { p = e - 91; q = L::RCOL; }
        double v = 0.0;
        for (int ii = 0; ii < npi; ii++) v += pair_G<WIDE>(outs + (size_t)ii * PS, 12 + p, q);
        red[NFR * L::FR + NPAIR * 36 + e] = v;
    }
}
VIWB_D void pair_reduce_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by;
    const WinMeta &m = bd.meta[bx];
    int *ab = (int *)smem;                  // bd.pitems_max ints
    if (mode == MODE_MARG) { if (m.mfused) pair_reduce_body<true>(bd, bx, tid, nt, mode, ab); return; }
    if (!m.fused || bd.work[bx].status != ST_RUNNING) return;
    if (m.has_common) pair_reduce_body<true>(bd, bx, tid, nt, mode, ab); else pair_reduce_body<false>(bd, bx, tid, nt, mode, ab);
}

// ------------------------------------------------------------------------------------------------ syrk_mma
// T = sum_k g_k w_k w_k^T (80 x 80, both triangles written, exactly symmetric), tvec = sum_k g_k gl_k w_k.
// solver: g_k = gamma_k; marginalisation: g_k = 1 / a_k for the landmarks hosted in frame 0 (gamma holds a_k, 0 = skip; marg_pivot_weight).
// One [80 x K] x [K x 81] product (column 80 of the right operand = gl): 10 x 11 tiles of 8 x 8, of which the 55 upper-triangular ones
// and the 10 of the tvec column are computed: five warps, warp v owns tile rows v and 9 - v (13 tiles each).  Chunks of 32 landmarks stream
// through two shared-memory buffers (cp.async); the row stride 88 makes every operand fetch two conflict-free wavefronts.
enum { SYRK_KC = 32, SYRK_LD = 88, SYRK_NT = 160 };
VIWB_HD size_t syrk_mma_smem_doubles() { return (size_t)2 * SYRK_KC * SYRK_LD + 2 * SYRK_KC; }
// 16-byte asynchronous global -> shared copy (cp.async), commit / wait by groups
VIWB_D void async_copy16(double *smem_dst, const double *gsrc) {
#ifdef VIWB_HOST_EMU
    smem_dst[0] = gsrc[0]; smem_dst[1] = gsrc[1];
#else
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(d), "l"(gsrc) : "memory");
#endif
}
VIWB_D void async_commit() {
#ifndef VIWB_HOST_EMU
    asm volatile("cp.async.commit_group;\n" ::: "memory");
#endif
}
template <int PENDING> VIWB_D void async_wait() {
#ifndef VIWB_HOST_EMU
    asm volatile("cp.async.wait_group %0;\n" ::"n"(PENDING) : "memory");
#endif
}
VIWB_D void syrk_mma_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by;
    const int w = bx;
    const WinMeta &m = bd.meta[w];
    if (mode == MODE_SOLVE && bd.work[w].status != ST_RUNNING) return;
    if (mode == MODE_MARG && m.margin_flag != 0) return;
    const double *W = bd.lm_W + (size_t)m.lm_off * VSUB, *gam = bd.lm_gamma + m.lm_off, *gl = bd.lm_g + m.lm_off;
    double *T = bd.Tvis + (size_t)w * VSUB * VSUB, *tv = bd.tvec + (size_t)w * VSUB;
#ifdef VIWB_HOST_EMU
    (void)smem; (void)tid; (void)nt;
    for (int i = 0; i < VSUB; i++) { for (int j = 0; j < VSUB; j++) T[i * VSUB + j] = 0.0; tv[i] = 0.0; }
    for (int k = 0; k < m.nlm; k++) {
        double g = gam[k];
        if (mode == MODE_MARG) g = marg_pivot_weight(g);
        if (g == 0.0) continue;                           // a landmark that takes no part: its row of W is not even read (it may never have been written)
        const double *r = W + (size_t)k * VSUB;
        for (int i = 0; i < VSUB; i++) { const double a = g * r[i]; for (int j = i; j < VSUB; j++) T[i * VSUB + j] += a * r[j]; tv[i] += a * gl[k]; }
    }
    for (int i = 0; i < VSUB; i++) for (int j = 0; j < i; j++) T[i * VSUB + j] = T[j * VSUB + i];
#else
    double *Wb[2] = {smem, smem + SYRK_KC * SYRK_LD};
    double *gkb[2] = {smem + 2 * SYRK_KC * SYRK_LD, smem + 2 * SYRK_KC * SYRK_LD + SYRK_KC};
    const int lane = tid & 31, wid = tid >> 5;
    const int tmA = wid, tmB = 9 - wid;                       // tile rows of this warp (tmA <= 4 < tmB)
    double accA[11][2], accB[6][2];
#pragma unroll
    for (int j = 0; j < 11; j++) { accA[j][0] = 0.0; accA[j][1] = 0.0; }
#pragma unroll
    for (int j = 0; j < 6; j++) { accB[j][0] = 0.0; accB[j][1] = 0.0; }
    auto stage = [&](int c, int p) {
        const int k0 = c * SYRK_KC, kc = (m.nlm - k0) < SYRK_KC ? (m.nlm - k0) : SYRK_KC;
        // rows with weight 0 (landmarks that take no part; marginalisation: not hosted in frame 0) are staged as zeros, never read: they may hold anything
        for (int e = tid; e < kc * (VSUB / 2); e += nt) {
            const int r = e / (VSUB / 2), cc = e - r * (VSUB / 2);
            if (gam[k0 + r] > 0.0) async_copy16(Wb[p] + r * SYRK_LD + 2 * cc, W + (size_t)(k0 + r) * VSUB + 2 * cc);
            else { Wb[p][r * SYRK_LD + 2 * cc] = 0.0; Wb[p][r * SYRK_LD + 2 * cc + 1] = 0.0; }
        }
        async_commit();
        for (int r = tid; r < SYRK_KC; r += nt) {
            double g = 0.0, gg = 0.0;
            if (r < kc) { g = gam[k0 + r]; if (mode == MODE_MARG) g = marg_pivot_weight(g); gg = gl[k0 + r]; }
            gkb[p][r] = g;
            Wb[p][r * SYRK_LD + VSUB] = gg;                   // column 80 of the right operand
            if (r >= kc) for (int q = 0; q < VSUB; q++) Wb[p][r * SYRK_LD + q] = 0.0;      // rows past the end of the window: zeros, not stale bytes
        }
    };
    for (int e = tid; e < 2 * SYRK_KC * 7; e += nt) { const int r = e / 7, q = e - 7 * r; smem[r * SYRK_LD + VSUB + 1 + q] = 0.0; }      // columns 81..87 of both buffers
    const int nchunk = (m.nlm + SYRK_KC - 1) / SYRK_KC;
    if (nchunk > 0) stage(0, 0);
    for (int c = 0, p = 0; c < nchunk; c++, p ^= 1) {
        if (c + 1 < nchunk) { stage(c + 1, p ^ 1); async_wait<1>(); } else async_wait<0>();
        __syncthreads();
        const double *Ws = Wb[p], *gk = gkb[p];
#pragma unroll 2
        for (int ks = 0; ks < SYRK_KC / 4; ks++) {
            const int k = 4 * ks + (lane & 3), col = lane >> 2;
            const double *row = Ws + k * SYRK_LD + col;
            const double g = gk[k];
            const double aA = g * row[8 * tmA], aB = g * row[8 * tmB];
#pragma unroll
            for (int j = 0; j < 11; j++) { const int tn = tmA + j; if (tn <= 10) dmma884(accA[j], aA, row[8 * tn]); }
#pragma unroll
            for (int j = 0; j < 6; j++) { const int tn = tmB + j; if (tn <= 10) dmma884(accB[j], aB, row[8 * tn]); }      // (register arrays want compile-time indices: the operand is fetched again)
        }
        __syncthreads();
    }
    // epilogue: lane l holds rows 8 tm + l/4, columns 8 tn + 2 (l%4) + {0, 1}
    const int mr = lane >> 2, n0 = 2 * (lane & 3);
    auto emit = [&](int tm, int tn, const double *v) {
        const int R = 8 * tm + mr, C = 8 * tn + n0;
        if (tn == 10) { if (n0 == 0) tv[R] = v[0]; return; }
        if (tn > tm) { T[R * VSUB + C] = v[0]; T[R * VSUB + C + 1] = v[1]; T[C * VSUB + R] = v[0]; T[(C + 1) * VSUB + R] = v[1]; return; }
        if (C >= R) { T[R * VSUB + C] = v[0]; T[C * VSUB + R] = v[0]; }
        if (C + 1 >= R) { T[R * VSUB + C + 1] = v[1]; T[(C + 1) * VSUB + R] = v[1]; }
    };
#pragma unroll
    for (int j = 0; j < 11; j++) if (tmA + j <= 10) emit(tmA, tmA + j, accA[j]);
#pragma unroll
    for (int j = 0; j < 6; j++) if (tmB + j <= 10) emit(tmB, tmB + j, accB[j]);
#endif
}

}  // namespace viwb
