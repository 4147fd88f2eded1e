// kernels_lin.cuh -- linearisation kernels: factor evaluation and gather-assembly of the normal equations.
//
// All kernels are written as block functions f(bd, bx, by, tid, nt, smem, mode) in strided-loop style with
// barriers only between phases, so the same source runs as a CUDA kernel and (nt = 1) in the CPU emulation.
//   setup      once per solve: IMU/wheel sqrt-information (imu_factor.h:75, wheel_factor.h:85), prior J^T J
//   lin_vis    one thread per visual factor: residual, Huber, tangent Jacobians -> 54-double record   (8a-5/6/7, a-12)
//   lm_reduce  13 threads per landmark: a = |J_l|^2, g_l, w = J_p^T J_l, Schur weight gamma, cost      (Schur, Appendix B)
//   lin_small  one block per window: IMU / wheel / plane factors and the prior residual + gradient   (8a-8..a-11)
//   (assembly of the normal equations: kernels_asm.cuh)
// mode 0 = solver linearisation at x_cand over the tangent layout, mode 1 = marginalisation at x_cur over the
// marginalisation layout (7 -> 6, plane quaternion counted 4; marginalization_factor.cpp:140-143).
#pragma once
#include "layout.cuh"
#include "factors.cuh"

namespace viwb {

enum { MODE_SOLVE = 0, MODE_MARG = 1, MODE_COST = 2 };      // MODE_COST: lin_vis_lm only -- the solver's decision-only round (costs at x_cand, no Jacobians)
enum { MLAY = 193 };   // marginalisation layout dimension over the fixed blocks
VIWB_HD int blk_moff(int b) { int t = blk_toff(b); return b > BLK_PR ? t + 1 : t; }

// MARGIN_SECOND_NEW marginalises the prior only (estimator.cpp:1819-1842); margin_flag < 0: nothing to marginalise
VIWB_HD bool marg_prior_only(const WinMeta &m, int mode) { return mode == MODE_MARG && m.margin_flag == 1; }
VIWB_HD bool marg_skip(const WinMeta &m, int mode) { return mode == MODE_MARG && m.margin_flag < 0; }
// Weight 1 / a of a dropped landmark's pivot a in the Schur sum T0 = sum w w^T / a.  The reference inverts the whole landmark block through its
// eigenvalues and discards every eigenvalue <= 1e-8 (marginalization_factor.cpp:282-287); a pivot under that cut is discarded here the same way.
// Such a pivot (a landmark seen only from its host's camera centre: no parallax) is rounding noise and so is its coupling w: its eigenvector is
// the landmark's own axis to O(|w|^2), so dropping it equals the eigen-cut, while dividing by it would inject w w^T / a in a direction set by rounding.
VIWB_HD double marg_pivot_weight(double a) { return a > 1e-8 ? 1.0 / a : 0.0; }

VIWB_HD const double *eval_state(const BatchDev &bd, int w, int mode) {
    return (mode == MODE_SOLVE ? bd.x_cand : bd.x_cur) + bd.meta[w].state_off;
}

// ------------------------------------------------------------------------------------------------ setup
VIWB_D void setup_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by; (void)smem; (void)mode;
    const int gi = bx * nt + tid, gstride = nt;   // gridDim.x handled by the launcher loop: items = bx*nt + tid
    (void)gstride;
    const int n_s = bd.nimu_total + bd.nwheel_total;
    if (gi < bd.nimu_total) {
        sqrt_info_upper(15, bd.imu_data + (size_t)gi * 287 + 62, bd.imu_S + (size_t)gi * 225);
    } else if (gi < n_s) {
        const int k = gi - bd.nimu_total;
        sqrt_info_upper(6, bd.wheel_data + (size_t)k * 78 + 25, bd.wheel_S + (size_t)k * 36);
    }
}
// wire format -> device tables, one block per window (runs once per upload, before anything reads the visual table)
VIWB_D void vis_expand_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by; (void)smem; (void)mode;
    const WinMeta &m = bd.meta[bx];
    for (int i = tid; i < m.nvis; i += nt) {
        const int f = m.vis_off + i, code = bd.vis_code[f];
        bd.vis_type[f] = code & 3; bd.vis_fi[f] = (code >> 2) & 15; bd.vis_fj[f] = (code >> 6) & 15; bd.vis_dup[f] = (unsigned char)((code >> 10) & 3); bd.vis_win[f] = bx;
        const double *hi = bd.obs_i + (size_t)bd.vis_oi[f] * 6, *hj = bd.obs_j + (size_t)f * 6;
        double *o = bd.vis_obs + (size_t)f * 12;
        o[0] = hi[0]; o[1] = hi[1]; o[2] = hi[2]; o[3] = hj[0]; o[4] = hj[1]; o[5] = hj[2]; o[6] = hi[3]; o[7] = hi[4]; o[8] = hj[3]; o[9] = hj[4]; o[10] = hi[5]; o[11] = hj[5];
    }
}
// prior A = J^T J, one block per prior
VIWB_D void prior_setup_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by; (void)smem; (void)mode;
    const PriorDev &p = bd.prior[bx];
    const int n = p.n;
    const double *J = bd.prior_J + p.J_off;
    double *A = bd.prior_A + p.J_off;
    for (int e = tid; e < n * n; e += nt) {
        const int i = e / n, j = e % n;
        double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;      // four partial sums (one dependent chain of n otherwise)
        int k = 0;
        for (; k + 3 < n; k += 4) { s0 += J[k * n + i] * J[k * n + j]; s1 += J[(k + 1) * n + i] * J[(k + 1) * n + j]; s2 += J[(k + 2) * n + i] * J[(k + 2) * n + j]; s3 += J[(k + 3) * n + i] * J[(k + 3) * n + j]; }
        for (; k < n; k++) s0 += J[k * n + i] * J[k * n + j];
        A[e] = (s0 + s1) + (s2 + s3);
    }
}

// ------------------------------------------------------------------------------------------------ lin_vis
// One thread per factor.  The records (VREC doubles per factor) are assembled in a shared-memory tile with an odd row stride
// and leave the block as one contiguous, fully coalesced stream (a thread storing its own record directly would touch 32
// different sectors per store instruction).
VIWB_HD size_t lin_vis_smem_doubles(int nt) { return (size_t)nt * (VREC | 1) + (nt + 7) / 8; }
VIWB_D void lin_vis_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by;
    const int ts = VREC | 1;
    double *tile = smem;
    unsigned char *act = reinterpret_cast<unsigned char *>(smem + (size_t)nt * ts);
    const int f = bx * nt + tid;
    bool on = f < bd.nvis_total;
    int w = 0, fi = 0;
    if (on) {
        w = bd.vis_win[f];
        if (mode == MODE_SOLVE && (bd.work[w].status != ST_RUNNING || bd.meta[w].fused)) on = false;      // fused windows: lin_vis_lm (kernels_fused.cuh)
    }
    if (on) {
        fi = bd.vis_fi[f];
        if (mode == MODE_MARG && (fi != 0 || bd.meta[w].margin_flag != 0 || bd.meta[w].mfused)) on = false;      // fused marginalisation: lin_vis_lm_wide
    }
    act[tid] = on ? 1 : 0;
    const int nrec = (bd.nvis_total - bx * nt) < nt ? (bd.nvis_total - bx * nt) : nt;
    if (on) {
        const WinMeta &m = bd.meta[w];
        const double *x = eval_state(bd, w, mode);
        double obs[12];
        for (int k = 0; k < 12; k++) obs[k] = bd.vis_obs[(size_t)f * 12 + k];      // (staging these through the tile measured slower)
        const int lm = bd.vis_lm[f];
        VisOut o;
        vis_eval(bd.vis_type[f], obs, x + 7 * fi, x + 7 * bd.vis_fj[f], x + blk_off(BLK_EX0), x + blk_off(BLK_EX1),
                 x[SFIX + lm], x[blk_off(BLK_TD)], m.S_vis, true, o);
        double half_rho;
        const double sc = huber_scale(o.r[0] * o.r[0] + o.r[1] * o.r[1], m.huber, half_rho);
        double *rec = tile + (size_t)tid * ts;
        rec[0] = o.r[0] * sc; rec[1] = o.r[1] * sc;
        for (int k = 0; k < 12; k++) { rec[REC_A + k] = o.JA[k] * sc; rec[REC_B + k] = o.JB[k] * sc; }
        rec[REC_L] = o.Jl[0] * sc; rec[REC_L + 1] = o.Jl[1] * sc;
        for (int k = 0; k < 12; k++) { rec[REC_E0 + k] = o.JE0[k] * sc; rec[REC_E1 + k] = o.JE1[k] * sc; }
        rec[REC_TD] = o.Jtd[0] * sc; rec[REC_TD + 1] = o.Jtd[1] * sc;
        bd.vis_cost[f] = half_rho;
    }
    VIWB_SYNC();
    double *out = bd.vis_rec + (size_t)bx * nt * VREC;
    for (int e = tid; e < nrec * VREC; e += nt) { const int r = e / VREC, q = e - r * VREC; if (act[r]) out[e] = tile[(size_t)r * ts + q]; }
}

// ------------------------------------------------------------------------------------------------ lm_reduce
// One warp per landmark, one lane per factor (chunks of 32 if a landmark has more): every lane streams its own record once
// (consecutive records -> fully used cache lines), forms its J_p^T J_lambda pieces in registers, and the warp combines them:
// a_k, g_k, the cost, the host-frame block and the common blocks by shuffle sums; the observing-frame blocks by the lanes that
// share a frame taking turns in lane order (fixed order -> deterministic).  LM_ROLES = threads per landmark for the launch.
#ifdef VIWB_HOST_EMU
enum { LM_ROLES = 1, LM_W = 1 };
#else
enum { LM_ROLES = 32, LM_W = 32 };
#endif
VIWB_D double lm_warp_sum(double v) {
#ifndef VIWB_HOST_EMU
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
#endif
    return v;
}
VIWB_D void lm_reduce_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by; (void)smem;
    const int gid = bx * nt + tid;
    const int k = gid / LM_ROLES, lane = gid % LM_ROLES;
    if (k >= bd.nlm_total) return;
    const int w = bd.lm_win[k];
    const WinWork &ww = bd.work[w];
    if (mode == MODE_SOLVE && (ww.status != ST_RUNNING || bd.meta[w].fused)) return;
    if (mode == MODE_MARG && bd.meta[w].mfused) return;
    const int f0 = bd.lm_fptr[k], f1 = bd.lm_fptr[k + 1];
    double *W = bd.lm_W + (size_t)k * VSUB;
    const bool skip = (mode == MODE_MARG) && (f0 == f1 || bd.vis_fi[f0] != 0 || bd.meta[w].margin_flag != 0);
    for (int p = lane; p < VSUB; p += LM_W) W[p] = 0.0;
    // a landmark that takes no part in the marginalisation still owns a row of W that syrk multiplies by its zero weight: the row must
    // hold numbers (a marginalise-only call on a recycled arena would otherwise multiply 0 by whatever an earlier batch left there)
    if (skip) { if (lane == 0) { bd.lm_gamma[k] = 0.0; bd.lm_a[k] = 0.0; bd.lm_g[k] = 0.0; } return; }
    if (f0 == f1) {      // a landmark without factors: contributes nothing
        if (lane == 0) { bd.lm_a[k] = 0.0; bd.lm_g[k] = 0.0; bd.lm_cost[k] = 0.0; bd.lm_gamma[k] = 0.0; if (ww.first) bd.lm_scale[k] = 1.0; }
        return;
    }
    VIWB_SYNCWARP();
    const int host = bd.vis_fi[f0];
    double a = 0.0, g = 0.0, c = 0.0, hacc[6] = {0, 0, 0, 0, 0, 0}, e0[6] = {0}, e1[6] = {0}, tdv = 0.0;
    for (int fb = f0; fb < f1; fb += LM_W) {
        const int f = fb + lane;
        const bool on = f < f1;
        int fj = -1;
        double bv[6] = {0, 0, 0, 0, 0, 0};
        if (on) {
            const int type = bd.vis_type[f];
            const double *rec = bd.vis_rec + (size_t)f * VREC;
            const double u0 = rec[REC_L], u1 = rec[REC_L + 1];
            a += u0 * u0 + u1 * u1; g += u0 * rec[0] + u1 * rec[1]; c += bd.vis_cost[f];
            if (type != 2) {
                for (int q = 0; q < 6; q++) hacc[q] += rec[REC_A + q] * u0 + rec[REC_A + 6 + q] * u1;
                for (int q = 0; q < 6; q++) bv[q] = rec[REC_B + q] * u0 + rec[REC_B + 6 + q] * u1;
                fj = bd.vis_fj[f];
            }
            for (int q = 0; q < 6; q++) e0[q] += rec[REC_E0 + q] * u0 + rec[REC_E0 + 6 + q] * u1;
            tdv += rec[REC_TD] * u0 + rec[REC_TD + 1] * u1;
            if (type != 0) for (int q = 0; q < 6; q++) e1[q] += rec[REC_E1 + q] * u0 + rec[REC_E1 + 6 + q] * u1;
        }
        // observing-frame blocks: lanes with the same frame add in lane order
#ifdef VIWB_HOST_EMU
        if (fj >= 0) for (int q = 0; q < 6; q++) W[6 * fj + q] += bv[q];
#else
        {
            const unsigned peers = __match_any_sync(0xffffffffu, fj);
            const int rank = __popc(peers & ((1u << lane) - 1u));
            const int rounds = __reduce_max_sync(0xffffffffu, fj >= 0 ? rank : 0);
            for (int r = 0; r <= rounds; r++) {
                if (fj >= 0 && rank == r) for (int q = 0; q < 6; q++) W[6 * fj + q] += bv[q];
                __syncwarp();
            }
        }
#endif
    }
    a = lm_warp_sum(a); g = lm_warp_sum(g); c = lm_warp_sum(c);
    for (int q = 0; q < 6; q++) hacc[q] = lm_warp_sum(hacc[q]);
    for (int q = 0; q < 6; q++) { e0[q] = lm_warp_sum(e0[q]); e1[q] = lm_warp_sum(e1[q]); }
    tdv = lm_warp_sum(tdv);
    if (lane != 0) return;
    for (int q = 0; q < 6; q++) W[6 * host + q] += hacc[q];
    for (int q = 0; q < 6; q++) { W[66 + q] = e0[q]; W[72 + q] = e1[q]; }
    W[78] = tdv;
    bd.lm_a[k] = a; bd.lm_g[k] = g; bd.lm_cost[k] = c;
    if (mode == MODE_MARG) { bd.lm_gamma[k] = a; return; }     // marginalisation keeps the pivot itself
    // Jacobi scale (first linearisation only) and the Schur weight for the mu this linearisation will be solved with:
    // scaled pivot h = c^2 a + mu * clamp(c^2 a); gamma = c^2 / h  (SURVEY Appendix B)
    double sc = bd.lm_scale[k];
    if (ww.first) { sc = bd.opt.jacobi_scaling ? 1.0 / (1.0 + sqrt(a)) : 1.0; bd.lm_scale[k] = sc; }
    const double s = sc * sc * a;
    double d2 = s; if (d2 < bd.opt.min_lm_diagonal) d2 = bd.opt.min_lm_diagonal; if (d2 > bd.opt.max_lm_diagonal) d2 = bd.opt.max_lm_diagonal;
    bd.lm_gamma[k] = sc * sc / (s + ww.mu_lin * d2);
}

// ------------------------------------------------------------------------------------------------ lin_small
// prior residual: r = r_lin + J_lin dx (marginalization_factor.cpp:361-380); dx in the prior's own column layout
VIWB_D void prior_dx(const PriorDev &p, const double *x, const double *x0, double *dx) {
    for (int i = 0; i < p.nb; i++) {
        const int b = p.block_id[i], size = blk_size(b), idx = p.block_idx[i], off = blk_off(b);
        if (size != 7) { for (int k = 0; k < size; k++) dx[idx + k] = x[off + k] - x0[off + k]; }
        else {
            for (int k = 0; k < 3; k++) dx[idx + k] = x[off + k] - x0[off + k];
            const Q4 dq = qinv(ldq(x0 + off + 3)) * ldq(x + off + 3);
            const double s = (dq.w >= 0) ? 2.0 : -2.0;          // quirk 8: sign flip when w < 0 (:374-377)
            dx[idx + 3] = s * dq.x; dx[idx + 4] = s * dq.y; dx[idx + 5] = s * dq.z;
        }
    }
}

// Small factors in two phases per group of SMALL_NSLOT: (A) one thread per factor evaluates the un-whitened residual and
// Jacobian into its shared-memory slot (the factors of a group run side by side in the lanes of one warp), (B) one warp per
// factor whitens one Jacobian column per lane (r <- S r, J <- S J with S upper triangular) and streams it to the record.
enum { SMALL_SLOT = 15 + 15 * 30, SMALL_NSLOT = 10, SMALL_S = 225 };
VIWB_HD size_t lin_small_smem_doubles(int nt) { const int W = nt < 32 ? nt : 32; return (size_t)SMALL_NSLOT * SMALL_SLOT + (size_t)(nt / W) * SMALL_S + nt + MAXPRI + 8; }
VIWB_D double whiten_store(const double *raw, const double *Sg, double *Ss, int rows, int ld, double *rec, int lane, int W) {
    // raw: [rows residual | rows x ld Jacobian] un-whitened in shared memory -> rec (global), returns this lane's part of 0.5 |r|^2.
    // The sqrt-information factor is first copied into the warp's shared-memory slice: every lane needs every entry of it.
    VIWB_SYNCWARP();
    for (int e = lane; e < rows * rows; e += W) Ss[e] = Sg[e];
    VIWB_SYNCWARP();
    const double *S = Ss;
    double c = 0.0;
    for (int col = lane; col <= ld; col += W) {
        for (int i = 0; i < rows; i++) {
            double a = 0.0;
            if (col < ld) { for (int k = i; k < rows; k++) a += S[i * rows + k] * raw[rows + k * ld + col]; rec[rows + i * ld + col] = a; }
            else { for (int k = i; k < rows; k++) a += S[i * rows + k] * raw[k]; rec[i] = a; c += 0.5 * a * a; }
        }
    }
    return c;
}
VIWB_D void lin_small_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by;
    const int w = bx;
    const WinMeta &m = bd.meta[w];
    WinWork &ww = bd.work[w];
    if (mode == MODE_SOLVE && ww.status != ST_RUNNING) return;
    if (marg_skip(m, mode)) return;
    const double *x = eval_state(bd, w, mode);
    const int W = nt < 32 ? nt : 32, nw = nt / W, wid = tid / W, lane = tid % W;
    double *Sw = smem + (size_t)SMALL_NSLOT * SMALL_SLOT + (size_t)wid * SMALL_S;      // this warp's copy of a factor's sqrt-information
    double *cost_part = smem + (size_t)SMALL_NSLOT * SMALL_SLOT + (size_t)nw * SMALL_S;      // [nt]
    double *dx = cost_part + nt;                                      // [MAXPRI]
    double c = 0.0;
    const int n_small = marg_prior_only(m, mode) ? 0 : m.nimu + m.nwheel + m.nplane;
    for (int t0 = 0; t0 < n_small; t0 += SMALL_NSLOT) {
        const int t1 = (t0 + SMALL_NSLOT < n_small) ? t0 + SMALL_NSLOT : n_small;
        // ---- A: evaluate
        for (int t = t0 + tid; t < t1; t += nt) {
            double *slot = smem + (size_t)(t - t0) * SMALL_SLOT;
            if (t < m.nimu) {
                const int f = m.imu_off + t, i = bd.imu_fi[f], j = bd.imu_fj[f];
                if (mode == MODE_MARG && !(i == 0 && j == 1)) continue;
                imu_eval(bd.imu_data + (size_t)f * 287, nullptr, m.G, x + 7 * i, x + 77 + 9 * i, x + 7 * j, x + 77 + 9 * j, true, slot, slot + 15);
            } else if (t < m.nimu + m.nwheel) {
                const int f = m.wheel_off + (t - m.nimu), i = bd.wheel_fi[f], j = bd.wheel_fj[f];
                if (mode == MODE_MARG && !(i == 0 && j == 1)) continue;
                wheel_eval(bd.wheel_data + (size_t)f * 78, nullptr, x + 7 * i, x + 7 * j, x + blk_off(BLK_EXW), x[blk_off(BLK_SX)], x[blk_off(BLK_SY)],
                           x[blk_off(BLK_SW)], x[blk_off(BLK_TDW)], true, slot, slot + 6);
            } else {
                const int f = m.plane_off + (t - m.nimu - m.nwheel), i = bd.plane_f[f];
                if (mode == MODE_MARG && i != 0) continue;
                double *rec = bd.plane_rec + (size_t)f * PLANE_REC;
                plane_eval(m.w_plane, x + 7 * i, x + blk_off(BLK_EXW), x + blk_off(BLK_PR), x[blk_off(BLK_PZ)], true, rec, rec + 3);
                for (int k = 0; k < 3; k++) c += 0.5 * rec[k] * rec[k];
            }
        }
        VIWB_SYNC();
        // ---- B: whiten
        for (int t = t0 + wid; t < t1; t += nw) {
            const double *slot = smem + (size_t)(t - t0) * SMALL_SLOT;
            if (t < m.nimu) {
                const int f = m.imu_off + t, i = bd.imu_fi[f], j = bd.imu_fj[f];
                if (mode == MODE_MARG && !(i == 0 && j == 1)) continue;
                c += whiten_store(slot, bd.imu_S + (size_t)f * 225, Sw, 15, 30, bd.imu_rec + (size_t)f * IMU_REC, lane, W);
            } else if (t < m.nimu + m.nwheel) {
                const int f = m.wheel_off + (t - m.nimu), i = bd.wheel_fi[f], j = bd.wheel_fj[f];
                if (mode == MODE_MARG && !(i == 0 && j == 1)) continue;
                c += whiten_store(slot, bd.wheel_S + (size_t)f * 36, Sw, 6, 22, bd.wheel_rec + (size_t)f * WHEEL_REC, lane, W);
            }
        }
        VIWB_SYNC();
    }
    if (m.prior_idx >= 0) {
        const PriorDev &p = bd.prior[m.prior_idx];
        const int n = p.n;
        if (tid == 0) prior_dx(p, x, bd.prior_x0 + p.x0_off, dx);
        VIWB_SYNC();
        const double *J = bd.prior_J + p.J_off;
        double *res = bd.prior_res + p.r_off, *g = bd.prior_g + p.r_off;
        for (int i = tid; i < n; i += nt) {      // thread per row, each walking its own row (measured slower: a warp per row with lanes along the row, 0.47 vs 0.34 ms per launch, r01zh; the same loop over a transposed copy so that neighbouring threads read neighbouring words, 0.38 vs 0.35, r02n)
            const double *Ji = J + (size_t)i * n;
            double s0 = bd.prior_r[p.r_off + i], s1 = 0.0, s2 = 0.0, s3 = 0.0;      // four partial sums: one dependent FMA chain of n otherwise
            int k = 0;
            for (; k + 3 < n; k += 4) { s0 += Ji[k] * dx[k]; s1 += Ji[k + 1] * dx[k + 1]; s2 += Ji[k + 2] * dx[k + 2]; s3 += Ji[k + 3] * dx[k + 3]; }
            for (; k < n; k++) s0 += Ji[k] * dx[k];
            const double s = (s0 + s1) + (s2 + s3);
            res[i] = s;
            c += 0.5 * s * s;
        }
        VIWB_SYNC();
        for (int i = tid; i < n; i += nt) {
            double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
            int k = 0;
            for (; k + 3 < n; k += 4) { s0 += J[k * n + i] * res[k]; s1 += J[(k + 1) * n + i] * res[k + 1]; s2 += J[(k + 2) * n + i] * res[k + 2]; s3 += J[(k + 3) * n + i] * res[k + 3]; }
            for (; k < n; k++) s0 += J[k * n + i] * res[k];
            g[i] = (s0 + s1) + (s2 + s3);
        }
    }
    cost_part[tid] = c;
    VIWB_SYNC();
    if (tid == 0) { double s = 0.0; for (int i = 0; i < nt; i++) s += cost_part[i]; ww.small_cost = s; }
}

}  // namespace viwb
