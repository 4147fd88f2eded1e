// layout.cuh -- device-resident data layout of a batch of windows (one Estimator::optimization() each).
//
// HBM layout (all FP64 unless noted; B windows, concatenated):
//   x_cur / x_cand      [sum(207 + nlm)]        parameter blocks, fixed-state layout of include/viwb.h + inverse depths
//   vis_*               visual factor table, sorted by landmark; vis_obs stays [nvis][12] as given
//   vis_rec             [nvis_total][54]        per-factor record written by lin_vis: r(2) A(12) B(12) Jl(2) Jtd(2) E0(12) E1(12); like vis_cost
//                       only allocated when some window's solve or marginalisation takes the unfused path
//   lm_*                per landmark: a = |J_l|^2, gl = J_l^T r, gamma = c^2/h (Schur weight), W [80] = J_p^T J_l over the
//                       "visual subspace" (11 poses x 6 | ex0 6 | ex1 6 | td 1 | pad)
//   imu_rec / wheel_rec / plane_rec   whitened residual + tangent Jacobian of the small factors
//   Hpk [B][192*193/2], gpk [B][192]  the active normal equations in the solve kernel's skyline order (assembled by gather, no atomics)
//   chol_plan           per distinct envelope: skyline row pointers and the Cholesky's trailing-update tiles per panel (int)
//   Tvis [B][80*80], tvec [B][80]     Schur sums  sum_k gamma_k w_k w_k^T  and  sum_k gamma_k w_k gl_k
//   per-window solver vectors (scale, D, scaled gradient, Gauss-Newton step) of length 192 + nlm
#pragma once
#include <stdint.h>
#include "vmath.cuh"

namespace viwb {

enum { NB = 32, NFR = 11, TFIX = 192, SFIX = 207, VSUB = 80, VREC = 54, IMU_REC = 15 + 15 * 30, WHEEL_REC = 6 + 6 * 22,
       PLANE_REC = 3 + 3 * 16, MAXPRI = 200 };
// record layout of lin_vis (VREC doubles per factor)
enum { REC_R = 0, REC_A = 2, REC_B = 14, REC_L = 26, REC_TD = 28, REC_E0 = 30, REC_E1 = 42 };
enum { BLK_SB0 = 11, BLK_EX0 = 22, BLK_EX1 = 23, BLK_EXW = 24, BLK_PR = 25, BLK_PZ = 26, BLK_SX = 27, BLK_SY = 28, BLK_SW = 29,
       BLK_TD = 30, BLK_TDW = 31 };

VIWB_HD int blk_size(int b) { return b < 11 ? 7 : b < 22 ? 9 : b < 25 ? 7 : b == 25 ? 4 : 1; }
VIWB_HD int blk_off(int b) { return b < 11 ? 7 * b : b < 22 ? 77 + 9 * (b - 11) : b < 25 ? 176 + 7 * (b - 22) : b == 25 ? 197 : 201 + (b - 26); }
VIWB_HD int blk_tsize(int b) { return b < 11 ? 6 : b < 22 ? 9 : b < 25 ? 6 : b == 25 ? 3 : 1; }
VIWB_HD int blk_toff(int b) { return b < 11 ? 6 * b : b < 22 ? 66 + 9 * (b - 11) : b < 25 ? 165 + 6 * (b - 22) : b == 25 ? 183 : 186 + (b - 26); }
VIWB_HD int blk_msize(int b) { int s = blk_size(b); return s == 7 ? 6 : s; }
// visual-subspace offset of a fixed block (-1 if the block is not touched by visual factors)
VIWB_HD int blk_voff(int b) { return b < 11 ? 6 * b : b == BLK_EX0 ? 66 : b == BLK_EX1 ? 72 : b == BLK_TD ? 78 : -1; }

enum { ASM_STRIDE = 108, ASM_CHUNK = 256, ITEM_FRAME = 0, ITEM_PAIR = 1, ITEM_COMMON = 2 };
// Fused path (solver linearisation of windows whose ex0 / ex1 / td are constant, "compact"): lin_vis_lm walks one HOST RUN per block -- the landmarks
// hosted in one frame, in landmark order, as tiles of whole landmarks -- and forms G = sum X^T X of every (host, observer) pair straight from the
// shared-memory tile (X = [A | B | r], 2 x 13; G: 13 x 13 inside three 8 x 8 FP64 tensor-core tiles), per chunk of PAIR_CHUNK records of the pair.
// Wide solver windows and every marginalisation keep landmark blocks (LmbDesc): lin_vis_lm_wide stores X records in frame-pair order, asm_pairs_wide
// turns them into the same chunk products.
enum { PAIR_CHUNK = 64, LMB_FACTORS = 128, NPAIR = NFR * (NFR - 1) / 2, PAIR_RED = NFR * 105 + NPAIR * 36 + 104 + 1 };      // PAIR_RED: the WIDE pair_reduce output (the compact one is a prefix-sized subset)
struct alignas(32) LmbDesc { int win, k0, k1, f0, nf, pad[3]; };      // window, global landmark range [k0, k1), first factor (global) and factor count (<= LMB_FACTORS)
// host run: window, host frame, its tiles [t0, t0 + ntile) in run_tile, and per observer frame j the pair item (global index into pitems / pair_out)
// of the first chunk of pair (host, j), -1 if the window has no such record
struct alignas(16) RunDesc { int win, host, t0, ntile, pfirst[NFR], pad; };
struct RunTile { int l0, nl, f0, nf; };      // entries [l0, l0 + nl) of run_lm and [f0, f0 + nf) of run_f (nf <= LMB_FACTORS)
struct AsmItem { int kind, win, a, b, lo, hi, phase, has_common, base; };      // base: fused path, offset (doubles) of the window's record region in xrec

struct PriorDev {       // one per window that has a valid prior
    int n, nb;
    int block_id[NB], block_idx[NB];
    int J_off;          // into prior_J (n*n row-major) and prior_A (n*n = J^T J, computed once per solve)
    int r_off;          // into prior_r (n), prior_res (n, current residual) and prior_g (n, J^T res)
    int x0_off;         // into prior_x0 (207)
};

struct WinMeta {        // read-only during a solve
    int state_off, lm_off, nlm;
    int vis_off, nvis;
    int imu_off, nimu, wheel_off, nwheel, plane_off, nplane;
    int prior_idx;      // -1: none
    int frame_count;
    int nf;             // active fixed tangent columns (compact)
    int margin_flag;
    int item_off, nitems, list_off;     // assembly items of the solver linearisation (kernels_asm.cuh); list entries are window-local
    int mitem_off, nmitems, mlist_off; // assembly items of the marginalisation linearisation (factors hosted in frame 0)
    int has_common;                     // any of ex0 / ex1 / td is an active column (solver); marginalisation always counts them
    int xrec_off, nxrec;                // fused path (wide solver windows): the window's record region in xrec (offset in DOUBLES), number of records
    int pitem_off, npitems;             // fused path: pair items (chunks of one frame pair's records), head item of a pair has phase 0
    int lmb_off, nlmb;                  // landmark blocks (whole landmarks, <= LMB_FACTORS factors) of lin_vis_lm_wide, solver (wide windows) and marginalisation
    int fused;                          // 1: this window's solver linearisation takes the fused path (regular factor table): host runs unless has_common
    int mxrec_off, nmxrec, mpitem_off, nmpitems;      // fused marginalisation (MARGIN_OLD, regular table): WIDE records of the factors hosted in frame 0, their pair items
    int mfused;
    short tcol[NB];     // compact column of fixed block b, -1 if constant / absent / unreferenced
    short efirst[TFIX]; // envelope of the reduced system: first structurally non-zero column of compact row i (<= i)
    int esize;          // number of stored entries = sum_i (i - efirst[i] + 1)
    int plan_off;       // the envelope's factorisation plan in chol_plan (kernels_solve.cuh; windows with one envelope share it)
    unsigned char flags[NB], mask[NB];
    double G[3], S_vis[4], w_plane[3], huber;
};

enum { ST_RUNNING = 0, ST_DONE = 1 };
enum { PH_INIT = 0, PH_CAND = 1 };

struct WinWork {        // solver state of one window (read-write)
    int status, term, phase;
    int iteration, num_iterations, successful, num_linear, num_invalid;
    int reuse, first;   // first: the pending linearisation is the first one (Jacobi scales are computed from it)
    int marg_status;    // 0 ok, <0 numeric problem on the marginalisation fast path
    int pad;
    double radius, mu, mu_lin;      // mu_lin: the mu the pending linearisation's Schur weights gamma were built with
    double x_cost, x_norm, step_norm, model_cost_change, dogleg_step_norm, alpha;
    double q_gg, q_gn, q_nn, l_g, l_n;   // v'Hv, v'Hn, n'Hn, g.v, g.n  with v = sgrad/D, n = gn/D (scaled space)
    double sgrad_norm, gn_norm, sgrad_dot_gn;
    double initial_cost, gradient_max_norm;
    double small_cost;  // cost of IMU/wheel/plane/prior at the evaluated point (written by lin_small)
};

struct Opts {
    int max_num_iterations, max_invalid, jacobi_scaling;
    double function_tolerance, gradient_tolerance, parameter_tolerance;
    double initial_radius, max_radius, min_radius, min_relative_decrease, min_lm_diagonal, max_lm_diagonal;
};

struct BatchDev {       // passed by value to every kernel
    int B, nvis_total, nlm_total, nimu_total, nwheel_total, nplane_total, nprior, nitems_solve, nitems_marg;
    int env_max, nf_max;    // largest esize and nf over the batch (size the solve kernel's shared memory)
    int marg_nmax;          // largest prior dimension any window of the batch produces (sizes the eigen-solver's shared memory)
    int n_unfused;          // windows whose solver linearisation runs lin_vis + lm_reduce + asm_items (the others: lin_vis_lm(_wide), WinMeta.fused)
    int n_fused_wide, n_fused_compact, n_munfused, n_mfused;      // fused solver windows by record width; marginalising windows by path
    int nlmb_total, npitems_total, nmpitems_total, pitems_max;
    int pout_stride;        // doubles per solver pair item in pair_out: 192 (all fused windows compact) or 640
    const int *mvis_pos;            // [nvis_total] marginalisation: window-local record slot of the factors hosted in frame 0 (-1 otherwise)
    const struct AsmItem *mpitems;  // [nmpitems_total]
    double *mpair_out;              // [nmpitems_total][640]
    const int *vis_pos;             // [nvis_total] wide solver windows: window-local position of the factor's X record in frame-pair order (-1: none)
    int nrun_total;                 // host runs of the compact solver windows, longest first (the blocks of lin_vis_lm)
    const struct RunDesc *run_desc; // [nrun_total]
    const struct RunTile *run_tile; // tiles of every run, consecutive per run
    const int *run_f;               // [nvis_total] compact windows: the window's factors (global index) in run order, at the window's vis_off
    const int *run_lm;              // [nlm_total][2] compact windows: landmark (global) and its first row in its tile, in run order, at the window's lm_off
    unsigned char *vis_dup;         // [nvis_total] 0: the factor alone observes its landmark from frame j; 1: first of two such factors (adds the next one's part); 2: second (adds nothing)
    const struct LmbDesc *lmb_desc; // [nlmb_total] landmark blocks of lin_vis_lm: everything the block needs to start, in one 32-byte load
    double *xrec;                   // [nxrec_total][XREC]
    const struct AsmItem *pitems;   // [npitems_total] kind = ITEM_PAIR, lo / hi = absolute record range in xrec
    double *pair_out;               // [npitems_total][PAIR_OUT] tile (0,0), (0,1), (1,1) of G in mma.m8n8k4 accumulator order
    double *pair_red;               // [B][PAIR_RED] per frame: diagonal block (21) + gradient (6); per pair a < b: off-diagonal block (36)  (pair_reduce)
    const WinMeta *meta;
    const int *chol_plan;           // factorisation plans of the batch's distinct envelopes (kernels_solve.cuh chol_plan_build), at WinMeta.plan_off
    WinWork *work;
    const PriorDev *prior;
    Opts opt;
    // states
    double *x_cur, *x_cand, *x_init, *x_before;
    // visual tables
    const int *vis_lm;              // landmark index local to the window
    int *vis_type, *vis_fi, *vis_fj, *vis_win;   // written on the device by vis_expand from the wire format below
    double *vis_obs;                // [nvis_total][12] exactly as the caller's table (rebuilt by vis_expand)
    // wire format of the visual table (what crosses PCIe): per factor one code word (type | fi << 2 | fj << 6 | dup << 10), the observer side of the
    // observation (pts_j, velocity_j, td_j) and an index into the table of host sides (pts_i, velocity_i, td_i), which every factor of a landmark shares
    const int *vis_code, *vis_oi;
    const double *obs_i, *obs_j;    // [nobs_i_total][6], [nvis_total][6]
    double *vis_rec;                // [nvis_total][VREC] if some window is unfused (n_unfused or n_munfused), else a placeholder
    double *vis_cost;               // [nvis_total] the same
    // assembly plan (static per batch): items = chunks of per-frame / per-frame-pair / common factor lists
    const struct AsmItem *items;    // solver items of all windows, then marginalisation items
    const int *asm_list;            // list entries: (window-local factor index << 1) | role; item.lo/hi are relative to meta.list_off / mlist_off
    double *asm_out;                // [nitems_total][ASM_STRIDE] partial sums written by asm_items
    // landmarks
    const int *lm_win, *lm_fptr;    // [nlm_total], [nlm_total+1] factor range (global factor indices, sorted by landmark)
    double *lm_a, *lm_g, *lm_gamma, *lm_scale, *lm_cost, *lm_W;   // lm_W [nlm_total][VSUB]
    int *lm_outlier;                // [nlm_total] outliersRejection verdict (kernels_marg.cuh: outlier_block)
    double out_focal, out_thresh;   // FOCAL_LENGTH and the pixel threshold of estimator.cpp:2183
    // small factors
    const int *imu_fi, *imu_fj, *imu_win, *wheel_fi, *wheel_fj, *wheel_win, *plane_f, *plane_win;
    const double *imu_data, *wheel_data;   // [n][287], [n][78]
    double *imu_S, *wheel_S;               // [n][225], [n][36] upper sqrt-info, built once per solve
    double *imu_rec, *wheel_rec, *plane_rec;
    // prior
    const double *prior_J, *prior_r, *prior_x0;
    double *prior_A, *prior_res, *prior_g;
    // normal equations
    double *Hpk, *gpk, *Tvis, *tvec;   // Hpk [B][TFIX*(TFIX+1)/2] packed active H, gpk [B][TFIX] compact gradient
    // solver vectors, per window at work_off = state_off - 15*w ... stored at vec_off = w*TFIX + lm_off
    double *v_scale, *v_D, *v_sgrad, *v_gn;
    double *v_wug, *v_wun;              // [nlm_total] per landmark w_k . u_g and w_k . (C y) of the current linearisation (solve)
    // marginalisation outputs
    double *marg_J, *marg_r, *marg_x0;  // [B][marg_nmax^2] (n x n, row stride n, at the head of the slot), [B][MAXPRI], [B][SFIX]
    int *marg_hdr;                      // [B][2 + 2*NB]: valid, n, nb, block_id[], block_idx[]
    double *marg_de, *marg_rot;         // [B][2 * MAXPRI] tridiagonal (d | e) -> eigenvalues; [B][2 * 3 nmax^2] rotation log (c, s) of the QL iteration
    int *marg_sweep;                    // [B][2 + 2 * 12 nmax] sweep log: count, rotations, then (l | m << 16, first rotation) per QL sweep
};

VIWB_HD int vec_off(const BatchDev &bd, int w) { return w * TFIX + bd.meta[w].lm_off; }

}  // namespace viwb
