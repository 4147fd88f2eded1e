// kernels_asm.cuh -- assembly of the normal equations without atomics and without a dense H in HBM.
//
// The factor graph of a window is static during a solve, so the host builds an assembly plan once per batch:
//   FRAME  item (frame a, chunk)      : list of (factor, role) touching pose a      -> F^T F (21), F^T [E0 E1 td] (78), F^T r (6)
//   PAIR   item (frames a<b, chunk)   : list of (factor, role of a)                 -> F_a^T F_b (36)
//   COMMON item (chunk)               : all factors                                 -> [E0 E1 td]^T [E0 E1 td] (91), ^T r (13)
// Lists are cut into chunks of ASM_CHUNK entries; chunk c of every list is "phase" c.  Items of one phase write
// disjoint blocks of H, so the consumer adds them phase by phase with plain stores (deterministic).
//   asm_items  : ASM_SPLIT warps per item, lanes over the item's outputs, records streamed from HBM/L2 (54 doubles per factor)
//   assemble_into(target) : called by the solve kernel (packed shared-memory triangle) and by the marginalisation
//                kernel (dense marginalisation layout): prior J^T J, IMU / wheel / plane J^T J factor by factor,
//                visual partial sums phase by phase.
#pragma once
#include "layout.cuh"
#include "factors.cuh"
#include "kernels_lin.cuh"

namespace viwb {

// slot table of a small factor: (block id, first column inside its Jacobian record), ascending columns
struct Slot { int blk, col; };
VIWB_D int imu_slots(int i, int j, Slot *s) { s[0].blk = i; s[0].col = 0; s[1].blk = BLK_SB0 + i; s[1].col = 6; s[2].blk = j; s[2].col = 15; s[3].blk = BLK_SB0 + j; s[3].col = 21; return 4; }
VIWB_D int wheel_slots(int i, int j, Slot *s) {
    s[0].blk = i; s[0].col = 0; s[1].blk = j; s[1].col = 6; s[2].blk = BLK_EXW; s[2].col = 12; s[3].blk = BLK_SX; s[3].col = 18;
    s[4].blk = BLK_SY; s[4].col = 19; s[5].blk = BLK_SW; s[5].col = 20; s[6].blk = BLK_TDW; s[6].col = 21; return 7;
}
VIWB_D int plane_slots(int i, Slot *s) { s[0].blk = i; s[0].col = 0; s[1].blk = BLK_EXW; s[1].col = 6; s[2].blk = BLK_PR; s[2].col = 12; s[3].blk = BLK_PZ; s[3].col = 15; return 4; }

// offset of common column c (0..12: ex0 6 | ex1 6 | td) inside a visual record, and its row stride
VIWB_HD int common_off(int c) { return c < 6 ? REC_E0 + c : c < 12 ? REC_E1 + (c - 6) : REC_TD; }
VIWB_HD int common_stride(int c) { return c < 12 ? 6 : 1; }
VIWB_HD void sym_unrank(int e, int &p, int &q) {   // e = p(p+1)/2 + q, 0 <= q <= p
    int pp = (int)((sqrtf(8.0f * (float)e + 1.0f) - 1.0f) * 0.5f);      // single-precision estimate, made exact by the two loops (e < 2^22)
    while ((pp + 1) * (pp + 2) / 2 <= e) pp++;
    while (pp * (pp + 1) / 2 > e) pp--;
    p = pp; q = e - pp * (pp + 1) / 2;
}

// ------------------------------------------------------------------------------------------------ asm_items
// grid: ceil(nitems * ASM_SPLIT / warps_per_block); mode selects the solver or the marginalisation item table.
enum { ASM_SPLIT = 4 };
VIWB_D void asm_items_block(const BatchDev &bd, int bx, int by, int tid, int nt, double *smem, int mode) {
    (void)by; (void)smem;
    const int W = nt < 32 ? nt : 32, wpb = nt / W, lane = tid % W;
    // Items with the common columns have up to 105 outputs: ASM_SPLIT warps share such an item (one slice of the outputs each, the
    // same list walk) instead of one warp walking the list four times.
    const int nitems = (mode == MODE_SOLVE) ? bd.nitems_solve : bd.nitems_marg;
    const int wi = bx * wpb + tid / W, it = wi / ASM_SPLIT, part = wi - it * ASM_SPLIT;
    if (it >= nitems) return;
    const int gi = (mode == MODE_SOLVE) ? it : bd.nitems_solve + it;
    const AsmItem item = bd.items[gi];
    if (mode == MODE_SOLVE && bd.work[item.win].status != ST_RUNNING) return;
    double *out = bd.asm_out + (size_t)gi * ASM_STRIDE;
    const WinMeta &wm = bd.meta[item.win];
    const int *list = bd.asm_list + (mode == MODE_SOLVE ? wm.list_off : wm.mlist_off);
    const double *recs = bd.vis_rec + (size_t)wm.vis_off * VREC;
    // outputs of this item; without common columns a FRAME item has only F^T F (21) and F^T r (6 -> stored at 99..104)
    int nout;
    if (item.kind == ITEM_FRAME) nout = item.has_common ? 105 : 27; else if (item.kind == ITEM_PAIR) nout = 36; else nout = 104;
    if (item.kind == ITEM_FRAME && !item.has_common && part == 0) for (int o = 21 + lane; o < 99; o += W) out[o] = 0.0;
    for (int o0 = lane + W * part; o0 < nout; o0 += W * ASM_SPLIT) {
        int o = o0;
        if (item.kind == ITEM_FRAME && !item.has_common && o0 >= 21) o = 99 + (o0 - 21);
        // operand kinds: 0 = frame slot of a, 1 = frame slot of b (PAIR), 2 = common column, 3 = residual
        int ka = 0, kb = 0, pa = 0, pb = 0;
        if (item.kind == ITEM_FRAME) {
            if (o < 21) { sym_unrank(o, pa, pb); ka = 0; kb = 0; }
            else if (o < 99) { pa = (o - 21) / 13; pb = (o - 21) % 13; ka = 0; kb = 2; }
            else { pa = o - 99; ka = 0; kb = 3; }
        } else if (item.kind == ITEM_PAIR) { pa = o / 6; pb = o % 6; ka = 0; kb = 1; }
        else { if (o < 91) { sym_unrank(o, pa, pb); ka = 2; kb = 2; } else { pa = o - 91; ka = 2; kb = 3; } }
        // role-independent parts of the record offsets
        const int ia_c = (ka == 2) ? common_off(pa) : pa, sa = (ka == 2) ? common_stride(pa) : 6;
        const int ib_c = (kb == 2) ? common_off(pb) : (kb == 3 ? 0 : pb), sb = (kb == 2) ? common_stride(pb) : (kb == 3 ? 1 : 6);
        double acc = 0.0;
        int e = item.lo;
        int nx[4] = {0, 0, 0, 0};                  // list entries of the next group, fetched one group ahead of the records they index
        if (e + 4 <= item.hi) for (int u = 0; u < 4; u++) nx[u] = list[e + u];
        for (; e + 4 <= item.hi; e += 4) {        // 4 independent gather chains in flight
            int en[4]; const double *rc[4]; double va[4], vb[4], wa[4], wb[4];
            for (int u = 0; u < 4; u++) en[u] = nx[u];
            if (e + 8 <= item.hi) for (int u = 0; u < 4; u++) nx[u] = list[e + 4 + u];
            for (int u = 0; u < 4; u++) {
                const int role = en[u] & 1;
                rc[u] = recs + (size_t)(en[u] >> 1) * VREC;
                const int ia = (ka == 0) ? (role ? REC_B : REC_A) + ia_c : ia_c;
                const int ib = (kb == 0) ? (role ? REC_B : REC_A) + ib_c : (kb == 1 ? (role ? REC_A : REC_B) + ib_c : ib_c);
                va[u] = rc[u][ia]; wa[u] = rc[u][ia + sa]; vb[u] = rc[u][ib]; wb[u] = rc[u][ib + sb];
            }
            for (int u = 0; u < 4; u++) acc += va[u] * vb[u] + wa[u] * wb[u];
        }
        for (; e < item.hi; e++) {
            const int ent = list[e], role = ent & 1;
            const double *rec = recs + (size_t)(ent >> 1) * VREC;
            const int ia = (ka == 0) ? (role ? REC_B : REC_A) + ia_c : ia_c;
            const int ib = (kb == 0) ? (role ? REC_B : REC_A) + ib_c : (kb == 1 ? (role ? REC_A : REC_B) + ib_c : ib_c);
            acc += rec[ia] * rec[ib] + rec[ia + sa] * rec[ib + sb];
        }
        out[o] = acc;
    }
}

// ------------------------------------------------------------------------------------------------ assemble_into
// A target provides:  int col(int blk, int k)  (-1 if that column is not part of the system),
//                     void add(int i, int j, double v)  for an unordered index pair (called once per pair per phase),
//                     void addg(int i, double v).
struct PackedTarget {      // solver: skyline lower triangle in shared memory over the compact active columns
    double *L, *g; const short *tcol; const short *rp, *fst;
    VIWB_DM int col(int blk, int k) const { return (tcol[blk] >= 0 && k < blk_tsize(blk)) ? tcol[blk] + k : -1; }
    VIWB_DM void add(int i, int j, double v) const { if (i < j) { const int t = i; i = j; j = t; } L[rp[i] - fst[i] + j] += v; }
    VIWB_DM void addg(int i, double v) const { g[i] += v; }
};
struct DenseTarget {       // marginalisation: dense symmetric matrix in the marginalisation layout (global memory)
    double *M, *g; int ld; const unsigned char *flags;
    VIWB_DM int col(int blk, int k) const { return ((flags[blk] & 1u) && k < blk_msize(blk)) ? blk_moff(blk) + k : -1; }
    VIWB_DM void add(int i, int j, double v) const { M[(size_t)i * ld + j] += v; if (i != j) M[(size_t)j * ld + i] += v; }
    VIWB_DM void addg(int i, double v) const { g[i] += v; }
};

// J^T J / J^T r of one small factor: J rows x ld (row-major) with `ns` parameter slots
template <typename Target>
VIWB_D void add_small_factor(const Target &t, const double *rec, int rows, int ld, const Slot *sl, int ns, int tid, int nt) {
    const double *res = rec, *J = rec + rows;
    // local column -> (block, k)
    for (int e = tid; e < ld * (ld + 1) / 2 + ld; e += nt) {
        if (e < ld * (ld + 1) / 2) {
            int p, q; sym_unrank(e, p, q);
            int bp = -1, kp = 0, bq = -1, kq = 0;
            for (int s = 0; s < ns; s++) { if (p >= sl[s].col) { bp = sl[s].blk; kp = p - sl[s].col; } if (q >= sl[s].col) { bq = sl[s].blk; kq = q - sl[s].col; } }
            const int ci = t.col(bp, kp), cj = t.col(bq, kq);
            if (ci < 0 || cj < 0) continue;
            double v = 0.0;
            for (int r = 0; r < rows; r++) v += J[r * ld + p] * J[r * ld + q];
            t.add(ci, cj, v);
        } else {
            const int p = e - ld * (ld + 1) / 2;
            int bp = -1, kp = 0;
            for (int s = 0; s < ns; s++) if (p >= sl[s].col) { bp = sl[s].blk; kp = p - sl[s].col; }
            const int ci = t.col(bp, kp);
            if (ci < 0) continue;
            double v = 0.0;
            for (int r = 0; r < rows; r++) v += J[r * ld + p] * res[r];
            t.addg(ci, v);
        }
    }
    VIWB_SYNC();
}

// common column c (0..12) -> (block, k)
VIWB_HD int common_blk(int c) { return c < 6 ? BLK_EX0 : c < 12 ? BLK_EX1 : BLK_TD; }
VIWB_HD int common_k(int c) { return c < 6 ? c : c < 12 ? c - 6 : 0; }

// Adds every contribution to the (zero-initialised by the caller) target.  All threads of the block must call it.
// imap: >= MAXPRI ints of block-shared scratch.  Every stage gives each matrix entry exactly one owner thread, and stages
// that may touch the same entries are separated by a barrier (no atomics; fixed summation order).
template <typename Target>
VIWB_D void assemble_into(const Target &t, const BatchDev &bd, int w, int mode, int tid, int nt, int *imap) {
    const WinMeta &m = bd.meta[w];
    const bool prior_only = marg_prior_only(m, mode);
    // ---- prior: A = J_lin^T J_lin (constant during the solve) and g = J_lin^T r, entry-parallel over the lower triangle
    if (m.prior_idx >= 0) {
        const PriorDev &pr = bd.prior[m.prior_idx];
        const double *A = bd.prior_A + pr.J_off, *g = bd.prior_g + pr.r_off;
        for (int bi = tid; bi < pr.nb; bi += nt) {
            const int ba = pr.block_id[bi];
            for (int p = 0; p < blk_msize(ba); p++) imap[pr.block_idx[bi] + p] = t.col(ba, p);
        }
        VIWB_SYNC();
        const int n = pr.n;
        for (int e = tid; e < n * (n + 1) / 2; e += nt) {
            int i, j; sym_unrank(e, i, j);
            const int ci = imap[i], cj = imap[j];
            if (ci >= 0 && cj >= 0) t.add(ci, cj, A[(size_t)i * n + j]);
        }
        for (int i = tid; i < n; i += nt) if (imap[i] >= 0) t.addg(imap[i], g[i]);
    }
    VIWB_SYNC();
    // ---- IMU: factor k joins frames (i, j = i + 1) (estimator.cpp:1528-1538), so factors of equal parity touch disjoint blocks:
    //      two barrier-separated passes instead of one per factor.  Wheel / plane factors share the wheel extrinsic and
    //      intrinsic blocks among all of them and stay one factor at a time.
    Slot sl[8];
    if (!prior_only) {
        bool chain = true;
        for (int k = 0; k < m.nimu; k++) { const int f = m.imu_off + k; if (bd.imu_fj[f] != bd.imu_fi[f] + 1) chain = false; }
        if (chain && mode == MODE_SOLVE) {
            const int per = 30 * 31 / 2 + 30;
            for (int par = 0; par < 2; par++) {
                for (int e = tid; e < m.nimu * per; e += nt) {
                    const int k = e / per, o = e - k * per, f = m.imu_off + k, i = bd.imu_fi[f];
                    if ((i & 1) != par) continue;
                    const double *res = bd.imu_rec + (size_t)f * IMU_REC, *J = res + 15;
                    // local column -> (block, k): [pose_i 6 | sb_i 9 | pose_j 6 | sb_j 9]
                    auto lc = [&](int p) { return p < 6 ? t.col(i, p) : p < 15 ? t.col(BLK_SB0 + i, p - 6) : p < 21 ? t.col(i + 1, p - 15) : t.col(BLK_SB0 + i + 1, p - 21); };
                    if (o < 465) {
                        int p, q; sym_unrank(o, p, q);
                        const int ci = lc(p), cj = lc(q);
                        if (ci < 0 || cj < 0) continue;
                        double v = 0.0;
                        for (int r = 0; r < 15; r++) v += J[r * 30 + p] * J[r * 30 + q];
                        t.add(ci, cj, v);
                    } else {
                        const int p = o - 465, ci = lc(p);
                        if (ci < 0) continue;
                        double v = 0.0;
                        for (int r = 0; r < 15; r++) v += J[r * 30 + p] * res[r];
                        t.addg(ci, v);
                    }
                }
                VIWB_SYNC();
            }
        } else {
            for (int k = 0; k < m.nimu; k++) {
                const int f = m.imu_off + k, i = bd.imu_fi[f], j = bd.imu_fj[f];
                if (mode == MODE_MARG && !(i == 0 && j == 1)) continue;
                const int ns = imu_slots(i, j, sl);
                add_small_factor(t, bd.imu_rec + (size_t)f * IMU_REC, 15, 30, sl, ns, tid, nt);
            }
        }
        for (int k = 0; k < m.nwheel; k++) {
            const int f = m.wheel_off + k, i = bd.wheel_fi[f], j = bd.wheel_fj[f];
            if (mode == MODE_MARG && !(i == 0 && j == 1)) continue;
            const int ns = wheel_slots(i, j, sl);
            add_small_factor(t, bd.wheel_rec + (size_t)f * WHEEL_REC, 6, 22, sl, ns, tid, nt);
        }
        for (int k = 0; k < m.nplane; k++) {
            const int f = m.plane_off + k, i = bd.plane_f[f];
            if (mode == MODE_MARG && i != 0) continue;
            const int ns = plane_slots(i, sl);      // plane_R: 3 tangent columns; its 4th marginalisation column stays zero
            add_small_factor(t, bd.plane_rec + (size_t)f * PLANE_REC, 3, 16, sl, ns, tid, nt);
        }
    }
    if (mode == MODE_SOLVE ? m.fused != 0 : m.mfused != 0) {
        // ---- fused path: pair_reduce (kernels_fused.cuh) has folded the pair chunks G = sum X^T X into per-frame diagonal blocks + gradients
        //      (+ the frame's block against the common columns ex0 | ex1 | td when the records are WIDE), per-pair off-diagonal blocks and the
        //      common block.  Exact zeros are frames / pairs without factors (their entries may lie outside the envelope) and are skipped.
        const bool wide = mode == MODE_MARG || m.has_common != 0;
        const int FR = wide ? 105 : 27;
        const double *red = bd.pair_red + (size_t)w * PAIR_RED;
        for (int e = tid; e < NFR * FR; e += nt) {
            const double v = red[e];
            if (v == 0.0) continue;
            const int f = e / FR, o = e - FR * f;
            if (o < 21) { int p, q; sym_unrank(o, p, q); const int ci = t.col(f, p), cj = t.col(f, q); if (ci >= 0 && cj >= 0) t.add(ci, cj, v); }
            else if (o < 27) { const int ci = t.col(f, o - 21); if (ci >= 0) t.addg(ci, v); }
            else { const int p = (o - 27) / 13, c = (o - 27) % 13; const int ci = t.col(f, p), cj = t.col(common_blk(c), common_k(c)); if (ci >= 0 && cj >= 0) t.add(ci, cj, v); }
        }
        for (int e = tid; e < NPAIR * 36; e += nt) {
            const double v = red[NFR * FR + e];
            if (v == 0.0) continue;
            int pi = e / 36, a = 0; const int o = e - 36 * pi;
            while (pi >= NFR - 1 - a) { pi -= NFR - 1 - a; a++; }
            const int ci = t.col(a, o / 6), cj = t.col(a + 1 + pi, o % 6);
            if (ci >= 0 && cj >= 0) t.add(ci, cj, v);
        }
        if (wide) for (int e = tid; e < 91 + 13; e += nt) {
            const double v = red[NFR * FR + NPAIR * 36 + e];
            if (v == 0.0) continue;
            if (e < 91) { int p, q; sym_unrank(e, p, q); const int ci = t.col(common_blk(p), common_k(p)), cj = t.col(common_blk(q), common_k(q)); if (ci >= 0 && cj >= 0) t.add(ci, cj, v); }
            else { const int c = e - 91; const int ci = t.col(common_blk(c), common_k(c)); if (ci >= 0) t.addg(ci, v); }
        }
        VIWB_SYNC();
        return;
    }
    // ---- visual partial sums: the chunks of one target (same frame / frame pair / common block) are consecutive items with
    //      phase 0, 1, 2, ...; the owner of entry o of the head item gathers the chunks, so one pass and no barriers
    const int ioff = (mode == MODE_SOLVE) ? m.item_off : bd.nitems_solve + m.mitem_off;
    const int ni = (mode == MODE_SOLVE) ? m.nitems : (m.margin_flag == 0 ? m.nmitems : 0);
    for (int e = tid; e < ni * ASM_STRIDE; e += nt) {
        const int ii = e / ASM_STRIDE, o = e - ii * ASM_STRIDE;
        const AsmItem &item = bd.items[ioff + ii];
        if (item.phase != 0) continue;
        double v = bd.asm_out[(size_t)(ioff + ii) * ASM_STRIDE + o];
        for (int c = 1; ii + c < ni && bd.items[ioff + ii + c].phase == c; c++) v += bd.asm_out[(size_t)(ioff + ii + c) * ASM_STRIDE + o];
        if (item.kind == ITEM_FRAME) {
            if (o < 21) { int p, q; sym_unrank(o, p, q); const int ci = t.col(item.a, p), cj = t.col(item.a, q); if (ci >= 0 && cj >= 0) t.add(ci, cj, v); }
            else if (o < 99) { const int p = (o - 21) / 13, c = (o - 21) % 13; const int ci = t.col(item.a, p), cj = t.col(common_blk(c), common_k(c)); if (ci >= 0 && cj >= 0 && item.has_common) t.add(ci, cj, v); }
            else if (o < 105) { const int ci = t.col(item.a, o - 99); if (ci >= 0) t.addg(ci, v); }
        } else if (item.kind == ITEM_PAIR) {
            if (o < 36) { const int ci = t.col(item.a, o / 6), cj = t.col(item.b, o % 6); if (ci >= 0 && cj >= 0) t.add(ci, cj, v); }
        } else {
            if (o < 91) { int p, q; sym_unrank(o, p, q); const int ci = t.col(common_blk(p), common_k(p)), cj = t.col(common_blk(q), common_k(q)); if (ci >= 0 && cj >= 0) t.add(ci, cj, v); }
            else if (o < 104) { const int c = o - 91; const int ci = t.col(common_blk(c), common_k(c)); if (ci >= 0) t.addg(ci, v); }
        }
    }
    VIWB_SYNC();
}

}  // namespace viwb
