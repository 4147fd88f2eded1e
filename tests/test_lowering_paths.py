"""The host lowering plans each window's solver linearisation -- compact (host runs of lin_vis_lm), wide (landmark blocks of lin_vis_lm_wide) or
unfused (lin_vis / lm_reduce / asm_items) -- and its marginalisation -- none, wide or unfused -- on its own (lower_count in viwb.cu).  One batch holds
every combination, each window's paths checked with the decision rule restated below.  Every window of the batch must give what it gives alone, bit for
bit, and agree with the CPU oracle; with VIWB_NO_FUSED=1 (every window unfused) it must still agree with the oracle.  The `emu` twin runs the device
source compiled for the host (tests/emu), the `gpu` twin libviwb.so."""
import numpy as np
import pytest

import parity_checks as pc
from viwb import abi, synth

LMB_FACTORS, PAIR_CHUNK = 128, 64
COMPACT, WIDE, UNFUSED, NONE = "compact", "wide", "unfused", "none"


@pytest.fixture(scope="module")
def emu_ctx():
    from emu import build_emu
    from viwb import lib as viwb_lib
    ctx = viwb_lib.Context(0, build_emu.build())
    yield ctx
    ctx.close()


@pytest.fixture(params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def ctx(request):
    return request.getfixturevalue("emu_ctx" if request.param == "emu" else "gpu_ctx")


def chunks(n, c=PAIR_CHUNK):
    return -(-int(n) // c)


def regular(prob):
    """Grouped by landmark, <= LMB_FACTORS factors per landmark, and per (landmark, observer) at most two two-frame factors, consecutive."""
    lm = prob.vis_landmark
    if np.any(np.diff(lm) < 0):
        return False
    for k in range(prob.num_landmarks):
        rows = np.flatnonzero(lm == k)
        if len(rows) > LMB_FACTORS:
            return False
        two = rows[prob.vis_type[rows] != abi.F_PROJ_1F2C]
        for j in set(prob.vis_frame_j[two].tolist()):
            r = two[prob.vis_frame_j[two] == j]
            if len(r) > 2 or (len(r) == 2 and r[1] != r[0] + 1):
                return False
    return True


def paths(prob, flag, allow_fused=True):
    """(solver path, marginalisation path) of the window.  Marginalisation: MARGIN_OLD of a full window (every window here has the IMU factor
    (0, 1), so frame 0 always takes part); MARGIN_SECOND_NEW without a prior marginalises nothing."""
    t, fi, fj = prob.vis_type, prob.vis_frame_i, prob.vis_frame_j
    two, one = t != abi.F_PROJ_1F2C, t == abi.F_PROJ_1F2C
    in_prior = {b for b, _ in prob.prior.blocks()} if prob.prior is not None and prob.prior.valid else set()
    used = {abi.BLK_EX_POSE0: len(t) > 0, abi.BLK_EX_POSE1: bool(np.any(t != abi.F_PROJ_2F1C)), abi.BLK_TD: len(t) > 0}
    has_common = any((u or b in in_prior) and prob.block_flags[b] & abi.BLOCK_PRESENT and not prob.block_flags[b] & abi.BLOCK_CONSTANT for b, u in used.items())
    pairs = lambda sel: sum(chunks(n) for n in np.unique(np.minimum(fi, fj)[sel] * 11 + np.maximum(fi, fj)[sel], return_counts=True)[1])
    npit = pairs(two) + (sum(chunks(n) for n in np.bincount(fi[one], minlength=11)) if has_common else 0)
    nmpit = pairs(two & (fi == 0)) + chunks(np.sum(one & (fi == 0)))
    marg = flag == abi.MARGIN_OLD and prob.frame_count == abi.WINDOW_SIZE
    assert not marg or np.any((prob.imu_frame_i == 0) & (prob.imu_frame_j == 1))
    fused = allow_fused and regular(prob)
    solve = (WIDE if has_common else COMPACT) if fused and npit > 0 else UNFUSED
    return solve, (WIDE if fused and nmpit > 0 else UNFUSED) if marg else NONE


def window(prob, rows=None, **kw):
    """The window with only the visual factors `rows` (indices, in that order); keyword arguments replace other fields."""
    rows = np.arange(len(prob.vis_type)) if rows is None else rows
    f = dict(frame_count=prob.frame_count, num_landmarks=prob.num_landmarks, block_flags=prob.block_flags, subset_mask=prob.subset_mask,
             vis_type=prob.vis_type[rows], vis_landmark=prob.vis_landmark[rows], vis_frame_i=prob.vis_frame_i[rows], vis_frame_j=prob.vis_frame_j[rows],
             vis_obs=prob.vis_obs[rows], imu_frame_i=prob.imu_frame_i, imu_frame_j=prob.imu_frame_j, imu_data=prob.imu_data,
             wheel_frame_i=prob.wheel_frame_i, wheel_frame_j=prob.wheel_frame_j, wheel_data=prob.wheel_data, plane_frame=prob.plane_frame,
             prior=prob.prior, globals_=prob.globals)
    f.update(kw)
    return abi.WindowProblem(**f)


def not_hosted_in_frame0(seq, cid):
    prob, st, _ = synth.make_window(cid, seq)
    return window(prob, np.flatnonzero(prob.vis_frame_i != 0)), st


@pytest.fixture(scope="module")
def cases(oracle):
    """[(name, problem, state, margin flag, (solver path, marginalisation path), oracle result)]"""
    out = []

    def add(name, prob, st, flag, expect):
        out.append((name, prob, st, flag, expect))

    p, s, _ = synth.make_window(2, 1)
    add("compact C2", p, s, abi.MARGIN_OLD, (COMPACT, WIDE))
    p, s, _ = synth.make_window(4, 2)
    add("wide C4", p, s, abi.MARGIN_OLD, (WIDE, WIDE))
    p, s, _ = synth.make_window(2, 3)
    add("shuffled C2", window(p, np.random.default_rng(7).permutation(len(p.vis_type))), s, abi.MARGIN_OLD, (UNFUSED, UNFUSED))
    p, s, _ = synth.make_window(2, 4)
    add("C2, MARGIN_SECOND_NEW", p, s, abi.MARGIN_SECOND_NEW, (COMPACT, NONE))
    p, s, _ = synth.make_window(2, 5)
    flags = p.block_flags.copy()
    flags[7:11] = 0
    flags[abi.BLK_SPEEDBIAS0 + 7:abi.BLK_SPEEDBIAS0 + 11] = 0
    add("C2, frame_count 6", window(p, np.flatnonzero(p.vis_frame_j <= 6), frame_count=6, block_flags=flags, imu_frame_i=p.imu_frame_i[:6],
                                    imu_frame_j=p.imu_frame_j[:6], imu_data=p.imu_data[:6]), s, abi.MARGIN_OLD, (COMPACT, NONE))
    p, s, _ = synth.make_window(2, 6)
    add("C2, one-frame factors only", window(p, np.flatnonzero(p.vis_type == abi.F_PROJ_1F2C)), s, abi.MARGIN_OLD, (UNFUSED, WIDE))
    p, s, _ = synth.make_window(2, 7)
    add("IMU only", window(p, [], num_landmarks=0), s[:abi.STATE_FIXED], abi.MARGIN_OLD, (UNFUSED, UNFUSED))
    seq = synth.Sequence(synth.make_config(2), 8, 12)
    p, s, _ = seq.window(0)
    a = oracle.gauge_reanchor(p, s, oracle.window_solve(p, s)[0])
    p, s, _ = seq.window(1, prior=oracle.marginalize(p, a, abi.MARGIN_OLD), prev_state=a)
    add("C2 with a prior", p, s, abi.MARGIN_OLD, (COMPACT, WIDE))
    # the remaining combinations
    p, s, _ = synth.make_window(4, 9)
    add("wide C4, MARGIN_SECOND_NEW", p, s, abi.MARGIN_SECOND_NEW, (WIDE, NONE))
    p, s, _ = synth.make_window(2, 10)
    add("shuffled C2, MARGIN_SECOND_NEW", window(p, np.random.default_rng(11).permutation(len(p.vis_type))), s, abi.MARGIN_SECOND_NEW, (UNFUSED, NONE))
    add("C2, nothing hosted in frame 0", *not_hosted_in_frame0(11, 2), abi.MARGIN_OLD, (COMPACT, UNFUSED))
    add("C4, nothing hosted in frame 0", *not_hosted_in_frame0(12, 4), abi.MARGIN_OLD, (WIDE, UNFUSED))
    return [(n, p, s, f, e, oracle.optimization(p, s, f)) for n, p, s, f, e in out]


def test_batch_holds_every_path(cases):
    for name, p, s, f, expect, _ in cases:
        assert paths(p, f) == expect, name
        assert paths(p, f, allow_fused=False) == (UNFUSED, UNFUSED if expect[1] != NONE else NONE), name
    assert {e for _, _, _, _, e, _ in cases} == {(a, b) for a in (COMPACT, WIDE, UNFUSED) for b in (WIDE, UNFUSED, NONE)}


def check_oracle(name, ref, state, summary):
    a0, sm0, _ = ref
    assert sm0.num_iterations == summary.num_iterations, name
    ep, er = synth.pose_errors(a0, state)
    assert ep <= pc.TIGHT_M and er <= pc.TIGHT_RAD, (name, ep, er)


def test_batch_matches_alone_and_oracle(ctx, cases):
    out_s, out_sum, out_pr = ctx.optimization_batch([c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases])
    for (name, p, s, f, _, ref), bs, bsum, bpr in zip(cases, out_s, out_sum, out_pr):
        a, sm, q = ctx.optimization(p, s, f)
        assert np.array_equal(a, bs), name
        assert [getattr(sm, k) for k, _ in abi.Summary._fields_] == [getattr(bsum, k) for k, _ in abi.Summary._fields_], name
        assert q.valid == bpr.valid and q.n == bpr.n and q.blocks() == bpr.blocks(), name
        assert np.array_equal(q.Jmat(), bpr.Jmat()) and np.array_equal(q.rvec(), bpr.rvec()), name
        check_oracle(name, ref, bs, bsum)


def test_no_fused(ctx, cases, monkeypatch):
    """VIWB_NO_FUSED=1, read by every batch build: the whole batch on the unfused path, whose rounds launch fewer kernels (no lin_vis_lm(_wide),
    asm_pairs_wide or pair_reduce)."""
    def run():
        n0 = ctx.launch_count()
        out = ctx.optimization_batch([c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases])
        return out, ctx.launch_count() - n0
    _, fused_launches = run()
    monkeypatch.setenv("VIWB_NO_FUSED", "1")
    (out_s, out_sum, _), launches = run()
    assert launches < fused_launches
    for (name, *_, ref), bs, bsum in zip(cases, out_s, out_sum):
        check_oracle(name, ref, bs, bsum)
