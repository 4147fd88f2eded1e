"""Marginalisation edges against an independent restatement of the reference's prior.

Every window's marginalisation (marg_prep, marg_tri / marg_ql / marg_apply or marg_eig, and the MODE_MARG branches of the linearisation kernels)
produces the prior the next window is anchored to; an error in it is not caught by the next solve, it propagates down the sequence.  Each case here
compares the library's prior with the oracle (oracle/vo_marg.c) and with `hp_marginalize`, a numpy restatement of
MarginalizationInfo::marginalize (marginalization_factor.cpp:282-306) that shares no code with either: equal kept dimension, equal block ids and
offsets, bit-equal linearisation point, and J^T J, J^T r within TIGHT of their max-abs.  The cases are MARGIN_SECOND_NEW with a prior that holds
pose 9, its pass-through, MARGIN_OLD with an incoming prior, landmarks seen only from their host's camera centre, a kept block with an exactly zero
row, the largest kept dimension next to a small one in one batch, and the unfused and one-kernel eigen paths.  The `emu` twin runs the device
source compiled for the host (tests/emu), the `gpu` twin libviwb.so."""
import dataclasses
import os
import subprocess
import sys

import numpy as np
import pytest

from test_lowering_paths import window
from viwb import abi, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TIGHT = 1e-6          # library vs oracle / hp_marginalize, relative to the max-abs of J^T J and of J^T r
SELF = 1e-8           # hp_marginalize vs oracle (the stationary window reaches 9.4e-9 on J^T r)
EPS = 1e-8            # marginalization_factor.h:81


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


# ------------------------------------------------------------------------------------------------ the reference's prior, restated
def hp_marginalize(A, b, m, n):
    """marginalization_factor.cpp:282-306 on the dense system (dropped dimensions first) of oracle.marginalize(..., want_system=True): Amm
    symmetrised and pseudo-inverted through its eigenvalues (> 1e-8 kept), the Schur complement formed in long double and rounded once, its
    eigen-decomposition cut the same way.  Returns the information form (J^T J, J^T r) of J = sqrt(S) V^T, r = sqrt(S^-1) V^T b, and n."""
    Amm = 0.5 * (A[:m, :m] + A[:m, :m].T)
    w, V = np.linalg.eigh(Amm)
    Vk = V[:, w > EPS]
    Amm_inv = (Vk / w[w > EPS]) @ Vk.T
    L = np.longdouble
    T = A[m:, :m].astype(L) @ Amm_inv.astype(L)
    An = (A[m:, m:].astype(L) - T @ A[:m, m:].astype(L)).astype(np.float64)
    bn = (b[m:].astype(L) - T @ b[:m].astype(L)).astype(np.float64)
    s, U = np.linalg.eigh(An)
    keep = s > EPS
    J = np.sqrt(s[keep])[:, None] * U[:, keep].T
    r = np.sqrt(1.0 / s[keep]) * (U[:, keep].T @ bn)
    return J.T @ J, J.T @ r, n


def rel(x, ref):
    return np.abs(x - ref).max() / np.abs(ref).max()


def oracle_prior(oracle, prob, state, flag):
    """(oracle prior, hp_marginalize's (J^T J, J^T r), Amm)"""
    q, A, b, (m, n) = oracle.marginalize(prob, state, flag, want_system=True)
    A0, b0, n0 = hp_marginalize(A, b, m, n)
    assert n0 == q.n
    return q, (A0, b0), A[:m, :m]


def check_prior(name, got, q, hp):
    assert got.valid and q.valid, name
    assert got.n == q.n, (name, got.n, q.n)
    assert got.blocks() == q.blocks(), (name, got.blocks(), q.blocks())
    assert np.array_equal(got.x0, q.x0), name
    A1, b1 = got.information()
    for what, (A0, b0) in (("oracle", q.information()), ("hp", hp)):
        assert rel(A1, A0) <= TIGHT and rel(b1, b0) <= TIGHT, (name, what, rel(A1, A0), rel(b1, b0))


def same_prior(a, b):
    if not (a.valid == b.valid and a.n == b.n and a.blocks() == b.blocks()):
        return False
    return not a.valid or (np.array_equal(a.x0, b.x0) and np.array_equal(a.Jmat(), b.Jmat()) and np.array_equal(a.rvec(), b.rvec()))


def shift_second_new(b):     # estimator.cpp:1843-1870: frame 10 takes the place of frame 9
    return 9 if b == 10 else 20 if b == 21 else b


def expected_blocks(kept):
    """[(new id, column offset)] of a prior keeping the blocks `kept` [(new id, id before the rename)], in ascending original id order"""
    out, off = [], 0
    for new, old in sorted(kept, key=lambda t: t[1]):
        out.append((new, off))
        off += abi.block_marg_size(old)
    return out


def reference_check(name, prob, state, flag, got, shift):
    """The library's prior against the reference's own MarginalizationInfo (compiled, or its stored results); skipped where neither has this call."""
    import viw_ref
    if not viw_ref.available():
        return
    try:
        ref = viw_ref.marginalize(prob, state, flag)
    except LookupError:
        return
    from test_reference_factors import _information_by_block
    assert ref["n"] == got.n, name
    ids0, A0, b0 = _information_by_block(ref["blocks"], ref["J"], ref["r"], shift)
    ids1, A1, b1 = _information_by_block(got.blocks(), got.Jmat(), got.rvec())
    assert ids0 == ids1, (name, ids0, ids1)
    assert rel(A1, A0) <= TIGHT and rel(b1, b0) <= TIGHT, (name, rel(A1, A0), rel(b1, b0))


# ------------------------------------------------------------------------------------------------ windows
def second_new_window(oracle, cid):
    """A MARGIN_OLD window, then the next one solved for MARGIN_SECOND_NEW: its prior holds pose 9 (the inputs of
    test_marginalization_second_new_matches_reference_code)."""
    seq = synth.Sequence(synth.make_config(cid), 3, 13)
    p, s, _ = seq.window(0)
    a, _, q = oracle.optimization(p, s, abi.MARGIN_OLD)
    p, s, _ = seq.window(1, prior=q, prev_state=a)
    a, _, _ = oracle.optimization(p, s, abi.MARGIN_SECOND_NEW, want_prior=False)
    return p, a


def with_frame10(prob, state, seed=0):
    """`prob` with its prior extended by pose 10 and speed-bias 10 (blocks 10 and 21), coupled to pose 9 and the prior's other blocks: a prior
    from MARGIN_OLD never holds them, but MARGIN_SECOND_NEW must rename them to 9 and 20 (estimator.cpp:1843-1870) when one does."""
    rng = np.random.default_rng(seed)
    q = prob.prior
    add = [b for b in (10, 21) if prob.block_flags[b] & abi.BLOCK_PRESENT]      # no speed-bias blocks without an IMU
    n, k = q.n, sum(abi.block_marg_size(b) for b in add)
    J = np.zeros((n + k, n + k))
    J[:n, :n] = q.Jmat()
    scale = np.abs(q.Jmat()).max()
    J[n:, :n] = rng.normal(0, 0.05 * scale, (k, n))
    J[n:, n:] = np.triu(rng.normal(0, 0.05 * scale, (k, k))) + np.eye(k) * 0.5 * scale
    r = np.r_[q.rvec(), rng.normal(0, 1.0, k)]
    x0 = q.x0.copy()
    blocks, off = q.blocks(), n
    for b in add:
        o, s = abi.block_offset(b), abi.block_size(b)
        x0[o:o + s] = state[o:o + s]
        blocks.append((b, off))
        off += abi.block_marg_size(b)
    prior = abi.PriorData.from_arrays(1, n + k, [b for b, _ in blocks], [i for _, i in blocks], x0, J, r)
    return window(prob, prior=prior)


def old_with_prior_window(oracle, cid):
    """The second window of a sequence, with the first one's MARGIN_OLD prior (the inputs of test_marginalization_matches_reference_code, k = 1)."""
    seq = synth.Sequence(synth.make_config(cid), 1, 13)
    p, s, _ = seq.window(0)
    a, _, q = oracle.optimization(p, s, abi.MARGIN_OLD)
    p, s, _ = seq.window(1, prior=q, prev_state=a)
    a, _, _ = oracle.optimization(p, s, abi.MARGIN_OLD, want_prior=False)
    return p, a


def stationary_window(baseline):
    """Mono C1 window whose frames 1 and 2 sit at frame 0's pose shifted by `baseline` (m, along the world y axis), the frame-0-hosted landmarks
    observed from frames 1 and 2 only.  At baseline 0 every such landmark's inverse-depth Jacobian is zero up to rounding."""
    p, s, _ = synth.make_window(1)
    s = s.copy()
    for f in (1, 2):
        s[7 * f:7 * f + 7] = s[0:7]
        s[7 * f + 1] += baseline
    rows = np.flatnonzero((p.vis_frame_i != 0) | np.isin(p.vis_frame_j, (1, 2)))
    return window(p, rows), s


def largest_config():
    """stereo + IMU + wheel + plane with both camera extrinsics estimated in full, the wheel extrinsic and td estimated"""
    return dataclasses.replace(synth.make_config(4), ex_subset_mask=0, estimate_ex_wheel=True, estimate_td=True)


def largest_window(oracle):
    """(problem, initial state, oracle-solved state) of the second window of a largest_config sequence, with the first window's prior"""
    seq = synth.Sequence(largest_config(), 5, 13)
    p, s, _ = seq.window(0)
    a, _, q = oracle.optimization(p, s, abi.MARGIN_OLD)
    p, s, _ = seq.window(1, prior=q, prev_state=a)
    a, _, _ = oracle.optimization(p, s, abi.MARGIN_OLD, want_prior=False)
    return p, s, a


def path_cases(oracle):
    """{name: (problem, state, flag)} of cases 1, 3 and 6, run again on the unfused and the one-kernel eigen paths"""
    out = {}
    for cid in (2, 4, 6):
        out["second_new_c%d" % cid] = second_new_window(oracle, cid) + (abi.MARGIN_SECOND_NEW,)
        out["old_prior_c%d" % cid] = old_with_prior_window(oracle, cid) + (abi.MARGIN_OLD,)
    p, a, flag = out["second_new_c2"]
    out["second_new_c2_frame10"] = (with_frame10(p, a, 2), a, flag)
    p, _, a = largest_window(oracle)
    out["largest"] = (p, a, abi.MARGIN_OLD)
    return out


@pytest.fixture(scope="module")
def cases(oracle):
    return path_cases(oracle)


# ------------------------------------------------------------------------------------------------ hp_marginalize itself
@pytest.mark.parametrize("cid", [1, 2, 3, 4, 6, "stationary"])
def test_hp_marginalize_matches_oracle(oracle, cid):
    """Two FP64 restatements of the same marginalisation, at SELF.  C3 (mono, extrinsic and td estimated) is the exception: its dropped block has
    a condition number of ~5e10 and its kept block eigenvalues from 1e-19 to 4e7, which limits any two FP64 eigen-solvers' agreement (measured
    7.1e-8 on J^T J and 1.5e-7 on J^T r); it is held to TIGHT."""
    if cid == "stationary":
        p, s = stationary_window(0.0)
    else:
        p, s, _ = synth.make_window(cid)
        s = oracle.window_solve(p, s)[0]
    q, (A0, b0), _ = oracle_prior(oracle, p, s, abi.MARGIN_OLD)
    A1, b1 = q.information()
    tol = TIGHT if cid == 3 else SELF
    assert rel(A0, A1) <= tol and rel(b0, b1) <= tol, (cid, rel(A0, A1), rel(b0, b1))


# ------------------------------------------------------------------------------------------------ 1. MARGIN_SECOND_NEW with pose 9 in the prior
@pytest.mark.parametrize("cid,frame10", [(2, False), (4, False), (6, False), (2, True), (6, True)])
def test_second_new_with_pose9(ctx, oracle, cases, cid, frame10):
    """The prior of a MARGIN_OLD window as it comes (pose 9 dropped, nothing renamed), and extended by blocks 10 and 21 (renamed to 9 and 20;
    not on C4, whose kept dimension would then be 106, beyond marg_cap)"""
    p, a, flag = cases["second_new_c%d" % cid]
    if frame10:
        p = with_frame10(p, a, cid)
    ids_in = [b for b, _ in p.prior.blocks()]
    assert 9 in ids_in and (10 in ids_in) == frame10 and (21 in ids_in) == (frame10 and cid != 6)
    got = ctx.marginalize(p, a, flag)
    q, hp, _ = oracle_prior(oracle, p, a, flag)
    check_prior(cid, got, q, hp)
    assert got.blocks() == expected_blocks([(shift_second_new(b), b) for b in ids_in if b != 9])
    # the linearisation point of the renamed blocks is the state of the frame they came from
    for b in ids_in:
        if b != 9:
            o, o2, k = abi.block_offset(b), abi.block_offset(shift_second_new(b)), abi.block_size(b)
            assert np.array_equal(got.x0[o2:o2 + k], a[o:o + k]), b
    # the produced prior, evaluated at a perturbed state: cost, gradient and Gauss-Newton matrix over the whole fixed state
    rng = np.random.default_rng(40 + cid)
    x = a.copy()
    for b, _ in got.blocks():
        o, k = abi.block_offset(b), abi.block_size(b)
        x[o:o + k] = got.x0[o:o + k]
    x[:abi.STATE_FIXED] += rng.normal(0, 0.01, abi.STATE_FIXED)
    for o in [7 * f + 3 for f in range(abi.NUM_FRAMES)] + [abi.block_offset(b) + 3 for b in (abi.BLK_EX_POSE0, abi.BLK_EX_POSE1, abi.BLK_EX_WHEEL)] + [abi.block_offset(abi.BLK_PLANE_R)]:
        x[o:o + 4] /= np.linalg.norm(x[o:o + 4])
    r1, J1 = ctx.prior_evaluate(got, x)
    r0, J0 = oracle.prior_evaluate(q, x)
    assert abs(r1 @ r1 - r0 @ r0) <= TIGHT * (r0 @ r0)
    assert rel(J1.T @ r1, J0.T @ r0) <= TIGHT and rel(J1.T @ J1, J0.T @ J0) <= TIGHT
    reference_check(cid, p, a, flag, got, shift_second_new)


# ------------------------------------------------------------------------------------------------ 2. pass-through
def without_pose9(q):
    """`q` with pose 9's columns taken out: J restricted to the other blocks, re-triangularised (J' = Q R, r' = Q^T r)"""
    kept = [(b, i) for b, i in q.blocks() if b != 9]
    cols = np.concatenate([np.arange(i, i + abi.block_marg_size(b)) for b, i in kept])
    Q, R = np.linalg.qr(q.Jmat()[:, cols])
    ids = [b for b, _ in kept]
    blocks = expected_blocks([(b, b) for b in ids])
    return abi.PriorData.from_arrays(1, len(cols), ids, [i for _, i in blocks], q.x0, R, Q.T @ q.rvec())


def test_second_new_pass_through(ctx, oracle, cases):
    p, a, flag = cases["second_new_c2"]
    prior = without_pose9(p.prior)
    assert prior.valid and 9 not in [b for b, _ in prior.blocks()]
    passing = window(p, prior=prior)
    none = window(p, prior=None)
    # alone
    got = ctx.marginalize(passing, a, abi.MARGIN_SECOND_NEW)
    assert same_prior(got, prior)
    assert same_prior(oracle.marginalize(passing, a, abi.MARGIN_SECOND_NEW), prior)
    assert not ctx.marginalize(none, a, abi.MARGIN_SECOND_NEW).valid
    # inside one batch with ordinary MARGIN_OLD windows
    old = [synth.make_window(2, 20)[:2], synth.make_window(4, 21)[:2]]
    probs, states = [passing, old[0][0], none, old[1][0]], [a, old[0][1], a, old[1][1]]
    flags = [abi.MARGIN_SECOND_NEW, abi.MARGIN_OLD, abi.MARGIN_SECOND_NEW, abi.MARGIN_OLD]
    out_s, _, out_pr = ctx.optimization_batch(probs, states, flags)
    assert same_prior(out_pr[0], prior)
    assert not out_pr[2].valid and out_pr[2].n == 0
    for k in (1, 3):
        s1, _, q1 = ctx.optimization(probs[k], states[k], flags[k])
        assert q1.valid and np.array_equal(s1, out_s[k]) and same_prior(q1, out_pr[k]), k


# ------------------------------------------------------------------------------------------------ 3. MARGIN_OLD with an incoming prior
@pytest.mark.parametrize("cid", [2, 4, 6])
def test_old_with_prior(ctx, oracle, cases, cid):
    p, a, flag = cases["old_prior_c%d" % cid]
    assert p.prior is not None and p.prior.valid
    got = ctx.marginalize(p, a, flag)
    q, hp, _ = oracle_prior(oracle, p, a, flag)
    check_prior(cid, got, q, hp)
    reference_check(cid, p, a, flag, got, lambda b: b - 1 if (1 <= b <= 10 or 12 <= b <= 21) else b)


# ------------------------------------------------------------------------------------------------ 4. landmarks without parallax
@pytest.mark.parametrize("baseline", [0.0, 0.05])
def test_stationary_landmarks(ctx, oracle, baseline):
    """Frames 1 and 2 at frame 0's camera centre: every frame-0-hosted landmark's pivot is rounding noise (<= 5e-24), far under the reference's
    1e-8 eigenvalue cut, and must be discarded as the cut discards it.  With a 5 cm baseline the same landmarks are well above the cut."""
    p, s = stationary_window(baseline)
    got = ctx.marginalize(p, s, abi.MARGIN_OLD)
    q, hp, Amm = oracle_prior(oracle, p, s, abi.MARGIN_OLD)
    w = np.linalg.eigvalsh(0.5 * (Amm + Amm.T))
    nlm0 = len(set(p.vis_landmark[p.vis_frame_i == 0].tolist()))
    assert nlm0 >= 50
    if baseline == 0.0:
        assert np.sum(w < 1e-12) >= nlm0, np.sort(w)[:nlm0 + 1]
    else:
        assert w.min() > 1e3 * EPS, w.min()
    check_prior(baseline, got, q, hp)


# ------------------------------------------------------------------------------------------------ 5. an exactly zero kept row
def test_zero_td_row(ctx, oracle):
    """td estimated while every observation's velocity is zero: td's Jacobian, its row and column of the kept block and its eigenvalue are
    exactly zero (marg_ql's deflation path, no rotation).  Householder reflections may mix rounding into it, so 1e-12 of the max-abs, not 0."""
    p, s, _ = synth.make_window(2, 22)
    flags = p.block_flags.copy()
    flags[abi.BLK_TD] = abi.BLOCK_PRESENT
    obs = p.vis_obs.copy()
    obs[:, 6:10] = 0.0
    p = window(p, vis_obs=obs, block_flags=flags)
    a = oracle.window_solve(p, s)[0]
    got = ctx.marginalize(p, a, abi.MARGIN_OLD)
    q, hp, _ = oracle_prior(oracle, p, a, abi.MARGIN_OLD)
    for name, prior in (("library", got), ("oracle", q)):
        td = dict(prior.blocks())[abi.BLK_TD]
        A, b = prior.information()
        assert np.abs(A[td]).max() <= 1e-12 * np.abs(A).max() and np.abs(A[:, td]).max() <= 1e-12 * np.abs(A).max(), name
        assert abs(b[td]) <= 1e-12 * np.abs(b).max(), name
    check_prior("zero td", got, q, hp)


# ------------------------------------------------------------------------------------------------ 6. the largest kept dimension
def test_largest_kept_dimension(ctx, oracle, cases):
    p, a, flag = cases["largest"]
    got = ctx.marginalize(p, a, flag)
    q, hp, _ = oracle_prior(oracle, p, a, flag)
    print("largest kept dimension: n = %d (marg_cap: 100)" % got.n)
    assert got.n >= 90
    check_prior("largest", got, q, hp)
    # next to a C6 window, whose kept block is much smaller: marg_J's per-window slot is nmax^2 with the n x n block at its head
    big = largest_window(oracle)[:2]
    c6p, c6s, _ = synth.make_window(6, 23)
    out_s, out_sum, out_pr = ctx.optimization_batch([big[0], c6p], [big[1], c6s], [abi.MARGIN_OLD] * 2)
    assert out_pr[1].valid and out_pr[1].n < got.n, (out_pr[1].n, got.n)
    for k, (pp, ss) in enumerate((big, (c6p, c6s))):
        s1, sm1, q1 = ctx.optimization(pp, ss, abi.MARGIN_OLD)
        assert np.array_equal(s1, out_s[k]) and same_prior(q1, out_pr[k]), k
        assert sm1.num_iterations == out_sum[k].num_iterations, k


# ------------------------------------------------------------------------------------------------ 7. the unfused and the one-kernel paths
def test_unfused_marginalization(ctx, oracle, cases, monkeypatch):
    """VIWB_NO_FUSED=1 (read by every batch build): the unfused marginalisation matches the oracle at the tight bound"""
    monkeypatch.setenv("VIWB_NO_FUSED", "1")
    for name, (p, a, flag) in cases.items():
        got = ctx.marginalize(p, a, flag)
        q, hp, _ = oracle_prior(oracle, p, a, flag)
        check_prior(name, got, q, hp)


def test_one_kernel_eigen_path(request, ctx, oracle, cases, tmp_path):
    """VIWB_MARG_ONE_KERNEL=1, read when the library loads, in a process of its own (tests/marg_one_kernel_worker.py): marg_eig runs
    tridiag_block + tql2_block, the statements of marg_tri / marg_ql / marg_apply in the same order.  The emulation build's priors must be
    bit-identical to the pipeline's.  The device build's differ at rounding level between the two kernels' code (not traced to an instruction
    yet), so there the one-kernel prior is held to the oracle at TIGHT with the pipeline's n, blocks and x0."""
    from emu import build_emu
    emu = request.node.callspec.params["ctx"] == "emu"
    out = str(tmp_path / "one_kernel.npz")
    env = dict(os.environ, VIWB_MARG_ONE_KERNEL="1")
    env.pop("VIWB_NO_FUSED", None)
    subprocess.run([sys.executable, os.path.join(ROOT, "tests", "marg_one_kernel_worker.py"), build_emu.build() if emu else "", out], check=True, env=env,
                   timeout=1200, cwd=ROOT)
    with np.load(out) as z:
        for name, (p, a, flag) in cases.items():
            got = ctx.marginalize(p, a, flag)
            one = abi.PriorData.from_arrays(*(z[name + "." + k] for k in ("valid", "n", "block_id", "block_idx", "x0", "J", "r")))
            if emu:
                assert same_prior(one, got), name
            else:
                q, hp, _ = oracle_prior(oracle, p, a, flag)
                check_prior(name, one, q, hp)
