"""Host runs of the compact solver windows (kernels_fused.cuh, lin_vis_lm): every (host, observer) pair's chunk products are formed from the
shared-memory tiles of the run of landmarks hosted in that frame.  Each case reshapes a synthetic C2 window (constant extrinsics and td: compact
records) so that one corner of the chunking / tiling is hit, checks with the host-run plan restated below that it is, and compares the normal
equations and a full solve with the CPU oracle.  The `emu` twin runs the device source compiled for the host (tests/emu), the `gpu` twin libviwb.so."""
import numpy as np
import pytest

import parity_checks as pc
from viwb import abi, synth

LMB_FACTORS, PAIR_CHUNK = 128, 64


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


def subset(prob, keep, order=None):
    """The window with only the visual factors `keep` (boolean mask), optionally in the given order."""
    idx = np.nonzero(keep)[0] if order is None else order
    return abi.WindowProblem(prob.frame_count, prob.num_landmarks, prob.block_flags, prob.subset_mask, prob.vis_type[idx], prob.vis_landmark[idx],
                             prob.vis_frame_i[idx], prob.vis_frame_j[idx], prob.vis_obs[idx], prob.imu_frame_i, prob.imu_frame_j, prob.imu_data,
                             prob.wheel_frame_i, prob.wheel_frame_j, prob.wheel_data, prob.plane_frame, globals_=prob.globals)


def host_runs(prob):
    """{host: [tiles]}, a tile being the list of factor indices it holds (the plan of host_runs in viwb.cu)."""
    cnt = np.bincount(prob.vis_landmark, minlength=prob.num_landmarks)
    first = np.full(prob.num_landmarks, -1)
    for i in range(len(prob.vis_landmark) - 1, -1, -1):
        first[prob.vis_landmark[i]] = i
    h0 = int(prob.vis_frame_i.min())
    runs = {}
    for h in range(11):
        tiles, n = [], 0
        for k in range(prob.num_landmarks):
            if (prob.vis_frame_i[first[k]] if cnt[k] else h0) != h:
                continue
            if not tiles or n + cnt[k] > LMB_FACTORS:
                tiles.append([])
                n = 0
            tiles[-1] += list(range(first[k], first[k] + cnt[k]))
            n += cnt[k]
        if tiles:
            runs[h] = tiles
    return runs


def pair_records(prob, h, j):
    return int(((prob.vis_frame_i == h) & (prob.vis_frame_j == j) & (prob.vis_type != abi.F_PROJ_1F2C)).sum())


def split_kstep(prob):
    """Some pair has an odd number of records before a tile boundary of its run: the k-step's second record is in the next tile."""
    for h, tiles in host_runs(prob).items():
        seen = np.zeros(11, int)
        for t in tiles[:-1]:
            for f in t:
                if prob.vis_type[f] != abi.F_PROJ_1F2C:
                    seen[prob.vis_frame_j[f]] += 1
            if (seen % 2 == 1).any():
                return True
    return False


def compare(ctx, oracle, prob, st):
    H0, g0, lm0, c0 = oracle.normal_equations(prob, st)
    H1, g1, lm1, c1 = ctx.normal_equations(prob, st)
    assert abs(c0 - c1) <= 1e-12 * c0
    assert np.abs(H0 - H1).max() <= 1e-12 * np.abs(H0).max()
    assert np.abs(g0 - g1).max() <= 1e-11 * np.abs(g0).max()
    assert np.abs(lm0 - lm1).max() <= 1e-11 * np.abs(lm0).max()
    s0, sm0 = oracle.window_solve(prob, st)
    s1, sm1 = ctx.window_solve(prob, st)
    assert sm0.num_iterations == sm1.num_iterations and sm0.num_successful_steps == sm1.num_successful_steps
    assert abs(sm0.final_cost - sm1.final_cost) <= 1e-7 * sm0.final_cost
    ep, er = synth.pose_errors(oracle.gauge_reanchor(prob, st, s0), ctx.gauge_reanchor(prob, st, s1))
    assert ep <= pc.TIGHT_M and er <= pc.TIGHT_RAD, (ep, er)


def c2():
    prob, st, _ = synth.make_window(2)
    assert all(prob.block_flags[b] & abi.BLOCK_CONSTANT for b in (abi.BLK_EX_POSE0, abi.BLK_EX_POSE1, abi.BLK_TD))      # compact records
    return prob, st


@pytest.mark.parametrize("n", [1, 64, 65, 129])
def test_pair_sizes(ctx, oracle, n):
    """Pair (0, 1) with exactly n records: one odd chunk, one full chunk, a full chunk + a one-record chunk, two full + one."""
    prob, st = c2()
    two01 = (prob.vis_frame_i == 0) & (prob.vis_frame_j == 1) & (prob.vis_type != abi.F_PROJ_1F2C)
    keep = ~two01
    keep[np.nonzero(two01)[0][:n]] = True
    sub = subset(prob, keep)
    assert pair_records(sub, 0, 1) == n
    compare(ctx, oracle, sub, st)


def test_long_run_and_split_kstep(ctx, oracle):
    """The bench window itself: frame 0's run has more than three tiles, and a k-step's two records fall into two tiles."""
    prob, st = c2()
    assert len(host_runs(prob)[0]) > 3
    assert split_kstep(prob)
    compare(ctx, oracle, prob, st)


def test_interleaved_hosts(ctx, oracle):
    """Landmark ids relabelled so that consecutive landmarks have different host frames: the runs are lists, not ranges."""
    prob, st = c2()
    perm = np.random.default_rng(5).permutation(prob.num_landmarks)        # new id of landmark k
    lm = perm[prob.vis_landmark]
    order = np.argsort(lm, kind="stable")
    sub = subset(prob, None, order)
    sub.vis_landmark = lm[order].astype(np.int32)
    st2 = st.copy()
    st2[abi.STATE_FIXED + perm] = st[abi.STATE_FIXED:]
    hosts = [sub.vis_frame_i[np.argmax(sub.vis_landmark == k)] for k in range(sub.num_landmarks) if (sub.vis_landmark == k).any()]
    assert sum(a != b for a, b in zip(hosts, hosts[1:])) > 50
    assert split_kstep(sub)
    compare(ctx, oracle, sub, st2)


def test_host_with_one_frame_factors_only(ctx, oracle):
    """Frame 3 hosts only one-frame stereo factors (a run without pairs); its landmarks that lose all factors ride in another run."""
    prob, st = c2()
    keep = ~((prob.vis_frame_i == 3) & (prob.vis_type != abi.F_PROJ_1F2C))
    sub = subset(prob, keep)
    assert (sub.vis_frame_i == 3).sum() > 0 and all(pair_records(sub, 3, j) == 0 for j in range(11))
    assert (np.bincount(sub.vis_landmark, minlength=sub.num_landmarks) == 0).any()
    assert 3 in host_runs(sub)
    compare(ctx, oracle, sub, st)


def test_mixed_batch(ctx, oracle):
    """Compact (host runs), wide (X records + asm_pairs_wide) and irregular (unfused: a table not grouped by landmark) windows in one batch."""
    compact, sc, _ = synth.make_window(2, 1)
    wide, sw, _ = synth.make_window(4, 2)
    base, si, _ = synth.make_window(2, 3)
    irregular = subset(base, None, np.random.default_rng(7).permutation(len(base.vis_type)))
    probs, sts = [compact, wide, irregular], [sc, sw, si]
    flags = [abi.MARGIN_OLD] * 3
    out_s, out_sum, _ = ctx.optimization_batch(probs, sts, flags)
    for p, s, f, bs, bsum in zip(probs, sts, flags, out_s, out_sum):
        a, sm, _ = ctx.optimization(p, s, f)
        assert np.array_equal(a, bs) and sm.num_iterations == bsum.num_iterations
        a0, sm0, _ = oracle.optimization(p, s, f)
        assert sm0.num_iterations == bsum.num_iterations
        ep, er = synth.pose_errors(a0, bs)
        assert ep <= pc.TIGHT_M and er <= pc.TIGHT_RAD, (ep, er)
