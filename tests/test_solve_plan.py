"""`not gpu`: the solve kernel's factorisation plan (kernels_solve.cuh chol_plan_build), built once per envelope by the host lowering.

The plan is checked against the envelope it was built from: the row pointers are the skyline's, every entry that receives a panel's
trailing update is listed in exactly one tile of that panel and nothing else is, and no listed tile is empty.  The builder is compiled
with g++ straight from the kernel header.  Then a batch mixing C1-C4 and C6 windows (several envelopes, some shared) is solved in the
emulation, and every window must come out bit-identical to itself solved alone."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "viw-fusion_b200", "python"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from viwb import abi, synth  # noqa: E402
from viwb import lib as viwb_lib  # noqa: E402

CSRC = os.path.join(ROOT, "viw-fusion_b200", "csrc")
NB = 8          # CHOL_NB

DRIVER = r"""
#include "kernels_solve.cuh"
#include <cstdio>
int main() {
    int n;
    while (scanf("%d", &n) == 1) {
        std::vector<short> e(n > 0 ? n : 1);
        for (int i = 0; i < n; i++) { int v; scanf("%d", &v); e[i] = (short)v; }
        std::vector<int> plan;
        viwb::chol_plan_build(e.data(), n, plan);
        printf("%zu", plan.size());
        for (int v : plan) printf(" %d", v);
        printf("\n");
    }
    return 0;
}
"""


@pytest.fixture(scope="module")
def plan_tool(tmp_path_factory):
    d = tmp_path_factory.mktemp("plan")
    src, exe = d / "plan.cpp", d / "plan"
    src.write_text(DRIVER)
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-DVIWB_HOST_EMU", "-x", "c++", "-Wno-unknown-pragmas", "-I", CSRC, "-o", str(exe), str(src)])

    def run(envs):
        text = "".join("%d %s\n" % (len(e), " ".join(str(int(v)) for v in e)) for e in envs)
        out = subprocess.run([str(exe)], input=text, capture_output=True, text=True, check=True).stdout.split("\n")
        plans = []
        for line in out[: len(envs)]:
            v = np.array([int(t) for t in line.split()], np.int64)
            assert v[0] == len(v) - 1
            plans.append(v[1:])
        return plans
    return run


def envelopes():
    rng = np.random.default_rng(7)
    out = [np.zeros(1, int), np.zeros(8, int), np.arange(9), np.zeros(17, int), np.arange(40), np.zeros(165, int)]
    for n in (5, 23, 64, 165, 192):
        out.append(np.array([rng.integers(0, i + 1) for i in range(n)]))                        # any first column <= i
        out.append(np.array([max(0, i - int(rng.integers(0, 12))) for i in range(n)]))          # a narrow band
    # the solver's shape: speed-bias blocks of 9 newest first, each coupling with its neighbour in the chain; then a dense visual block
    e, col = [], 0
    for f in range(11):
        e += [max(0, col - 9)] * 9
        col += 9
    e += [0] * 6 * 11 + [99 - 9 * 3] * 13
    out.append(np.minimum(np.array(e), np.arange(len(e))))
    return out


def check_plan(e, plan):
    n = len(e)
    npan = (n + NB - 1) // NB
    head = n + 1 + npan + 1
    rp = np.concatenate([[0], np.cumsum(np.arange(n) - e + 1)])
    assert np.array_equal(plan[: n + 1], rp)
    toff = plan[n + 1: head]
    tiles = plan[head:].astype(np.uint32)
    assert toff[0] == 0 and np.all(np.diff(toff) >= 0) and toff[-1] == len(tiles)
    for p in range(npan):
        r0 = min(n, (p + 1) * NB)
        reach = lambda i: i == n or e[i] < r0       # noqa: E731
        want = {(i, k) for i in range(r0, n + 1) if reach(i) for k in range(r0, min(i, n - 1) + 1) if reach(k)}
        got, seen_tiles = [], set()
        for wd in tiles[toff[p]: toff[p + 1]]:
            ti, tk, on = int(wd & 0xFF), int((wd >> 8) & 0xFF), int(wd >> 16)
            assert on != 0, "empty tile listed"
            assert tk <= ti and (ti, tk) not in seen_tiles
            seen_tiles.add((ti, tk))
            for a in range(4):
                for b in range(4):
                    if (on >> (4 * a + b)) & 1:
                        got.append((r0 + 4 * ti + a, r0 + 4 * tk + b))
        assert len(got) == len(set(got)), "an entry listed twice"
        assert set(got) == want, "panel %d: %d entries missing, %d extra" % (p, len(want - set(got)), len(set(got) - want))


def test_plan_covers_the_envelope(plan_tool):
    envs = envelopes()
    for e, plan in zip(envs, plan_tool(envs)):
        check_plan(e, plan)


def test_mixed_batch_matches_single_windows():
    from emu import build_emu
    ctx = viwb_lib.Context(0, build_emu.build())
    probs, sts = [], []
    for cid, seq in ((1, 0), (2, 1), (3, 2), (4, 3), (6, 4), (2, 5)):
        p, s, _ = synth.make_window(cid, seq)
        probs.append(p)
        sts.append(s)
    flags = [abi.MARGIN_OLD] * len(probs)
    out_s, out_sum, out_pr = ctx.optimization_batch(probs, sts, flags)
    for p, s, f, bs, bsum, bpr in zip(probs, sts, flags, out_s, out_sum, out_pr):
        a, sm, q = ctx.optimization(p, s, f)
        assert np.array_equal(a, bs)
        assert sm.num_iterations == bsum.num_iterations and sm.final_cost == bsum.final_cost
        assert q.n == bpr.n and np.array_equal(q.Jmat(), bpr.Jmat()) and np.array_equal(q.rvec(), bpr.rvec())
    ctx.close()
