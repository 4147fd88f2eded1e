"""The solve kernel's launch: three C2 windows per SM, and results that do not depend on the block size.

`not gpu`: the shared memory the lowering asks for a C2 benchmark window fits three blocks in an H100 SM (228 KB, 1 KB reserved per block), and
the carve (kernels_solve.cuh `carve`, compiled with g++ straight from the header) keeps apart every two regions that are live at the same time.
`gpu`: the device holds three such blocks per SM, C4 windows (two per SM at either size) launch 384 threads, and the same C2 batch solved by a -DSOLVE_NT=384 build of the library (two windows per SM)
comes out bit-identical: the kernel's sums are stated over one virtual thread layout whatever the block size."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "viw-fusion_b200", "python"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from viwb import abi, synth  # noqa: E402
from viwb import lib as viwb_lib  # noqa: E402

CSRC = os.path.join(ROOT, "viw-fusion_b200", "csrc")
SM_BYTES, BLOCK_RESERVED = 228 * 1024, 1024          # H100: shared memory per SM, and what the runtime reserves per block


def c2_windows(distinct=2, copies=2, config=2):
    """Steady-state windows as the benchmark builds them: window 1 of each sequence with the prior the oracle marginalised from window 0."""
    import viw_oracle as vo
    cfg = synth.make_config(config)
    probs, states = [], []
    rng = np.random.default_rng(5)
    for i in range(distinct):
        seq = synth.Sequence(cfg, i, 12)
        p0, st0, _ = seq.window(0)
        a0, _, q0 = vo.optimization(p0, st0, abi.MARGIN_OLD)
        p, st, _ = seq.window(1, prior=q0, prev_state=a0)
        for c in range(copies):
            x = st.copy()
            if c:
                x[abi.STATE_FIXED:] *= 1.0 + rng.normal(0, 0.02, len(x) - abi.STATE_FIXED)
            probs.append(p)
            states.append(x)
    return probs, states


def test_c2_window_fits_three_per_sm():
    from emu import build_emu
    ctx = viwb_lib.Context(0, build_emu.build())
    probs, states = c2_windows()
    b = ctx.batch(probs, states)
    nt, smem, _ = b.solve_launch(occupancy=False)
    b.destroy()
    ctx.close()
    assert nt == 256
    assert 3 * (smem + BLOCK_RESERVED) <= SM_BYTES, smem


CARVE_DRIVER = r"""
#include "kernels_solve.cuh"
#include <cstdio>
int main() {
    int nt, esize, nf_max;
    while (scanf("%d %d %d", &nt, &esize, &nf_max) == 3) {
        std::vector<double> sm(viwb::solve_smem_doubles(nt, esize, nf_max));
        viwb::SolveSmem s; viwb::carve(s, sm.data(), nt, esize, nf_max);
        auto o = [&](const void *p) { return (long)((const char *)p - (const char *)sm.data()); };
        printf("%zu %ld %ld %ld %ld %ld %ld %ld %ld %ld %ld %ld %ld %ld %ld %d\n", sm.size() * 8, o(s.L), o(s.g), o(s.ug), o(s.u), o(s.Hu), o(s.xo),
               o(s.Pt), o(s.uvis), o(s.chol), o(s.y), o(s.red), o(s.vmap), o(s.fst), o(s.rp), s.ldp);
    }
    return 0;
}
"""


def test_carve_keeps_live_regions_apart(tmp_path):
    src, exe = tmp_path / "carve.cpp", tmp_path / "carve"
    src.write_text(CARVE_DRIVER)
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-DVIWB_HOST_EMU", "-x", "c++", "-Wno-unknown-pragmas", "-I", CSRC, "-o", str(exe), str(src)])
    cases = [(nt, nf * (nf + 1) // 2, nf) for nt in (1, 256, 384) for nf in (1, 7, 8, 9, 40, 165, 192)] + [(256, 7620, 165), (256, 7621, 165)]
    out = subprocess.run([str(exe)], input="".join("%d %d %d\n" % c for c in cases), capture_output=True, text=True, check=True).stdout.split("\n")
    for (nt, esize, nf), line in zip(cases, out):
        v = [int(t) for t in line.split()]
        total, off = v[0], dict(zip(["L", "g", "ug", "u", "Hu", "xo", "Pt", "uvis", "chol", "y", "red", "vmap", "fst", "rp"], v[1:15]))
        ldp = v[15]
        P = max(4, (nf + 3) // 4 * 4)
        rows = (nf + 1 - 8 + 3) // 4 * 4 if nf > 8 else 4          # the first panel's trailing rows, rhs included, in whole 4-row tiles
        fac = min((nt + 31) // 32, (rows + 31) // 32)                # warps that hold panel rows
        assert ldp >= rows and ldp % 4 == 0 and off["Pt"] % 16 == 0
        size = {"L": 8 * esize, "g": 8 * nf, "ug": 8 * nf, "u": 8 * nf, "Hu": 8 * nf, "xo": 8 * nf, "Pt": 8 * 8 * ldp, "uvis": 8 * 160,
                "chol": 8 * 48 * fac, "y": 8 * nf, "red": 8 * 5 * 16, "vmap": 2 * nf, "fst": 2 * nf, "rp": 2 * (nf + 1)}
        size["imap"], off["imap"] = 4 * 200, off["Hu"]             # assemble_into's int scratch (MAXPRI) sits in Hu until the Cauchy point
        for k in size:
            assert 0 <= off[k] and off[k] + size[k] <= total, (k, nt, nf)

        def apart(a, b):
            assert off[a] + size[a] <= off[b] or off[b] + size[b] <= off[a], (a, b, nt, esize, nf)
        always = ["L", "y", "red", "vmap", "fst", "rp"]
        live_together = [["g", "imap"],                  # assembly
                         ["ug", "Hu", "uvis"],           # Cauchy point
                         ["Pt", "chol"],                 # Cholesky
                         ["xo"],                         # back-substitution
                         ["u", "uvis"],                  # landmark back-substitution
                         ["u", "Hu"]]                    # quadratic forms
        for i, a in enumerate(always):
            for b in always[i + 1:] + [r for phase in live_together for r in phase]:
                apart(a, b)
        for phase in live_together:
            for i, a in enumerate(phase):
                for b in phase[i + 1:]:
                    apart(a, b)


@pytest.mark.gpu
def test_c2_three_blocks_resident():
    ctx = viwb_lib.Context(0)
    probs, states = c2_windows()
    b = ctx.batch(probs, states)
    nt, smem, bps = b.solve_launch()
    b.destroy()
    ctx.close()
    assert nt == 256 and bps == 3, (nt, smem, bps)


@pytest.mark.gpu
def test_wide_windows_keep_their_warps():
    """C4 windows fit two blocks per SM at either block size: the launch takes the 384-thread kernel, 24 resident warps instead of 16."""
    ctx = viwb_lib.Context(0)
    probs, states = c2_windows(distinct=1, copies=1, config=4)
    b = ctx.batch(probs, states)
    nt, smem, bps = b.solve_launch()
    b.destroy()
    ctx.close()
    assert nt == 384 and bps == 2, (nt, smem, bps)


@pytest.mark.gpu
def test_block_size_does_not_change_results(tmp_path):
    lib384 = tmp_path / "libviwb_nt384.so"
    mk = open(os.path.join(CSRC, "Makefile")).read()
    flags = [ln.split("?=", 1)[1].split() for ln in mk.splitlines() if ln.startswith("NVCCFLAGS")][0]
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc] + flags + ["-DSOLVE_NT=384", "-shared", "-o", str(lib384), os.path.join(CSRC, "viwb.cu")], cwd=CSRC)
    probs, states = c2_windows(distinct=3, copies=2)
    flags_m = [abi.MARGIN_OLD] * len(probs)
    outs = []
    for path in (None, str(lib384)):
        ctx = viwb_lib.Context(0, path) if path else viwb_lib.Context(0)
        b = ctx.batch(probs, states)
        nt = b.solve_launch(occupancy=False)[0]
        b.destroy()
        outs.append((nt, ctx.optimization_batch(probs, states, flags_m)))
        ctx.close()
    (nt_a, (sa, suma, pa)), (nt_b, (sb, sumb, pb)) = outs
    assert (nt_a, nt_b) == (256, 384)
    for x, y in zip(sa, sb):
        assert np.array_equal(x, y)
    for x, y in zip(suma, sumb):
        assert x.num_iterations == y.num_iterations and x.num_linear_solves == y.num_linear_solves and x.final_cost == y.final_cost
    for x, y in zip(pa, pb):
        assert x.n == y.n and np.array_equal(x.Jmat(), y.Jmat()) and np.array_equal(x.rvec(), y.rvec())
