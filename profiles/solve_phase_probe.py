"""Where the time of the solve kernel goes: clock64() cycles per phase of one trust-region iteration, from the measurement build
libviwb_phases.so (make -C viw-fusion_b200/csrc phases), over the bench's C2 batch (33 x 48 = 1584 windows).

Thread 0 of each window's block reads the SM clock at the barrier-delimited phase boundaries; only launches that compute a step are
counted.  The Cholesky is split per panel into thread 0's warp factoring the diagonal block, the panel solve up to its barrier and the
trailing update up to the next one; the back-substitution per block into the block solve and the row update up to its barrier.  Per phase the table gives the mean cycles per such launch over the batch, the p90 over the windows of each window's own
mean per launch, and the mean / p90 over the windows of the cycles summed over a whole solve.  The card's name, power limit and SM
clocks are read in the same call.
Usage (GPU): python profiles/solve_phase_probe.py [path/to/libviwb_phases.so] [--runs 3] [--json OUT]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "viw-fusion_b200", "python"))
import bench  # noqa: E402
from viwb import abi, lib  # noqa: E402

PHASES = ["prologue + phase A", "assembly", "D + scaling", "Cauchy (symv + landmarks 1)", "Schur subtraction", "Cholesky: diagonal block",
          "Cholesky: panel solve", "Cholesky: trailing update", "back-substitution: block solve", "back-substitution: row update",
          "landmark pass 2", "reload + symv + forms", "dogleg + candidate"]


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    return dict(zip(q.split(","), [v.strip() for v in out.strip().splitlines()[0].split(",")]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("lib", nargs="?", default=os.path.join(ROOT, "viw-fusion_b200", "csrc", "libviwb_phases.so"))
    ap.add_argument("--runs", type=int, default=3, help="timed batch runs (whole solves of every window)")
    ap.add_argument("--distinct", type=int, default=33)
    ap.add_argument("--copies", type=int, default=48)
    ap.add_argument("--json", default="", help="also write the table here")
    args = ap.parse_args()
    ctx = lib.Context(0, os.path.abspath(args.lib))
    L = ctx.lib
    if not hasattr(L, "viwb_solve_probe_read"):
        raise SystemExit("%s has no phase probe: build it with make -C viw-fusion_b200/csrc phases" % args.lib)
    slots = L.viwb_solve_probe_slots()
    nph = len(PHASES)
    assert slots == nph + 2, slots
    cfg, seqs, first = bench.make_windows(0, args.distinct, args.copies, 2)
    a0, _, q0 = ctx.optimization_batch([f[0] for f in first], [f[1] for f in first], [abi.MARGIN_OLD] * len(first))
    probs, states = bench.replicate(seqs, q0, a0, args.copies, 0)
    B = len(probs)
    batch = ctx.batch(probs, states, [abi.MARGIN_OLD] * B)
    for _ in range(2):
        batch.run()
    batch.download()
    info = gpu_info()
    ctx._ck(L.viwb_solve_probe_clear(ctx.h), "viwb_solve_probe_clear")
    for _ in range(args.runs):
        batch.run()
    _, sums, _ = batch.download()
    raw = np.zeros(B * slots, np.uint64)
    ctx._ck(L.viwb_solve_probe_read(ctx.h, C.c_int(B), raw.ctypes.data_as(C.POINTER(C.c_ulonglong))), "viwb_solve_probe_read")
    info_after = gpu_info()
    raw = raw.reshape(B, slots).astype(np.float64)
    cyc, steps, fact = raw[:, :nph], raw[:, nph], raw[:, nph + 1]
    per_launch_w = cyc / np.maximum(steps, 1)[:, None]
    per_window = cyc / args.runs
    mean_launch = cyc.sum(0) / steps.sum()
    total = mean_launch.sum()
    rows = []
    print("solve phase probe: %s, B=%d windows, %d runs, %.2f step launches and %.2f factorisations per window and solve" % (
        os.path.basename(args.lib), B, args.runs, steps.sum() / B / args.runs, fact.sum() / B / args.runs))
    print("GPU: %s, power limit %s, SM clock %s (max %s); after: SM clock %s" % (
        info["name"], info["power.limit"], info["clocks.sm"], info["clocks.max.sm"], info_after["clocks.sm"]))
    print("%-30s %12s %12s %7s %14s %14s" % ("phase", "mean/launch", "p90/launch", "share", "mean/window", "p90/window"))
    for p, name in enumerate(PHASES):
        r = {"phase": name, "mean_per_launch": float(mean_launch[p]), "p90_per_launch": float(np.percentile(per_launch_w[:, p], 90)),
             "share": float(mean_launch[p] / total), "mean_per_window": float(per_window[:, p].mean()),
             "p90_per_window": float(np.percentile(per_window[:, p], 90))}
        rows.append(r)
        print("%-30s %12.0f %12.0f %6.1f%% %14.0f %14.0f" % (name, r["mean_per_launch"], r["p90_per_launch"], 100 * r["share"],
                                                        r["mean_per_window"], r["p90_per_window"]))
    tw = per_window.sum(1)
    print("%-30s %12.0f %12.0f %7s %14.0f %14.0f" % ("total", total, np.percentile(per_launch_w.sum(1), 90), "", tw.mean(), np.percentile(tw, 90)))
    print("iterations of window 0: %d" % sums[0].num_iterations)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"lib": os.path.basename(args.lib), "gpu": info, "gpu_after": info_after, "B": B, "runs": args.runs,
                       "steps_per_window": float(steps.sum() / B / args.runs), "phases": rows, "total_per_launch": float(total)}, f, indent=1)
    batch.destroy()
    ctx.close()


if __name__ == "__main__":
    main()
