"""What solving the resident FeatureManager's windows where they are costs, against the host round trip it replaces: at 1584 stereo streams x
~150 rows (the rows of one synth sequence, config 2, 752x480), twin lists take the same adds, triangulations, slides and removeFailures, and at
every NON_LINEAR tick
  (a) the host chain: window -> Batch(...) (viwb_batch_create) -> run -> download -> outliers -> set_depth -> remove_outliers -> predict
  (b) the device chain: Features.batch (viwb_features_batch_create) -> run -> set_depth_from -> remove_outliers_from -> predict_from
run one after the other, the order alternating from tick to tick.  Each call is timed by the host clock around the call and a synchronise of the
context's stream; the per-tick total is the sum of a chain's calls.  Also viwb_h2d_bytes per tick of each chain, and a check that both chains
leave the same removed ids and predictions.  The windows carry the IMU tables of the sequence's synth window, ex0 / ex1 / td constant, the
decisions' margin flags.  Prints one JSON line with the card's name and power limit read in the same run.  There is no CPU path: without a CUDA
device the script fails.
Usage (GPU box): python profiles/features_batch_probe.py   (FM_STREAMS env)"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in ("", "viw-fusion_b200/python", "oracle", "tests"):
    sys.path.insert(0, os.path.join(ROOT, p))
from viwb import abi, lib  # noqa: E402
import features_checks as fc  # noqa: E402

F = int(os.environ.get("FM_STREAMS", "1584"))
TICKS, MEASURED = 17, 6                     # ticks 0..10 fill the window (INITIAL), the last MEASURED are NON_LINEAR ticks
VIS_CAP = 2500

if not torch.cuda.is_available():
    raise SystemExit("features_batch_probe: no CUDA device")
card = torch.cuda.get_device_name(0)
power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()

sc = fc.Script(2, 0, TICKS + 1)
ctx = lib.Context(0)
stream = torch.cuda.Stream()
ctx.set_stream(stream.cuda_stream)
fa, fb = (ctx.features(F, 160, True, 10.0 / fc.FOCAL, fc.FOCAL) for _ in range(2))


def timed(fn, rec, name):
    t0 = time.perf_counter()
    out = fn()
    stream.synchronize()
    rec[name] = (time.perf_counter() - t0) * 1e3
    return out


def bare_problems(t):
    p = sc.s.window(max(0, min(t - 10, sc.frames - 11)), perturb=False)[0]
    flags = p.block_flags.copy()
    for b in (abi.BLK_EX_POSE0, abi.BLK_EX_POSE1, abi.BLK_TD):
        flags[b] |= abi.BLOCK_PRESENT | abi.BLOCK_CONSTANT
    return p, dict(block_flags=flags, subset_mask=p.subset_mask, imu_frame_i=p.imu_frame_i, imu_frame_j=p.imu_frame_j, imu_data=p.imu_data, globals_=p.globals)


def host_chain(states, margin, common, fc_, rec):
    tabs, inv, _ = timed(lambda: fa.window(VIS_CAP), rec, "window")
    probs = [abi.WindowProblem(fc_, tb["num_landmarks"], vis_type=tb["vis_type"], vis_landmark=tb["vis_landmark"], vis_frame_i=tb["vis_frame_i"],
                               vis_frame_j=tb["vis_frame_j"], vis_obs=tb["vis_obs"], **common) for tb in tabs]
    b = timed(lambda: ctx.batch(probs, [np.concatenate([states[s], inv[s]]) for s in range(F)], margin), rec, "batch_create")
    timed(b.run, rec, "run")
    solved, _, _ = timed(lambda: b.download(want_priors=False), rec, "download")
    verdicts = timed(b.outliers, rec, "outliers")
    timed(lambda: fa.set_depth([x[abi.STATE_FIXED:] for x in solved]), rec, "set_depth")
    removed = timed(lambda: fa.remove_outliers(verdicts), rec, "remove_outliers")
    pred = timed(lambda: fa.predict(np.array([x[:abi.STATE_FIXED] for x in solved]), [fc_] * F), rec, "predict")
    b.destroy()
    return removed, pred, np.array([x[:abi.STATE_FIXED] for x in solved])


def device_chain(states, margin, common, fc_, rec):
    probs = [abi.WindowProblem(fc_, 0, **common) for _ in range(F)]
    b = timed(lambda: fb.batch(probs, states, margin), rec, "batch_create")
    timed(b.run, rec, "run")
    timed(lambda: fb.set_depth_from(b), rec, "set_depth")
    removed = timed(lambda: fb.remove_outliers_from(b), rec, "remove_outliers")
    pred = timed(lambda: fb.predict_from(b, [fc_] * F), rec, "predict")
    solved, _, _ = b.download(want_priors=False)           # (untimed: the next tick's states for the slide)
    b.destroy()
    return removed, pred, np.array([x[:abi.STATE_FIXED] for x in solved])


res = {"host": {}, "device": {}}
h2d = {"host": [], "device": []}
for t in range(TICKS):
    fc_ = min(t, 10)
    rows_t = [fc.rows_of(sc.image(t), True)] * F
    states = np.array([sc.state(t)] * F)
    nonlin = t > 10
    for fs in (fa, fb):
        fs.add([fc_] * F, [0.0] * F, rows_t)
    dec = fa.decisions()
    assert np.array_equal(dec["margin_flag"], fb.decisions()["margin_flag"])
    if nonlin:
        for fs in (fa, fb):
            fs.triangulate(states)
        _, common = bare_problems(t)
        margin = [int(x) for x in dec["margin_flag"]]
        out = {}
        for which in (("host", "device") if t % 2 else ("device", "host")):
            rec = {}
            h0 = ctx.h2d_bytes()
            out[which] = (host_chain if which == "host" else device_chain)(states, margin, common, fc_, rec)
            h2d[which].append(ctx.h2d_bytes() - h0)
            if t >= TICKS - MEASURED:
                for k, v in rec.items():
                    res[which].setdefault(k, []).append(v)
                res[which].setdefault("tick_total", []).append(sum(rec.values()))
        (ra, pa, sa), (rb, pb, sb) = out["host"], out["device"]
        assert all(np.array_equal(x, y) for x, y in zip(ra, rb)) and sa.tobytes() == sb.tobytes()
        assert all(x[0].tobytes() == y[0].tobytes() and x[1].tobytes() == y[1].tobytes() for x, y in zip(pa, pb))
        states = sa
    mats = [np.array([m] * F) for m in fc.cam_mats(states[0])]
    for fs in (fa, fb):
        fs.slide([fc_] * F, [1 if nonlin else 0] * F, *mats)
        if nonlin:
            fs.remove_failures()
fa.close(); fb.close()
summ = {w: {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v)), "n": len(v)} for k, v in r.items()} for w, r in res.items()}
print(json.dumps({"what": "NON_LINEAR tick: host chain vs viwb_features_batch_create chain, stereo, max_rows 160, host clock + stream synchronise",
                  "card": card, "power_limit": power, "streams": F, "ms": summ,
                  "h2d_bytes_per_tick": {w: {"median": float(np.median(v[-MEASURED:])), "min": int(np.min(v[-MEASURED:])), "max": int(np.max(v[-MEASURED:]))} for w, v in h2d.items()}}))
