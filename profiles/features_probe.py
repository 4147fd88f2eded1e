"""What the resident FeatureManager costs on the device: each viwb_features_* call of one NON_LINEAR tick (add, decisions, triangulate, window,
set_depth, remove_outliers, predict, slide, remove_failures) and the whole sequence, at 1584 streams x 150 rows, CUDA events on the context's
stream around each call (uploads and downloads inside the bracket).  Beside it, the host-side equivalent it replaces: the restated
FeatureManager of oracle/features_oracle.py (an untuned Python host, not the reference's C++) run over the same rows for a few streams, per
stream.  Every stream sees the rows of one synth sequence (stereo, config 2).  Prints one JSON line with the card's name and power limit.
There is no CPU path: without a CUDA device the script fails.
Usage (GPU box): python profiles/features_probe.py   (FM_STREAMS, FM_HOST_STREAMS env)"""
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
from viwb import lib  # noqa: E402
import features_checks as fc  # noqa: E402
import features_oracle as fmo  # noqa: E402

F = int(os.environ.get("FM_STREAMS", "1584"))
HOST_F = int(os.environ.get("FM_HOST_STREAMS", "8"))
TICKS, MEASURED = 16, 5                     # ticks 0..10 fill the window (INITIAL), the last MEASURED are NON_LINEAR ticks
VIS_CAP = 2500

if not torch.cuda.is_available():
    raise SystemExit("features_probe: no CUDA device")
card = torch.cuda.get_device_name(0)
power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()

sc = fc.Script(2, 0, TICKS + 1)
ctx = lib.Context(0)
stream = torch.cuda.Stream()
ctx.set_stream(stream.cuda_stream)
fs = ctx.features(F, 160, True, 10.0 / fc.FOCAL, fc.FOCAL)
refs = [fmo.FeatureManagerRef(True, 10.0 / fc.FOCAL, fc.FOCAL) for _ in range(HOST_F)]
rng = np.random.default_rng(0)


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream); out = fn(); e1.record(stream)
    stream.synchronize()
    return e0.elapsed_time(e1), out


res, host_ms, rows = {}, [], []
for t in range(TICKS):
    fc_ = min(t, 10)
    image = sc.image(t)
    rows_t = [fc.rows_of(image, True)] * F
    state = sc.state(t)
    states = np.array([state] * F)
    mats = [np.array([m] * F) for m in fc.cam_mats(state)]
    nonlin = t > 10
    calls = {}
    calls["add"] = timed(lambda: fs.add([fc_] * F, [0.0] * F, rows_t))[0]
    calls["decisions"], dec = timed(fs.decisions)
    if nonlin:
        calls["triangulate"] = timed(lambda: fs.triangulate(states))[0]
        calls["window"], (tabs, inv, _) = timed(lambda: fs.window(VIS_CAP))
        xs = [v * (1.0 + 1e-3 * rng.standard_normal(len(v))) for v in inv]
        verdicts = [(rng.uniform(size=len(v)) < 0.03).astype(np.uint8) for v in inv]
        calls["set_depth"] = timed(lambda: fs.set_depth(xs))[0]
        calls["remove_outliers"], removed = timed(lambda: fs.remove_outliers(verdicts))
        calls["predict"] = timed(lambda: fs.predict(states, [fc_] * F))[0]
    calls["slide"] = timed(lambda: fs.slide([fc_] * F, [1 if nonlin else 0] * F, *mats))[0]
    if nonlin:
        calls["remove_failures"] = timed(fs.remove_failures)[0]
    # the restated host FeatureManager over the same rows, same order of calls
    t0 = time.perf_counter()
    for r in refs:
        kf = r.add_feature_check_parallax(fc_, image, 0.0)
        if nonlin:
            r.triangulate(state)
            table, x, _ = r.window()
            r.set_depth(x)
            r.remove_outlier(r.outlier_ids(np.zeros(len(x), np.uint8)))
            r.predict(state, fc_)
        r.slide(fc_, kf, nonlin, fc.cam_mats(state))
        if nonlin:
            r.remove_failures()
    h = (time.perf_counter() - t0) * 1e3 / HOST_F
    if t >= TICKS - MEASURED:
        for k, v in calls.items():
            res.setdefault(k, []).append(v)
        res.setdefault("tick_total", []).append(sum(calls.values()))
        host_ms.append(h)
        rows.append(len(image))
prof_names = {}
ctx.set_profiling(True)                                 # kernel times of one more NON_LINEAR tick
fs.add([10] * F, [0.0] * F, [fc.rows_of(sc.image(TICKS), True)] * F); fs.decisions(); fs.triangulate(states)
tabs, inv, _ = fs.window(VIS_CAP); fs.set_depth(inv); fs.remove_outliers([np.zeros(len(v), np.uint8) for v in inv]); fs.predict(states, [10] * F)
fs.slide([10] * F, [1] * F, *mats); fs.remove_failures(); fs.download()
prof = {k: v[0] for k, v in ctx.profile().items() if k.startswith("fm_")}
ctx.set_profiling(False)
fs.close()
summ = {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v)), "n": len(v)} for k, v in res.items()}
print(json.dumps({"what": "viwb_features_* per NON_LINEAR tick, stereo, max_rows 160", "card": card, "power_limit": power, "streams": F,
                  "rows_per_stream_mean": float(np.mean(rows)), "landmarks_per_stream": int(len(inv[0])), "tracked_per_stream": int(dec["last_track_num"][0]), "ms": summ, "kernel_ms": prof,
                  "host_python_restatement_ms_per_stream": {"median": float(np.median(host_ms)), "streams_timed": HOST_F}}))
