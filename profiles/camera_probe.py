"""What the camera model costs on the device: a pinhole session (EuRoC's cam0/cam1_pinhole calibrations) and an MEI session (EuRoC's
cam0/cam1_mei calibrations, camodocal::CataCamera) at the bench shape, ticked alternately in one process, the order swapped every tick.  Every tick
after the second is preceded by viwb_tracker_feedback (one row in twenty removed, every row tracked at least twice predicted), so the session runs
the estimator's loop and trk_feedback projects through the camera model.  Timed ticks (CUDA events on the context's stream around
viwb_tracker_feedback and viwb_tracker_track) alternate with profiled ticks (viwb_set_profiling: trk_merge, trk_stereo, trk_feedback, the kernels
that lift or project).  Prints one JSON line with the card's name and power limit, and whether the two models' ranges overlap.  There is no CPU
path: without a CUDA device the script fails.
Usage (GPU box): python profiles/camera_probe.py   (CAM_STREAMS, CAM_TICKS env; default 1584 stereo streams x 150 rows, 752 x 480)"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "viw-fusion_b200", "python"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from viwb import lib  # noqa: E402
import camera_checks as cc  # noqa: E402
import camera_oracle as co  # noqa: E402
import parity_checks as pc  # noqa: E402

F = int(os.environ.get("CAM_STREAMS", "1584"))
TICKS = int(os.environ.get("CAM_TICKS", "20"))             # measured ticks per session, half timed, half profiled
WARM = 4
W, H, MAX_CNT, MIN_DIST = 752, 480, 150, 30
PIN0 = (461.1586, 459.7529, 362.6593, 248.5236, -0.2847798, 0.08245052, -1.0946e-06, 4.78701e-06)     # config/euroc/cam0_pinhole.yaml
PIN1 = (457.5874, 456.1340, 379.9994, 255.2381, -0.2836831, 0.07395907, 1.9359e-04, 1.7618e-05)       # config/euroc/cam1_pinhole.yaml
KERNELS = ("trk_merge", "trk_stereo", "trk_feedback")

if not torch.cuda.is_available():
    raise SystemExit("camera_probe: no CUDA device")
card = torch.cuda.get_device_name(0)
power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()

# every stream sees the same camera (the work per stream does not depend on what the others see): one image per tick, stride 0 over the streams
seq = pc.camera_sequence(300, W, H, WARM + TICKS)
left = [np.broadcast_to(a[None], (F, H, W)) for a in seq[0]]
right = [np.broadcast_to(a[None], (F, H, W)) for a in seq[1]]

ctx = lib.Context(0)
stream = torch.cuda.Stream()
ctx.set_stream(stream.cuda_stream)
sessions = {"pinhole": {"cam0": PIN0, "trk": ctx.tracker(F, W, H, PIN0, PIN1, MAX_CNT, MIN_DIST, True)},
            "mei": {"cam0": cc.EUROC_CAM0, "trk": ctx.tracker(F, W, H, cc.lib_camera(cc.EUROC_CAM0), cc.lib_camera(cc.EUROC_CAM1), MAX_CNT, MIN_DIST, True)}}
res = {m: {"feedback_ms": [], "tick_ms": [], "rows_mean": []} | {k + "_ms": [] for k in KERNELS} for m in sessions}


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream); fn(); e1.record(stream)
    stream.synchronize()
    return e0.elapsed_time(e1)


def plan(cam, out, motion):
    """per stream: ids to remove (one row in twenty) and the camera-frame prediction of every row tracked at least twice, at the coming motion"""
    n_left, ids, cnt, feat = out[:4]
    rm, pred = [], []
    for f in range(F):
        n = int(n_left[f])
        rows = np.nonzero(cnt[f, :n] >= 2)[0]
        un = co.lift_projective(cam, feat[f, rows, 2:4] + np.float32(motion)).astype(np.float64)
        pred.append((ids[f, rows].copy(), np.column_stack([un, np.ones(len(rows))]) * 5.0))
        rm.append(ids[f, :n][::20].copy())
    return rm, pred


for t in range(WARM + TICKS):
    profiled = t >= WARM and (t - WARM) % 2 == 1
    for m in (list(sessions) if t % 2 == 0 else list(sessions)[::-1]):
        s = sessions[m]
        trk = s["trk"]
        if t >= 2:
            rm, pred = plan(s["cam0"], s["out"], seq[2][t])
        if profiled:
            ctx.set_profiling(True)
        fb = timed(lambda: trk.feedback(rm, pred)) if t >= 2 else 0.0
        tk = timed(lambda: trk.track(0.05 * (t + 1), left[t], right[t]))
        s["out"] = [a.copy() for a in trk.download()]
        if profiled:
            prof = ctx.profile()
            ctx.set_profiling(False)
            for k in KERNELS:
                res[m][k + "_ms"].append(prof.get(k, (float("nan"), 0))[0])
        elif t >= WARM:
            res[m]["feedback_ms"].append(fb); res[m]["tick_ms"].append(tk); res[m]["rows_mean"].append(float(s["out"][0].mean()))
for s in sessions.values():
    s["trk"].close()
summ = {m: {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v)), "n": len(v)} for k, v in r.items()} for m, r in res.items()}
overlap = {k: bool(summ["pinhole"][k]["min"] <= summ["mei"][k]["max"] and summ["mei"][k]["min"] <= summ["pinhole"][k]["max"]) for k in res["mei"] if k != "rows_mean"}
line = json.dumps({"what": "pinhole vs MEI sessions, stereo 752x480, MAX_CNT 150, FLOW_BACK 1, feedback before every tick", "card": card, "power_limit": power,
                   "streams": F, "ms": summ, "ranges_overlap": overlap})
print(line)
