"""What the Kannala-Brandt camera model costs on the device, beside the pinhole and MEI models: one session per model (EuRoC's pinhole and MEI
calibrations, a Kalibr-style 752 x 480 Kannala-Brandt pair) at the bench shape, ticked alternately in one process, the order rotated every
tick.  Every tick after the second is preceded by viwb_tracker_feedback (one row in twenty removed, every row tracked at least twice
predicted), so trk_feedback projects through the camera model.  Timed ticks (CUDA events on the context's stream around viwb_tracker_feedback
and viwb_tracker_track) alternate with profiled ticks (viwb_set_profiling: trk_merge, trk_stereo, trk_feedback).  `undistort` is the
undistort kernel of viwb_undistort_velocity_camera over streams x 150 pixels of the image, per model, profiled.
With CAM_PARENT_LIB naming another build of libviwb.so (the parent commit's, say), its pinhole and MEI sessions run in the same process,
alternated with the others, as `pinhole@parent` / `mei@parent`.  Prints one JSON line with the card's name and power limit.  There is no CPU
path: without a CUDA device the script fails.
Usage (GPU box): python profiles/camera_kb_probe.py   (CAM_STREAMS, CAM_TICKS, CAM_PARENT_LIB env; default 1584 stereo streams x 150 rows)"""
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
import kb_camera_checks as kc  # noqa: E402
import kb_oracle as ko  # noqa: E402
import parity_checks as pc  # noqa: E402

F = int(os.environ.get("CAM_STREAMS", "1584"))
TICKS = int(os.environ.get("CAM_TICKS", "20"))             # measured ticks per session, half timed, half profiled
WARM = 4
W, H, MAX_CNT, MIN_DIST = 752, 480, 150, 30
PIN0 = (461.1586, 459.7529, 362.6593, 248.5236, -0.2847798, 0.08245052, -1.0946e-06, 4.78701e-06)     # config/euroc/cam0_pinhole.yaml
PIN1 = (457.5874, 456.1340, 379.9994, 255.2381, -0.2836831, 0.07395907, 1.9359e-04, 1.7618e-05)       # config/euroc/cam1_pinhole.yaml
KB0 = kc.KB_752
KB1 = KB0._replace(k2=-1.1937e-02, k3=1.0571e-02, mu=235.83, u0=379.5)
KERNELS = ("trk_merge", "trk_stereo", "trk_feedback")

if not torch.cuda.is_available():
    raise SystemExit("camera_kb_probe: no CUDA device")
card = torch.cuda.get_device_name(0)
power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()

seq = pc.camera_sequence(300, W, H, WARM + TICKS)
left = [np.broadcast_to(a[None], (F, H, W)) for a in seq[0]]
right = [np.broadcast_to(a[None], (F, H, W)) for a in seq[1]]

stream = torch.cuda.Stream()
ctxs = {"": lib.Context(0)}
if os.environ.get("CAM_PARENT_LIB"):
    ctxs["@parent"] = lib.Context(0, os.environ["CAM_PARENT_LIB"])
for c in ctxs.values():
    c.set_stream(stream.cuda_stream)
sessions = {}
for tag, ctx in ctxs.items():
    sessions["pinhole" + tag] = {"ctx": ctx, "cam0": PIN0, "trk": ctx.tracker(F, W, H, PIN0, PIN1, MAX_CNT, MIN_DIST, True)}
    sessions["mei" + tag] = {"ctx": ctx, "cam0": cc.EUROC_CAM0,
                             "trk": ctx.tracker(F, W, H, cc.lib_camera(cc.EUROC_CAM0), cc.lib_camera(cc.EUROC_CAM1), MAX_CNT, MIN_DIST, True)}
    if tag == "":
        sessions["kb"] = {"ctx": ctx, "cam0": KB0, "trk": ctx.tracker(F, W, H, kc.lib_camera(KB0), kc.lib_camera(KB1), MAX_CNT, MIN_DIST, True)}
res = {m: {"feedback_ms": [], "tick_ms": [], "rows_mean": [], "undistort_ms": []} | {k + "_ms": [] for k in KERNELS} for m in sessions}
rng = np.random.default_rng(1)
upx = np.column_stack([rng.uniform(0, W, F * MAX_CNT), rng.uniform(0, H, F * MAX_CNT)]).astype(np.float32)


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream); fn(); e1.record(stream)
    stream.synchronize()
    return e0.elapsed_time(e1)


def plan(cam, out, motion):
    n_left, ids, cnt, feat = out[:4]
    rm, pred = [], []
    for f in range(F):
        n = int(n_left[f])
        rows = np.nonzero(cnt[f, :n] >= 2)[0]
        un = ko.lift_projective(cam, feat[f, rows, 2:4] + np.float32(motion)).astype(np.float64)
        pred.append((ids[f, rows].copy(), np.column_stack([un, np.ones(len(rows))]) * 5.0))
        rm.append(ids[f, :n][::20].copy())
    return rm, pred


names = list(sessions)
for t in range(WARM + TICKS):
    profiled = t >= WARM and (t - WARM) % 2 == 1
    k0 = t % len(names)
    for m in names[k0:] + names[:k0]:
        s = sessions[m]
        trk, ctx = s["trk"], s["ctx"]
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
            cam = s["cam0"]
            ctx.set_profiling(True)
            ctx.undistort_velocity(cam if type(cam) is tuple else kc.lib_camera(cam), upx, None, None, 0.05, want_velocity=False)
            prof = ctx.profile()
            ctx.set_profiling(False)
            res[m]["undistort_ms"].append(prof.get("undistort", (float("nan"), 0))[0])
        elif t >= WARM:
            res[m]["feedback_ms"].append(fb); res[m]["tick_ms"].append(tk); res[m]["rows_mean"].append(float(s["out"][0].mean()))
for s in sessions.values():
    s["trk"].close()
summ = {m: {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v)), "n": len(v)} for k, v in r.items()} for m, r in res.items()}
line = json.dumps({"what": "pinhole vs MEI vs Kannala-Brandt sessions, stereo 752x480, MAX_CNT 150, FLOW_BACK 1, feedback before every tick; undistort over "
                   "streams x 150 pixels", "card": card, "power_limit": power, "streams": F, "ms": summ})
print(line)
