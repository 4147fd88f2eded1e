"""What the estimator -> tracker feedback costs on the device: viwb_tracker_feedback (removeOutliers + setPrediction on every stream) and one
viwb_tracker_track that consumes the resident prediction, against the same tick fed the same pixels through predict_pts from the host.  One session,
the two kinds of tick alternated after warm-up, CUDA events on the context's stream around each call (the upload of the id lists, resp. of the pixel
array, is inside the bracket; the host-side id lookup and projection the caller needs for predict_pts is reported apart).  Prints one JSON line with
the card's name and power limit.  There is no CPU path: without a CUDA device the script fails.
Usage (GPU box): python profiles/feedback_probe.py   (FB_STREAMS, FB_TICKS env; default 1584 streams x 150 rows, the C2 batch shape)"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "viw-fusion_b200", "python"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from viwb import lib  # noqa: E402
import feedback_oracle as fbo  # noqa: E402
import feature_oracle as fo  # noqa: E402
import parity_checks as pc  # noqa: E402

F = int(os.environ.get("FB_STREAMS", "1584"))
TICKS = int(os.environ.get("FB_TICKS", "12"))             # measured ticks, half of each kind
W, H, MAX_CNT, MIN_DIST = 752, 480, 150, 30
CAM0 = (461.1586, 459.7529, 362.6593, 248.5236, -0.2847798, 0.08245052, -1.0946e-06, 4.78701e-06)     # config/euroc/cam0_pinhole.yaml
CAM1 = (457.5874, 456.1340, 379.9994, 255.2381, -0.2836831, 0.07395907, 1.9359e-04, 1.7618e-05)       # config/euroc/cam1_pinhole.yaml
WARM = 4

if not torch.cuda.is_available():
    raise SystemExit("feedback_probe: no CUDA device")
card = torch.cuda.get_device_name(0)
power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()

# every stream sees the same camera (the work per stream does not depend on what the others see): one image per tick, stride 0 over the streams
seq = pc.camera_sequence(300, W, H, WARM + TICKS)
left = [np.broadcast_to(a[None], (F, H, W)) for a in seq[0]]
right = [np.broadcast_to(a[None], (F, H, W)) for a in seq[1]]

ctx = lib.Context(0)
stream = torch.cuda.Stream()
ctx.set_stream(stream.cuda_stream)
trk = ctx.tracker(F, W, H, CAM0, CAM1, MAX_CNT, MIN_DIST, True)
rng = np.random.default_rng(0)


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream); fn(); e1.record(stream)
    stream.synchronize()
    return e0.elapsed_time(e1)


def plan(out, motion):
    """per stream: ids to remove (one row in twenty) and the prediction of every row tracked at least twice, at the coming tick's image motion"""
    n_left, ids, cnt, feat = out[:4]
    rm, pred, pp = [], [], np.zeros((F, MAX_CNT, 2), np.float32)
    t0 = time.perf_counter()
    for f in range(F):
        n = int(n_left[f])
        rows = np.nonzero(cnt[f, :n] >= 2)[0]
        px = feat[f, rows, 2:4] + np.float32(motion)
        pts = np.column_stack([fo.lift_projective(CAM0, px).astype(np.float64), np.ones(len(rows))]) * 5.0
        pred.append((ids[f, rows].copy(), pts))
        rm.append(ids[f, :n][::20].copy())
    plan_s = time.perf_counter() - t0
    t0 = time.perf_counter()                       # what a caller of predict_pts does instead: id lookup, spaceToPlane, fall-back to prev_pts
    for f in range(F):
        n = int(n_left[f])
        pp[f, :n] = feat[f, :n, 2:4]
        rows = np.nonzero(cnt[f, :n] >= 2)[0]
        pp[f, rows] = fbo.space_to_plane(CAM0, pred[f][1]).astype(np.float32)
    return rm, pred, pp, time.perf_counter() - t0


res = {"feedback_ms": [], "track_resident_ms": [], "track_host_fed_ms": [], "host_lookup_ms": []}
for t in range(WARM + TICKS):
    if t < 2:
        trk.track(0.05 * (t + 1), left[t], right[t])
    else:
        rm, pred, pp, host_s = plan(out, seq[2][t])
        resident = t % 2 == 0
        if resident:
            fb = timed(lambda: trk.feedback(rm, pred))
            tk = timed(lambda: trk.track(0.05 * (t + 1), left[t], right[t]))
        else:
            tk = timed(lambda: trk.track(0.05 * (t + 1), left[t], right[t], pp, np.ones(F, np.uint8)))
        if t >= WARM:
            if resident:
                res["feedback_ms"].append(fb); res["track_resident_ms"].append(tk)
            else:
                res["track_host_fed_ms"].append(tk); res["host_lookup_ms"].append(host_s * 1e3)
    out = [a.copy() for a in trk.download()]
ctx.set_profiling(True)                             # the feedback kernel alone: CUDA events around the launch
rm, pred, pp, _ = plan(out, seq[2][-1])
trk.feedback(rm, pred); trk.download()
prof = ctx.profile()
ctx.set_profiling(False)
trk.close()
summ = {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v)), "n": len(v)} for k, v in res.items()}
print(json.dumps({"what": "viwb_tracker_feedback and the tick after it, stereo 752x480, MAX_CNT 150, FLOW_BACK 1", "card": card, "power_limit": power,
                  "streams": F, "rows_mean": float(out[0].mean()), "ms": summ, "trk_feedback_kernel_ms": prof.get("trk_feedback", (None, 0))[0],
                  "predict_pts_upload_bytes": F * MAX_CNT * 8}))
