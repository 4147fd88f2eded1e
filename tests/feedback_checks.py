"""Checks of the estimator -> tracker feedback (estimator.cpp:841-843): viwb_predict_pts (Estimator::predictPtsInNextFrame) and
viwb_tracker_feedback (FeatureTracker::removeOutliers + setPrediction on the resident sessions), parameterised by the context like
parity_checks.py: tests/test_feedback.py runs each on the emulation build and, marked gpu, on libviwb.so.  The restatements they compare
with (oracle/feedback_oracle.py) are pinned to the reference's compiled code by the first two checks."""
import ctypes as C

import numpy as np

import parity_checks as pc
from viwb import synth
from viwb.lib import ViwbError

W, H, MAX_CNT, MIN_DIST = 320, 240, 60, 20
CAM0 = (461.1586 * W / 752, 459.7529 * W / 752, W / 2 - 3.2, H / 2 + 1.7, -0.2847798, 0.08245052, -1.0946e-06, 4.78701e-06)
CAM1 = (457.5874 * W / 752, 456.1340 * W / 752, W / 2 + 4.1, H / 2 - 2.6, -0.2836831, 0.07395907, 1.9359e-04, 1.7618e-05)


# ------------------------------------------------------------------------------------------------ predictPtsInNextFrame
def predict_case(cid, seed, frame_count=10, n=80):
    """A window state of configuration `cid` and a feature list with every kind of row the reference tells apart: 1, 2, 3 and >= 4 observations,
    non-positive depths, tracks that ended before frame_count, tracks that reach it."""
    rng = np.random.default_rng(seed)
    prob, st, gt = synth.Sequence(synth.make_config(cid), 1, 11).window(0)
    state = np.array(gt[:207], np.float64)
    num_obs = rng.integers(1, 8, n).astype(np.int32)
    num_obs[:8] = [1, 1, 2, 2, 3, 3, 4, 5]
    ends_now = rng.uniform(size=n) < 0.7
    ends_now[:8] = True
    start = np.where(ends_now, frame_count - num_obs + 1, rng.integers(0, max(frame_count - 7, 1), n)).astype(np.int32)
    start = np.clip(start, 0, 10).astype(np.int32)
    pt0 = np.column_stack([rng.uniform(-0.8, 0.8, n), rng.uniform(-0.5, 0.5, n), np.ones(n)])
    depth = rng.uniform(1.5, 20.0, n)
    depth[8:14] = [-1.0, 0.0, -5.0, -1.0, 0.0, -0.2]
    return state, frame_count, start, num_obs, pt0, depth


def _close(a, b, rtol):
    return np.abs(a - b).max() <= rtol * max(np.abs(b).max(), 1e-300) if a.size else True


def check_predict_restatement_vs_reference_code(cid):
    """oracle/feedback_oracle.py:predict_pts_in_next_frame against Estimator::predictPtsInNextFrame itself (compiled, or its stored results)"""
    import feedback_oracle as fbo
    import viw_ref_feedback as vrf
    seen_valid = 0
    for fc in (10, 5, 2, 1, 0):
        args = predict_case(cid, 40 + cid, fc)
        pts, valid = fbo.predict_pts_in_next_frame(*args)
        ref = vrf.predict_pts(*args)
        assert np.array_equal(valid, ref["valid"]), (cid, fc)
        assert _close(pts, ref["pts_cam"], 1e-12), (cid, fc, np.abs(pts - ref["pts_cam"]).max())
        assert ref["has_prediction"] == (fc >= 2) and (fc >= 2 or not valid.any())          # :2083 returns before setPrediction
        seen_valid += int(valid.sum())
        if fc == 10:                                             # each kind of row decided as estimator.cpp:2094-2099 decides it
            state, _, start, num_obs, pt0, depth = args
            want = (depth > 0) & (num_obs >= 2) & (start + num_obs - 1 == fc)
            assert np.array_equal(valid.astype(bool), want) and valid[:8].tolist() == [0, 0, 1, 1, 1, 1, 1, 1] and not valid[8:14].any()
    assert seen_valid > 30


def feedback_case(seed, n=48, remove_all=False, has_prediction=True):
    """Rows of a tracker (pixels, ids, track counts), a remove set and a prediction map that overlap them partly; both lists also name ids
    the tracker does not hold, and the remove list names one id twice."""
    import feature_oracle as fo
    rng = np.random.default_rng(seed)
    prev = np.column_stack([rng.uniform(5, W - 5, n), rng.uniform(5, H - 5, n)]).astype(np.float32)
    ids = np.sort(rng.choice(400, n, replace=False)).astype(np.int32)
    cnt = rng.integers(1, 30, n).astype(np.int32)
    remove = ids.copy() if remove_all else np.concatenate([rng.choice(ids, n // 5, replace=False), [1000, 1001, ids[0], ids[0]]]).astype(np.int32)
    pid = np.concatenate([rng.choice(ids, n // 2, replace=False), [2000, 2001]]).astype(np.int32)
    rng.shuffle(pid)
    target = np.column_stack([rng.uniform(5, W - 5, len(pid)), rng.uniform(5, H - 5, len(pid))]).astype(np.float32)
    depth = rng.uniform(1.0, 30.0, len(pid))
    pts_cam = np.column_stack([fo.lift_projective(CAM0, target).astype(np.float64), np.ones(len(pid))]) * depth[:, None]
    return prev, ids, cnt, remove, has_prediction, pid, pts_cam


def restated_feedback(cam, prev, ids, cnt, remove, has_prediction, pid, pts_cam):
    import feedback_oracle as fbo
    r = fbo.FeatureTrackerRef(cam, None, MAX_CNT, MIN_DIST)
    r.prev_pts, r.ids, r.track_cnt = np.array(prev, np.float32), [int(i) for i in ids], [int(c) for c in cnt]
    r.remove_outliers(remove)
    if has_prediction:
        r.set_prediction_from_map({int(i): p for i, p in zip(pid, pts_cam)})
    return r


def check_feedback_restatement_vs_reference_code():
    """FeatureTrackerRef.remove_outliers / set_prediction_from_map against FeatureTracker::removeOutliers / setPrediction themselves: rows, order
    and counts identical, predict_pts the same floats bit for bit"""
    import viw_ref_feedback as vrf
    for cam in (CAM0, (300.0, 301.0, 160.0, 120.0, 0.0, 0.0, 0.0, 0.0)):                     # with distortion, and m_noDistortion
        for seed, kw in ((1, {}), (2, {"remove_all": True}), (3, {"has_prediction": False}), (4, {"n": 1})):
            case = feedback_case(seed, **kw)
            ref = vrf.tracker_feedback(cam, W, H, *case)
            r = restated_feedback(cam, *case)
            assert np.array_equal(np.asarray(r.ids, np.int32), ref["ids"]) and np.array_equal(np.asarray(r.track_cnt, np.int32), ref["track_cnt"])
            assert np.array_equal(r.prev_pts.reshape(-1, 2), ref["prev_pts"]) and r.hasPrediction == ref["has_prediction"]
            if case[4]:
                assert r.predict_pts.tobytes() == ref["predict_pts"].astype(np.float32).tobytes(), (seed, np.abs(r.predict_pts - ref["predict_pts"]).max())
            if kw.get("remove_all"):
                assert len(ref["ids"]) == 0
            elif len(case[1]) > 1:
                assert 0 < len(ref["ids"]) < len(case[1])


def check_predict_pts(ctx, cid):
    """viwb_predict_pts against the restatement and against the reference's code: valid flags identical, pts_cam to 1e-9 relative"""
    import feedback_oracle as fbo
    import viw_ref_feedback as vrf
    for fc in (10, 2, 1):
        args = predict_case(cid, 40 + cid, fc)
        got, valid = ctx.predict_pts(*args)
        pts, want = fbo.predict_pts_in_next_frame(*args)
        assert np.array_equal(valid, want) and _close(got, pts, 1e-9), (cid, fc)
        if vrf.available():
            ref = vrf.predict_pts(*args)
            assert np.array_equal(valid, ref["valid"]) and _close(got, ref["pts_cam"], 1e-9), (cid, fc)
    empty = ctx.predict_pts(args[0], 10, np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros((0, 3)), np.zeros(0))
    assert empty[0].shape == (0, 3)
    for bad_fc, bad_start in ((11, 0), (-1, 0), (10, 11), (10, -1)):
        try:
            ctx.predict_pts(args[0], bad_fc, np.array([bad_start], np.int32), np.array([2], np.int32), np.ones((1, 3)), np.ones(1))
            raise AssertionError("frame_count %d / start_frame %d accepted" % (bad_fc, bad_start))
        except ViwbError:
            pass


# ------------------------------------------------------------------------------------------------ sessions
def cam_points(cam, px, depth):
    """camera-frame points that PinholeCamera::spaceToPlane sends to the pixels `px` (to the accuracy of the 8-step undistortion)"""
    import feature_oracle as fo
    px = np.asarray(px, np.float32).reshape(-1, 2)
    return np.column_stack([fo.lift_projective(cam, px).astype(np.float64), np.ones(len(px))]) * np.asarray(depth, np.float64).reshape(-1, 1)


def _compare_tick(t, f, out, r, stereo, tol_px=1e-2):
    n_left, ids, cnt, feat, n_right, ids_r, feat_r = out
    rid, rcnt, rpts, run, rvel, rid_r, rpts_r, run_r, rvel_r = r
    n = int(n_left[f])
    assert n == len(rid), (t, f, n, len(rid))
    assert np.array_equal(ids[f, :n], rid) and np.array_equal(cnt[f, :n], rcnt), (t, f)
    if n:
        assert np.abs(feat[f, :n, 2:4] - rpts).max() <= tol_px, (t, f, np.abs(feat[f, :n, 2:4] - rpts).max())
    if stereo:
        m = int(n_right[f])
        assert m == len(rid_r) and np.array_equal(ids_r[f, :m], rid_r), (t, f, m, len(rid_r))
        if m:
            assert np.abs(feat_r[f, :m, 2:4] - rpts_r).max() <= tol_px


def _reference_agrees(ref, cam, remove, predict):
    """where the reference is compiled: FeatureTracker::removeOutliers / setPrediction themselves on the restatement's rows (called past the
    stored-result layer: these rows come out of cv2's flow and are not inputs a stored result could be keyed on)"""
    import viw_ref
    import viw_ref_feedback as vrf
    if not viw_ref.live():
        return None
    pid = np.array(list(predict.keys()) if predict is not None else [], np.int32)
    pts = np.array([predict[int(i)] for i in pid], np.float64).reshape(-1, 3)
    return vrf.tracker_feedback.__wrapped__(cam, W, H, ref.prev_pts, np.asarray(ref.ids, np.int32), np.asarray(ref.track_cnt, np.int32), np.asarray(list(remove), np.int32),
                                predict is not None, pid, pts)


def apply_feedback(trk, refs, removes, predicts):
    """one estimator tick's feedback on the library's sessions and on the restated trackers (removes[f]: ids; predicts[f]: {id: pts_cam} or None)"""
    for ref, rm, pr in zip(refs, removes, predicts):
        want = _reference_agrees(ref, ref.cam[0], rm, pr)
        ref.remove_outliers(rm)
        if pr is not None:
            ref.set_prediction_from_map(pr)
        if want is not None:
            assert np.array_equal(np.asarray(ref.ids, np.int32), want["ids"]) and np.array_equal(ref.prev_pts.reshape(-1, 2), want["prev_pts"])
            assert pr is None or ref.predict_pts.tobytes() == want["predict_pts"].tobytes()
    trk.feedback(removes, None if all(p is None for p in predicts) else
                 [None if p is None else (np.array(list(p.keys()), np.int32), np.array(list(p.values()), np.float64).reshape(-1, 3)) for p in predicts])


def check_tracker_feedback(ctx):
    """After viwb_tracker_feedback, track + download equal the restated FeatureTracker driven through remove_outliers + set_prediction_from_map +
    track_image on every tick: ids, track counts, row order identical, pixels within the session tolerance."""
    import feedback_oracle as fbo
    streams, ticks = 2, 6
    seqs = [pc.camera_sequence(80 + f, W, H, ticks) for f in range(streams)]
    refs = [fbo.FeatureTrackerRef(CAM0, CAM1, MAX_CNT, MIN_DIST, True) for _ in range(streams)]
    trk = ctx.tracker(streams, W, H, CAM0, CAM1, MAX_CNT, MIN_DIST, True)
    rng = np.random.default_rng(17)
    removed = [set(), set()]
    for t in range(ticks):
        left, right = np.stack([seqs[f][0][t] for f in range(streams)]), np.stack([seqs[f][1][t] for f in range(streams)])
        trk.track(0.05 * (t + 1), left, right)
        out = trk.download()
        for f in range(streams):
            _compare_tick(t, f, out, refs[f].track_image(0.05 * (t + 1), seqs[f][0][t], seqs[f][1][t]), True)
            assert not (set(int(i) for i in out[1][f, : out[0][f]]) & removed[f]), (t, f)
        if t + 1 == ticks:
            break
        ids0, ids1 = list(refs[0].ids), list(refs[1].ids)

        def predicted(f, rows):          # the true image motion of the coming tick for `rows` of stream f
            prev = refs[f].prev_pts[rows] + np.float32(seqs[f][2][t + 1])
            return {int(refs[f].ids[i]): p for i, p in zip(rows, cam_points(CAM0, prev, rng.uniform(2, 20, len(rows))))}
        if t == 1:       # stream 0: ids it holds and ids it does not, one twice; a prediction for half of the rows.  stream 1: empty list, no prediction
            rm = [[ids0[3], ids0[10], ids0[3], 777777, -5], []]
            pr = [predicted(0, np.arange(0, len(ids0), 2)), None]
            pr[0][888888] = np.array([0.1, 0.2, 3.0])
        elif t == 2:     # stream 0 loses every row, stream 1 keeps all of them and is predicted in full
            rm = [ids0, [424242]]
            pr = [None, predicted(1, np.arange(len(ids1)))]
        elif t == 3:     # removal alone: the next tick runs the plain path
            rm, pr = [[ids0[0]], [ids1[-1], ids1[0]]], [None, None]
        else:            # prediction alone, both streams
            rm, pr = [[], []], [predicted(0, np.arange(len(ids0))), predicted(1, np.arange(1, len(ids1), 3))]
        for f in range(streams):
            removed[f] |= set(int(i) for i in rm[f])
        apply_feedback(trk, refs, rm, pr)
        # the download between feedback and the next tick still holds the last tick's rows
        again = trk.download()
        assert np.array_equal(again[0], out[0]) and np.array_equal(again[1], out[1])
    assert refs[0].stats["predicted"] == 3 and refs[1].stats["predicted"] == 3, (refs[0].stats, refs[1].stats)
    trk.close()


def check_fallback_rows_static_scene(ctx):
    """setPrediction's fall-back rows are prev_pts bit for bit: on a static scene the seeded flow of such a row starts at the point itself and stays
    there, so the tracked pixel equals the previous one exactly; a predicted row starts a hair off (float projection of the lifted pixel)."""
    import feedback_oracle as fbo
    img = pc.camera_sequence(91, W, H, 1)[0][0]
    trk = ctx.tracker(1, W, H, CAM0, None, MAX_CNT, MIN_DIST, True)
    ref = fbo.FeatureTrackerRef(CAM0, None, MAX_CNT, MIN_DIST, True)
    trk.track(0.05, img[None])
    n0, ids, cnt, feat = [a.copy() for a in trk.download()[:4]]
    ref.track_image(0.05, img)
    n = int(n0[0])
    before = {int(ids[0, j]): feat[0, j, 2:4].copy() for j in range(n)}
    rows = np.arange(0, n, 2)
    pred = {int(ids[0, j]): p for j, p in zip(rows, cam_points(CAM0, feat[0, rows, 2:4] + np.float32(0.3), np.full(len(rows), 4.0)))}
    apply_feedback(trk, [ref], [[int(ids[0, 1])]], [pred])
    trk.track(0.10, img[None])
    out = trk.download()
    _compare_tick(1, 0, out, ref.track_image(0.10, img), False)
    assert ref.stats == {"predicted": 1, "repeated": 0}
    kept = 0
    for j in range(int(out[0][0])):
        fid = int(out[1][0, j])
        if fid in before and fid not in pred:
            assert out[3][0, j, 2:4].tobytes() == before[fid].tobytes(), (fid, out[3][0, j, 2:4], before[fid])
            kept += 1
    assert kept >= n // 4 and int(ids[0, 1]) not in set(int(i) for i in out[1][0, : out[0][0]])
    trk.close()


def check_closed_loop(ctx, ticks=7, streams=2):
    """The loop the reference runs per frame (estimator.cpp:827-870) on resident sessions: each tick a seeded subset of the returned ids is removed
    and the next frame's points are predicted by viwb_predict_pts from a constant-velocity window state, then handed back by
    viwb_tracker_feedback.  The restated tracker, fed by the restated prediction, must agree on every tick."""
    import feedback_oracle as fbo
    seqs = [pc.camera_sequence(60 + f, W, H, ticks) for f in range(streams)]
    refs = [fbo.FeatureTrackerRef(CAM0, CAM1, MAX_CNT, MIN_DIST, True) for _ in range(streams)]
    trk = ctx.tracker(streams, W, H, CAM0, CAM1, MAX_CNT, MIN_DIST, True)
    rng = np.random.default_rng(23)
    depth, fc = 6.0, 10
    removed = [set() for _ in range(streams)]
    last_un = [[{}, {}] for _ in range(streams)]            # id -> undistorted point at the previous tick: [library's rows, restatement's rows]
    top_id, n_predicted = [-1] * streams, 0
    for t in range(ticks):
        left, right = np.stack([seqs[f][0][t] for f in range(streams)]), np.stack([seqs[f][1][t] for f in range(streams)])
        trk.track(0.05 * (t + 1), left, right)
        out = trk.download()
        rm, pr_lib, pr_ref = [], [], []
        for f in range(streams):
            r = refs[f].track_image(0.05 * (t + 1), seqs[f][0][t], seqs[f][1][t])
            _compare_tick(t, f, out, r, True)
            n = int(out[0][f])
            now = set(int(i) for i in out[1][f, :n])
            assert not (now & removed[f]), (t, f)                                  # a removed id never comes back
            fresh = [i for i in now if i > top_id[f]]
            assert t == 0 or len(fresh) > 0                                        # n_id keeps counting: removal makes room for new corners
            top_id[f] = max(top_id[f], max(now))
            rm.append([int(i) for i in rng.choice(out[1][f, :n], max(n // 8, 1), replace=False)] + [10 ** 6 + t])
            removed[f] |= set(rm[-1])
            # the caller's feature list of the last two frames: a track seen at both ticks has two observations starting at frame fc - 1, a new
            # corner one observation at frame fc.  The camera moved parallel to the image plane by the tick's image motion at depth `depth`.
            state = np.zeros(207); state[3 + 7 * np.arange(11) + 3] = 1.0; state[182] = 1.0
            delta = np.array([-seqs[f][2][t][0] * depth / CAM0[0], -seqs[f][2][t][1] * depth / CAM0[1], 0.0])
            state[7 * fc: 7 * fc + 3] = delta
            preds = []
            for which, (ids_now, un_now) in enumerate(((out[1][f, :n], out[3][f, :n, 0:2]), (r[0], r[3]))):
                old = last_un[f][which]
                two = np.array([int(i) in old for i in ids_now], bool)
                start, nobs = np.where(two, fc - 1, fc).astype(np.int32), np.where(two, 2, 1).astype(np.int32)
                pt0 = np.array([list(old[int(i)]) + [1.0] if int(i) in old else [un_now[k][0], un_now[k][1], 1.0] for k, i in enumerate(ids_now)], np.float64).reshape(-1, 3)
                dep = np.full(len(ids_now), depth)
                pts, valid = ctx.predict_pts(state, fc, start, nobs, pt0, dep) if which == 0 else fbo.predict_pts_in_next_frame(state, fc, start, nobs, pt0, dep)
                assert np.array_equal(valid.astype(bool), two)
                preds.append({int(i): p for i, p, v in zip(ids_now, pts, valid) if v})
                last_un[f][which] = {int(i): un_now[k].astype(np.float64) for k, i in enumerate(ids_now)}
            pr_lib.append(preds[0] if preds[0] else None); pr_ref.append(preds[1] if preds[1] else None)
            n_predicted += len(preds[0])
        if t + 1 < ticks:
            for f in range(streams):
                refs[f].remove_outliers(rm[f])
                if pr_ref[f] is not None:
                    refs[f].set_prediction_from_map(pr_ref[f])
            trk.feedback(rm, [None if p is None else (np.array(list(p.keys()), np.int32), np.array(list(p.values()))) for p in pr_lib])
    for f in range(streams):
        assert refs[f].stats["predicted"] == ticks - 2 and refs[f].stats["repeated"] == 0, refs[f].stats      # the seeded pass ran and held
    assert n_predicted >= streams * (ticks - 2) * MAX_CNT // 3
    trk.close()


def check_unchanged_path(ctx):
    """A session that never calls feedback launches what it launched before there was one, and a tick that consumes a resident prediction is the
    tick fed the same pixels through predict_pts: same launches, same downloads bit for bit."""
    import feedback_oracle as fbo
    ticks = 4
    seq = pc.camera_sequence(66, W, H, ticks)
    a, b = (ctx.tracker(2, W, H, CAM0, CAM1, MAX_CNT, MIN_DIST, True) for _ in range(2))
    ref = fbo.FeatureTrackerRef(CAM0, CAM1, MAX_CNT, MIN_DIST, True)
    rng = np.random.default_rng(5)
    for t in range(ticks):
        left, right = np.stack([seq[0][t]] * 2), np.stack([seq[1][t]] * 2)
        pp = hp = None
        if t >= 2:        # stream 0 predicted for two rows in three, stream 1 not at all
            rows = np.array([i for i in range(len(ref.ids)) if i % 3])
            pred = {int(ref.ids[i]): p for i, p in zip(rows, cam_points(CAM0, ref.prev_pts[rows] + np.float32(seq[2][t]), rng.uniform(2, 9, len(rows))))}
            ref.set_prediction_from_map(pred)
            # the host-fed twin: setPrediction restated on the library's own rows of the last tick (its prev_pts, to the bit)
            pp, hp = np.zeros((2, MAX_CNT, 2), np.float32), np.array([1, 0], np.uint8)
            for j in range(int(ob[0][0])):
                fid = int(ob[1][0, j])
                pp[0, j] = fbo.space_to_plane(CAM0, pred[fid])[0].astype(np.float32) if fid in pred else ob[3][0, j, 2:4]
            a.feedback(None, [(np.array(list(pred.keys()), np.int32), np.array(list(pred.values()))), None])
        l0 = ctx.launch_count(); a.track(0.05 * (t + 1), left, right); oa = [x.copy() for x in a.download()]
        l1 = ctx.launch_count(); b.track(0.05 * (t + 1), left, right, pp, hp); ob = [x.copy() for x in b.download()]
        l2 = ctx.launch_count()
        assert l1 - l0 == l2 - l1, (t, l1 - l0, l2 - l1)
        if t == 1:
            assert 17 <= l2 - l1 <= 19, l2 - l1                    # a stereo, flow-back tick without a prediction
        for x, y in zip(oa, ob):
            assert x.tobytes() == y.tobytes(), t
        _compare_tick(t, 0, oa, ref.track_image(0.05 * (t + 1), seq[0][t], seq[1][t]), True)
    assert ref.stats["predicted"] == 2
    a.close(); b.close()


def check_feedback_errors(ctx):
    """Every argument error is VIWB_ERR_INVALID with a message, and the session works afterwards"""
    import feedback_oracle as fbo
    seq = pc.camera_sequence(67, W, H, 3)
    trk = ctx.tracker(1, W, H, CAM0, None, MAX_CNT, MIN_DIST, True)
    ref = fbo.FeatureTrackerRef(CAM0, None, MAX_CNT, MIN_DIST, True)
    L, INVALID = ctx.lib, -1
    one = lambda v, ty=np.int32: np.array([v], ty)
    vp = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)

    def raw(n_rm=None, rm=None, n_pr=None, pid=None, pts=None, hp=None):
        return L.viwb_tracker_feedback(trk.hnd, vp(n_rm), vp(rm), vp(n_pr), vp(pid), vp(pts), vp(hp))
    assert L.viwb_tracker_feedback(None, None, None, None, None, None, None) == INVALID
    assert raw(one(0)) == INVALID and b"no tick" in L.viwb_last_error(ctx.h)                 # before the first tick
    trk.track(0.05, seq[0][0][None]); ref.track_image(0.05, seq[0][0])
    ids = trk.download()[1][0].copy()
    assert raw(one(-1), one(0)) == INVALID and b"negative" in L.viwb_last_error(ctx.h)
    assert raw(None, None, one(-1), one(0), np.ones(3), one(1, np.uint8)) == INVALID
    assert raw(one(1), None) == INVALID and b"remove_ids" in L.viwb_last_error(ctx.h)
    assert raw(None, None, one(1), None, np.ones(3), one(1, np.uint8)) == INVALID
    assert raw(None, None, one(1), one(0), None, one(1, np.uint8)) == INVALID
    assert raw(None, None, one(1), one(0), np.ones(3), None) == INVALID and b"has_prediction" in L.viwb_last_error(ctx.h)
    assert raw() == 0                                                                        # both halves absent: nothing to do
    # none of the refused calls touched the rows: a real feedback now, then a tick given predict_pts as well is refused and leaves the session as it was
    pred = {int(ids[2]): cam_points(CAM0, ref.prev_pts[2] + np.float32(seq[2][1]), [5.0])[0]}
    apply_feedback(trk, [ref], [[int(ids[0])]], [pred])
    try:
        trk.track(0.10, seq[0][1][None], None, np.zeros((1, MAX_CNT, 2), np.float32), one(1, np.uint8))
        raise AssertionError("predict_pts accepted beside a pending resident prediction")
    except ViwbError as e:
        assert "pending" in str(e)
    assert raw(one(0)) == INVALID and b"pending" in L.viwb_last_error(ctx.h)                  # removal alone under a pending prediction
    trk.track(0.10, seq[0][1][None])
    _compare_tick(1, 0, trk.download(), ref.track_image(0.10, seq[0][1]), False)
    assert ref.stats["predicted"] == 1
    trk.track(0.15, seq[0][2][None])                                                         # hasPrediction was cleared: the plain path again
    _compare_tick(2, 0, trk.download(), ref.track_image(0.15, seq[0][2]), False)
    assert ref.stats["predicted"] == 1
    trk.close()
