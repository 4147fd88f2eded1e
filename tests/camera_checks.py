"""Checks of the MEI camera model (camodocal::CataCamera) beside the pinhole one: the restatements (oracle/camera_oracle.py) against the
reference's compiled CataCamera.cc, then viwb_undistort_velocity_camera, viwb_tracker_create_camera sessions and viwb_tracker_feedback on
MEI sessions, parameterised by the context like parity_checks.py: tests/test_camera_models.py runs each library check on the emulation build (`not gpu`) and, marked gpu, on libviwb.so."""
import ctypes as C

import numpy as np

import camera_oracle as co
import feedback_oracle as fbo
import parity_checks as pc
from viwb import lib as viwb_lib

f32 = np.float32

# MEI calibrations shipped with the reference (camodocal yaml, model_type: MEI), 752 x 480
EUROC_CAM0 = co.Mei(3.6313355285286337e+00, 1.1757726639872075e+00, 1.5491281051140213e+01, -8.1237172954550494e-04, 6.7297684030310243e-04,
                    2.1387619122017772e+03, 2.1315886210259278e+03, 3.6119856633263799e+02, 2.4827644773395667e+02)       # config/euroc/cam0_mei.yaml
EUROC_CAM1 = co.Mei(8.1261505894146113e-01, -3.4247886078397966e-01, 1.7108792755973357e-01, -6.6653144364906686e-04, 7.2311255846767091e-04,
                    8.3406249735437791e+02, 8.3140606765916948e+02, 3.7432007355249738e+02, 2.5422391621480082e+02)       # config/euroc/cam1_mei.yaml
MYNT_LEFT = co.Mei(1.4456544769803834e+00, -3.4363053357673362e-01, 6.2347376791548004e-02, 1.2608078788285675e-03, -2.1374139252651483e-04,
                   8.9594371861807986e+02, 8.9741581479032754e+02, 3.7221680816143993e+02, 2.3833534175557006e+02)         # config/mynteye/left_mei.yaml
# synthetic sets for the branches the calibrations do not reach
XI_ONE = co.Mei(1.0, -0.21, 0.04, 3e-4, -2e-4, 410.0, 408.5, 371.3, 243.9)            # the xi == 1 branch of liftProjective
NO_DIST = co.Mei(0.87, 0.0, 0.0, 0.0, 0.0, 512.0, 509.25, 377.5, 236.0)              # m_noDistortion
WIDE = co.Mei(2.5, -0.08, 0.006, 2e-4, 1e-4, 190.0, 191.0, 376.0, 240.0)              # 1 + (1 - xi^2) rho^2 < 0 beyond ~83 px from the centre
CAMERAS = {"euroc_cam0": EUROC_CAM0, "euroc_cam1": EUROC_CAM1, "mynteye_left": MYNT_LEFT, "xi_one": XI_ONE, "no_distortion": NO_DIST, "wide": WIDE}
CW, CH = 752, 480

W, H, MAX_CNT, MIN_DIST = 320, 240, 60, 20
PIN1 = (457.5874 * W / 752, 456.1340 * W / 752, W / 2 + 4.1, H / 2 - 2.6, -0.2836831, 0.07395907, 1.9359e-04, 1.7618e-05)


def scaled(cam):
    """a 752 x 480 MEI calibration for the W x H session images"""
    return cam._replace(gamma1=cam.gamma1 * W / CW, gamma2=cam.gamma2 * H / CH, u0=cam.u0 * W / CW, v0=cam.v0 * H / CH)


def lib_camera(cam):
    """the viwb.lib.Camera of an oracle camera (camera_oracle.Mei or a pinhole 8-tuple)"""
    return viwb_lib.Camera.mei(*cam) if isinstance(cam, co.Mei) else viwb_lib.Camera.pinhole(*cam)


def same_floats(a, b):
    """bit-identical outside NaN, NaN in the same places (NaN bit patterns differ between x86 and CUDA)"""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb)) and a[~na].tobytes() == b[~nb].tobytes()


def pixel_set(seed, n=400):
    """pixels over the whole image, a few beyond it, the principal points of every calibration and the image corners"""
    rng = np.random.default_rng(seed)
    pts = np.column_stack([rng.uniform(-40, CW + 40, n), rng.uniform(-40, CH + 40, n)])
    fixed = [[c.u0, c.v0] for c in CAMERAS.values()] + [[0, 0], [CW - 1, 0], [0, CH - 1], [CW - 1, CH - 1]]
    return np.concatenate([pts, fixed]).astype(f32)


def space_set(cam, seed, n=300):
    """camera-frame points: rays of image pixels at several depths, random points around the camera (behind it as well), and the rays with
    P(2) + xi |P| <= 0 (z = 0 exactly where xi == 1)"""
    rng = np.random.default_rng(seed)
    px = pixel_set(seed, n // 2)
    with np.errstate(all="ignore"):
        un = co.lift_projective(cam, px).astype(np.float64)
    rays = np.column_stack([un, np.ones(len(un))]) * rng.uniform(0.5, 40.0, (len(un), 1))
    rays = rays[np.isfinite(rays).all(1)]
    free = rng.normal(0, 3.0, (n // 2, 3))
    behind = [[0.0, 0.0, -1.0], [0.3, -0.2, -5.0], [1e-3, 2e-3, -1.0], [0.0, 0.0, 0.0]]
    return np.concatenate([rays, free, behind])


# ------------------------------------------------------------------------------------------------ the restatements against the reference
def check_restatement_vs_reference_code():
    """lift_projective_mei and space_to_plane_mei against CataCamera::liftProjective (through FeatureTracker::undistortedPts) and
    CataCamera::spaceToPlane compiled from the reference (or their stored results): every float identical, NaN / inf in the same places"""
    import viw_ref_camera as vrc
    seen = {"nan_lift": 0, "nonpositive_z": 0}
    for k, (name, cam) in enumerate(CAMERAS.items()):
        px = pixel_set(10 + k)
        mine = co.lift_projective(cam, px)
        assert same_floats(mine, vrc.camera_undistorted_pts(cam, CW, CH, px)), name
        seen["nan_lift"] += int(np.isnan(mine).any(1).sum())
        P = space_set(cam, 30 + k)
        uv = co.space_to_plane(cam, P)
        assert same_floats(uv, vrc.camera_space_to_plane(cam, CW, CH, P)), name
        with np.errstate(all="ignore"):
            seen["nonpositive_z"] += int((P[:, 2] + cam.xi * np.sqrt((P[:, 0] ** 2 + P[:, 1] ** 2) + P[:, 2] ** 2) <= 0).sum())
        if name.startswith(("euroc", "mynteye")):
            inside = (px[:, 0] >= 0) & (px[:, 0] < CW) & (px[:, 1] >= 0) & (px[:, 1] < CH)
            assert np.isfinite(mine[inside]).all(), name                          # the real calibrations lift their whole image
    assert seen["nan_lift"] > 20 and seen["nonpositive_z"] >= 4, seen          # the sqrt of a negative number and the rays behind the mirror were reached


def feedback_case(cam, seed, n=48, has_prediction=True):
    """rows of a tracker, a remove set and a prediction map over them (ids the tracker does not hold included), the predictions on rays of
    `cam` (a few behind the camera)"""
    rng = np.random.default_rng(seed)
    prev = np.column_stack([rng.uniform(5, W - 5, n), rng.uniform(5, H - 5, n)]).astype(f32)
    ids = np.sort(rng.choice(400, n, replace=False)).astype(np.int32)
    cnt = rng.integers(1, 30, n).astype(np.int32)
    remove = np.concatenate([rng.choice(ids, n // 5, replace=False), [1000, ids[0], ids[0]]]).astype(np.int32)
    pid = np.concatenate([rng.choice(ids, n // 2, replace=False), [2000]]).astype(np.int32)
    rng.shuffle(pid)
    target = np.column_stack([rng.uniform(5, W - 5, len(pid)), rng.uniform(5, H - 5, len(pid))]).astype(f32)
    pts_cam = np.column_stack([co.lift_projective(cam, target).astype(np.float64), np.ones(len(pid))]) * rng.uniform(1.0, 30.0, (len(pid), 1))
    pts_cam[:3] = [[0.1, 0.2, -4.0], [0.0, 0.0, -1.0], [-0.4, 0.3, 2.0]]
    return prev, ids, cnt, remove, has_prediction, pid, pts_cam


def restated_feedback(cam, prev, ids, cnt, remove, has_prediction, pid, pts_cam):
    r = co.FeatureTrackerRef(cam, None, MAX_CNT, MIN_DIST)
    r.prev_pts, r.ids, r.track_cnt = np.array(prev, f32), [int(i) for i in ids], [int(c) for c in cnt]
    r.remove_outliers(remove)
    if has_prediction:
        r.set_prediction_from_map({int(i): p for i, p in zip(pid, pts_cam)})
    return r


def check_feedback_restatement_vs_reference_code():
    """removeOutliers + setPrediction with an MEI m_camera[0]: the restated tracker against the reference's: rows identical, predict_pts the
    same floats"""
    import viw_ref_camera as vrc
    for k, cam in enumerate((scaled(EUROC_CAM0), scaled(EUROC_CAM1), scaled(XI_ONE), scaled(NO_DIST))):
        for seed, kw in ((1 + 10 * k, {}), (2 + 10 * k, {"has_prediction": False})):
            case = feedback_case(cam, seed, **kw)
            ref = vrc.camera_tracker_feedback(cam, W, H, *case)
            r = restated_feedback(cam, *case)
            assert np.array_equal(np.asarray(r.ids, np.int32), ref["ids"]) and np.array_equal(np.asarray(r.track_cnt, np.int32), ref["track_cnt"])
            assert np.array_equal(r.prev_pts.reshape(-1, 2), ref["prev_pts"]) and r.hasPrediction == ref["has_prediction"]
            if case[4]:
                assert same_floats(r.predict_pts, ref["predict_pts"].astype(f32)), (k, seed)


def check_track_image_vs_reference_code(cv2):
    """The reference's own trackImage() with CataCamera m_camera entries (and removeOutliers / setPrediction between ticks) against
    FeatureTrackerRef with the same MEI cameras: every row identical, both hasPrediction outcomes, stereo and mono"""
    import viw_ref
    import viw_ref_camera as vrc
    cam0, cam1 = scaled(EUROC_CAM0), scaled(EUROC_CAM1)
    ticks = 6
    for stereo in (True, False):
        left, right, motion = pc.camera_sequence(81, W, H, ticks)
        ref = vrc.ReferenceFeatureTracker(cam0, cam1 if stereo else None, W, H, MAX_CNT, MIN_DIST, True)
        mine = co.FeatureTrackerRef(cam0, cam1 if stereo else None, MAX_CNT, MIN_DIST, True, use_cv_detector=True, order_fn=viw_ref.std_sort_order)
        for t in range(ticks):
            if t == 2:                       # a prediction through the estimator's path: removeOutliers, then setPrediction over CataCamera::spaceToPlane
                rows = np.arange(0, len(mine.ids), 2)
                pts = np.column_stack([co.lift_projective(cam0, mine.prev_pts[rows] + f32(motion[t])).astype(np.float64), np.ones(len(rows))]) * 5.0
                pred = {int(mine.ids[i]): p for i, p in zip(rows, pts)}
                rm = [int(mine.ids[1]), int(mine.ids[3]), 99999]
                for tr in (ref, mine):
                    tr.remove_outliers(rm); tr.set_prediction_from_map(pred)
            if t == 4:                       # one outside the image: fewer than 10 successes, the full-pyramid repeat
                pred = (mine.prev_pts + f32([W + 30.0, H + 30.0])).astype(f32)
                ref.set_prediction(pred); mine.set_prediction(pred)
            ids0, cnt0, f0, idr0, fr0 = ref.track_image(0.05 * (t + 1), left[t], right[t] if stereo else None)
            ids1, cnt1, pts1, un1, vel1, idr1, ptsr1, unr1, velr1 = mine.track_image(0.05 * (t + 1), left[t], right[t] if stereo else None)
            assert np.array_equal(ids0, ids1) and np.array_equal(cnt0, cnt1), (stereo, t)
            assert np.array_equal(f0[:, 2:4], pts1) and same_floats(f0[:, 0:2], un1) and same_floats(f0[:, 4:6], vel1), (stereo, t)
            assert np.array_equal(idr0, idr1)
            if stereo:
                assert np.array_equal(fr0[:, 2:4], ptsr1) and same_floats(fr0[:, 0:2], unr1) and same_floats(fr0[:, 4:6], velr1), (stereo, t)
        assert mine.stats == {"predicted": 2, "repeated": 1}, mine.stats


# ------------------------------------------------------------------------------------------------ viwb_undistort_velocity_camera
def check_undistort_velocity_camera(ctx):
    """MEI: un_pts bit-identical to the restatement (and to the reference's code or its stored results), velocities bit-identical to the
    reference's rounding of those points.  PINHOLE through the new entry: viwb_undistort_velocity to the bit."""
    import viw_ref_camera as vrc
    rng = np.random.default_rng(6)
    dt = 0.05
    for k, (name, cam) in enumerate(CAMERAS.items()):
        px = pixel_set(10 + k)
        n = len(px)
        want = co.lift_projective(cam, px)
        prev = (np.nan_to_num(want) + rng.normal(0, 0.01, (n, 2))).astype(f32)
        has = (rng.uniform(size=n) < 0.8).astype(np.uint8)
        un, vel = ctx.undistort_velocity(lib_camera(cam), px, prev, has, dt)
        assert same_floats(un, want), name
        if vrc.available():
            assert same_floats(un, vrc.camera_undistorted_pts(cam, CW, CH, px)), name
        with np.errstate(all="ignore"):
            want_vel = np.where(has[:, None] > 0, ((want - prev).astype(np.float64) / dt).astype(f32), f32(0))
        assert same_floats(vel, want_vel), name
        un2, vel2 = ctx.undistort_velocity(lib_camera(cam), px, None, None, dt)
        assert same_floats(un2, want) and not vel2.any()
    pin = (461.1586, 459.7529, 362.6593, 248.5236, -0.2847798, 0.08245052, -1.0946e-06, 4.78701e-06)      # config/euroc/cam0_pinhole.yaml
    px = pixel_set(3)
    prev = rng.normal(0, 0.3, (len(px), 2)).astype(f32)
    for c in (pin, pin[:4] + (0.0, 0.0, 0.0, 0.0)):
        a = ctx.undistort_velocity(c, px, prev, None, dt)
        b = ctx.undistort_velocity(viwb_lib.Camera.pinhole(*c), px, prev, None, dt)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()


# ------------------------------------------------------------------------------------------------ sessions
def _lift_matches(cam, feat, n):
    """the session's normalised points are the restated lift of the session's own pixels: bit for bit for MEI; a pinhole camera keeps the
    library's contracted lift (one float ulp)"""
    if n == 0:
        return True
    got, want = feat[:n, 0:2], co.lift_projective(cam, feat[:n, 2:4])
    return same_floats(got, want) if isinstance(cam, co.Mei) else np.abs(got - want).max() <= 2e-7


def check_mei_session(ctx, cam0, cam1, streams=2, ticks=5, predict=True):
    """viwb_tracker_create_camera sessions against FeatureTrackerRef with the same cameras: ids, track counts and row order identical on every
    tick, pixels within the session tolerance (1e-2 px); the downloaded normalised points equal the restated lift of the downloaded pixels.
    Stream 0 is given the true motion as prediction, the last stream one outside the image (the full-pyramid repeat)."""
    stereo = cam1 is not None
    seqs = [pc.camera_sequence(70 + f, W, H, ticks) for f in range(streams)]
    refs = [co.FeatureTrackerRef(cam0, cam1, MAX_CNT, MIN_DIST, True) for _ in range(streams)]
    trk = ctx.tracker(streams, W, H, lib_camera(cam0), lib_camera(cam1) if stereo else None, MAX_CNT, MIN_DIST, True)
    followed = 0
    for t in range(ticks):
        left = np.stack([seqs[f][0][t] for f in range(streams)])
        right = np.stack([seqs[f][1][t] for f in range(streams)]) if stereo else None
        pp = hp = None
        if predict and t >= 2:
            pp, hp = np.zeros((streams, MAX_CNT, 2), f32), np.zeros(streams, np.uint8)
            for f in ([0, streams - 1] if streams > 1 else [0]):
                prev = refs[f].prev_pts
                pred = (prev + (seqs[f][2][t] if f == 0 else f32([W + 37.0, H + 29.0]))).astype(f32)
                pp[f, : len(prev)] = pred; hp[f] = 1
                refs[f].set_prediction(pred)
        trk.track(0.05 * (t + 1), left, right, pp, hp)
        out = trk.download()
        for f in range(streams):
            r = refs[f].track_image(0.05 * (t + 1), seqs[f][0][t], seqs[f][1][t] if stereo else None)
            _compare_tick(t, f, out, r, stereo)
            assert _lift_matches(cam0, out[3][f], int(out[0][f])), (t, f)
            if stereo:
                assert _lift_matches(cam1, out[6][f], int(out[4][f])), (t, f)
            followed += int((r[1] > 1).sum())
    assert followed >= streams * (ticks - 1) * MAX_CNT // 3, followed
    if predict and ticks > 2:
        assert refs[0].stats["predicted"] == ticks - 2
        if streams > 1:
            assert refs[-1].stats["repeated"] == ticks - 2, refs[-1].stats
    trk.close()


def _compare_tick(t, f, out, r, stereo, tol_px=1e-2):
    n_left, ids, cnt, feat, n_right, ids_r, feat_r = out
    rid, rcnt, rpts, run, rvel, rid_r, rpts_r, run_r, rvel_r = r
    n = int(n_left[f])
    assert n == len(rid) and np.array_equal(ids[f, :n], rid) and np.array_equal(cnt[f, :n], rcnt), (t, f, n, len(rid))
    if n:
        assert np.abs(feat[f, :n, 2:4] - rpts).max() <= tol_px, (t, f, np.abs(feat[f, :n, 2:4] - rpts).max())
    if stereo:
        m = int(n_right[f])
        assert m == len(rid_r) and np.array_equal(ids_r[f, :m], rid_r), (t, f, m, len(rid_r))
        if m:
            assert np.abs(feat_r[f, :m, 2:4] - rpts_r).max() <= tol_px


def check_mei_sessions(ctx):
    check_mei_session(ctx, scaled(EUROC_CAM0), scaled(EUROC_CAM1))                             # the EuRoC MEI stereo pair
    check_mei_session(ctx, scaled(MYNT_LEFT), None, streams=2, ticks=4)                        # mono
    check_mei_session(ctx, scaled(EUROC_CAM1), PIN1, streams=1, ticks=4, predict=False)        # an MEI left camera beside a pinhole right one


def check_mei_feedback(ctx):
    """viwb_tracker_feedback on MEI sessions: a session given the prediction through feedback (removeOutliers + setPrediction over
    CataCamera::spaceToPlane on the device) downloads, tick after tick, what a twin session fed the restated setPrediction's pixels through
    predict_pts downloads, bit for bit -- the device's predict_pts are the restatement's, fall-back rows (prev_pts) included -- and both
    agree with the restated tracker.  A static scene then shows the fall-back rows bit-equal to prev_pts."""
    cam0, cam1 = scaled(EUROC_CAM0), scaled(EUROC_CAM1)
    ticks = 5
    seq = pc.camera_sequence(66, W, H, ticks)
    a, b = (ctx.tracker(1, W, H, lib_camera(cam0), lib_camera(cam1), MAX_CNT, MIN_DIST, True) for _ in range(2))
    ref = co.FeatureTrackerRef(cam0, cam1, MAX_CNT, MIN_DIST, True)
    rng = np.random.default_rng(5)
    ob = None
    for t in range(ticks):
        pp = hp = None
        if t >= 2:
            rm = [int(ref.ids[0]), int(ref.ids[5]), 31337]
            rows = np.array([i for i in range(len(ref.ids)) if i % 3 and i not in (0, 5)])
            pts = np.column_stack([co.lift_projective(cam0, ref.prev_pts[rows] + f32(seq[2][t])).astype(np.float64), np.ones(len(rows))])
            pred = {int(ref.ids[i]): p for i, p in zip(rows, pts * rng.uniform(2, 9, (len(rows), 1)))}
            # the host-fed twin: removeOutliers + setPrediction restated on the library's own rows of the last tick
            twin = restated_feedback(cam0, ob[3][0, : ob[0][0], 2:4], ob[1][0, : ob[0][0]], ob[2][0, : ob[0][0]], rm, True, np.array(list(pred.keys()), np.int32),
                                     np.array(list(pred.values())))
            ref.remove_outliers(rm); ref.set_prediction_from_map(pred)
            a.feedback([rm], [(np.array(list(pred.keys()), np.int32), np.array(list(pred.values())))])
            # b removes the same ids through feedback and takes the prediction through predict_pts
            b.feedback([rm], None)
            pp, hp = np.zeros((1, MAX_CNT, 2), f32), np.ones(1, np.uint8)
            pp[0, : len(twin.predict_pts)] = twin.predict_pts
            fallback = np.array([int(i) not in pred for i in twin.ids])
            assert fallback.any() and twin.predict_pts[fallback].tobytes() == twin.prev_pts[fallback].tobytes()
        a.track(0.05 * (t + 1), seq[0][t][None], seq[1][t][None]); oa = [x.copy() for x in a.download()]
        b.track(0.05 * (t + 1), seq[0][t][None], seq[1][t][None], pp, hp); ob = [x.copy() for x in b.download()]
        for x, y in zip(oa, ob):
            assert x.tobytes() == y.tobytes(), t
        _compare_tick(t, 0, oa, ref.track_image(0.05 * (t + 1), seq[0][t], seq[1][t]), True)
    assert ref.stats["predicted"] == ticks - 2
    a.close(); b.close()
    # static scene: a row without a prediction is seeded at prev_pts and stays there, to the bit
    img = pc.camera_sequence(91, W, H, 1)[0][0]
    trk = ctx.tracker(1, W, H, lib_camera(cam0), None, MAX_CNT, MIN_DIST, True)
    trk.track(0.05, img[None])
    n0, ids, _, feat = [x.copy() for x in trk.download()[:4]]
    n = int(n0[0])
    rows = np.arange(0, n, 2)
    pts = np.column_stack([co.lift_projective(cam0, feat[0, rows, 2:4] + f32(0.3)).astype(np.float64), np.ones(len(rows))]) * 4.0
    trk.feedback(None, [(ids[0, rows], pts)])
    trk.track(0.10, img[None])
    out = trk.download()
    before = {int(ids[0, j]): feat[0, j, 2:4].tobytes() for j in range(n) if j % 2}
    kept = sum(1 for j in range(int(out[0][0])) if int(out[1][0, j]) in before and out[3][0, j, 2:4].tobytes() == before[int(out[1][0, j])])
    assert kept >= n // 4, (kept, n)
    trk.close()


def check_mei_closed_loop(ctx, ticks=6, streams=2):
    """The reference's per-frame loop (estimator.cpp:827-870) on MEI sessions: each tick a seeded subset of the returned ids is removed and the
    next frame's points are predicted by viwb_predict_pts from a constant-velocity window state, then handed back by viwb_tracker_feedback,
    where CataCamera::spaceToPlane projects them.  The restated tracker, fed by the restated prediction, must agree on every tick."""
    cam0, cam1 = scaled(EUROC_CAM0), scaled(EUROC_CAM1)
    focal = cam0.gamma1 / (1.0 + cam0.xi)                  # pixels per unit of the normalised plane near the centre
    seqs = [pc.camera_sequence(60 + f, W, H, ticks) for f in range(streams)]
    refs = [co.FeatureTrackerRef(cam0, cam1, MAX_CNT, MIN_DIST, True) for _ in range(streams)]
    trk = ctx.tracker(streams, W, H, lib_camera(cam0), lib_camera(cam1), MAX_CNT, MIN_DIST, True)
    rng = np.random.default_rng(29)
    depth, fc = 6.0, 10
    last_un = [[{}, {}] for _ in range(streams)]
    removed = [set() for _ in range(streams)]
    n_predicted = 0
    for t in range(ticks):
        left, right = np.stack([seqs[f][0][t] for f in range(streams)]), np.stack([seqs[f][1][t] for f in range(streams)])
        trk.track(0.05 * (t + 1), left, right)
        out = trk.download()
        rm, pr_lib, pr_ref = [], [], []
        for f in range(streams):
            r = refs[f].track_image(0.05 * (t + 1), seqs[f][0][t], seqs[f][1][t])
            _compare_tick(t, f, out, r, True)
            n = int(out[0][f])
            assert _lift_matches(cam0, out[3][f], n)
            assert not (set(int(i) for i in out[1][f, :n]) & removed[f]), (t, f)
            rm.append([int(i) for i in rng.choice(out[1][f, :n], max(n // 8, 1), replace=False)])
            removed[f] |= set(rm[-1])
            state = np.zeros(207); state[3 + 7 * np.arange(11) + 3] = 1.0; state[182] = 1.0
            state[7 * fc: 7 * fc + 3] = [-seqs[f][2][t][0] * depth / focal, -seqs[f][2][t][1] * depth / focal, 0.0]
            preds = []
            for which, (ids_now, un_now) in enumerate(((out[1][f, :n], out[3][f, :n, 0:2]), (r[0], r[3]))):
                old = last_un[f][which]
                two = np.array([int(i) in old for i in ids_now], bool)
                start, nobs = np.where(two, fc - 1, fc).astype(np.int32), np.where(two, 2, 1).astype(np.int32)
                pt0 = np.array([list(old[int(i)]) + [1.0] if int(i) in old else [un_now[k][0], un_now[k][1], 1.0] for k, i in enumerate(ids_now)], np.float64).reshape(-1, 3)
                dep = np.full(len(ids_now), depth)
                pts, valid = ctx.predict_pts(state, fc, start, nobs, pt0, dep) if which == 0 else fbo.predict_pts_in_next_frame(state, fc, start, nobs, pt0, dep)
                preds.append({int(i): p for i, p, v in zip(ids_now, pts, valid) if v})
                last_un[f][which] = {int(i): un_now[k].astype(np.float64) for k, i in enumerate(ids_now)}
            assert preds[0].keys() == preds[1].keys()
            pr_lib.append(preds[0] or None); pr_ref.append(preds[1] or None)
            n_predicted += len(preds[0])
        if t + 1 < ticks:
            for f in range(streams):
                refs[f].remove_outliers(rm[f])
                if pr_ref[f] is not None:
                    refs[f].set_prediction_from_map(pr_ref[f])
            trk.feedback(rm, [None if p is None else (np.array(list(p.keys()), np.int32), np.array(list(p.values()))) for p in pr_lib])
    for f in range(streams):
        assert refs[f].stats["predicted"] == ticks - 2, refs[f].stats
    assert n_predicted >= streams * (ticks - 2) * MAX_CNT // 3, n_predicted
    trk.close()


# ------------------------------------------------------------------------------------------------ the pinhole path and the ABI
def check_pinhole_through_camera_entry(ctx):
    """A seeded pinhole session created through viwb_tracker_create_camera downloads, tick after tick, what one created through
    viwb_tracker_create downloads, bit for bit, with the same launches"""
    cam0 = (461.1586 * W / 752, 459.7529 * W / 752, W / 2 - 3.2, H / 2 + 1.7, -0.2847798, 0.08245052, -1.0946e-06, 4.78701e-06)
    seq = pc.camera_sequence(72, W, H, 4)
    a = ctx.tracker(2, W, H, cam0, PIN1, MAX_CNT, MIN_DIST, True)
    b = ctx.tracker(2, W, H, viwb_lib.Camera.pinhole(*cam0), viwb_lib.Camera.pinhole(*PIN1), MAX_CNT, MIN_DIST, True)
    for t in range(4):
        left, right = np.stack([seq[0][t]] * 2), np.stack([seq[1][t]] * 2)
        l0 = ctx.launch_count(); a.track(0.05 * (t + 1), left, right); oa = [x.copy() for x in a.download()]
        l1 = ctx.launch_count(); b.track(0.05 * (t + 1), left, right); ob = [x.copy() for x in b.download()]
        assert l1 - l0 == ctx.launch_count() - l1
        for x, y in zip(oa, ob):
            assert x.tobytes() == y.tobytes(), t
        assert oa[0][0] > 0
    a.close(); b.close()


def check_camera_errors(ctx):
    """An unknown model and a NULL camera are VIWB_ERR_INVALID with a message, on both new entries, and the context stays usable"""
    L, INVALID = ctx.lib, -1
    px = pixel_set(1, 8)
    un = np.zeros((len(px), 2), f32)
    vp = lambda x: x.ctypes.data_as(C.c_void_p)
    bad = viwb_lib.Camera.mei(*EUROC_CAM0); bad.model = 7
    assert L.viwb_undistort_velocity_camera(ctx.h, C.byref(bad), C.c_int(len(px)), vp(px), None, None, C.c_double(0.05), vp(un), None) == INVALID
    assert b"unknown" in L.viwb_last_error(ctx.h)
    assert L.viwb_undistort_velocity_camera(ctx.h, None, C.c_int(len(px)), vp(px), None, None, C.c_double(0.05), vp(un), None) == INVALID
    assert b"NULL" in L.viwb_last_error(ctx.h)
    cfg = viwb_lib.TrackerConfig(MAX_CNT, MIN_DIST, 1, 1)
    h = C.c_void_p()
    good = viwb_lib.Camera.mei(*scaled(EUROC_CAM0))
    for cams in ((viwb_lib.Camera * 2)(good, bad), (viwb_lib.Camera * 2)(bad, good), None):
        assert L.viwb_tracker_create_camera(ctx.h, C.c_int(1), C.c_int(W), C.c_int(H), C.byref(cfg), cams, C.byref(h)) == INVALID and not h.value
        assert (b"unknown" if cams is not None else b"NULL") in L.viwb_last_error(ctx.h)
    un2, _ = ctx.undistort_velocity(viwb_lib.Camera.mei(*EUROC_CAM0), px)
    assert same_floats(un2, co.lift_projective(EUROC_CAM0, px))
    check_mei_session(ctx, scaled(EUROC_CAM1), None, streams=1, ticks=2, predict=False)
