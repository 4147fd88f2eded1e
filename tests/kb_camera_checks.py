"""Checks of the Kannala-Brandt camera model (camodocal::EquidistantCamera) beside the pinhole and MEI ones: the restatement (oracle/vo_kb.c
through oracle/kb_oracle.py) against the reference's compiled EquidistantCamera.cc and its eigen-solver against LAPACK, then
viwb_undistort_velocity_camera, viwb_tracker_create_camera sessions and viwb_tracker_feedback with Kannala-Brandt cameras, parameterised by
the context like camera_checks.py: tests/test_camera_kb.py runs each library check on the emulation build (`not gpu`) and, marked gpu, on
libviwb.so.

The library's floats are the restatement's bit for bit, except that the GPU's sin / cos / acos / atan2 (within 2 ulp; glibc's within 1) may
move a double across a float rounding boundary: such values may differ by one float ulp, and the checks print how many did."""
import ctypes as C

import numpy as np

import camera_checks as cc
import feedback_oracle as fbo
import kb_oracle as ko
import parity_checks as pc
from viwb import lib as viwb_lib

f32 = np.float32

# realistic fisheye calibrations (Kalibr `equidistant` magnitudes): a 752 x 480 global-shutter camera and an 848 x 800 fisheye pair
KB_752 = ko.Kb(-1.2755e-02, 1.1638e-02, -8.9673e-03, 2.1014e-03, 236.41, 236.12, 371.75, 243.5)
KB_848_L = ko.Kb(-5.0261e-03, 4.1237e-02, -3.8435e-02, 6.6239e-03, 285.72, 286.08, 424.25, 399.5)
KB_848_R = ko.Kb(-3.4126e-03, 3.7913e-02, -3.5120e-02, 5.7180e-03, 284.91, 285.37, 427.5, 398.75)
# edge sets
NPOW1 = ko.Kb(0.0, 0.0, 0.0, 0.0, 240.0, 239.5, 376.0, 240.0)                     # npow 1: theta = |p_u|
NPOW7 = ko.Kb(-1.2e-02, 1.1e-02, -9.0e-03, 0.0, 236.4, 236.1, 371.75, 243.5)       # k5 = 0
K2_ZERO = ko.Kb(0.0, 1.1e-02, -9.0e-03, 2.1e-03, 236.4, 236.1, 371.75, 243.5)      # npow 7 with k5 dropped: the reference's quirk
NO_ROOT = ko.Kb(-0.5, 0.0, 0.0, 0.0, 240.0, 240.0, 376.0, 240.0)                  # r(theta) <= 0.544: no non-negative real root beyond ~130 px
CAMERAS = {"kb_752": (KB_752, 752, 480), "kb_848_left": (KB_848_L, 848, 800), "kb_848_right": (KB_848_R, 848, 800), "npow1": (NPOW1, 752, 480),
           "npow7": (NPOW7, 752, 480), "k2_zero": (K2_ZERO, 752, 480), "no_root": (NO_ROOT, 752, 480)}
# refused: the coefficient at npow is 0 (k4 == 0 with k5 != 0; k2 == k4 == k5 == 0 with k3 != 0)
REFUSED = [ko.Kb(-1.2e-02, 1.1e-02, 0.0, 2.1e-03, 236.4, 236.1, 371.75, 243.5), ko.Kb(0.0, 1.1e-02, 0.0, 0.0, 236.4, 236.1, 371.75, 243.5)]

W, H, MAX_CNT, MIN_DIST = cc.W, cc.H, cc.MAX_CNT, cc.MIN_DIST


def scaled(cam, cw=752, ch=480):
    """a cw x ch calibration for the W x H session images"""
    return cam._replace(mu=cam.mu * W / cw, mv=cam.mv * H / ch, u0=cam.u0 * W / cw, v0=cam.v0 * H / ch)


def lib_camera(cam):
    return viwb_lib.Camera.kannala_brandt(*cam) if isinstance(cam, ko.Kb) else cc.lib_camera(cam)


def pixel_set(cam, w, h, seed, n=400):
    """pixels over the whole image and a margin beyond it, the principal point and the image corners"""
    rng = np.random.default_rng(seed)
    pts = np.column_stack([rng.uniform(-40, w + 40, n), rng.uniform(-40, h + 40, n)])
    fixed = [[cam.u0, cam.v0], [0, 0], [w - 1, 0], [0, h - 1], [w - 1, h - 1]]
    return np.concatenate([pts, fixed]).astype(f32)


def space_set(cam, w, h, seed, n=300):
    """camera-frame points: rays of image pixels at several depths, random points around the camera (behind it as well), the optical axis"""
    rng = np.random.default_rng(seed)
    un = ko.lift_projective(cam, pixel_set(cam, w, h, seed, n // 2)).astype(np.float64)
    rays = np.column_stack([un, np.ones(len(un))]) * rng.uniform(0.5, 40.0, (len(un), 1))
    rays = rays[np.isfinite(rays).all(1)]
    return np.concatenate([rays, rng.normal(0, 3.0, (n // 2, 3)), [[0.0, 0.0, 1.0], [0.0, 0.0, -2.0], [0.3, -0.2, -5.0], [1e-3, 0.0, 0.0]]])


def ulp_diff(a, b):
    """per element: 0 where a and b are the same float (NaN where both are NaN), else the distance in float ulps (NaN vs number: huge)"""
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    na, nb = np.isnan(a), np.isnan(b)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)           # monotone integer image of the floats
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    d = np.abs(ia - ib)
    return np.where(na & nb, 0, np.where(na | nb, 1 << 40, d))


def within_one_ulp(got, want, what, report):
    """got == want bit for bit, except rows that differ by one float ulp; their count goes to `report`"""
    d = ulp_diff(got, want).reshape(len(got), -1)
    assert d.max(initial=0) <= 1, (what, int(d.max()))
    report[what] = report.get(what, 0) + int((d.max(1) > 0).sum())


# ------------------------------------------------------------------------------------------------ the restatement against the reference
def check_restatement_vs_reference_code():
    """kb_oracle's lift and projection against EquidistantCamera::liftProjective (through FeatureTracker::undistortedPts) and spaceToPlane
    compiled from the reference (or their stored results): every float identical, NaN / inf in the same places.  The edge sets are reached."""
    import viw_ref_kb as vrk
    seen = {"past_90": 0, "principal_point": 0, "fallback": 0}
    for k, (name, (cam, w, h)) in enumerate(CAMERAS.items()):
        px = pixel_set(cam, w, h, 10 + k)
        mine, theta = ko.lift_projective_kb(cam, px, want_theta=True)
        assert cc.same_floats(mine, vrk.camera_kb_undistorted_pts(cam, w, h, px)), name
        P = space_set(cam, w, h, 30 + k)
        assert cc.same_floats(ko.space_to_plane(cam, P), vrk.camera_kb_space_to_plane(cam, w, h, P)), name
        seen["past_90"] += int((theta > np.pi / 2).sum())
        mx = (px[:, 0].astype(np.float64) - cam.u0) / cam.mu
        my = (px[:, 1].astype(np.float64) - cam.v0) / cam.mv
        seen["principal_point"] += int((np.hypot(mx, my) < 1e-10).sum())
        if name == "no_root":
            norm = np.hypot(mx, my)                          # theta = |p_u| beyond the maximum 0.544 of r(theta)
            far = norm > 0.6
            assert np.allclose(theta[far], norm[far], rtol=1e-12, atol=0), name
            seen["fallback"] += int(far.sum())
    assert seen["past_90"] > 20 and seen["principal_point"] >= len(CAMERAS) and seen["fallback"] > 50, seen


def check_eigenvalues_vs_lapack():
    """The restated EigenSolver against LAPACK's (numpy.linalg.eigvals) on the companion matrices of every set over a range of |p_u|: every
    eigenvalue that is simple and separated from the others by at least 1e-3 agrees to 1e-12 of max(1, |lambda|)"""
    checked = 0
    for name, (cam, w, h) in CAMERAS.items():
        if ko.npow(cam) == 1:
            continue
        for norm in np.concatenate([[0.0, 1e-12, 1e-6], np.linspace(0.01, 3.5, 40)]):
            A = ko.companion(cam, norm)
            mine, status = ko.eigenvalues(A)
            assert status == 0, (name, norm)
            lap = np.linalg.eigvals(A)
            for lam in mine:
                others = np.sort(np.abs(mine - lam))[1] if len(mine) > 1 else np.inf
                if others < 1e-3:
                    continue
                assert np.abs(lap - lam).min() <= 1e-12 * max(1.0, abs(lam)), (name, norm, lam, lap)
                checked += 1
    assert checked > 1000, checked


# ------------------------------------------------------------------------------------------------ viwb_undistort_velocity_camera
def check_undistort_velocity_camera(ctx):
    """un_pts equal the restatement (and the reference's code or its stored results) under the one-ulp bar; velocities are the rounding of
    the library's own points, bit for bit"""
    import viw_ref_kb as vrk
    rng = np.random.default_rng(6)
    dt = 0.05
    report = {}
    for k, (name, (cam, w, h)) in enumerate(CAMERAS.items()):
        px = pixel_set(cam, w, h, 10 + k)
        n = len(px)
        want = ko.lift_projective(cam, px)
        prev = (np.nan_to_num(want) + rng.normal(0, 0.01, (n, 2))).astype(f32)
        has = (rng.uniform(size=n) < 0.8).astype(np.uint8)
        un, vel = ctx.undistort_velocity(lib_camera(cam), px, prev, has, dt)
        within_one_ulp(un, want, "undistort", report)
        if vrk.available():
            within_one_ulp(un, vrk.camera_kb_undistorted_pts(cam, w, h, px), "undistort vs reference code", report)
        with np.errstate(all="ignore"):
            own = np.where(has[:, None] > 0, ((un - prev).astype(np.float64) / dt).astype(f32), f32(0))
        assert cc.same_floats(vel, own), name
        un2, vel2 = ctx.undistort_velocity(lib_camera(cam), px, None, None, dt)
        assert un2.tobytes() == un.tobytes() and not vel2.any()
    print("Kannala-Brandt undistort rows one float ulp from the restatement:", report)


# ------------------------------------------------------------------------------------------------ sessions
def _lift_within(cam, feat, n, report):
    if n == 0:
        return
    got, want = feat[:n, 0:2], ko.lift_projective(cam, feat[:n, 2:4])
    if isinstance(cam, ko.Kb):
        within_one_ulp(got, want, "session lift", report)
    else:
        assert cc._lift_matches(cam, feat, n)


def check_kb_session(ctx, cam0, cam1, streams=2, ticks=5, predict=True, report=None):
    """viwb_tracker_create_camera sessions against the restated tracker with the same cameras: ids, track counts and row order identical on
    every tick, pixels within 1e-2 px; the downloaded normalised points equal the restated lift of the downloaded pixels (one-ulp bar).
    Stream 0 is given the true motion as prediction, the last stream one outside the image (the full-pyramid repeat)."""
    report = {} if report is None else report
    stereo = cam1 is not None
    seqs = [pc.camera_sequence(70 + f, W, H, ticks) for f in range(streams)]
    refs = [ko.FeatureTrackerRef(cam0, cam1, MAX_CNT, MIN_DIST, True) for _ in range(streams)]
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
            cc._compare_tick(t, f, out, r, stereo)
            _lift_within(cam0, out[3][f], int(out[0][f]), report)
            if stereo:
                _lift_within(cam1, out[6][f], int(out[4][f]), report)
            followed += int((r[1] > 1).sum())
    assert followed >= streams * (ticks - 1) * MAX_CNT // 3, followed
    if predict and ticks > 2:
        assert refs[0].stats["predicted"] == ticks - 2
        if streams > 1:
            assert refs[-1].stats["repeated"] == ticks - 2, refs[-1].stats
    trk.close()
    return report


def check_kb_sessions(ctx):
    report = {}
    check_kb_session(ctx, scaled(KB_848_L, 848, 800), scaled(KB_848_R, 848, 800), report=report)          # a fisheye stereo pair
    check_kb_session(ctx, scaled(KB_752), None, streams=2, ticks=4, report=report)                         # mono
    check_kb_session(ctx, scaled(KB_752), cc.PIN1, streams=1, ticks=4, predict=False, report=report)       # Kannala-Brandt left, pinhole right
    check_kb_session(ctx, scaled(K2_ZERO), scaled(NPOW7), streams=1, ticks=3, predict=False, report=report)   # the degree-7 polynomials
    print("Kannala-Brandt session rows one float ulp from the restated lift:", report)


def _restated_feedback(cam, prev, ids, cnt, remove, has_prediction, pid, pts_cam):
    r = ko.FeatureTrackerRef(cam, None, MAX_CNT, MIN_DIST)
    r.prev_pts, r.ids, r.track_cnt = np.array(prev, f32), [int(i) for i in ids], [int(c) for c in cnt]
    r.remove_outliers(remove)
    if has_prediction:
        r.set_prediction_from_map({int(i): p for i, p in zip(pid, pts_cam)})
    return r


def check_kb_feedback(ctx):
    """viwb_tracker_feedback on Kannala-Brandt sessions: a session given the prediction through feedback (removeOutliers + setPrediction over
    EquidistantCamera::spaceToPlane on the device) downloads, tick after tick, what a twin session fed the restated setPrediction's pixels
    through predict_pts downloads, bit for bit, and both agree with the restated tracker"""
    cam0, cam1 = scaled(KB_848_L, 848, 800), scaled(KB_848_R, 848, 800)
    ticks = 5
    seq = pc.camera_sequence(66, W, H, ticks)
    a, b = (ctx.tracker(1, W, H, lib_camera(cam0), lib_camera(cam1), MAX_CNT, MIN_DIST, True) for _ in range(2))
    ref = ko.FeatureTrackerRef(cam0, cam1, MAX_CNT, MIN_DIST, True)
    rng = np.random.default_rng(5)
    ob = None
    for t in range(ticks):
        pp = hp = None
        if t >= 2:
            rm = [int(ref.ids[0]), int(ref.ids[5]), 31337]
            rows = np.array([i for i in range(len(ref.ids)) if i % 3 and i not in (0, 5)])
            pts = np.column_stack([ko.lift_projective(cam0, ref.prev_pts[rows] + f32(seq[2][t])).astype(np.float64), np.ones(len(rows))])
            pred = {int(ref.ids[i]): p for i, p in zip(rows, pts * rng.uniform(2, 9, (len(rows), 1)))}
            twin = _restated_feedback(cam0, ob[3][0, : ob[0][0], 2:4], ob[1][0, : ob[0][0]], ob[2][0, : ob[0][0]], rm, True,
                                      np.array(list(pred.keys()), np.int32), np.array(list(pred.values())))
            ref.remove_outliers(rm); ref.set_prediction_from_map(pred)
            a.feedback([rm], [(np.array(list(pred.keys()), np.int32), np.array(list(pred.values())))])
            b.feedback([rm], None)
            pp, hp = np.zeros((1, MAX_CNT, 2), f32), np.ones(1, np.uint8)
            pp[0, : len(twin.predict_pts)] = twin.predict_pts
        a.track(0.05 * (t + 1), seq[0][t][None], seq[1][t][None]); oa = [x.copy() for x in a.download()]
        b.track(0.05 * (t + 1), seq[0][t][None], seq[1][t][None], pp, hp); ob = [x.copy() for x in b.download()]
        for x, y in zip(oa, ob):
            assert x.tobytes() == y.tobytes(), t
        cc._compare_tick(t, 0, oa, ref.track_image(0.05 * (t + 1), seq[0][t], seq[1][t]), True)
    assert ref.stats["predicted"] == ticks - 2
    a.close(); b.close()


def check_kb_closed_loop(ctx, ticks=6, streams=2):
    """The reference's per-frame loop (estimator.cpp:827-870) on Kannala-Brandt sessions: each tick a seeded subset of the returned ids is
    removed and the next frame's points are predicted by viwb_predict_pts from a constant-velocity window state, then handed back by
    viwb_tracker_feedback, where EquidistantCamera::spaceToPlane projects them.  The restated tracker, fed by the restated prediction, must
    agree on every tick."""
    cam0, cam1 = scaled(KB_848_L, 848, 800), scaled(KB_848_R, 848, 800)
    focal = cam0.mu                                         # pixels per radian near the centre
    seqs = [pc.camera_sequence(60 + f, W, H, ticks) for f in range(streams)]
    refs = [ko.FeatureTrackerRef(cam0, cam1, MAX_CNT, MIN_DIST, True) for _ in range(streams)]
    trk = ctx.tracker(streams, W, H, lib_camera(cam0), lib_camera(cam1), MAX_CNT, MIN_DIST, True)
    rng = np.random.default_rng(29)
    depth, fc = 6.0, 10
    last_un = [[{}, {}] for _ in range(streams)]
    n_predicted = 0
    for t in range(ticks):
        left, right = np.stack([seqs[f][0][t] for f in range(streams)]), np.stack([seqs[f][1][t] for f in range(streams)])
        trk.track(0.05 * (t + 1), left, right)
        out = trk.download()
        rm, pr_lib, pr_ref = [], [], []
        for f in range(streams):
            r = refs[f].track_image(0.05 * (t + 1), seqs[f][0][t], seqs[f][1][t])
            cc._compare_tick(t, f, out, r, True)
            n = int(out[0][f])
            rm.append([int(i) for i in rng.choice(out[1][f, :n], max(n // 8, 1), replace=False)])
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


# ------------------------------------------------------------------------------------------------ the refusal
def check_kb_errors(ctx):
    """The refused parameter sets are VIWB_ERR_INVALID with a message from both entries, no session is made, and the context stays usable"""
    L, INVALID = ctx.lib, -1
    px = pixel_set(KB_752, 752, 480, 1, 8)
    un = np.zeros((len(px), 2), f32)
    vp = lambda x: x.ctypes.data_as(C.c_void_p)
    cfg = viwb_lib.TrackerConfig(MAX_CNT, MIN_DIST, 1, 1)
    good = lib_camera(scaled(KB_752))
    for cam in REFUSED:
        assert ko.refused(cam)
        bad = lib_camera(cam)
        assert L.viwb_undistort_velocity_camera(ctx.h, C.byref(bad), C.c_int(len(px)), vp(px), None, None, C.c_double(0.05), vp(un), None) == INVALID
        assert b"Kannala-Brandt" in L.viwb_last_error(ctx.h)
        for cams in ((viwb_lib.Camera * 2)(good, bad), (viwb_lib.Camera * 2)(bad, good)):
            h = C.c_void_p()
            assert L.viwb_tracker_create_camera(ctx.h, C.c_int(1), C.c_int(W), C.c_int(H), C.byref(cfg), cams, C.byref(h)) == INVALID and not h.value
            assert b"Kannala-Brandt" in L.viwb_last_error(ctx.h)
    assert not any(ko.refused(c) for c, _, _ in CAMERAS.values())
    un2, _ = ctx.undistort_velocity(lib_camera(KB_752), px)
    within_one_ulp(un2, ko.lift_projective(KB_752, px), "after the refusal", {})
    check_kb_session(ctx, scaled(KB_752), None, streams=1, ticks=2, predict=False)
