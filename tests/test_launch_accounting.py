"""viwb_launch_count per entry point.  Every family of calls below launches a fixed number of kernels; the `emu` test pins that number on the
emulation build (tests/emu), so that a change to the host code cannot drop or add a launch unnoticed.  The `gpu` test runs the same calls on
libviwb.so with the profiler on: each family must launch the same number of kernels there, and the profile must report every one of them, i.e.
the sum of the profile's launches equals the launch count, over kernel names that bench.py knows."""
import numpy as np
import pytest

import features_checks as fc
import feedback_checks as fbc
import parity_checks as pc
from viwb import abi, synth
from viwb import lib as viwb_lib

W, H = fbc.W, fbc.H


def _images(seed, ticks, streams):
    """left / right frames of a camera panning over a texture: [tick] -> (left [streams, H, W], right [streams, H, W])"""
    out = []
    for t in range(ticks):
        left = np.stack([np.ascontiguousarray(synth.texture_image(H + 40, W + 40, seed + s)[2 * t: 2 * t + H, 3 * t: 3 * t + W]) for s in range(streams)])
        right = np.stack([np.ascontiguousarray(np.roll(x, -4, axis=1)) for x in left])
        out.append((left, right))
    return out


def factor_evaluate(ctx, ftype):
    prob, st, _ = synth.make_window(4)
    st = st.copy()
    if ftype <= abi.F_PROJ_1F2C:
        f = int(np.flatnonzero(prob.vis_type == ftype)[0])
        fi, fj, lm = prob.vis_frame_i[f], prob.vis_frame_j[f], 32 + prob.vis_landmark[f]
        blocks = {abi.F_PROJ_2F1C: [fi, fj, 22, lm, 30], abi.F_PROJ_2F2C: [fi, fj, 22, 23, lm, 30], abi.F_PROJ_1F2C: [22, 23, lm, 30]}[ftype]
        consts = prob.vis_obs[f]
    elif ftype == abi.F_IMU:
        blocks, consts = [prob.imu_frame_i[0], 11 + prob.imu_frame_i[0], prob.imu_frame_j[0], 11 + prob.imu_frame_j[0]], prob.imu_data[0]
    elif ftype == abi.F_WHEEL:
        blocks, consts = [prob.wheel_frame_i[0], prob.wheel_frame_j[0], 24, 27, 28, 29, 31], prob.wheel_data[0]
    else:
        blocks, consts = [prob.plane_frame[0], 24, 25, 26], None
    params = [pc.block_ptr(st, b) for b in blocks]
    return lambda: ctx.factor_evaluate(ftype, prob.globals, consts, params)


def prior_evaluate(ctx):
    prob, st, _ = synth.make_window(4)
    prior = ctx.marginalize(prob, st, abi.MARGIN_OLD)
    return lambda: ctx.prior_evaluate(prior, st)


def preintegration(ctx, wheel):
    rng = np.random.default_rng(5)
    lens = [10, 1, 7]
    dts = [np.full(k, 0.005) for k in lens]
    a = [rng.normal(0, 1.0, (k + 1, 3)) for k in lens]
    g = [rng.normal(0, 0.5, (k + 1, 3)) for k in lens]
    if wheel:
        return lambda: ctx.wheel_preintegrate(dts, a, g, np.ones((3, 3)), np.zeros(3), np.array([0.01, 0.004]))
    return lambda: ctx.imu_preintegrate(dts, a, g, np.zeros((3, 3)), np.zeros((3, 3)), np.array([0.1, 0.01, 1e-3, 1e-4]))


def alignment(ctx, linear):
    case = pc.alignment_case(1, F=6)
    n = len(case["dts"])
    rec = ctx.imu_preintegrate(case["dts"], case["accs"], case["gyrs"], np.zeros((n, 3)), np.zeros((n, 3)), case["noise"])
    if linear:
        return lambda: ctx.linear_alignment(case["R"], case["T"], rec, None, case["tic"], None, None, case["g_norm"])
    return lambda: ctx.solve_gyroscope_bias(case["R"], rec)


def points(ctx, which):
    rng = np.random.default_rng(9)
    state, frame_count, start, num_obs, pt0, depth = fbc.predict_case(2, 3)
    n = 20
    if which == "triangulate":
        return lambda: ctx.triangulate(state, np.arange(n) % 2, np.arange(n) % 9, rng.normal(0, 0.3, (n, 2)), rng.normal(0, 0.3, (n, 2)))
    if which == "shift_depth":
        uv = np.column_stack([rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), np.ones(n)])
        return lambda: ctx.shift_depth(uv, rng.uniform(1, 9, n), np.eye(3).reshape(9), np.zeros(3), np.eye(3).reshape(9), np.ones(3))
    return lambda: ctx.predict_pts(state, frame_count, start, num_obs, pt0, depth)


def undistort(ctx, model):
    cam = viwb_lib.Camera.pinhole(*fbc.CAM0) if model == "pinhole" else viwb_lib.Camera.mei(2.5, -0.08, 0.006, 2e-4, 1e-4, 190.0, 191.0, 160.0, 120.0)
    pts = np.random.default_rng(2).uniform(10, 200, (40, 2)).astype(np.float32)
    return lambda: ctx.undistort_velocity(cam, pts, pts * 0.001, np.ones(40, np.uint8))


def lk(ctx, which):
    ims = pc.lk_images(1, W, H)
    p = np.ascontiguousarray(ims[2][:50], np.float32)
    if which == "lk_track":
        return lambda: ctx.lk_track(ims[0], ims[1], p)
    if which == "track_checked":
        return lambda: ctx.track_checked(ims[0], ims[1], p, 0, True)
    lb = ctx.lk_batch(2, W, H, 64, stereo=True, flow_back=True)
    pts, n = np.zeros((2, 64, 2), np.float32), np.array([50, 30], np.int32)
    pts[0, :50], pts[1, :30] = p, p[:30]
    imgs = np.stack([ims[0], ims[0]]), np.stack([ims[1], ims[1]])
    lb.upload(prev=imgs[0], cur=imgs[1], right=imgs[1], prev_pts=pts, n_prev=n, stereo_pts=pts, n_stereo=n)
    return lambda: (lb.run(), lb.download())


def detection(ctx, which):
    img = synth.texture_image(H, W, 4)
    rng = np.random.default_rng(11)
    pts, cnt = pc._tracked_points(rng, W, H, 30, 64)
    if which == "set_mask":
        return lambda: ctx.set_mask(W, H, pts[:30], cnt[:30], 20)
    if which == "good_features":
        return lambda: ctx.good_features_to_track(img, 60, 0.01, 20)
    det = ctx.detector(2, W, H, 64, 20)
    return lambda: det.detect(np.stack([img, img]), np.stack([pts, pts]), np.stack([cnt, cnt]), np.array([30, 0], np.int32), 60)


def tracker(ctx, feedback):
    frames = _images(30, 4, 2)
    trk = ctx.tracker(2, W, H, fbc.CAM0, fbc.CAM1, fbc.MAX_CNT, fbc.MIN_DIST, True)
    for t in range(3):                      # a session with tracks
        trk.track(0.05 * (t + 1), *frames[t])
    n_left, ids, *_ = trk.download()
    if not feedback:
        return lambda: (trk.track(0.2, *frames[3]), trk.download())
    pred = [(ids[f, : n_left[f]].copy(), np.tile([0.1, 0.05, 1.0], (int(n_left[f]), 1))) for f in range(2)]

    def run():
        trk.feedback([ids[f, :2].tolist() for f in range(2)], pred)
        trk.track(0.2, *frames[3])
        trk.download()
    return run


def features(ctx):
    sc = fc.Script(2, 3, 14)
    fs = ctx.features(1, 160, True, 10.0 / fc.FOCAL)
    for t in range(10):
        fs.add([t], [0.0], [fc.rows_of(sc.image(t), True)])
    st = np.array([sc.state(10)])

    def run():
        fs.add([10], [0.0], [fc.rows_of(sc.image(10), True)])
        fs.decisions()
        fs.triangulate(st)
        _, inv, _ = fs.window(4000)
        fs.set_depth(inv)
        fs.remove_outliers([np.zeros(len(v), np.uint8) for v in inv])
        fs.predict(st, [10])
        fs.slide([10], [1], *[np.array([m]) for m in fc.cam_mats(sc.state(10))])
        fs.remove_failures()
        fs.download()
    return run


def optimization(ctx, cid):
    prob, st, _ = synth.make_window(cid)
    return lambda: ctx.optimization(prob, st, abi.MARGIN_OLD)


def batch_calls(ctx, which):
    prob, st, _ = synth.make_window(2)
    if which == "normal_equations":
        return lambda: ctx.normal_equations(prob, st)
    b = ctx.batch([prob], [st])
    b.run()
    return lambda: b.outliers()


def empty_calls(ctx):
    """every entry point called with n == 0 launches nothing"""
    st = np.zeros(abi.STATE_FIXED)
    z2, zi = np.zeros((0, 2)), np.zeros(0, np.int32)

    def run():
        ctx.triangulate(st, zi, zi, z2, z2)
        ctx.shift_depth(np.zeros((0, 3)), np.zeros(0), np.eye(3).reshape(9), np.zeros(3), np.eye(3).reshape(9), np.zeros(3))
        ctx.predict_pts(st, 5, zi, zi, np.zeros((0, 3)), np.zeros(0))
        ctx.undistort_velocity(fbc.CAM0, np.zeros((0, 2), np.float32))
        ctx.imu_preintegrate([], [], [], np.zeros((0, 3)), np.zeros((0, 3)), np.ones(4))
        ctx.wheel_preintegrate([], [], [], np.zeros((0, 3)), np.zeros(0), np.ones(2))
        ctx.lk_track(np.zeros((H, W), np.uint8), np.zeros((H, W), np.uint8), np.zeros((0, 2), np.float32))
        ctx.track_checked(np.zeros((H, W), np.uint8), np.zeros((H, W), np.uint8), np.zeros((0, 2), np.float32))
    return run


# family -> (setup(ctx) returning the counted call, its launches)
FAMILIES = {
    **{f"factor_evaluate_{t}": ((lambda t: lambda ctx: factor_evaluate(ctx, t))(t), 1) for t in range(6)},
    "prior_evaluate": (prior_evaluate, 1),
    "imu_preintegrate": (lambda ctx: preintegration(ctx, False), 1),
    "wheel_preintegrate": (lambda ctx: preintegration(ctx, True), 1),
    "solve_gyroscope_bias": (lambda ctx: alignment(ctx, False), 1),
    "linear_alignment": (lambda ctx: alignment(ctx, True), 1),
    "triangulate": (lambda ctx: points(ctx, "triangulate"), 1),
    "shift_depth": (lambda ctx: points(ctx, "shift_depth"), 1),
    "predict_pts": (lambda ctx: points(ctx, "predict_pts"), 1),
    "undistort_pinhole": (lambda ctx: undistort(ctx, "pinhole"), 1),
    "undistort_mei": (lambda ctx: undistort(ctx, "mei"), 1),
    "lk_track": (lambda ctx: lk(ctx, "lk_track"), 7),
    "track_checked": (lambda ctx: lk(ctx, "track_checked"), 9),
    "lk_batch": (lambda ctx: lk(ctx, "lk_batch"), 12),
    "set_mask": (lambda ctx: detection(ctx, "set_mask"), 2),
    "good_features_to_track": (lambda ctx: detection(ctx, "good_features"), 2),
    "detector_tick": (lambda ctx: detection(ctx, "detector"), 4),
    "tracker_tick": (lambda ctx: tracker(ctx, False), 19),
    "tracker_tick_feedback": (lambda ctx: tracker(ctx, True), 23),
    "features_round": (features, 12),
    "optimization_c2": (lambda ctx: optimization(ctx, 2), 55),
    "optimization_c4": (lambda ctx: optimization(ctx, 4), 63),
    "batch_outliers": (lambda ctx: batch_calls(ctx, "outliers"), 1),
    "debug_normal_equations": (lambda ctx: batch_calls(ctx, "normal_equations"), 7),
    "empty_calls": (empty_calls, 0),
}


def launches(ctx, setup):
    call = setup(ctx)
    n0 = ctx.launch_count()
    call()
    return ctx.launch_count() - n0


@pytest.fixture(scope="module")
def emu_ctx():
    from emu import build_emu
    ctx = viwb_lib.Context(0, build_emu.build())
    yield ctx
    ctx.close()


@pytest.mark.parametrize("family", list(FAMILIES))
def test_launch_count(emu_ctx, family):
    setup, want = FAMILIES[family]
    assert launches(emu_ctx, setup) == want


# the kernels the families above launch, under the names the profiler reports (bench.py keys its models on them)
PROFILE_NAMES = {
    "eval_factor", "prior_eval", "imu_preint", "wheel_preint", "gyro_bias", "align", "triangulate", "shift_depth", "predict_pts", "undistort",
    "lk_pyr_down", "lk_track", "lk_post", "det_order", "det_mask", "det_corners", "det_select",
    "trk_pred_setup", "trk_pred_check", "trk_advance", "trk_merge", "trk_stereo", "trk_feedback",
    "fm_add_check", "fm_add_apply", "fm_triangulate", "fm_window_count", "fm_window_write", "fm_set_depth", "fm_predict", "fm_compact", "fm_pack",
    "vis_expand", "setup", "lin_vis_lm", "lin_vis_lm_wide", "lin_small", "asm_pairs_wide", "pair_reduce", "syrk_mma", "solve", "reanchor",
    "lin_vis_lm_wide_marg", "lin_small_marg", "asm_pairs_wide_marg", "pair_reduce_marg", "syrk_mma_marg", "marg_prep", "marg_tri", "marg_ql", "marg_apply", "outlier",
}


@pytest.mark.gpu
def test_profile_reports_every_launch(gpu_ctx):
    setups = {family: setup(gpu_ctx) for family, (setup, _) in FAMILIES.items()}
    gpu_ctx.set_profiling(True)
    try:
        total = 0
        for family, call in setups.items():
            n0 = gpu_ctx.launch_count()
            call()
            got = gpu_ctx.launch_count() - n0
            assert got == FAMILIES[family][1], family
            total += got
        prof = gpu_ctx.profile()
    finally:
        gpu_ctx.set_profiling(False)
    assert sum(n for _, n in prof.values()) == total
    assert set(prof) == PROFILE_NAMES
