"""The LK tracker, the detector and the session tracker at the image sizes of the reference's shipped configurations (KITTI odometry / raw,
simulation, KAIST, RealSense) and at the sizes where buildOpticalFlowPyramid gains or loses a level, with a belt of points along every border.

What is new about these sizes: the device row pitch (w + 15) & ~15 differs from the width, TMA tiles overhang a right edge that is not
16-byte aligned (the unit zero-fills those columns), pyrDown has odd-size tails and the detector reads the tracker's resident images with a
stride other than the width.  The bars are tighter than the ones of parity_checks.py: status identical on every point, at most 3 % of the
points both sides track more than 1e-4 px apart and none more than 1e-2 px (float accumulation order alone moves a few points by a few 1e-3 px),
`err` within 1e-2.  On the GPU the TMA staging is also held bit for bit to the reflect-101 staging (VIWB_LK_NO_TMA), which changes only the
bytes that reach shared memory, never the arithmetic."""
import ctypes as C

import numpy as np

import parity_checks as pc
from viwb import synth

# (width, height, levels of buildOpticalFlowPyramid(winSize 21, maxLevel 3) = its return value + 1)
SHIPPED = [(752, 480, 4),            # EuRoC-sized control
           (1241, 376, 4),           # kitti_odom/*, kitti_raw/kitti_10_03: odd width, level 3 has 47 rows
           (1226, 370, 4),           # kitti_raw/cam_09_30: width not a multiple of 16
           (600, 600, 4),            # simulation: width not a multiple of 16, level 3 is 75 x 75
           (1280, 560, 4),           # kaist
           (640, 512, 4)]            # realsense_d435i and others
BOUNDARY = [(300, 84, 2), (300, 85, 3), (320, 168, 3), (320, 169, 4)]      # a level exists only if it is wider and taller than 21 px
GEOMETRIES = SHIPPED + BOUNDARY

TOL_FINE, TOL_SHARE, TOL_MAX, TOL_ERR = 1e-4, 0.03, 1e-2, 1e-2
CALL_SHAPES = ((3, 0), (1, 4), (0, 0))          # (maxLevel, flags) of check_lk: full pyramid, OPTFLOW_USE_INITIAL_FLOW at maxLevel 1, no pyramid
BELT_DIST = sorted({d * 2 ** L for d in (0.3, 1, 1.5, 3, 6, 9.5, 10.5, 11.5, 13, 17, 23, 29, 37, 45, 53) for L in range(4)})
FRACS = (0.0, 0.25, 0.5, 0.75)


def pyramid_levels(w, h):
    import cv2
    n, _ = cv2.buildOpticalFlowPyramid(np.zeros((h, w), np.uint8), (21, 21), 3)
    return n + 1


def border_belt(w, h, per_edge=64):
    """Points at the BELT_DIST distances (every level's scale of the window radius and beyond) from each of the four edges.  Along an edge the
    other coordinate takes all 16 residues mod 16 with fractional parts 0, .25, .5, .75 (per_edge >= 64), so that the 16-byte aligned tile
    origins (ipx - 1) & ~15 and (inx - 4) & ~15 go through every offset, right edges that are not 16-aligned included."""
    out = []
    for edge in range(4):                          # left, right, top, bottom
        across, along = (w, h) if edge < 2 else (h, w)
        dists = [d for d in BELT_DIST if d <= across - 1]
        blocks = max(1, (along - 16) // 16)
        for i in range(per_edge):
            d = dists[i % len(dists)]
            r, frac = i % 16, FRACS[(i // 16) % 4]
            a = 16 * ((i * 11) % blocks) + r + frac
            c = d if edge % 2 == 0 else across - 1 - d
            out.append((c, a) if edge < 2 else (a, c))
    return np.array(out, np.float32)


def lk_points(w, h, seed=0):
    """lk_images' pair (a blurred texture and its affine warp, ~3 px shift plus 1 % scale) and its goodFeaturesToTrack corners plus the belt"""
    img0, img1, pts = pc.lk_images(seed, w, h)
    return img0, img1, np.vstack([pts, border_belt(w, h)]).astype(np.float32)


def same_bits(x, y):
    x, y = np.asarray(x), np.asarray(y)
    return x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()


def agreement(tag, st_ref, st, p_ref, p, err_ref=None, err=None, min_both=40):
    """the section's bars; returns the numbers the assertion is made on"""
    st_ref, st = np.asarray(st_ref).reshape(-1).astype(np.uint8), np.asarray(st).reshape(-1).astype(np.uint8)
    p_ref, p = np.asarray(p_ref, np.float32).reshape(-1, 2), np.asarray(p, np.float32).reshape(-1, 2)
    both = (st_ref == 1) & (st == 1)
    d = np.abs(p_ref[both].astype(np.float64) - p[both]).max(axis=1) if both.any() else np.zeros(0)
    row = {"case": tag, "points": len(st), "both": int(both.sum()), "status_mismatch": int((st_ref != st).sum()),
           "max_dpos": float(d.max()) if len(d) else 0.0, "beyond_1e-4": int((d > TOL_FINE).sum()),
           "share_beyond": float((d > TOL_FINE).mean()) if len(d) else 0.0}
    if err is not None:
        e = np.abs(np.asarray(err_ref).reshape(-1)[both].astype(np.float64) - np.asarray(err).reshape(-1)[both])      # (err is undefined where status is 0)
        row["max_derr"] = float(e.max()) if len(e) else 0.0
    print("LK", row)
    assert row["status_mismatch"] == 0, row
    assert row["both"] >= min_both, row
    assert row["max_dpos"] <= TOL_MAX and row["share_beyond"] <= TOL_SHARE, row
    assert row.get("max_derr", 0.0) <= TOL_ERR, row
    return row


# ------------------------------------------------------------------------------------------------ raw C entry points (strided images)
def _vp(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def lk_track_raw(ctx, a, b, pts, init=None, max_level=3, flags=0):
    """viwb_lk_track on two uint8 views with strides[1] == 1 and the row stride of the view (Context.lk_track makes them contiguous)"""
    assert a.dtype == np.uint8 and a.strides[1] == 1 and a.strides == b.strides and a.shape == b.shape
    h, w = a.shape
    p0 = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    p1 = np.array(init if init is not None else p0, np.float32, copy=True).reshape(-1, 2)
    st, err = np.zeros(len(p0), np.uint8), np.zeros(len(p0), np.float32)
    ctx._ck(ctx.lib.viwb_lk_track(ctx.h, _vp(a), _vp(b), C.c_int(w), C.c_int(h), C.c_int(a.strides[0]), _vp(p0), _vp(p1), C.c_int(len(p0)), C.c_int(21),
                                  C.c_int(max_level), C.c_int(30), C.c_float(0.01), C.c_int(flags), C.c_float(1e-4), _vp(st), _vp(err)), "viwb_lk_track")
    return p1, st, err


def track_checked_raw(ctx, a, b, pts, mode, flow_back):
    assert a.dtype == np.uint8 and a.strides[1] == 1 and a.strides == b.strides and a.shape == b.shape
    h, w = a.shape
    p0 = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    p1, st = np.zeros_like(p0), np.zeros(len(p0), np.uint8)
    ctx._ck(ctx.lib.viwb_track_checked(ctx.h, _vp(a), _vp(b), C.c_int(w), C.c_int(h), C.c_int(a.strides[0]), _vp(p0), _vp(p1), C.c_int(len(p0)), C.c_int(mode),
                                       C.c_int(1 if flow_back else 0), _vp(st)), "viwb_track_checked")
    return p1, st


def layouts(imgs, seed):
    """uint8 [F, h, w] -> {layout: view of the same pixels}: tight (stride w); the device pitch (w + 15) & ~15 with the streams exactly
    pitch * h apart (one strided copy for all of them); stride w + 7 as a region of a wider buffer.  Padding bytes are random, so a
    kernel that took pitch padding for pixels would change its result."""
    F, h, w = imgs.shape
    rng = np.random.default_rng(seed)
    pitch = (w + 15) & ~15
    out = {"tight": np.ascontiguousarray(imgs)}
    buf = rng.integers(0, 256, (F, h, pitch), dtype=np.uint8)
    buf[:, :, :w] = imgs
    out["pitch"] = buf[:, :, :w]
    wide = rng.integers(0, 256, (F, h + 2, w + 7), dtype=np.uint8)
    wide[:, 1:h + 1, 3:w + 3] = imgs
    out["roi"] = wide[:, 1:h + 1, 3:w + 3]
    assert out["pitch"].strides[1] == pitch and out["roi"].strides[1] == w + 7
    return out


# ------------------------------------------------------------------------------------------------ 2. LK against OpenCV
def check_lk_vs_opencv(ctx, w, h, levels, label, seed=0):
    import cv2
    assert pyramid_levels(w, h) == levels, (w, h, pyramid_levels(w, h), levels)          # the table above cannot drift from OpenCV
    img0, img1, pts = lk_points(w, h, seed)
    crit = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 30, 0.01)
    rows = []
    for ml, flags in CALL_SHAPES:
        init = (pts + np.float32([2.0, -1.5])) if flags else None
        p_cv, st_cv, err_cv = cv2.calcOpticalFlowPyrLK(img0, img1, pts.reshape(-1, 1, 2), None if init is None else init.reshape(-1, 1, 2).copy(),
                                                       winSize=(21, 21), maxLevel=ml, criteria=crit, flags=flags)
        p_g, st_g, err_g = ctx.lk_track(img0, img1, pts, init, max_level=ml, flags=flags)
        rows.append(agreement("%s %dx%d lk_track(maxLevel %d, flags %d)" % (label, w, h, ml, flags), st_cv, st_g, p_cv, p_g, err_cv, err_g))
    return rows


def check_track_checked_vs_reference(ctx, w, h, label, seed=1):
    img0, img1, pts = lk_points(w, h, seed)
    rows = []
    for mode in (0, 1):
        for fb in (True, False):
            p_ref, st_ref = pc.ref_track_checked(img0, img1, pts, mode, fb)
            p_g, st_g = ctx.track_checked(img0, img1, pts, mode=mode, flow_back=fb)
            rows.append(agreement("%s %dx%d track_checked(mode %d, flow_back %d)" % (label, w, h, mode, fb), st_ref, st_g, p_ref, p_g))
    return rows


def batch_inputs(w, h, streams=2, seed=10):
    """two ticks of `streams` stereo streams (lk_images pairs with the belt, 4 px disparity, a second tick shifted by (2, -3) px), ragged counts"""
    ims = [lk_points(w, h, seed + s) for s in range(streams)]
    maxn = max(len(i[2]) for i in ims)
    img0 = np.stack([i[0] for i in ims]); img1 = np.stack([i[1] for i in ims])
    right = np.stack([np.ascontiguousarray(np.roll(i[1], -4, axis=1)) for i in ims])
    img2 = np.stack([np.ascontiguousarray(np.roll(np.roll(i[1], 2, axis=0), -3, axis=1)) for i in ims])
    right2 = np.stack([np.ascontiguousarray(np.roll(i, -4, axis=1)) for i in img2])
    pts = np.zeros((streams, maxn, 2), np.float32); n = np.zeros(streams, np.int32)
    for s in range(streams):
        p = ims[s][2][: len(ims[s][2]) - 9 * s]            # ragged counts
        n[s] = len(p); pts[s, : n[s]] = p
    return maxn, (img0, img1, right, img2, right2), pts, n


def run_lk_batch(ctx, w, h, maxn, images, pts, n, streams=2):
    """-> [(cur_pts, status, right_pts, status_right) of tick 1, of tick 2]; tick 2 tracks tick 1's output points from the resident image"""
    img0, img1, right, img2, right2 = images
    lb = ctx.lk_batch(streams, w, h, maxn, stereo=True, flow_back=True)
    try:
        lb.upload(prev=img0, cur=img1, right=right, prev_pts=pts, n_prev=n, stereo_pts=pts, n_stereo=n)
        lb.run()
        t1 = [a.copy() for a in lb.download()]
        lb.upload(cur=img2, right=right2, prev_pts=t1[0], n_prev=n, stereo_pts=t1[0], n_stereo=n)
        lb.run()
        t2 = [a.copy() for a in lb.download()]
    finally:
        lb.close()
    return [t1, t2]


def check_lk_batch_vs_reference(ctx, w, h, label):
    streams = 2
    maxn, images, pts, n = batch_inputs(w, h, streams)
    img0, img1, right, img2, right2 = images
    got = run_lk_batch(ctx, w, h, maxn, images, pts, n, streams)
    rows = []
    for tick, (prev, cur, rgt, p_in) in enumerate([(img0, img1, right, pts), (img1, img2, right2, got[0][0])]):
        cur_pts, st, rp, sr = got[tick]
        for s in range(streams):
            k = int(n[s])
            p_ref, st_ref = pc.ref_track_checked(prev[s], cur[s], p_in[s, :k], 0, True)
            rows.append(agreement("%s %dx%d lk_batch tick %d stream %d temporal" % (label, w, h, tick + 1, s), st_ref, st[s, :k], p_ref, cur_pts[s, :k]))
            q_ref, sq_ref = pc.ref_track_checked(cur[s], rgt[s], p_in[s, :k], 1, True)
            rows.append(agreement("%s %dx%d lk_batch tick %d stream %d stereo" % (label, w, h, tick + 1, s), sq_ref, sr[s, :k], q_ref, rp[s, :k]))
    return rows


# ------------------------------------------------------------------------------------------------ 3. TMA staging against reflect staging (GPU)
def session_cameras(w, h):
    cam0 = (461.1586 * w / 752, 459.7529 * w / 752, w / 2 - 3.2, h / 2 + 1.7, -0.2847798, 0.08245052, -1.0946e-06, 4.78701e-06)
    cam1 = (457.5874 * w / 752, 456.1340 * w / 752, w / 2 + 4.1, h / 2 - 2.6, -0.2836831, 0.07395907, 1.9359e-04, 1.7618e-05)
    return cam0, cam1


def run_tracker_session(ctx, w, h, left_seq, right_seq, motion, ticks, max_cnt, min_dist, streams=2, stereo=True, predict_from=2):
    """a stereo session fed by camera_sequence frames; from tick `predict_from` stream 0 gets its true image motion as a prediction and the
    last stream one outside the image -> every array of download(), cut to the valid rows, per tick"""
    cam0, cam1 = session_cameras(w, h)
    trk = ctx.tracker(streams, w, h, cam0, cam1 if stereo else None, max_cnt, min_dist, True)
    out = []
    try:
        prev = None
        for t in range(ticks):
            left = np.stack([left_seq[f][t] for f in range(streams)])
            right = np.stack([right_seq[f][t] for f in range(streams)]) if stereo else None
            pp = hp = None
            if prev is not None and t >= predict_from:
                pp, hp = np.zeros((streams, max_cnt, 2), np.float32), np.ones(streams, np.uint8)
                for f in range(streams):
                    k = int(prev[0][f])
                    pp[f, :k] = prev[3][f, :k, 2:4] + (motion[f][t] if f == 0 else np.float32([w + 37.0, h + 29.0]))
            trk.track(0.05 * (t + 1), left, right, pp, hp)
            d = [a.copy() for a in trk.download()]
            prev = d
            rows = {}
            for f in range(streams):
                k, m = int(d[0][f]), int(d[4][f]) if stereo else 0
                rows[f] = (k, d[1][f, :k], d[2][f, :k], d[3][f, :k], m, d[5][f, :m] if stereo else None, d[6][f, :m] if stereo else None)
            out.append(rows)
    finally:
        trk.close()
    return out


def staging_outputs(ctx, w, h):
    """every output the TMA path can influence, at one geometry: {name: array}"""
    out = {}
    img0, img1, pts = lk_points(w, h, 2)
    for ml, flags in CALL_SHAPES:
        init = (pts + np.float32([2.0, -1.5])) if flags else None
        for k, a in enumerate(ctx.lk_track(img0, img1, pts, init, max_level=ml, flags=flags)):
            out["lk_track(%d, %d)[%d]" % (ml, flags, k)] = a
    for mode in (0, 1):
        for fb in (True, False):
            for k, a in enumerate(ctx.track_checked(img0, img1, pts, mode=mode, flow_back=fb)):
                out["track_checked(%d, %d)[%d]" % (mode, fb, k)] = a
    maxn, images, bpts, n = batch_inputs(w, h, 2, seed=20)
    for tick, res in enumerate(run_lk_batch(ctx, w, h, maxn, images, bpts, n)):
        for k, a in enumerate(res):
            for s in range(2):
                out["lk_batch tick %d [%d] stream %d" % (tick + 1, k, s)] = a[s, : n[s]]
    seqs = [pc.camera_sequence(80 + f, w, h, 4) for f in range(2)]
    sess = run_tracker_session(ctx, w, h, [s[0] for s in seqs], [s[1] for s in seqs], [s[2] for s in seqs], 4, 150, 20)
    for t, rows in enumerate(sess):
        for f, r in rows.items():
            for k, a in enumerate(r):
                out["tracker tick %d stream %d [%d]" % (t, f, k)] = np.asarray(a)
    return out


def check_tma_matches_reflect(make_ctx, w, h):
    """make_ctx(no_tma) -> a fresh Context whose LK batches are built with (no_tma False) or without TMA staging"""
    res = {}
    for no_tma in (False, True):
        ctx = make_ctx(no_tma)
        try:
            res[no_tma] = staging_outputs(ctx, w, h)
        finally:
            ctx.close()
    a, b = res[False], res[True]
    assert a.keys() == b.keys()
    for key in a:
        x, y = np.asarray(a[key]), np.asarray(b[key])
        assert same_bits(x, y), "%dx%d %s: TMA staging differs from reflect staging (VIWB_LK_NO_TMA); %d of %d values differ" % (
            w, h, key, int((x != y).sum()) if x.shape == y.shape else -1, x.size)
    print("TMA %dx%d: %d output arrays bit-identical with and without TMA staging" % (w, h, len(a)))
    return len(a)


# ------------------------------------------------------------------------------------------------ 4. strides and pitch padding
def check_strides(ctx, w, h, label, ticks=3, max_cnt=120, min_dist=20):
    """tight, device-pitch and w + 7 strides with random padding: viwb_lk_track, viwb_lk_batch_upload / run, viwb_tracker_track and
    viwb_detector_detect give bit-identical results"""
    streams = 2
    img0, img1, pts = lk_points(w, h, 4)
    res = {}
    for name, (v0, v1) in {k: (a[0], a[1]) for k, a in layouts(np.stack([img0, img1]), 1).items()}.items():
        r = {}
        for ml, flags in CALL_SHAPES:
            init = (pts + np.float32([2.0, -1.5])) if flags else None
            r["lk_track(%d, %d)" % (ml, flags)] = lk_track_raw(ctx, v0, v1, pts, init, ml, flags)
        r["track_checked"] = track_checked_raw(ctx, v0, v1, pts, 0, True)
        res[name] = r
    maxn, images, bpts, n = batch_inputs(w, h, streams, seed=30)
    lay = [layouts(im, 40 + i) for i, im in enumerate(images)]
    for name in res:
        got = run_lk_batch(ctx, w, h, maxn, [L[name] for L in lay], bpts, n, streams)
        res[name]["lk_batch"] = [a[s, : n[s]] for t in got for a in t for s in range(streams)]
    seqs = [pc.camera_sequence(90 + f, w, h, ticks) for f in range(streams)]
    left = [layouts(np.stack([seqs[f][0][t] for f in range(streams)]), 50 + t) for t in range(ticks)]
    right = [layouts(np.stack([seqs[f][1][t] for f in range(streams)]), 60 + t) for t in range(ticks)]
    cam0, cam1 = session_cameras(w, h)
    rng = np.random.default_rng(15)
    cap = 192
    dpts, dcnt, dn = np.zeros((streams, cap, 2), np.float32), np.zeros((streams, cap), np.int32), np.array([60, 0], np.int32)
    dpts[0, :60] = np.column_stack([rng.uniform(1, w - 2, 60), rng.uniform(1, h - 2, 60)]); dcnt[0, :60] = rng.integers(1, 15, 60)
    for name in res:
        trk = ctx.tracker(streams, w, h, cam0, cam1, max_cnt, min_dist, True)
        det = ctx.detector(streams, w, h, cap, min_dist)
        out = []
        try:
            for t in range(ticks):
                trk.track(0.05 * (t + 1), left[t][name], right[t][name])
                d = trk.download()
                out += [d[1][f, : d[0][f]].copy() for f in range(streams)] + [d[3][f, : d[0][f]].copy() for f in range(streams)]
                out += [d[6][f, : d[4][f]].copy() for f in range(streams)]
                keep, n_keep, new_pts, n_new, _ = det.detect(left[t][name], dpts, dcnt, dn, max_cnt)
                out += [keep[f, : n_keep[f]].copy() for f in range(streams)] + [new_pts[f, : n_new[f]].copy() for f in range(streams)]
        finally:
            trk.close(); det.close()
        res[name]["tracker + detector"] = out
    for name in ("pitch", "roi"):
        for key, ref in res["tight"].items():
            got = res[name][key]
            assert len(got) == len(ref)
            for i, (x, y) in enumerate(zip(ref, got)):
                assert same_bits(x, y), "%s %dx%d: %s output %d differs between stride %d and %s layout" % (label, w, h, key, i, w, name)


# ------------------------------------------------------------------------------------------------ 5. the detector
DETECTOR_GEOMETRIES = [(1241, 376, 200, 30), (1226, 370, 150, 30), (600, 600, 150, 30), (1280, 560, 150, 30)]


def fisheye_mask(w, h):
    m = np.full((h, w), 255, np.uint8)
    m[:, : w // 5] = 0; m[h - 40:, :] = 128           # only 255 counts as free
    return m


def check_detector_geometry(ctx, w, h, max_cnt, min_dist, label):
    """goodFeaturesToTrack, setMask + goodFeaturesToTrack on host images (a fisheye-style base mask on stream 0) and on the tracker's resident
    images (three ticks, both left slots): identical to feature_oracle, and resident == host"""
    import feature_oracle as fo
    F, cap = 2, 256
    img = synth.texture_image(h, w, 70)
    ref = fo.good_features_to_track(img, max_cnt, 0.01, float(min_dist))
    got = ctx.good_features_to_track(img, max_cnt, 0.01, float(min_dist), capacity=1024)
    assert ref.shape == got.shape and np.array_equal(ref, got), (label, w, h, len(ref), len(got))
    rng = np.random.default_rng(16)
    imgs = np.stack([synth.texture_image(h, w, 71 + f) for f in range(F)])
    pts, cnt, n = np.zeros((F, cap, 2), np.float32), np.zeros((F, cap), np.int32), np.array([90, 20], np.int32)
    for f in range(F):
        pts[f], cnt[f] = pc._tracked_points(rng, w, h, int(n[f]), cap)
    base = np.stack([fisheye_mask(w, h), np.full((h, w), 255, np.uint8)])
    det = ctx.detector(F, w, h, cap, min_dist)
    lb = ctx.lk_batch(F, w, h, cap, stereo=False, flow_back=True)
    try:
        keep, n_keep, new_pts, n_new, mask = det.detect(imgs, pts, cnt, n, max_cnt, base_masks=base, want_mask=True)
        for f in range(F):
            m0, k0, c0 = fo.detect(imgs[f], pts[f, : n[f]], cnt[f, : n[f]], max_cnt, min_dist, base_mask=base[f])
            assert n_keep[f] == len(k0) and np.array_equal(keep[f, : n_keep[f]], k0), (label, f)
            assert np.array_equal(mask[f], m0), (label, f)
            assert n_new[f] == len(c0) and np.array_equal(new_pts[f, : n_new[f]], c0), (label, f, int(n_new[f]), len(c0))
        img1 = np.stack([np.roll(imgs[f], (1, 2), axis=(0, 1)) for f in range(F)])
        for tick, cur in enumerate([img1, imgs, img1]):              # the tracker alternates its two left slots
            lb.upload(prev=imgs if tick == 0 else None, cur=cur, prev_pts=pts, n_prev=n)
            lb.run(); lb.download()
            a = [x.copy() for x in det.detect(None, pts, cnt, n, max_cnt, resident=lb)[:4]]
            b = [x.copy() for x in det.detect(cur, pts, cnt, n, max_cnt)[:4]]
            assert np.array_equal(a[1], b[1]) and np.array_equal(a[3], b[3]), (label, tick)
            for f in range(F):
                _, k0, c0 = fo.detect(cur[f], pts[f, : n[f]], cnt[f, : n[f]], max_cnt, min_dist)
                assert np.array_equal(a[0][f, : a[1][f]], k0) and np.array_equal(a[2][f, : a[3][f]], c0), (label, tick, f)
                assert np.array_equal(b[0][f, : b[1][f]], k0) and np.array_equal(b[2][f, : b[3][f]], c0), (label, tick, f)
    finally:
        det.close(); lb.close()


# ------------------------------------------------------------------------------------------------ 6. sessions against the restated trackImage()
def check_session(ctx, w, h, label, streams, ticks, max_cnt, min_dist, stereo, predict=True):
    """viwb_tracker_track against FeatureTrackerRef (cv2's LK underneath): ids, row order and track counts identical every tick; pixels at the
    LK bars of this file over all rows of the session; undistorted points and velocities within check_tracker_session's bounds"""
    import feature_oracle as fo
    cam0, cam1 = session_cameras(w, h)
    seqs = [pc.camera_sequence(70 + f, w, h, ticks) for f in range(streams)]
    refs = [fo.FeatureTrackerRef(cam0, cam1 if stereo else None, max_cnt, min_dist, True) for _ in range(streams)]
    trk = ctx.tracker(streams, w, h, cam0, cam1 if stereo else None, max_cnt, min_dist, True)
    dt = 0.05
    tol_un = 1.5 * TOL_MAX / cam0[0]
    dl, dr = [], []
    try:
        for t in range(ticks):
            left = np.stack([seqs[f][0][t] for f in range(streams)])
            right = np.stack([seqs[f][1][t] for f in range(streams)]) if stereo else None
            pp = hp = None
            if predict and t >= 2:
                pp, hp = np.zeros((streams, max_cnt, 2), np.float32), np.zeros(streams, np.uint8)
                for f in ([0, streams - 1] if streams > 1 else [0]):
                    prev = refs[f].prev_pts
                    pred = (prev + (seqs[f][2][t] if f == 0 else np.float32([w + 37.0, h + 29.0]))).astype(np.float32)
                    pp[f, : len(prev)] = pred; hp[f] = 1
                    refs[f].set_prediction(pred)
            trk.track(dt * (t + 1), left, right, pp, hp)
            n_left, ids, cnt, feat, n_right, ids_r, feat_r = trk.download()
            for f in range(streams):
                rid, rcnt, rpts, run, rvel, rid_r, rpts_r, run_r, rvel_r = refs[f].track_image(dt * (t + 1), seqs[f][0][t], seqs[f][1][t] if stereo else None)
                n = int(n_left[f])
                assert n == len(rid), (label, t, f, n, len(rid))
                assert np.array_equal(ids[f, :n], rid) and np.array_equal(cnt[f, :n], rcnt), (label, t, f)
                dl.append(np.abs(feat[f, :n, 2:4].astype(np.float64) - rpts).max(axis=1) if n else np.zeros(0))
                assert np.abs(feat[f, :n, 0:2] - run).max(initial=0) <= tol_un and np.abs(feat[f, :n, 4:6] - rvel).max(initial=0) <= 2 * tol_un / dt, (label, t, f)
                if stereo:
                    m = int(n_right[f])
                    assert m == len(rid_r) and np.array_equal(ids_r[f, :m], rid_r), (label, t, f, m, len(rid_r))
                    dr.append(np.abs(feat_r[f, :m, 2:4].astype(np.float64) - rpts_r).max(axis=1) if m else np.zeros(0))
                    assert np.abs(feat_r[f, :m, 0:2] - run_r).max(initial=0) <= tol_un and np.abs(feat_r[f, :m, 4:6] - rvel_r).max(initial=0) <= 2 * tol_un / dt
    finally:
        trk.close()
    rows = []
    for side, ds in (("left", dl), ("right", dr)):
        if not ds:
            continue
        d = np.concatenate(ds)
        row = {"case": "%s %dx%d session %s" % (label, w, h, side), "rows": len(d), "max_dpos": float(d.max()), "beyond_1e-4": int((d > TOL_FINE).sum()),
               "share_beyond": float((d > TOL_FINE).mean())}
        print("SESSION", row)
        assert len(d) >= ticks * max_cnt // 3, row
        assert row["max_dpos"] <= TOL_MAX and row["share_beyond"] <= TOL_SHARE, row
        rows.append(row)
    if predict and ticks > 2:
        assert refs[0].stats["predicted"] == ticks - 2 and refs[0].stats["repeated"] == 0, refs[0].stats
        if streams > 1:
            assert refs[-1].stats["repeated"] == ticks - 2, refs[-1].stats
    return rows
