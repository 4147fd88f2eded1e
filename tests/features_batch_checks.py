"""Checks of viwb_features_batch_create and the feedback calls that read its batch (viwb_features_set_depth_batch / remove_outliers_batch /
predict_batch), parameterised by the context: tests/test_features_batch.py runs each on the emulation build and, marked gpu, on libviwb.so.
The yardstick is the host chain the new calls replace: viwb_features_window + viwb_batch_create, and set_depth / remove_outliers / predict fed
what viwb_batch_download and viwb_batch_outliers return.  Everything is compared bit for bit."""
import numpy as np

from viwb import abi
from viwb.lib import ViwbError

import features_checks as fc
from test_lowering_paths import paths

FOCAL = fc.FOCAL
CONSTANT_COMMON, FREE_TD = "ex0/ex1/td constant", "td free"


def _imu_tables(sc, k, frame_count, cache):
    """the IMU tables and block layout of the synth window of frames k..k+10 of the script's sequence, cut to the frames up to frame_count"""
    if k not in cache:
        cache[k] = sc.s.window(k, perturb=False)[0]
    p = cache[k]
    keep = (p.imu_frame_i <= frame_count) & (p.imu_frame_j <= frame_count)
    return p, dict(imu_frame_i=p.imu_frame_i[keep], imu_frame_j=p.imu_frame_j[keep], imu_data=p.imu_data[keep])


def _block_flags(p, layout):
    fl = p.block_flags.copy()
    for b in (abi.BLK_EX_POSE0, abi.BLK_EX_POSE1, abi.BLK_TD):
        fl[b] |= abi.BLOCK_PRESENT | abi.BLOCK_CONSTANT
    if layout == FREE_TD:
        fl[abi.BLK_TD] = abi.BLOCK_PRESENT
    return fl


def same_prior(a, b):
    if a.valid != b.valid or a.n != b.n or a.blocks() != b.blocks():
        return False
    n = a.n
    return not a.valid or (a.J[: n * n].tobytes() == b.J[: n * n].tobytes() and a.r[:n].tobytes() == b.r[:n].tobytes() and a.x0.tobytes() == b.x0.tobytes())


def same_lists(fa, fb, what):
    for s, (x, y) in enumerate(zip(fa.download(), fb.download())):
        for k in x:
            assert x[k].tobytes() == y[k].tobytes(), (what, s, k)


def compare_batches(host, dev, what):
    """download (states, summaries, priors), num_landmarks and outliers of a viwb_batch_create batch and a viwb_features_batch_create one"""
    assert dev.num_landmarks == host.num_landmarks, (what, dev.num_landmarks, host.num_landmarks)
    sa, ma, pa = host.download()
    sb, mb, pb = dev.download()
    for w in range(host.B):
        assert sa[w].tobytes() == sb[w].tobytes(), (what, w, "states")
        assert bytes(ma[w]) == bytes(mb[w]), (what, w, "summary")
        assert same_prior(pa[w], pb[w]), (what, w, "prior")
    oa, ob = host.outliers(), dev.outliers()
    assert all(x.tobytes() == y.tobytes() for x, y in zip(oa, ob)), (what, "outliers")
    return sa, pa, oa


# ------------------------------------------------------------------------------------------------ the scripts, twin lists
def run_twins(ctx, cid, ticks=16, min_parallax=10.0 / FOCAL, seed=0, seen=None):
    """Three streams of one script configuration; stream 1 loses every row on some ticks and a third of them on others, stream 2 runs two frames
    behind (other frame_counts).  Twin lists fa / fb take the same adds, triangulations, slides and removeFailures.  At every NON_LINEAR tick fa's
    windows are exported and built by viwb_batch_create, fb's by viwb_features_batch_create, both with the IMU tables of the sequence's synth
    window, the decisions' margin flags and, from the second window of a stream on, the prior its previous window produced; the block layout
    alternates between ex0 / ex1 / td constant and td free.  The batches must agree bit for bit, then fa takes the host chain's feedback and fb
    the batch calls, and the lists, removed ids and predictions must agree bit for bit.  seen collects the (layout, solve path, marginalisation)."""
    script = [fc.Script(cid, seed + s, ticks + 3) for s in range(3)]
    stereo = script[0].cfg.stereo
    F = 3
    fa, fb = (ctx.features(F, 160, stereo, min_parallax, FOCAL) for _ in range(2))
    seen = seen if seen is not None else set()
    caches = [{} for _ in range(F)]
    priors = [None] * F
    nonlin = False
    for t in range(ticks):
        src_t = [t, t, max(0, t - 2)]
        fcs = [min(t, 10), min(t, 10), min(max(0, t - 2), 10)]
        images = []
        for s in range(F):
            drop = ()
            if s == 1 and t % 7 == 5:
                drop = set(tid for tid, _, _ in script[s].rows[t])
            elif s == 1 and t % 7 == 3:
                drop = set(tid for k, (tid, _, _) in enumerate(script[s].rows[t]) if k % 3 == 0)
            images.append(script[s].image(src_t[s], drop) if (s < 2 or t >= 2) else {})
        td = [0.001 * t, -0.002 * t, 0.0]
        rows = [fc.rows_of(im, stereo) for im in images]
        for fs in (fa, fb):
            fs.add(fcs, td, rows)
        da, db = fa.decisions(), fb.decisions()
        assert all(da[k].tobytes() == db[k].tobytes() for k in da), t
        states = np.array([script[s].state(src_t[s]) for s in range(F)])
        if nonlin:
            for fs in (fa, fb):
                fs.triangulate(states)
            same_lists(fa, fb, ("triangulate", t))
            layout = CONSTANT_COMMON if t % 2 == 0 else FREE_TD
            tabs, inv, _ = fa.window(4000)
            flags = [int(x) for x in da["margin_flag"]]
            host_probs, bare_probs = [], []
            for s in range(F):
                k = max(0, min(src_t[s] - 10, script[s].frames - 11))
                p, imu = _imu_tables(script[s], k, fcs[s], caches[s])
                common = dict(block_flags=_block_flags(p, layout), subset_mask=p.subset_mask, prior=priors[s], globals_=p.globals, **imu)
                host_probs.append(abi.WindowProblem(fcs[s], tabs[s]["num_landmarks"], vis_type=tabs[s]["vis_type"], vis_landmark=tabs[s]["vis_landmark"],
                                                    vis_frame_i=tabs[s]["vis_frame_i"], vis_frame_j=tabs[s]["vis_frame_j"], vis_obs=tabs[s]["vis_obs"], **common))
                bare_probs.append(abi.WindowProblem(fcs[s], 0, **common))
                sol, marg = paths(host_probs[s], flags[s])
                if flags[s] == abi.MARGIN_SECOND_NEW and fcs[s] == abi.WINDOW_SIZE and priors[s] is not None and priors[s].valid and \
                        abi.WINDOW_SIZE - 1 in [b for b, _ in priors[s].blocks()]:
                    marg = "second_new"
                seen.add((layout, sol, marg))
            host = ctx.batch(host_probs, [np.concatenate([states[s], inv[s]]) for s in range(F)], flags)
            dev = fb.batch(bare_probs, states, flags)
            for b in (host, dev):
                b.run()
            solved, pri, verdicts = compare_batches(host, dev, ("batch", t))
            priors = [pri[s] if pri[s].valid else None for s in range(F)]
            # feedback: the host chain on fa, the batch calls on fb
            fa.set_depth([x[abi.STATE_FIXED:] for x in solved])
            fb.set_depth_from(dev)
            same_lists(fa, fb, ("set_depth", t))
            ra, rb = fa.remove_outliers(verdicts), fb.remove_outliers_from(dev)
            assert all(np.array_equal(x, y) for x, y in zip(ra, rb)), t
            same_lists(fa, fb, ("remove_outliers", t))
            pa = fa.predict(np.array([x[:abi.STATE_FIXED] for x in solved]), fcs)
            pb = fb.predict_from(dev, fcs)
            for x, y in zip(pa, pb):
                assert (x is None) == (y is None) and (x is None or (x[0].tobytes() == y[0].tobytes() and x[1].tobytes() == y[1].tobytes())), t
            states = np.array([x[:abi.STATE_FIXED] for x in solved])
            host.destroy(); dev.destroy()
        mats = [fc.cam_mats(states[s]) for s in range(F)]
        for fs in (fa, fb):
            fs.slide(fcs, [1 if nonlin else 0] * F, *[np.array([m[i] for m in mats]) for i in range(4)])
            if nonlin:
                fs.remove_failures()
        same_lists(fa, fb, ("tick", t))
        nonlin = nonlin or fcs[0] == 10
    fa.close(); fb.close()
    return seen


def check_scripts(ctx, ticks=16):
    """mono config 1 and stereo configs 2 and 4 (4 at a parallax threshold that only a tick without rows passes, so that MARGIN_SECOND_NEW windows
    with a prior follow MARGIN_OLD ones); both solve paths, both block layouts, the wide marginalisation and MARGIN_SECOND_NEW must occur"""
    seen = set()
    run_twins(ctx, 1, ticks, 10.0 / FOCAL, 0, seen)
    run_twins(ctx, 2, ticks, 10.0 / FOCAL, 10, seen)
    run_twins(ctx, 4, ticks, 1.0, 20, seen)
    sol = {s for _, s, _ in seen}
    marg = {m for _, _, m in seen}
    assert {"compact", "wide"} <= sol and {"wide", "second_new"} <= marg and {l for l, _, _ in seen} == {CONSTANT_COMMON, FREE_TD}, seen
    assert ("ex0/ex1/td constant", "compact") in {(l, s) for l, s, _ in seen} and ("td free", "wide") in {(l, s) for l, s, _ in seen}, seen
    return seen


# ------------------------------------------------------------------------------------------------ closed loop with the tracker
def check_closed_loop(ctx, ticks=16, streams=2):
    """check_closed_loop of features_checks.py twice, on twin trackers and lists: twin a through the host chain (window, viwb_batch_create, download,
    outliers, set_depth, remove_outliers, predict), twin b through viwb_features_batch_create and the batch calls.  On every tick the trackers'
    rows, the lists, decisions, solved states, removed ids and predictions are bit-identical, so viwb_tracker_feedback gets the same arguments."""
    import feedback_checks as fbc
    import parity_checks as pc
    from viwb import synth
    W, H, MAX_CNT = fbc.W, fbc.H, fbc.MAX_CNT
    seqs = [pc.camera_sequence(70 + f, W, H, ticks) for f in range(streams)]
    trk = [ctx.tracker(streams, W, H, fbc.CAM0, fbc.CAM1, MAX_CNT, fbc.MIN_DIST, True) for _ in range(2)]
    fs = [ctx.features(streams, MAX_CNT, True, 10.0 / FOCAL, FOCAL) for _ in range(2)]
    prob2, _, gt2 = synth.make_window(2, 0)
    states = np.array([gt2[:abi.STATE_FIXED]] * streams)
    nonlin, n_pred, n_removed = False, 0, 0
    fc0 = max(0, 14 - ticks)
    for t in range(ticks):
        fcnt = min(t + fc0, 10)
        left, right = np.stack([seqs[f][0][t] for f in range(streams)]), np.stack([seqs[f][1][t] for f in range(streams)])
        outs = []
        for k in range(2):
            trk[k].track(0.05 * (t + 1), left, right)
            outs.append([x.copy() for x in trk[k].download()])
            fs[k].add_tracked(trk[k], [fcnt] * streams, [0.0] * streams)
        for f in range(streams):                            # the rows each session hands over (entries past the counts are undefined)
            ia, ib = fc._tracker_image(outs[0], f, True), fc._tracker_image(outs[1], f, True)
            assert list(ia) == list(ib) and all(ia[i][0].tobytes() == ib[i][0].tobytes() and (ia[i][1] is None) == (ib[i][1] is None) and
                       (ia[i][1] is None or ia[i][1].tobytes() == ib[i][1].tobytes()) for i in ia), (t, f)
        da, db = fs[0].decisions(), fs[1].decisions()
        assert all(da[k].tobytes() == db[k].tobytes() for k in da), t
        same_lists(fs[0], fs[1], ("add_tracked", t))
        if nonlin:
            for f_ in fs:
                f_.triangulate(states)
            flags = [int(x) for x in da["margin_flag"]]
            tabs, inv, _ = fs[0].window(3000)
            extra = dict(imu_frame_i=prob2.imu_frame_i, imu_frame_j=prob2.imu_frame_j, imu_data=prob2.imu_data, globals_=prob2.globals)
            probs = [abi.WindowProblem(10, tb["num_landmarks"], prob2.block_flags, prob2.subset_mask, vis_type=tb["vis_type"], vis_landmark=tb["vis_landmark"],
                                       vis_frame_i=tb["vis_frame_i"], vis_frame_j=tb["vis_frame_j"], vis_obs=tb["vis_obs"], **extra) for tb in tabs]
            host = ctx.batch(probs, [np.concatenate([states[f], inv[f]]) for f in range(streams)], flags)
            dev = fs[1].batch([abi.WindowProblem(10, 0, prob2.block_flags, prob2.subset_mask, **extra) for _ in range(streams)], states, flags)
            host.run(); dev.run()
            solved, _, _ = host.download(want_priors=False)
            sb, _, _ = dev.download(want_priors=False)
            assert all(x.tobytes() == y.tobytes() for x, y in zip(solved, sb)), t
            verdicts = host.outliers()
            states = np.array([x[:abi.STATE_FIXED] for x in solved])
            fs[0].set_depth([x[abi.STATE_FIXED:] for x in solved])
            fs[1].set_depth_from(dev)
            ra, rb = fs[0].remove_outliers(verdicts), fs[1].remove_outliers_from(dev)
            assert all(np.array_equal(x, y) for x, y in zip(ra, rb)), t
            pa, pb = fs[0].predict(states, [fcnt] * streams), fs[1].predict_from(dev, [fcnt] * streams)
            assert all(x[0].tobytes() == y[0].tobytes() and x[1].tobytes() == y[1].tobytes() for x, y in zip(pa, pb)), t
            host.destroy(); dev.destroy()
            n_removed += sum(len(r) for r in ra); n_pred += sum(len(p[0]) for p in pa)
            trk[0].feedback([[int(i) for i in r] for r in ra], pa)
            trk[1].feedback([[int(i) for i in r] for r in rb], pb)
        mats = [fc.cam_mats(states[f]) for f in range(streams)]
        for f_ in fs:
            f_.slide([fcnt] * streams, [1 if nonlin else 0] * streams, *[np.array([m[k] for m in mats]) for k in range(4)])
            if nonlin:
                f_.remove_failures()
        same_lists(fs[0], fs[1], ("tick", t))
        nonlin = nonlin or fcnt == 10
    assert n_pred > 0 and n_removed > 0
    for x in fs + trk:
        x.close()


# ------------------------------------------------------------------------------------------------ bytes and launches
def _filled_lists(ctx, F, ticks=12, stereo_cid=2, max_features=0):
    sc = fc.Script(stereo_cid, 3, ticks + 2)
    fs = ctx.features(F, 160, sc.cfg.stereo, 10.0 / FOCAL, max_features=max_features)
    for t in range(ticks):
        fs.add([min(t, 10)] * F, [0.0] * F, [fc.rows_of(sc.image(t), sc.cfg.stereo)] * F)
        if t < ticks - 1:
            fs.slide([min(t, 10)] * F, [0] * F)
    fs.triangulate(np.array([sc.state(ticks - 1)] * F))
    p, _, _ = sc.s.window(max(0, ticks - 11), perturb=False)
    bare = abi.WindowProblem(10, 0, p.block_flags, p.subset_mask, imu_frame_i=p.imu_frame_i, imu_frame_j=p.imu_frame_j, imu_data=p.imu_data, globals_=p.globals)
    return fs, sc, bare


def check_h2d_bytes(ctx):
    """the new create uploads less than viwb_batch_create of the same windows, by at least the observations (48 B per factor and 48 B per
    landmark) and the landmark states (8 B per landmark), less the two arrays it adds -- the fixed states apart and each window's offsets (8 B
    per window) -- and their alignment (up to 255 B each)"""
    F = 3
    fs, sc, bare = _filled_lists(ctx, F)
    st = np.array([sc.state(11)] * F)
    tabs, inv, _ = fs.window(4000)
    probs = [abi.WindowProblem(10, tb["num_landmarks"], bare.block_flags, bare.subset_mask, vis_type=tb["vis_type"], vis_landmark=tb["vis_landmark"],
                               vis_frame_i=tb["vis_frame_i"], vis_frame_j=tb["vis_frame_j"], vis_obs=tb["vis_obs"], imu_frame_i=bare.imu_frame_i,
                               imu_frame_j=bare.imu_frame_j, imu_data=bare.imu_data, globals_=bare.globals) for tb in tabs]
    h0 = ctx.h2d_bytes()
    host = ctx.batch(probs, [np.concatenate([st[s], inv[s]]) for s in range(F)], [0] * F)
    h1 = ctx.h2d_bytes()
    dev = fs.batch([bare] * F, st, [0] * F)
    h2 = ctx.h2d_bytes()
    nvis, nlm = sum(len(tb["vis_type"]) for tb in tabs), sum(tb["num_landmarks"] for tb in tabs)
    assert nvis > 0 and dev.num_landmarks == host.num_landmarks
    payload = 48 * nvis + 48 * nlm + 8 * nlm
    assert (h1 - h0) - (h2 - h1) >= payload - 8 * F - 2 * 255, (h1 - h0, h2 - h1, payload)
    host.destroy(); dev.destroy(); fs.close()
    return h1 - h0, h2 - h1


def check_launches_do_not_depend_on_streams(ctx):
    """every new call launches the same number of kernels for 1 and for 5 streams"""
    counts = []
    for F in (1, 5):
        fs, sc, bare = _filled_lists(ctx, F)
        st = np.array([sc.state(11)] * F)
        c = []
        l0 = ctx.launch_count()
        b = fs.batch([bare] * F, st, [0] * F)
        c.append(ctx.launch_count() - l0)
        b.run()
        for call in (lambda: fs.set_depth_from(b), lambda: fs.remove_outliers_from(b), lambda: fs.predict_from(b, [10] * F)):
            l0 = ctx.launch_count()
            call()
            c.append(ctx.launch_count() - l0)
        counts.append(c)
        b.destroy(); fs.close()
    assert counts[0] == counts[1] and counts[0] == [4, 1, 3, 2], counts      # count + digest + fill + vis_expand; set_depth; outlier + compact + pack; predict + pack


# ------------------------------------------------------------------------------------------------ errors
def check_errors(ctx):
    """each refusal is VIWB_ERR_INVALID with a message and leaves the lists (and a batch given to it) as they were"""
    F = 2
    fs, sc, bare = _filled_lists(ctx, F, max_features=2000)
    st = np.array([sc.state(11)] * F)
    state = {"before": fs.download()}

    def unchanged(what):
        for x, y in zip(state["before"], fs.download()):
            for k in x:
                assert x[k].tobytes() == y[k].tobytes(), (what, k)

    def refused(fn, text, *a):
        try:
            fn(*a)
        except ViwbError as e:
            assert text in str(e) and "failed with -1:" in str(e), (text, str(e))      # VIWB_ERR_INVALID
        else:
            raise AssertionError("accepted: " + text)
        unchanged(text)
    n_batches = ctx.launch_count()
    # a problem with visual rows or landmarks
    tabs, inv, _ = fs.window(4000)
    tb = tabs[1]
    with_rows = abi.WindowProblem(10, tb["num_landmarks"], bare.block_flags, bare.subset_mask, vis_type=tb["vis_type"], vis_landmark=tb["vis_landmark"],
                                  vis_frame_i=tb["vis_frame_i"], vis_frame_j=tb["vis_frame_j"], vis_obs=tb["vis_obs"])
    refused(fs.batch, "problem 1 carries visual rows", [bare, with_rows], st, [0] * F)
    refused(fs.batch, "problem 0 carries visual rows", [abi.WindowProblem(10, 3, bare.block_flags), bare], st, [0] * F)
    # a list observation beyond the problem's frame_count
    refused(fs.batch, "bad visual factor table", [bare, abi.WindowProblem(5, 0, bare.block_flags, bare.subset_mask)], st, [0] * F)
    assert ctx.launch_count() - n_batches <= 2 * 2          # the refused creates ran at most their count and digest launches: no batch was built
    # batches of another features object and of viwb_batch_create
    b = fs.batch([bare] * F, st, [0] * F)
    b.run()
    other = ctx.features(F, 160, True, 10.0 / FOCAL)
    ob = other.batch([bare] * F, st, [0] * F)
    probs = [abi.WindowProblem(10, t_["num_landmarks"], bare.block_flags, bare.subset_mask, vis_type=t_["vis_type"], vis_landmark=t_["vis_landmark"],
                               vis_frame_i=t_["vis_frame_i"], vis_frame_j=t_["vis_frame_j"], vis_obs=t_["vis_obs"]) for t_ in fs.window(4000)[0]]
    hb = ctx.batch(probs, [np.concatenate([st[s], inv[s]]) for s in range(F)])
    for wrong, what in ((ob, "another features object"), (hb, "viwb_batch_create")):
        refused(fs.set_depth_from, "not built from these lists", wrong)
        refused(fs.remove_outliers_from, "not built from these lists", wrong)
        refused(fs.predict_from, "not built from these lists", wrong, [10] * F)
    state_b = b.download()[0]
    # lists changed since the create: set_depth / remove_outliers refuse, predict (fixed states only) runs
    fs.slide([9] * F, [0] * F)                              # frame_count 9: no stream slides, but it counts as a change
    state["before"] = fs.download()
    refused(fs.set_depth_from, "the lists changed since the batch was built", b)
    refused(fs.remove_outliers_from, "the lists changed since the batch was built", b)
    fs.predict_from(b, [10] * F)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(state_b, b.download()[0]))
    # an add error still unread
    big = (np.arange(10 ** 6, 10 ** 6 + 160, dtype=np.int32), np.zeros((160, 6), np.float32))
    none = (np.zeros(0, np.int32), np.zeros((0, 6), np.float32))
    for _ in range(13):                                     # 13 * 160 new ids overflow max_features = 2000 on stream 1
        fs.add([10] * F, [0.0] * F, [none, big])
        big = (big[0] + 160, big[1])
    n0 = ctx.launch_count()
    try:                                                    # (the lists cannot be read before: the read would report the error)
        fs.batch([bare] * F, st, [0] * F)
        raise AssertionError("built over an unread add error")
    except ViwbError as e:
        assert "stream 1: the list would exceed max_features" in str(e) and "failed with -1:" in str(e), str(e)
    assert ctx.launch_count() == n0                         # refused before any launch
    fs.batch([bare] * F, st, [0] * F).destroy()             # reported once: the lists build again
    for x in (b, ob, hb):
        x.destroy()
    other.close(); fs.close()
    # more than VIWB_MAX_LANDMARKS landmarks in a stream
    big = ctx.features(2, 1024, False, 0.02, max_features=1100)
    rows = (np.arange(1001, dtype=np.int32), np.tile(np.float32([0.1, 0.2, 300, 200, 0, 0]), (1001, 1)))
    few = (np.arange(5, dtype=np.int32), np.tile(np.float32([0.1, 0.2, 300, 200, 0, 0]), (5, 1)))
    for t in range(4):
        big.add([t, t], [0.0, 0.0], [few, rows])
    kept = big.download()
    try:
        big.batch([abi.WindowProblem(3, 0, bare.block_flags)] * 2, np.array([sc.state(11)] * 2))
        raise AssertionError("1001 landmarks built")
    except ViwbError as e:
        assert "VIWB_MAX_LANDMARKS" in str(e) and "stream 1" in str(e), str(e)
    assert all(x[k].tobytes() == y[k].tobytes() for x, y in zip(kept, big.download()) for k in x)
    big.close()
