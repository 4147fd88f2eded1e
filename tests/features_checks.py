"""Checks of the resident FeatureManager (viwb_features_*), parameterised by the context like parity_checks.py: tests/test_features.py runs each on
the emulation build and, marked gpu, on libviwb.so.  The library is held to the restatement of oracle/features_oracle.py after every call, and
its triangulated / shifted depths and predictions to viwb_triangulate / viwb_shift_depth / viwb_predict_pts on the downloaded list."""
import numpy as np

from viwb import abi, synth
from viwb.lib import ViwbError

import features_oracle as fmo

FOCAL = 460.0


# ------------------------------------------------------------------------------------------------ scripts
class Script:
    """featureFrame rows of a synth.Sequence: ids are track indices, {x, y} the noisy normalised observations (float), p_u / p_v their pixels,
    velocities the finite difference of x, y over the camera period (0 for a track's first frame), right rows for the stereo observations."""

    def __init__(self, cid, seq, frames):
        self.cfg = synth.make_config(cid)
        if cid == 1:
            self.cfg.landmarks_all_frames, self.cfg.tracks_per_frame = 0, 120
        self.s = synth.Sequence(self.cfg, seq, frames)
        self.frames, self.dt = frames, 1.0 / self.cfg.cam_rate
        self.rows = [[] for _ in range(frames)]
        for tid, tr in enumerate(self.s.tracks):
            prev = None
            for f, pl, pr in tr["obs"]:
                def six(p, q):
                    x, y = np.float32(p[0]), np.float32(p[1])
                    vx = np.float32((float(x) - float(q[0])) / self.dt) if q is not None else np.float32(0)
                    vy = np.float32((float(y) - float(q[1])) / self.dt) if q is not None else np.float32(0)
                    return np.array([x, y, self.cfg.fx * float(x) + self.cfg.cx, self.cfg.fy * float(y) + self.cfg.cy, vx, vy], np.float32)
                self.rows[f].append((tid, six(pl, prev[0] if prev else None), None if pr is None else six(pr, prev[1] if prev and prev[1] is not None else None)))
                prev = (pl, pr)

    def image(self, t, drop=()):
        return {tid: (l, r if self.cfg.stereo else None) for tid, l, r in self.rows[t] if tid not in drop}

    def state(self, t):
        return self.s.gt_state(max(0, min(t - 10, self.frames - 11)), [])[:abi.STATE_FIXED]


def rows_of(image, stereo):
    ids = np.array(sorted(image), np.int32)[::-1].copy()            # any row order: the map sorts them
    feat = np.array([image[i][0] for i in ids], np.float32).reshape(-1, 6)
    if not stereo:
        return (ids, feat)
    rid = np.array([i for i in ids if image[i][1] is not None], np.int32)
    return (ids, feat, rid, np.array([image[i][1] for i in rid], np.float32).reshape(-1, 6))


def cam_mats(state):
    """the camera poses of slideWindowOld (estimator.cpp:2053-2059): marginalised frame 0 and the new frame 0 (frame 1 before the slide)"""
    def pose(i):
        R = fmo.fbo.q_to_R(state[7 * i + 3: 7 * i + 7]) @ fmo.fbo.q_to_R(state[179:183])
        return R, state[7 * i: 7 * i + 3] + fmo.fbo.q_to_R(state[7 * i + 3: 7 * i + 7]) @ state[176:179]
    (R0, P0), (R1, P1) = pose(0), pose(1)
    return R0.reshape(9), P0, R1.reshape(9), P1


def compare_lists(fs, refs, what, depth_exact=True):
    got = fs.download()
    for s, (g, r) in enumerate(zip(got, refs)):
        w = r.as_arrays()
        assert np.array_equal(g["ids"], w["ids"]), (what, s, len(g["ids"]), len(w["ids"]))
        for k in ("start_frame", "num_obs", "solve_flag"):
            assert np.array_equal(g[k], w[k]), (what, s, k)
        for k, v in enumerate(w["num_obs"]):
            assert g["obs"][k, :v].tobytes() == w["obs"][k, :v].tobytes() and g["cur_td"][k, :v].tobytes() == w["cur_td"][k, :v].tobytes(), (what, s, k)
            assert np.array_equal(g["is_stereo"][k, :v], w["is_stereo"][k, :v]), (what, s, k)
        if depth_exact:
            assert g["depth"].tobytes() == w["depth"].tobytes(), (what, s)
        else:
            assert np.allclose(g["depth"], w["depth"], rtol=1e-9, atol=0), (what, s)
    return got


def sync_depths(got, refs):
    """after a triangulation or a depth shift (held to 1e-9): the restatement continues from the library's depths"""
    for g, r in zip(got, refs):
        for f, d in zip(r.feature, g["depth"]):
            f.estimated_depth = float(d)


# ------------------------------------------------------------------------------------------------ the scripted sequence
def run_script(ctx, cid, ticks=32, min_parallax=10.0 / FOCAL, seed=0, stats=None, reference=True):
    """Three streams of one configuration through the estimator's per-frame order: INITIAL ticks 0..10 (add, removeBack at frame_count 10), then
    NON_LINEAR ticks (add, triangulate, window, setDepth with some negative depths, removeOutlier, predict, removeBackShiftDepth / removeFront,
    removeFailures).  Stream 1 sees no rows on some ticks and drops a third of them on others.  Stream 2 runs at other frame_counts: frame 0's
    rows at frame_count 0 and 1, none at 2, then one set of new ids four times at frame_count 3 (40 and more long tracks, none eligible for
    parallax), then from frame_count 4 on a third id range that follows the sequence.  reference: also solve stream 0's first NON_LINEAR window
    and hold every stream to the reference's own FeatureManager (the scripts of check_scripts have stored results)."""
    script = [Script(cid, seed + s, ticks + 3) for s in range(3)]

    def stream2(t):
        if t < 2:
            return 0, script[2].image(0)
        if t == 2:
            return 2, {}
        if t < 7:
            return 3, {i + 100000: v for i, v in script[2].image(3).items()}
        return min(t - 3, 10), {i + 200000: v for i, v in script[2].image(t).items()}
    stereo = script[0].cfg.stereo
    F = 3
    fs = ctx.features(F, 160, stereo, min_parallax, FOCAL)
    refs = [fmo.FeatureManagerRef(stereo, min_parallax, FOCAL) for _ in range(F)]
    rng = np.random.default_rng(100 + cid)
    import viw_ref_features as vrf
    ops, recs = [[] for _ in range(F)], [[] for _ in range(F)]       # each stream's script for the reference's FeatureManager, and the restatement's records

    def note(s, op, depth=False, add=None):
        a = refs[s].as_arrays()
        rec = {"n": len(a["ids"]), "digest": vrf.list_digest(a)}
        if depth:
            rec["depth"] = a["depth"]
        if add is not None:
            rec["stats"], rec["avg"] = np.array([1 if add else 0, refs[s].last_track_num, refs[s].long_track_num, refs[s].new_feature_num], np.int32), refs[s].last_average_parallax
        ops[s].append(op); recs[s].append(rec)
    stats = stats if stats is not None else {}
    nonlin = [False] * F
    fcs = [0] * F
    seen_reappear = 0
    removed_before = [set() for _ in range(F)]
    for t in range(ticks):
        src_t = [t, t, max(0, t - 3)]
        fc2, im2 = stream2(t)
        fc = [min(t, 10), min(t, 10), fc2]
        images = []
        for s in range(2):
            drop = ()
            if s == 1 and t % 7 == 5:
                drop = set(tid for tid, _, _ in script[s].rows[t])
            elif s == 1 and t % 7 == 3:
                drop = set(tid for k, (tid, _, _) in enumerate(script[s].rows[t]) if k % 3 == 0)
            images.append(script[s].image(t, drop))
        images.append(im2)
        td = [0.001 * t, -0.002 * t, 0.0]
        kf = [refs[s].add_feature_check_parallax(fc[s], images[s], td[s]) for s in range(F)]
        for s in range(F):
            stats[refs[s].reason] = stats.get(refs[s].reason, 0) + 1
            new_ids = set(images[s]) & removed_before[s]
            seen_reappear += len(new_ids)
            removed_before[s] -= new_ids
        fs.add(fc, td, [rows_of(im, stereo) for im in images])
        d = fs.decisions()
        for s in range(F):
            assert d["margin_flag"][s] == (0 if kf[s] else 1), (t, s, refs[s].reason)
            assert (d["last_track_num"][s], d["long_track_num"][s], d["new_feature_num"][s]) == (refs[s].last_track_num, refs[s].long_track_num, refs[s].new_feature_num)
            assert d["last_average_parallax"][s] == refs[s].last_average_parallax, (t, s)
        got = compare_lists(fs, refs, ("add", t))
        for s in range(F):
            r = rows_of(images[s], True)
            note(s, (vrf.ADD, fc[s], td[s], r[0], r[1], r[2] if stereo else np.zeros(0, np.int32), r[3] if stereo else np.zeros((0, 6), np.float32)), add=kf[s])
        states = np.array([script[s].state(src_t[s]) for s in range(F)])
        if any(nonlin):
            # triangulate, held bit for bit to viwb_triangulate on the downloaded list and to 1e-9 to the restatement
            want = []
            for s in range(F):
                g = got[s]
                sel = [k for k in range(len(g["ids"])) if g["depth"][k] <= 0 and ((stereo and g["is_stereo"][k, 0]) or g["num_obs"][k] > 1)]
                st_flag = np.array([1 if (stereo and g["is_stereo"][k, 0]) else 0 for k in sel], np.int32)
                p0 = np.array([g["obs"][k, 0, 0:2] for k in sel], np.float64).reshape(-1, 2)
                p1 = np.array([g["obs"][k, 0, 6:8] if f else g["obs"][k, 1, 0:2] for k, f in zip(sel, st_flag)], np.float64).reshape(-1, 2)
                want.append((sel, ctx.triangulate(states[s], st_flag, g["start_frame"][sel], p0, p1) if sel else np.zeros(0)))
                refs[s].triangulate(states[s])
            fs.triangulate(states)
            got = compare_lists(fs, refs, ("triangulate", t), depth_exact=False)
            for s in range(F):
                assert got[s]["depth"][want[s][0]].tobytes() == want[s][1].tobytes(), (t, s)
            sync_depths(got, refs)
            for s in range(F):
                note(s, (vrf.TRIANGULATE, fc[s], states[s]), depth=True)
            # the window's visual table, bit for bit
            tables, inv, lids = fs.window(4000)
            for s in range(F):
                wt, wi, wl = refs[s].window()
                for k in wt:
                    assert np.asarray(tables[s][k]).tobytes() == np.asarray(wt[k]).tobytes(), (t, s, k)
                assert inv[s].tobytes() == wi.tobytes() and np.array_equal(lids[s], wl), (t, s)
            if t == 11 and reference:                             # stream 0's first NON_LINEAR window: solved, and re-assembled by the reference's optimization()
                check_exported_window(ctx, script[0], t, tables[0], inv[0], 0 if kf[0] else 1)
                stats["solved"] = stats.get("solved", 0) + 1
            # setDepth with a solver-like perturbation and a few negative depths; outliers; prediction
            xs, verdicts = [], []
            for s in range(F):
                x = inv[s] * (1.0 + rng.normal(0, 1e-3, len(inv[s])))
                x[rng.uniform(size=len(x)) < 0.04] *= -1.0
                xs.append(x)
                verdicts.append((rng.uniform(size=len(x)) < 0.05).astype(np.uint8))
            fs.set_depth(xs)
            for s in range(F):
                refs[s].set_depth(xs[s])
                note(s, (vrf.SET_DEPTH, xs[s]), depth=True)
            compare_lists(fs, refs, ("set_depth", t))
            removed = fs.remove_outliers(verdicts)
            for s in range(F):
                ids = refs[s].outlier_ids(verdicts[s])
                assert np.array_equal(removed[s], np.array(ids, np.int32)), (t, s)
                refs[s].remove_outlier(ids)
                note(s, (vrf.REMOVE_OUTLIER, np.array(ids, np.int32)))
                removed_before[s] |= set(ids)
                stats["outliers"] = stats.get("outliers", 0) + len(ids)
            got = compare_lists(fs, refs, ("remove_outliers", t))
            pred = fs.predict(states, fc)
            for s in range(F):
                r = refs[s].predict(states[s], fc[s])
                assert (pred[s] is None) == (r is None), (t, s)
                if r is not None:
                    assert np.array_equal(pred[s][0], r[0]) and np.allclose(pred[s][1], r[1], rtol=1e-9, atol=1e-12), (t, s)
                    g = got[s]
                    pts, valid = ctx.predict_pts(states[s], fc[s], g["start_frame"], g["num_obs"], np.column_stack([g["obs"][:, 0, 0:2].astype(np.float64), np.ones(len(g["ids"]))]),
                                                 g["depth"])
                    assert np.array_equal(pred[s][0], g["ids"][valid.astype(bool)]) and pred[s][1].tobytes() == pts[valid.astype(bool)].tobytes(), (t, s)
                    stats["predicted"] = stats.get("predicted", 0) + len(r[0])
        # slide (with the flag of the add) and, in NON_LINEAR, removeFailures
        mats = [cam_mats(states[s]) for s in range(F)]
        want = []
        for s in range(F):
            g = got[s]
            sel = [k for k in range(len(g["ids"])) if g["start_frame"][k] == 0 and g["num_obs"][k] - 1 >= 2] if (nonlin[s] and kf[s] and fc[s] == 10) else []
            uv = np.column_stack([g["obs"][sel, 0, 0:2].astype(np.float64), np.ones(len(sel))]) if sel else np.zeros((0, 3))
            want.append((g["ids"][sel], ctx.shift_depth(uv, g["depth"][sel], *mats[s]) if sel else np.zeros(0)))
            refs[s].slide(fc[s], kf[s], nonlin[s], mats[s])
        fs.slide(fc, [1 if x else 0 for x in nonlin], np.array([m[0] for m in mats]), np.array([m[1] for m in mats]), np.array([m[2] for m in mats]),
                 np.array([m[3] for m in mats]))
        got = compare_lists(fs, refs, ("slide", t), depth_exact=False)
        for s in range(F):
            if len(want[s][0]):
                stats["shifted"] = stats.get("shifted", 0) + len(want[s][0])
                pos = {int(i): k for k, i in enumerate(got[s]["ids"])}
                assert got[s]["depth"][[pos[int(i)] for i in want[s][0]]].tobytes() == want[s][1].tobytes(), (t, s)
        sync_depths(got, refs)
        for s in range(F):
            note(s, (vrf.SLIDE, fc[s], 1 if nonlin[s] else 0) + tuple(mats[s]), depth=True)
        if any(nonlin):
            before = sum(len(r.feature) for r in refs)
            fs.remove_failures()
            for s in range(F):                              # every call runs on every stream (a stream still INITIAL was given depths too)
                refs[s].remove_failures()
                note(s, (vrf.REMOVE_FAILURES,))
            stats["failures"] = stats.get("failures", 0) + before - sum(len(r.feature) for r in refs)
            compare_lists(fs, refs, ("remove_failures", t))
        for s in range(F):
            if fc[s] == 10:
                nonlin[s] = True
            fcs[s] = fc[s]
    stats["reappeared"] = stats.get("reappeared", 0) + seen_reappear
    fs.close()
    if reference:
        for s in range(F):
            pin_to_reference(ops[s], recs[s], stereo, min_parallax)
        stats["pinned"] = stats.get("pinned", 0) + F
    return stats


def pin_to_reference(ops, recs, stereo, min_parallax):
    """the reference's own FeatureManager (compiled, or its stored results) through the same calls: after every call the same list (ids, order,
    start frames, observations, cur_td, stereo and solve flags, by digest), the same statistics and last_average_parallax bit for bit, depths
    to 1e-9 (the restatement continues from the library's triangulated / shifted depths, the reference from its own)"""
    import viw_ref_features as vrf
    got = vrf.features_script(vrf.script_digest(ops), stereo, min_parallax, 5.0, lambda: ops)
    assert len(got) == len(recs)
    for i, (g, w) in enumerate(zip(got, recs)):
        assert g["n"] == w["n"] and g["digest"] == w["digest"], (i, ops[i][0], g["n"], w["n"])
        if "stats" in w:
            assert np.array_equal(g["stats"], w["stats"]) and g["avg"] == w["avg"], (i, g["stats"], w["stats"], g["avg"], w["avg"])
        if "depth" in w:
            assert np.allclose(g["depth"], w["depth"], rtol=1e-9, atol=0), (i, ops[i][0])


def check_exported_window(ctx, sc, t, table, inv, flag):
    """An exported visual table with the IMU / wheel / plane tables of the synth window it belongs to: solved by the library like the oracle (pose
    bar 1e-4, same iteration count), and handed with the library's solution to the reference's own Estimator::optimization(), which re-assembles
    the problem with its own loop over the feature list: no structure, vector2double or visual-row mismatch."""
    import viw_oracle as vo
    import viw_ref_features as vrf
    prob, st0, _ = sc.s.window(t - 10)
    p = abi.WindowProblem(10, table["num_landmarks"], prob.block_flags, prob.subset_mask, vis_type=table["vis_type"], vis_landmark=table["vis_landmark"],
                          vis_frame_i=table["vis_frame_i"], vis_frame_j=table["vis_frame_j"], vis_obs=table["vis_obs"], imu_frame_i=prob.imu_frame_i,
                          imu_frame_j=prob.imu_frame_j, imu_data=prob.imu_data, wheel_frame_i=prob.wheel_frame_i, wheel_frame_j=prob.wheel_frame_j,
                          wheel_data=prob.wheel_data, plane_frame=prob.plane_frame, prior=None, globals_=prob.globals)
    from test_reference_factors import _as_the_estimator_holds_it
    state = _as_the_estimator_holds_it(np.concatenate([np.asarray(st0[:abi.STATE_FIXED], np.float64), inv]))   # the window as para_* hold it
    a1, sm1, _ = ctx.optimization(p, state, flag)
    a0, sm0, _ = vo.optimization(p, state, flag)
    ep, er = synth.pose_errors(a0, a1)
    assert ep <= 1e-4 and er <= 1e-4 and sm0.num_iterations == sm1.num_iterations, (ep, er, sm0.num_iterations, sm1.num_iterations)
    if vrf.available():
        rec = vrf.features_estimator_record(p, state, a1, flag)
        assert rec["structure_mismatches"] == 0 and rec["vector2double_mismatches"] == 0 and rec["visual_row_mismatches"] == 0, rec
        assert rec["proj_2f1c"] == int(np.sum(table["vis_type"] == 0)), rec


def check_scripts(ctx):
    """mono (config 1) and stereo (configs 2 and 4) scripts; together they reach every clause of the keyframe rule, outliers, failures, shifted
    depths, predictions and outlier ids that come back as new features"""
    stats = {}
    run_script(ctx, 1, 32, 10.0 / FOCAL, 0, stats)
    run_script(ctx, 2, 30, 10.0 / FOCAL, 10, stats)
    run_script(ctx, 4, 30, 1.0, 20, stats)
    for k in ("frame_count", "last_track", "long_track", "new_features", "parallax", "no_eligible", "non_keyframe", "outliers", "failures", "shifted",
              "predicted", "reappeared", "solved", "pinned"):
        assert stats.get(k, 0) > 0, (k, stats)
    return stats


# ------------------------------------------------------------------------------------------------ fed by the resident tracker
def _tracker_image(out, f, stereo):
    n_left, ids, _, feat, n_right, ids_r, feat_r = out
    right = {int(ids_r[f, j]): feat_r[f, j].copy() for j in range(int(n_right[f]))} if stereo else {}
    return {int(ids[f, j]): (feat[f, j].copy(), right.get(int(ids[f, j]))) for j in range(int(n_left[f]))}


def check_closed_loop(ctx, ticks=16, streams=2):
    """Tracker tick -> add_tracked -> triangulate -> window -> set_depth -> remove_outliers -> predict -> viwb_tracker_feedback -> slide ->
    remove_failures on two stereo streams, the exported windows solved by ctx.batch (viwb_batch_create / run / download) with the IMU tables of a
    synth window, their depths set from the solution and their outliers from Batch.outliers (viwb_batch_outliers).  add_tracked must equal add fed the rows viwb_tracker_download returns for the same tick (lists and
    decisions bit for bit), and both the restatement fed those rows; the removed ids and predictions go back into the tracker sessions.  The first
    tick runs at frame_count max(0, 14 - ticks), so that at least three ticks run NON_LINEAR after the window filled."""
    import feedback_checks as fbc
    import parity_checks as pc
    W, H, MAX_CNT = fbc.W, fbc.H, fbc.MAX_CNT
    seqs = [pc.camera_sequence(70 + f, W, H, ticks) for f in range(streams)]
    trk = ctx.tracker(streams, W, H, fbc.CAM0, fbc.CAM1, MAX_CNT, fbc.MIN_DIST, True)
    fa = ctx.features(streams, MAX_CNT, True, 10.0 / FOCAL, FOCAL)
    fb = ctx.features(streams, MAX_CNT, True, 10.0 / FOCAL, FOCAL)
    refs = [fmo.FeatureManagerRef(True, 10.0 / FOCAL, FOCAL) for _ in range(streams)]
    rng = np.random.default_rng(31)
    prob2, _, gt2 = synth.make_window(2, 0)                 # the IMU / wheel tables and block layout of a stereo window
    states = np.array([gt2[:abi.STATE_FIXED]] * streams)
    nonlin, n_pred, n_removed = False, 0, 0
    fc0 = max(0, 14 - ticks)
    for t in range(ticks):
        fc = min(t + fc0, 10)
        left, right = np.stack([seqs[f][0][t] for f in range(streams)]), np.stack([seqs[f][1][t] for f in range(streams)])
        trk.track(0.05 * (t + 1), left, right)
        out = [x.copy() for x in trk.download()]
        images = [_tracker_image(out, f, True) for f in range(streams)]
        td = [0.0] * streams
        l0 = ctx.launch_count()
        fa.add_tracked(trk, [fc] * streams, td)
        assert ctx.launch_count() - l0 == 2
        fb.add([fc] * streams, td, [rows_of(im, True) for im in images])
        kf = [refs[f].add_feature_check_parallax(fc, images[f], 0.0) for f in range(streams)]
        da, db = fa.decisions(), fb.decisions()
        for k in da:
            assert da[k].tobytes() == db[k].tobytes(), (t, k)
        assert [int(x) for x in da["margin_flag"]] == [0 if k else 1 for k in kf], t
        assert all(da["last_average_parallax"][f] == refs[f].last_average_parallax for f in range(streams)), t
        ga = compare_lists(fa, refs, ("add_tracked", t))
        gb = compare_lists(fb, refs, ("add", t))
        for x, y in zip(ga, gb):
            for k in x:
                assert x[k].tobytes() == y[k].tobytes(), (t, k)
        removed, preds = [[] for _ in range(streams)], [None] * streams
        if nonlin:
            for fs in (fa, fb):
                fs.triangulate(states)
            for f, r in enumerate(refs):
                r.triangulate(states[f])
            got = compare_lists(fa, refs, ("triangulate", t), depth_exact=False)
            sync_depths(got, refs)
            tabs = [fs.window(3000) for fs in (fa, fb)]
            problems = []
            for f in range(streams):
                wt, wi, _ = refs[f].window()
                assert all(np.asarray(tabs[0][0][f][k]).tobytes() == np.asarray(wt[k]).tobytes() for k in wt), (t, f)
                assert all(np.asarray(tabs[1][0][f][k]).tobytes() == np.asarray(wt[k]).tobytes() for k in wt), (t, f)
                tb = tabs[0][0][f]
                problems.append(abi.WindowProblem(10, tb["num_landmarks"], prob2.block_flags, prob2.subset_mask, vis_type=tb["vis_type"], vis_landmark=tb["vis_landmark"],
                                                  vis_frame_i=tb["vis_frame_i"], vis_frame_j=tb["vis_frame_j"], vis_obs=tb["vis_obs"],
                                                  imu_frame_i=prob2.imu_frame_i, imu_frame_j=prob2.imu_frame_j, imu_data=prob2.imu_data, globals_=prob2.globals))
            # the exported windows solved as one viwb_batch (solve + re-anchoring + marginalisation), depths and outliers from it
            batch = ctx.batch(problems, [np.concatenate([states[f], tabs[0][1][f]]) for f in range(streams)], [int(x) for x in da["margin_flag"]])
            batch.run()
            solved, summ, _ = batch.download(want_priors=False)
            verdicts = batch.outliers()
            batch.destroy()
            xs = [np.asarray(solved[f][abi.STATE_FIXED:]) for f in range(streams)]
            states = np.array([np.asarray(solved[f][:abi.STATE_FIXED]) for f in range(streams)])
            assert all(np.isfinite(x).all() for x in xs) and all(sm.num_iterations >= 1 for sm in summ), t
            for fs in (fa, fb):
                fs.set_depth(xs)
            rm = fa.remove_outliers(verdicts)
            assert all(np.array_equal(a, b) for a, b in zip(rm, fb.remove_outliers(verdicts)))
            for f in range(streams):
                ids = refs[f].outlier_ids(verdicts[f])
                assert np.array_equal(rm[f], ids)
                refs[f].set_depth(xs[f]); refs[f].remove_outlier(ids)
                removed[f] = [int(i) for i in rm[f]]
                n_removed += len(ids)
            preds = fa.predict(states, [fc] * streams)
            for f in range(streams):
                r = refs[f].predict(states[f], fc)
                assert np.array_equal(preds[f][0], r[0]) and np.allclose(preds[f][1], r[1], rtol=1e-9, atol=1e-12)
                n_pred += len(r[0])
            fb.predict(states, [fc] * streams)
            trk.feedback(removed, preds)
        mats = [cam_mats(states[f]) for f in range(streams)]
        for fs in (fa, fb):
            fs.slide([fc] * streams, [1 if nonlin else 0] * streams, *[np.array([m[k] for m in mats]) for k in range(4)])
        for f in range(streams):
            refs[f].slide(fc, kf[f], nonlin, mats[f])
        got = compare_lists(fa, refs, ("slide", t), depth_exact=False)
        sync_depths(got, refs)
        if nonlin:
            for fs in (fa, fb):
                fs.remove_failures()
            for r in refs:
                r.remove_failures()
        ga = compare_lists(fa, refs, ("tick", t))
        for x, y in zip(ga, fb.download()):
            for k in x:
                assert x[k].tobytes() == y[k].tobytes(), (t, k)
        nonlin = nonlin or fc == 10
    assert n_pred > 0 and n_removed > 0
    fa.close(); fb.close(); trk.close()


def check_launches_do_not_depend_on_streams(ctx):
    """every call launches the same kernels for 1 and for 5 streams"""
    counts = []
    for F in (1, 5):
        sc = Script(2, 3, 14)
        fs = ctx.features(F, 160, True, 10.0 / FOCAL)
        c = []
        for t in range(12):
            fc = min(t, 10)
            l0 = ctx.launch_count()
            fs.add([fc] * F, [0.0] * F, [rows_of(sc.image(t), True)] * F)
            fs.triangulate(np.array([sc.state(t)] * F))
            tabs, inv, _ = fs.window(4000)
            fs.set_depth(inv)
            fs.remove_outliers([np.zeros(len(v), np.uint8) for v in inv])
            fs.predict(np.array([sc.state(t)] * F), [fc] * F)
            fs.slide([fc] * F, [1] * F, *[np.array([m] * F) for m in cam_mats(sc.state(t))])
            fs.remove_failures()
            c.append(ctx.launch_count() - l0)
        counts.append(c)
        fs.close()
    assert counts[0] == counts[1] and counts[0][-1] == 12, counts          # add 2, triangulate 1, window 2, set_depth 1, remove_outliers 2, predict 2, slide 1, remove_failures 1


def check_errors(ctx):
    """every error rule is VIWB_ERR_INVALID with a message, and a download afterwards shows every list as it was"""
    sc = Script(2, 5, 14)
    fs = ctx.features(2, 160, True, 10.0 / FOCAL, max_features=300)
    for t in range(4):
        fs.add([t, t], [0.0, 0.0], [rows_of(sc.image(t), True), rows_of(sc.image(t), True)])
    state = {"before": fs.download()}

    def unchanged(what):
        for x, y in zip(state["before"], fs.download()):
            for k in x:
                assert x[k].tobytes() == y[k].tobytes(), (what, k)

    def refused(fn, text, *a):
        try:
            fn(*a)
        except ViwbError as e:
            assert text in str(e), (text, str(e))
        else:
            raise AssertionError("accepted: " + text)
        unchanged(text)
    im = sc.image(4)
    ids, feat, rid, rfeat = rows_of(im, True)
    dup = (np.concatenate([ids, ids[:1]]), np.concatenate([feat, feat[:1]]), rid, rfeat)
    refused(fs.add, "duplicate left id", [4, 4], [0.0, 0.0], [rows_of(im, True), dup])
    refused(fs.add, "without a left row", [4, 4], [0.0, 0.0], [(ids[1:], feat[1:], rid, rfeat), rows_of(im, True)])
    big = (np.arange(161, dtype=np.int32), np.zeros((161, 6), np.float32))
    refused(fs.add, "max_rows", [4, 4], [0.0, 0.0], [big, rows_of(im, True)])
    refused(fs.add, "frame_count", [11, 4], [0.0, 0.0], [rows_of(im, True)] * 2)
    many = (np.arange(10 ** 6, 10 ** 6 + 160, dtype=np.int32), np.zeros((160, 6), np.float32))      # 160 new ids on a list of more than 140
    d0 = fs.decisions()
    fs.add([4, 4], [0.0, 0.0], [rows_of(im, True), many])
    fs.add([4, 4], [0.0, 0.0], [rows_of(im, True), rows_of(im, True)])          # queued behind the failed add, no synchronising call between
    refused(fs.download, "stream 1: the list would exceed max_features")          # the first failure is reported, and neither add changed a list
    d1 = fs.decisions()                                                            # the decisions are still those of the last applied add
    assert all(d0[k].tobytes() == d1[k].tobytes() for k in d0)
    for t in range(4, 11):                                          # a twelfth observation
        fs.add([t, t], [0.0, 0.0], [rows_of(sc.image(3), True)] * 2)
    fs.decisions()
    state["before"] = fs.download()
    fs.add([10, 10], [0.0, 0.0], [rows_of(sc.image(3), True)] * 2)
    refused(fs.decisions, "more than 11 observations")
    refused(fs.window, "more than vis_cap", 10)
    refused(fs.set_depth, "changed since the last", [np.zeros(0)] * 2)
    tabs, inv, _ = fs.window(4000)
    fs.slide([10, 10], [0, 0])
    state["before"] = fs.download()
    refused(fs.remove_outliers, "changed since the last", [np.zeros(len(v), np.uint8) for v in inv])
    other = ctx.features(3, 160, True, 0.02)
    trk = ctx.tracker(2, 64, 48, (50.0, 50.0, 32.0, 24.0, 0, 0, 0, 0), None, 40, 10, True)
    refused(other.add_tracked, "another stream count", trk, [0, 0, 0], [0.0] * 3)
    other.close(); trk.close()
    from viwb import lib as viwb_lib
    ctx2 = viwb_lib.Context(0, ctx.lib._name)
    trk2 = ctx2.tracker(2, 64, 48, (50.0, 50.0, 32.0, 24.0, 0, 0, 0, 0), None, 40, 10, True)
    refused(fs.add_tracked, "another context", trk2, [0, 0], [0.0] * 2)
    trk2.close(); ctx2.close(); fs.close()
    # more than VIWB_MAX_LANDMARKS landmarks in an export
    big = ctx.features(1, 1024, False, 0.02, max_features=1100)
    rows = (np.arange(1001, dtype=np.int32), np.tile(np.float32([0.1, 0.2, 300, 200, 0, 0]), (1001, 1)))
    for t in range(4):
        big.add([t], [0.0], [rows])
    kept = big.download()
    try:
        big.window(20000)
        raise AssertionError("1001 landmarks exported")
    except ViwbError as e:
        assert "VIWB_MAX_LANDMARKS" in str(e) and "stream 0" in str(e), str(e)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(kept[0].values(), big.download()[0].values()))
    big.close()
