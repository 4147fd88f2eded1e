"""TEST INFRASTRUCTURE ONLY -- ctypes binding of oracle/_ref/libviw_ref_features.so (oracle/features.mk): the reference's OWN FeatureManager
(estimator/feature_manager.cpp, compiled unmodified) driven through a scripted sequence of calls.  features_script answers from
tests/golden/reference where the reference is not compiled (viw_ref's stored-result mechanism).

A script is a list of operations, each a tuple (kind, arguments...):
  (ADD, frame_count, td, ids, feat [n, 6], ids_right, feat_right [m, 6])   addFeatureCheckParallax with the image map of these rows
  (TRIANGULATE, frame_count, state [207])                                     triangulate(frame_count, Ps, Rs, tic, ric) of the window state
  (SET_DEPTH, x)                                                              setDepth(x)
  (REMOVE_OUTLIER, ids)                                                       removeOutlier(set(ids))
  (SLIDE, frame_count, shift_depth, marg_R [9], marg_P, new_R [9], new_P)     slideWindow's FeatureManager part with the flag of the last ADD:
                                                                              frame_count == WINDOW_SIZE only; keyframe -> removeBackShiftDepth if
                                                                              shift_depth else removeBack; otherwise removeFront(frame_count)
  (REMOVE_FAILURES,)                                                          removeFailures()
After every operation the record holds the list size, a digest of the list without depths (list_digest), the depths after the operations that
change them, and the statistics after an ADD."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np

import viw_ref

LIB = os.path.join(viw_ref.HERE, "_ref", "libviw_ref_features.so")
ADD, TRIANGULATE, SET_DEPTH, REMOVE_OUTLIER, SLIDE, REMOVE_FAILURES = range(6)
_lib = None


def available():
    return viw_ref.available()


def lib():
    global _lib
    if _lib is None:
        viw_ref.lib()                                       # builds / loads _ref/libviw_ref.so, which this library links against
        if os.path.isdir(viw_ref.REF_SRC):
            subprocess.check_call(["make", "-C", viw_ref.HERE, "-s", "-f", "features.mk"], env=viw_ref.MAKE_ENV)
        _lib = C.CDLL(LIB)
        _lib.ref_fm_create.restype = C.c_void_p
        _lib.ref_fm_create.argtypes = [C.c_int, C.c_double, C.c_double]
        for name in ("ref_fm_destroy", "ref_fm_add", "ref_fm_triangulate", "ref_fm_set_depth", "ref_fm_remove_outlier", "ref_fm_remove_back_shift_depth",
                     "ref_fm_remove_back", "ref_fm_remove_front", "ref_fm_remove_failures", "ref_fm_size", "ref_fm_dump"):
            getattr(_lib, name).restype = C.c_int if name == "ref_fm_size" else None
    return _lib


def list_digest(a):
    """48-bit digest of a list in viwb_features_download's per-stream form, depths excluded (ids, start frames, observation counts, solve flags,
    and every observation slot's floats, cur_td and stereo flag, zeros past num_obs)"""
    h = hashlib.sha1()
    for k, dt in (("ids", np.int32), ("start_frame", np.int32), ("num_obs", np.int32), ("solve_flag", np.int32)):
        h.update(np.ascontiguousarray(a[k], dt).tobytes())
    n = len(a["ids"])
    obs, td, ster = np.zeros((n, 11, 12), np.float32), np.zeros((n, 11)), np.zeros((n, 11), np.uint8)
    for k, v in enumerate(np.asarray(a["num_obs"])):
        obs[k, :v], td[k, :v], ster[k, :v] = a["obs"][k, :v], a["cur_td"][k, :v], a["is_stereo"][k, :v]
        obs[k, :v, 6:] *= ster[k, :v, None]
    for x in (obs, td, ster):
        h.update(x.tobytes())
    return float(int.from_bytes(h.digest()[:6], "little"))


def script_digest(ops):
    """the key of a script for the stored results: per operation its kind, scalars and the size / sum / absolute sum of each array"""
    out = []
    for op in ops:
        out.append(float(op[0]))
        for v in op[1:]:
            a = np.asarray(v, np.float64).ravel()
            out += [float(a.size), float(a.sum()), float(np.abs(a).sum())] if a.size != 1 or np.ndim(v) else [float(a[0])]
    return np.array(out)


_ip = lambda x: x.ctypes.data_as(C.c_void_p)


def _dump(h):
    L = lib()
    n = L.ref_fm_size(C.c_void_p(h))
    a = dict(ids=np.zeros(n, np.int32), start_frame=np.zeros(n, np.int32), num_obs=np.zeros(n, np.int32), depth=np.zeros(n), solve_flag=np.zeros(n, np.int32),
             obs=np.zeros((n, 11, 12), np.float32), cur_td=np.zeros((n, 11)), is_stereo=np.zeros((n, 11), np.uint8))
    if n:
        L.ref_fm_dump(C.c_void_p(h), *[_ip(a[k]) for k in ("ids", "start_frame", "num_obs", "depth", "solve_flag", "obs", "cur_td", "is_stereo")])
    return a


@viw_ref._stored
def features_script(digest, stereo, min_parallax, init_depth, ops_fn):
    """The reference's FeatureManager through the script ops_fn() (whose key is `digest` = script_digest(ops)) -> one record per operation:
    dict(n, digest, [depth], [stats = keyframe, last_track_num, long_track_num, new_feature_num], [avg])"""
    L = lib()
    h = L.ref_fm_create(int(stereo), float(min_parallax), float(init_depth))
    recs, keyframe = [], True
    try:
        for op in ops_fn():
            k, rec = op[0], {}
            if k == ADD:
                _, fc, td, ids, feat, ids_r, feat_r = op
                ids, ids_r = np.ascontiguousarray(ids, np.int32), np.ascontiguousarray(ids_r, np.int32)
                feat, feat_r = np.ascontiguousarray(feat, np.float32).reshape(-1, 6), np.ascontiguousarray(feat_r, np.float32).reshape(-1, 6)
                stats, avg = np.zeros(4, np.int32), C.c_double(0.0)
                L.ref_fm_add(C.c_void_p(h), C.c_int(fc), C.c_double(td), C.c_int(len(ids)), _ip(ids), _ip(feat), C.c_int(len(ids_r)), _ip(ids_r), _ip(feat_r),
                             _ip(stats), C.byref(avg))
                keyframe = bool(stats[0])
                rec["stats"], rec["avg"] = stats, avg.value
            elif k == TRIANGULATE:
                st = np.ascontiguousarray(op[2], np.float64)
                L.ref_fm_triangulate(C.c_void_p(h), C.c_int(op[1]), _ip(st))
            elif k == SET_DEPTH:
                x = np.ascontiguousarray(op[1], np.float64)
                L.ref_fm_set_depth(C.c_void_p(h), C.c_int(len(x)), _ip(x))
            elif k == REMOVE_OUTLIER:
                ids = np.ascontiguousarray(op[1], np.int32)
                L.ref_fm_remove_outlier(C.c_void_p(h), C.c_int(len(ids)), _ip(ids))
            elif k == SLIDE:
                _, fc, shift, mR, mP, nR, nP = op
                if fc == 10:
                    if keyframe and shift:
                        m = [np.ascontiguousarray(v, np.float64) for v in (mR, mP, nR, nP)]
                        L.ref_fm_remove_back_shift_depth(C.c_void_p(h), *[_ip(v) for v in m])
                    elif keyframe:
                        L.ref_fm_remove_back(C.c_void_p(h))
                    else:
                        L.ref_fm_remove_front(C.c_void_p(h), C.c_int(fc))
            elif k == REMOVE_FAILURES:
                L.ref_fm_remove_failures(C.c_void_p(h))
            a = _dump(h)
            rec["n"], rec["digest"] = len(a["ids"]), list_digest(a)
            if k in (TRIANGULATE, SET_DEPTH, SLIDE):
                rec["depth"] = a["depth"]
            recs.append(rec)
    finally:
        L.ref_fm_destroy(C.c_void_p(h))
    return recs


@viw_ref._stored
def features_estimator_record(problem, state, state_solved, flag):
    """viw_ref.estimator_optimization's assembly record of a window whose visual table came out of viwb_features_window (stored under its own
    name, so that the existing stored results stay as they are)"""
    return viw_ref.estimator_optimization.__wrapped__(problem, state, state_solved, flag)["record"]
