"""TEST INFRASTRUCTURE ONLY -- ctypes binding of oracle/_ref/libviw_ref_feedback.so (oracle/feedback.mk): the reference's OWN
Estimator::predictPtsInNextFrame, FeatureTracker::removeOutliers and FeatureTracker::setPrediction, compiled unmodified.  predict_pts and
tracker_feedback answer from tests/golden/reference where the reference is not compiled (viw_ref's stored-result mechanism)."""
import ctypes as C
import os
import subprocess

import numpy as np

import viw_ref

LIB = os.path.join(viw_ref.HERE, "_ref", "libviw_ref_feedback.so")
_lib = None


def available():
    return viw_ref.available()


def lib():
    global _lib
    if _lib is None:
        viw_ref.lib()                                       # builds / loads _ref/libviw_ref.so, which this library links against
        if os.path.isdir(viw_ref.REF_SRC):
            subprocess.check_call(["make", "-C", viw_ref.HERE, "-s", "-f", "feedback.mk"], env=viw_ref.MAKE_ENV)
        _lib = C.CDLL(LIB)
    return _lib


_dp = viw_ref._dp
_ip = lambda x: x.ctypes.data_as(C.POINTER(C.c_int32))
_fp = lambda x: x.ctypes.data_as(C.POINTER(C.c_float))
_up = lambda x: x.ctypes.data_as(C.POINTER(C.c_uint8))


@viw_ref._stored
def predict_pts(state, frame_count, start_frame, num_obs, pt0, depth):
    """The reference's predictPtsInNextFrame on a feature list (ids 0..n-1) -> dict(pts_cam [n, 3], valid [n], has_prediction)"""
    st = np.ascontiguousarray(state, np.float64)
    sf, no = np.ascontiguousarray(start_frame, np.int32), np.ascontiguousarray(num_obs, np.int32)
    p0, dep = np.ascontiguousarray(pt0, np.float64).reshape(-1, 3), np.ascontiguousarray(depth, np.float64)
    n = len(sf)
    out, valid, hp = np.zeros((max(n, 1), 3)), np.zeros(max(n, 1), np.uint8), C.c_int32(0)
    rc = lib().ref_predict_pts(_dp(st), C.c_int(frame_count), C.c_int(n), _ip(sf), _ip(no), _dp(p0), _dp(dep), _dp(out), _up(valid), C.byref(hp))
    if rc:
        raise RuntimeError("ref_predict_pts rc=%d" % rc)
    return {"pts_cam": out[:n].copy(), "valid": valid[:n].copy(), "has_prediction": bool(hp.value)}


@viw_ref._stored
def tracker_feedback(cam, width, height, prev_pts, ids, track_cnt, remove_ids, has_prediction, pred_ids, pred_pts_cam):
    """removeOutliers(remove_ids), then setPrediction({pred_ids: pred_pts_cam}) when has_prediction, on a FeatureTracker holding the given rows
    -> dict(prev_pts, ids, track_cnt, predict_pts, has_prediction)"""
    c = np.ascontiguousarray(cam, np.float64)
    pp = np.ascontiguousarray(prev_pts, np.float32).reshape(-1, 2)
    i_, t_ = np.ascontiguousarray(ids, np.int32), np.ascontiguousarray(track_cnt, np.int32)
    rm, pid = np.ascontiguousarray(remove_ids, np.int32).reshape(-1), np.ascontiguousarray(pred_ids, np.int32).reshape(-1)
    pc = np.ascontiguousarray(pred_pts_cam, np.float64).reshape(-1, 3)
    n = len(i_)
    cap = max(n, 1)
    n_out, hp = C.c_int32(0), C.c_int32(0)
    prev_o, ids_o, cnt_o, pred_o = np.zeros((cap, 2), np.float32), np.zeros(cap, np.int32), np.zeros(cap, np.int32), np.zeros((cap, 2), np.float32)
    rc = lib().ref_tracker_feedback(_dp(c), C.c_int(width), C.c_int(height), C.c_int(n), _fp(pp), _ip(i_), _ip(t_), C.c_int(len(rm)), _ip(rm), C.c_int(1 if has_prediction else 0),
                                    C.c_int(len(pid)), _ip(pid), _dp(pc), C.byref(n_out), _fp(prev_o), _ip(ids_o), _ip(cnt_o), _fp(pred_o), C.byref(hp))
    if rc:
        raise RuntimeError("ref_tracker_feedback rc=%d" % rc)
    m = n_out.value
    return {"prev_pts": prev_o[:m].copy(), "ids": ids_o[:m].copy(), "track_cnt": cnt_o[:m].copy(), "predict_pts": pred_o[:m].copy(), "has_prediction": bool(hp.value)}


class ReferenceFeatureTracker(viw_ref.ReferenceFeatureTracker):
    """viw_ref.ReferenceFeatureTracker (the reference's trackImage on cv2) with the reference's own removeOutliers / setPrediction between ticks;
    needs the compiled reference (viw_ref.live())"""

    def remove_outliers(self, ids):
        a = np.ascontiguousarray(list(ids), np.int32).reshape(-1)
        lib().ref_tracker_remove_outliers(self.h, C.c_int(len(a)), _ip(a))

    def set_prediction_from_map(self, predict):
        ids = np.ascontiguousarray(list(predict.keys()), np.int32).reshape(-1)
        pts = np.ascontiguousarray([predict[int(i)] for i in ids], np.float64).reshape(-1, 3)
        lib().ref_tracker_set_prediction_map(self.h, C.c_int(len(ids)), _ip(ids), _dp(pts))
