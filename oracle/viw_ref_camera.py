"""TEST INFRASTRUCTURE ONLY -- ctypes binding of oracle/_ref/libviw_ref_camera.so (oracle/camera.mk): the reference's OWN camodocal::CataCamera
(camera_models/src/camera_models/CataCamera.cc, compiled unmodified) under FeatureTracker::undistortedPts, spaceToPlane, removeOutliers +
setPrediction, and trackImage().  A camera is a camera_oracle.Mei or a pinhole 8-tuple.  The @viw_ref._stored functions answer from
tests/golden/reference where the reference is not compiled."""
import ctypes as C
import os
import subprocess

import numpy as np

import camera_oracle as co
import viw_ref
import viw_ref_feedback

LIB = os.path.join(viw_ref.HERE, "_ref", "libviw_ref_camera.so")
_lib = None


def available():
    return viw_ref.available()


def lib():
    global _lib
    if _lib is None:
        viw_ref.lib()                                       # builds / loads _ref/libviw_ref.so, which this library links against
        if os.path.isdir(viw_ref.REF_SRC):
            subprocess.check_call(["make", "-C", viw_ref.HERE, "-s", "-f", "camera.mk"], env=viw_ref.MAKE_ENV)
        _lib = C.CDLL(LIB)
    return _lib


def camera_args(cam):
    """(model, p[9]) as viwb_camera lays them out"""
    if isinstance(cam, co.Mei):
        return 1, np.array([float(v) for v in cam], np.float64)
    return 0, np.array([float(v) for v in cam] + [0.0], np.float64)


_dp = viw_ref._dp
_ip = lambda x: x.ctypes.data_as(C.POINTER(C.c_int32))
_fp = lambda x: x.ctypes.data_as(C.POINTER(C.c_float))


@viw_ref._stored
def camera_undistorted_pts(cam, width, height, pts):
    """FeatureTracker::undistortedPts(pts, camera) -> float32 [n, 2]"""
    model, p = camera_args(cam)
    q = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    out = np.zeros((max(len(q), 1), 2), np.float32)
    rc = lib().ref_camera_undistorted_pts(C.c_int(model), _dp(p), C.c_int(width), C.c_int(height), C.c_int(len(q)), _fp(q), _fp(out))
    if rc:
        raise RuntimeError("ref_camera_undistorted_pts rc=%d" % rc)
    return out[: len(q)].copy()


@viw_ref._stored
def camera_space_to_plane(cam, width, height, P):
    """camera->spaceToPlane -> float64 [n, 2]"""
    model, p = camera_args(cam)
    P = np.ascontiguousarray(P, np.float64).reshape(-1, 3)
    uv = np.zeros((max(len(P), 1), 2))
    rc = lib().ref_camera_space_to_plane(C.c_int(model), _dp(p), C.c_int(width), C.c_int(height), C.c_int(len(P)), _dp(P), _dp(uv))
    if rc:
        raise RuntimeError("ref_camera_space_to_plane rc=%d" % rc)
    return uv[: len(P)].copy()


@viw_ref._stored
def camera_tracker_feedback(cam, width, height, prev_pts, ids, track_cnt, remove_ids, has_prediction, pred_ids, pred_pts_cam):
    """viw_ref_feedback.tracker_feedback with m_camera[0] = cam"""
    model, p = camera_args(cam)
    pp = np.ascontiguousarray(prev_pts, np.float32).reshape(-1, 2)
    i_, t_ = np.ascontiguousarray(ids, np.int32), np.ascontiguousarray(track_cnt, np.int32)
    rm, pid = np.ascontiguousarray(remove_ids, np.int32).reshape(-1), np.ascontiguousarray(pred_ids, np.int32).reshape(-1)
    pc = np.ascontiguousarray(pred_pts_cam, np.float64).reshape(-1, 3)
    cap = max(len(i_), 1)
    n_out, hp = C.c_int32(0), C.c_int32(0)
    prev_o, ids_o, cnt_o, pred_o = np.zeros((cap, 2), np.float32), np.zeros(cap, np.int32), np.zeros(cap, np.int32), np.zeros((cap, 2), np.float32)
    rc = lib().ref_camera_tracker_feedback(C.c_int(model), _dp(p), C.c_int(width), C.c_int(height), C.c_int(len(i_)), _fp(pp), _ip(i_), _ip(t_), C.c_int(len(rm)), _ip(rm),
                                           C.c_int(1 if has_prediction else 0), C.c_int(len(pid)), _ip(pid), _dp(pc), C.byref(n_out), _fp(prev_o), _ip(ids_o), _ip(cnt_o),
                                           _fp(pred_o), C.byref(hp))
    if rc:
        raise RuntimeError("ref_camera_tracker_feedback rc=%d" % rc)
    m = n_out.value
    return {"prev_pts": prev_o[:m].copy(), "ids": ids_o[:m].copy(), "track_cnt": cnt_o[:m].copy(), "predict_pts": pred_o[:m].copy(), "has_prediction": bool(hp.value)}


class ReferenceFeatureTracker(viw_ref_feedback.ReferenceFeatureTracker):
    """The reference's own trackImage() (viw_ref.ReferenceFeatureTracker, with removeOutliers / setPrediction) whose m_camera entries are the
    given cameras of either model; needs the compiled reference (viw_ref.live())"""

    def __init__(self, cam0, cam1, width, height, max_cnt, min_dist, flow_back=True):
        pin = (1.0, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0)            # placeholders, exchanged below
        super().__init__(pin, None if cam1 is None else pin, width, height, max_cnt, min_dist, flow_back)
        for c, cam in enumerate((cam0, cam1)):
            if cam is not None:
                model, p = camera_args(cam)
                assert lib().ref_tracker_set_camera(self.h, C.c_int(c), C.c_int(model), _dp(p), C.c_int(width), C.c_int(height)) == 0
