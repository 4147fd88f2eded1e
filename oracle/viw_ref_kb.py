"""TEST INFRASTRUCTURE ONLY -- ctypes binding of oracle/_ref/libviw_ref_kb.so (oracle/kb.mk): the reference's OWN camodocal::EquidistantCamera
(camera_models/src/camera_models/EquidistantCamera.cc, compiled unmodified) under FeatureTracker::undistortedPts and spaceToPlane.  A camera
is a kb_oracle.Kb.  The @viw_ref._stored functions answer from tests/golden/reference where the reference is not compiled."""
import ctypes as C
import os
import subprocess

import numpy as np

import viw_ref

LIB = os.path.join(viw_ref.HERE, "_ref", "libviw_ref_kb.so")
_lib = None


def available():
    return viw_ref.available()


def lib():
    global _lib
    if _lib is None:
        viw_ref.lib()                                       # builds / loads _ref/libviw_ref.so, which this library links against
        if os.path.isdir(viw_ref.REF_SRC):
            subprocess.check_call(["make", "-C", viw_ref.HERE, "-s", "-f", "kb.mk", "ref"], env=viw_ref.MAKE_ENV)
        _lib = C.CDLL(LIB)
    return _lib


_dp = viw_ref._dp
_fp = lambda x: x.ctypes.data_as(C.POINTER(C.c_float))


@viw_ref._stored
def camera_kb_undistorted_pts(cam, width, height, pts):
    """FeatureTracker::undistortedPts(pts, EquidistantCamera) -> float32 [n, 2]"""
    p = np.array([float(v) for v in cam], np.float64)
    q = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    out = np.zeros((max(len(q), 1), 2), np.float32)
    rc = lib().ref_kb_undistorted_pts(_dp(p), C.c_int(width), C.c_int(height), C.c_int(len(q)), _fp(q), _fp(out))
    if rc:
        raise RuntimeError("ref_kb_undistorted_pts rc=%d" % rc)
    return out[: len(q)].copy()


@viw_ref._stored
def camera_kb_space_to_plane(cam, width, height, P):
    """EquidistantCamera::spaceToPlane -> float64 [n, 2]"""
    p = np.array([float(v) for v in cam], np.float64)
    P = np.ascontiguousarray(P, np.float64).reshape(-1, 3)
    uv = np.zeros((max(len(P), 1), 2))
    rc = lib().ref_kb_space_to_plane(_dp(p), C.c_int(width), C.c_int(height), C.c_int(len(P)), _dp(P), _dp(uv))
    if rc:
        raise RuntimeError("ref_kb_space_to_plane rc=%d" % rc)
    return uv[: len(P)].copy()
