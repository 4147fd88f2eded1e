"""TEST INFRASTRUCTURE ONLY -- CPU restatement of camodocal's Kannala-Brandt camera (camodocal::EquidistantCamera) where FeatureTracker calls a
camera, through oracle/libvo_kb.so (vo_kb.c, built by oracle/kb.mk with -ffp-contract=off; glibc's sin / cos / acos / atan2):

  * EquidistantCamera::liftProjective + backprojectSymmetric (under FeatureTracker::undistortedPts)   EquidistantCamera.cc:428-442, 716-818
  * EquidistantCamera::spaceToPlane (under FeatureTracker::setPrediction)                             EquidistantCamera.cc:451-461
  * EigenSolver<MatrixXd>::eigenvalues of backprojectSymmetric's companion matrix (Eigen 3.3, restated)

A camera is a `Kb` (EquidistantCamera::Parameters' order), a `camera_oracle.Mei` or a pinhole 8-tuple; lift_projective / space_to_plane
follow the model they are given, and FeatureTrackerRef takes any of them per camera.  Only tests/, __graft_entry__.smoke() and profiles/ may
import this file; the product never does.  Pinned to the reference's compiled EquidistantCamera.cc by tests/test_camera_kb.py (through
oracle/viw_ref_kb.py), its eigen-solver to LAPACK by the same tests."""
import ctypes as C
import os
import subprocess
from collections import namedtuple

import numpy as np

import camera_oracle as co
import feedback_oracle as fbo

f32 = np.float32
HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "libvo_kb.so")

Kb = namedtuple("Kb", "k2 k3 k4 k5 mu mv u0 v0")

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB) or os.path.getmtime(LIB) < os.path.getmtime(os.path.join(HERE, "vo_kb.c")):
            subprocess.check_call(["make", "-C", HERE, "-s", "-f", "kb.mk", "libvo_kb.so"])
        _lib = C.CDLL(LIB)
    return _lib


_dp = lambda x: x.ctypes.data_as(C.POINTER(C.c_double))
_fp = lambda x: x.ctypes.data_as(C.POINTER(C.c_float))


def params(cam):
    return np.array([float(v) for v in cam], np.float64)


def npow(cam):
    """backprojectSymmetric's polynomial degree: 9, less 2 for every zero k_i wherever it sits"""
    return int(lib().vo_kb_npow(_dp(params(cam))))


def refused(cam):
    """the parameter sets whose companion matrix would divide by zero (the coefficient at npow is 0 while npow > 1)"""
    n = npow(cam)
    return n > 1 and [0.0, 1.0, 0.0, cam.k2, 0.0, cam.k3, 0.0, cam.k4, 0.0, cam.k5][n] == 0.0


def companion(cam, norm):
    """backprojectSymmetric's companion matrix for |p_u| = norm (None when npow == 1)"""
    A = np.zeros(81)
    n = int(lib().vo_kb_companion(_dp(params(cam)), C.c_double(norm), _dp(A)))
    return None if n == 1 else A[: n * n].reshape(n, n).T.copy()


def eigenvalues(A):
    """the restated EigenSolver<MatrixXd>(A).eigenvalues() -> (complex [n], status 0 = converged, 1 = no convergence, 2 = non-finite)"""
    A = np.asarray(A, np.float64)
    n = len(A)
    a = np.ascontiguousarray(A.T).ravel()
    wr, wi = np.zeros(n), np.zeros(n)
    rc = lib().vo_kb_eigenvalues(_dp(a), C.c_int(n), _dp(wr), _dp(wi))
    return wr + 1j * wi, int(rc)


def lift_projective_kb(cam, pts, want_theta=False):
    """EquidistantCamera::liftProjective, then b.x() / b.z(), b.y() / b.z() narrowed to cv::Point2f; with want_theta also the theta of
    backprojectSymmetric"""
    p = np.ascontiguousarray(pts, f32).reshape(-1, 2)
    un, th = np.zeros((len(p), 2), f32), np.zeros(len(p))
    lib().vo_kb_lift(_dp(params(cam)), C.c_int(len(p)), _fp(p), _fp(un), _dp(th))
    return (un, th) if want_theta else un


def space_to_plane_kb(cam, P):
    """EquidistantCamera::spaceToPlane: camera-frame points [n, 3] -> pixels [n, 2] in double"""
    P = np.ascontiguousarray(P, np.float64).reshape(-1, 3)
    uv = np.zeros((len(P), 2))
    lib().vo_kb_space_to_plane(_dp(params(cam)), C.c_int(len(P)), _dp(P), _dp(uv))
    return uv


def lift_projective(cam, pts):
    return lift_projective_kb(cam, pts) if isinstance(cam, Kb) else co.lift_projective(cam, pts)


def space_to_plane(cam, P):
    return space_to_plane_kb(cam, P) if isinstance(cam, Kb) else co.space_to_plane(cam, P)


_PLACEHOLDER = (1.0, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0)


class FeatureTrackerRef(fbo.FeatureTrackerRef):
    """feedback_oracle.FeatureTrackerRef whose cameras may be of any model, Kannala-Brandt included -- camera_oracle.FeatureTrackerRef's
    construction: the base class runs the tick with a placeholder pinhole camera (trackImage touches the camera only in undistortedPts), and
    the lift, the velocities and the id -> point maps are then formed here with the session's own cameras.  setPrediction projects through
    camera 0's model."""

    def __init__(self, cam0, cam1=None, *args, **kw):
        super().__init__(_PLACEHOLDER, None if cam1 is None else _PLACEHOLDER, *args, **kw)
        self.models = (cam0, cam1)

    def track_image(self, cur_time, img, img1=None):
        prev_map, prev_map_r, dt = self.prev_un_pts_map, self.prev_un_right_pts_map, cur_time - self.prev_time
        ids, cnt, pts, _, _, ids_r, pts_r, _, _ = super().track_image(cur_time, img, img1)
        idl = [int(i) for i in ids]
        un = lift_projective(self.models[0], pts)                                     # feature_tracker.cpp:207-208
        vel = self._velocity(idl, un, prev_map, dt)
        self.prev_un_pts_map = {fid: un[i] for i, fid in enumerate(idl)}
        un_r, vel_r = np.zeros((0, 2), f32), np.zeros((0, 2), f32)
        if img1 is not None and self.stereo:                                          # :254-268
            idr = [int(i) for i in ids_r]
            if len(pts_r):
                un_r = lift_projective(self.models[1], pts_r)
                vel_r = self._velocity(idr, un_r, prev_map_r, dt)
            self.prev_un_right_pts_map = {fid: un_r[i] for i, fid in enumerate(idr)}
        return ids, cnt, pts, un, vel, ids_r, pts_r, un_r, vel_r

    def set_prediction_from_map(self, predict):
        """feature_tracker.cpp:715-736 with m_camera[0]->spaceToPlane of camera 0's model"""
        self.hasPrediction = True
        out = np.zeros((len(self.ids), 2), f32)
        for i, fid in enumerate(self.ids):
            out[i] = space_to_plane(self.models[0], predict[fid])[0].astype(f32) if fid in predict else self.prev_pts[i]
        self.predict_pts = out
