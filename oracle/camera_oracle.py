"""TEST INFRASTRUCTURE ONLY -- CPU restatement (numpy) of camodocal's MEI camera model (camodocal::CataCamera, the unified omnidirectional model
with mirror parameter xi) where FeatureTracker calls a camera:

  * CataCamera::liftProjective (under FeatureTracker::undistortedPts)   camera_models/src/camera_models/CataCamera.cc:556-626, m_inv_K* :319-323,
                                                                         m_noDistortion :307-317; feature_tracker.cpp:606-617
  * CataCamera::spaceToPlane (under FeatureTracker::setPrediction)      CataCamera.cc:636-659; feature_tracker.cpp:715-736
  * CataCamera::distortion                                               CataCamera.cc:766-782

A camera is an `Mei` (CataCamera's parameters in its constructor / yaml order, CataCamera.cc:300-303) or a pinhole 8-tuple (fx, fy, cx, cy,
k1, k2, p1, p2); lift_projective / space_to_plane follow the model they are given, and FeatureTrackerRef takes either model per camera.
numpy rounds every operation on its own, as the reference's build (-ffp-contract=off, SSE2) does, so the floats are the reference's bit for bit.
Only tests/, __graft_entry__.smoke() and profiles/ may import this file; the product never does.  Pinned to the reference's compiled
CataCamera.cc by tests/test_camera_models.py (through oracle/viw_ref_camera.py)."""
from collections import namedtuple

import numpy as np

import feature_oracle as fo
import feedback_oracle as fbo

f32 = np.float32

Mei = namedtuple("Mei", "xi k1 k2 p1 p2 gamma1 gamma2 u0 v0")


def mei_distortion(cam, x, y):
    """CataCamera::distortion (CataCamera.cc:766-782)"""
    k1, k2, p1, p2 = (float(v) for v in (cam.k1, cam.k2, cam.p1, cam.p2))
    mx2, my2, mxy = x * x, y * y, x * y
    rho2 = mx2 + my2
    rad = k1 * rho2 + k2 * rho2 * rho2
    return x * rad + 2.0 * p1 * mxy + p2 * (rho2 + 2.0 * mx2), y * rad + 2.0 * p2 * mxy + p1 * (rho2 + 2.0 * my2)


def mei_no_distortion(cam):
    """m_noDistortion (CataCamera.cc:307-317)"""
    return cam.k1 == 0.0 and cam.k2 == 0.0 and cam.p1 == 0.0 and cam.p2 == 0.0


def lift_projective_mei(cam, pts):
    """CataCamera::liftProjective (recursive distortion model n = 8, the xi == 1 branch and 1 - xi (rho^2 + 1) / (xi + sqrt(1 + (1 - xi^2) rho^2))
    otherwise), then b.x() / b.z(), b.y() / b.z() narrowed to cv::Point2f.  NaN / inf where the reference has them."""
    xi, g1, g2, u0, v0 = (float(v) for v in (cam.xi, cam.gamma1, cam.gamma2, cam.u0, cam.v0))
    p = np.asarray(pts, f32).reshape(-1, 2)
    with np.errstate(all="ignore"):
        mxd, myd = (1.0 / g1) * p[:, 0].astype(np.float64) + (-u0 / g1), (1.0 / g2) * p[:, 1].astype(np.float64) + (-v0 / g2)
        mx, my = mxd.copy(), myd.copy()
        if not mei_no_distortion(cam):
            for _ in range(8):
                dx, dy = mei_distortion(cam, mx, my)
                mx, my = mxd - dx, myd - dy
        if xi == 1.0:
            z = (1.0 - mx * mx - my * my) / 2.0
        else:
            rho2 = mx * mx + my * my
            z = 1.0 - xi * (rho2 + 1.0) / (xi + np.sqrt(1.0 + (1.0 - xi * xi) * rho2))
        return np.column_stack([(mx / z).astype(f32), (my / z).astype(f32)])


def space_to_plane_mei(cam, P):
    """CataCamera::spaceToPlane: z = P(2) + xi |P| with |P| = sqrt((x^2 + y^2) + z^2), then the distortion and gamma * p_d + (u0, v0).
    Camera-frame points [n, 3] -> pixels [n, 2] in double."""
    xi, g1, g2, u0, v0 = (float(v) for v in (cam.xi, cam.gamma1, cam.gamma2, cam.u0, cam.v0))
    P = np.asarray(P, np.float64).reshape(-1, 3)
    with np.errstate(all="ignore"):
        z = P[:, 2] + xi * np.sqrt((P[:, 0] * P[:, 0] + P[:, 1] * P[:, 1]) + P[:, 2] * P[:, 2])
        x, y = P[:, 0] / z, P[:, 1] / z
        if not mei_no_distortion(cam):
            dx, dy = mei_distortion(cam, x, y)
            x, y = x + dx, y + dy
        return np.column_stack([g1 * x + u0, g2 * y + v0])


def lift_projective(cam, pts):
    """undistortedPts' lift through the camera's model: lift_projective_mei or feature_oracle.lift_projective (pinhole)"""
    return lift_projective_mei(cam, pts) if isinstance(cam, Mei) else fo.lift_projective(cam, pts)


def space_to_plane(cam, P):
    """setPrediction's projection through the camera's model: space_to_plane_mei or feedback_oracle.space_to_plane (pinhole)"""
    return space_to_plane_mei(cam, P) if isinstance(cam, Mei) else fbo.space_to_plane(cam, P)


_PLACEHOLDER = (1.0, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0)


class FeatureTrackerRef(fbo.FeatureTrackerRef):
    """feedback_oracle.FeatureTrackerRef (the restated trackImage with removeOutliers / setPrediction) whose cameras may be of either model.
    trackImage touches the camera only in undistortedPts, whose points feed nothing but the returned rows, ptsVelocity and the id -> point maps
    (feature_tracker.cpp:207-208, 254-268): the base class runs the tick with a placeholder pinhole camera, and the lift, the velocities and the
    maps are then formed here with the session's own cameras, as the base class forms them.  setPrediction projects through camera 0's model."""

    def __init__(self, cam0, cam1=None, *args, **kw):
        super().__init__(_PLACEHOLDER, None if cam1 is None else _PLACEHOLDER, *args, **kw)
        self.models = (cam0, cam1)

    def track_image(self, cur_time, img, img1=None):
        prev_map, prev_map_r, dt = self.prev_un_pts_map, self.prev_un_right_pts_map, cur_time - self.prev_time
        ids, cnt, pts, _, _, ids_r, pts_r, _, _ = super().track_image(cur_time, img, img1)
        idl = [int(i) for i in ids]
        un = lift_projective(self.models[0], pts)                                     # :207-208
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
