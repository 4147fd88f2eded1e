"""TEST INFRASTRUCTURE ONLY -- CPU restatement (numpy) of the estimator's way back into the feature tracker (estimator.cpp:841-843):

  * Estimator::predictPtsInNextFrame()            vins_estimator/src/estimator/estimator.cpp:2066-2113
  * FeatureTracker::removeOutliers()              vins_estimator/src/featureTracker/feature_tracker.cpp:739-755
  * FeatureTracker::setPrediction()               feature_tracker.cpp:715-736, over PinholeCamera::spaceToPlane
                                                  (camera_models/src/camera_models/PinholeCamera.cc:520-542, distortion :646-662)

Only tests/, __graft_entry__.smoke() and profiles/ may import this file; the product never does.  Pinned to the reference's compiled code by
tests/test_feedback.py (through oracle/viw_ref_feedback.py)."""
import numpy as np

import feature_oracle as fo

f32 = np.float32


def q_to_R(q):
    """Eigen::Quaterniond(w, x, y, z).toRotationMatrix() for q = [x, y, z, w]"""
    x, y, z, w = (float(v) for v in q)
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz, txx, txy, txz, tyy, tyz, tzz = tx * w, ty * w, tz * w, tx * x, ty * x, tz * x, ty * y, tz * y, tz * z
    return np.array([[1 - (tyy + tzz), txy - twz, txz + twy], [txy + twz, 1 - (txx + tzz), tyz - twx], [txz - twy, tyz + twx, 1 - (txx + tyy)]])


def pose44(state, i):
    """Estimator::getPoseInWorldFrame(index, T) (:2073-2078) from the window's pose block i"""
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = q_to_R(state[7 * i + 3: 7 * i + 7]), state[7 * i: 7 * i + 3]
    return T


def predict_pts_in_next_frame(state, frame_count, start_frame, num_obs, pt0, depth):
    """estimator.cpp:2080-2113 over a feature list given as arrays (start_frame, feature_per_frame.size(), feature_per_frame[0].point,
    estimated_depth).  Returns (pts_cam [n, 3], valid [n] uint8): valid marks the ids the reference inserts into predictPts."""
    state = np.asarray(state, np.float64)
    n = len(start_frame)
    pts_cam, valid = np.zeros((n, 3)), np.zeros(n, np.uint8)
    if frame_count < 2:
        return pts_cam, valid
    curT, prevT = pose44(state, frame_count), pose44(state, frame_count - 1)
    nextT = curT @ (np.linalg.inv(prevT) @ curT)
    ric, tic = q_to_R(state[179:183]), state[176:179]
    for k in range(n):
        if depth[k] > 0:
            first = int(start_frame[k])
            last = first + int(num_obs[k]) - 1
            if num_obs[k] >= 2 and last == frame_count:
                pts_j = ric @ (depth[k] * np.asarray(pt0[k], np.float64)) + tic
                pts_w = q_to_R(state[7 * first + 3: 7 * first + 7]) @ pts_j + state[7 * first: 7 * first + 3]
                pts_local = nextT[:3, :3].T @ (pts_w - nextT[:3, 3])
                pts_cam[k] = ric.T @ (pts_local - tic)
                valid[k] = 1
    return pts_cam, valid


def space_to_plane(cam, P):
    """PinholeCamera::spaceToPlane (PinholeCamera.cc:520-542): camera-frame points [n, 3] -> pixels [n, 2] in double.
    cam = (fx, fy, cx, cy, k1, k2, p1, p2)."""
    fx, fy, cx, cy, k1, k2, p1, p2 = (float(v) for v in cam)
    P = np.asarray(P, np.float64).reshape(-1, 3)
    x, y = P[:, 0] / P[:, 2], P[:, 1] / P[:, 2]
    xd, yd = x, y
    if not (k1 == 0.0 and k2 == 0.0 and p1 == 0.0 and p2 == 0.0):
        mx2, my2, mxy = x * x, y * y, x * y
        rho2 = mx2 + my2
        rad = k1 * rho2 + k2 * rho2 * rho2
        xd = x + (x * rad + 2.0 * p1 * mxy + p2 * (rho2 + 2.0 * mx2))
        yd = y + (y * rad + 2.0 * p2 * mxy + p1 * (rho2 + 2.0 * my2))
    return np.column_stack([fx * xd + cx, fy * yd + cy])


class FeatureTrackerRef(fo.FeatureTrackerRef):
    """feature_oracle.FeatureTrackerRef with the two members the estimator calls between ticks"""

    def remove_outliers(self, remove_ids):
        """feature_tracker.cpp:739-755: reduceVector(prev_pts / ids / track_cnt) by membership in the std::set"""
        remove = set(int(i) for i in remove_ids)
        status = np.array([i not in remove for i in self.ids], bool)
        self.prev_pts = self.prev_pts[status] if len(status) else self.prev_pts
        self.ids = [i for i, s in zip(self.ids, status) if s]
        self.track_cnt = [c for c, s in zip(self.track_cnt, status) if s]

    def set_prediction_from_map(self, predict):
        """feature_tracker.cpp:715-736.  predict: {id: pts_cam} (std::map<int, Eigen::Vector3d>)"""
        self.hasPrediction = True
        out = np.zeros((len(self.ids), 2), f32)
        for i, fid in enumerate(self.ids):
            if fid in predict:
                out[i] = space_to_plane(self.cam[0], predict[fid])[0].astype(f32)          # cv::Point2f(tmp_uv.x(), tmp_uv.y())
            else:
                out[i] = self.prev_pts[i]
        self.predict_pts = out
