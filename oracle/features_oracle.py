"""TEST INFRASTRUCTURE ONLY -- a line-by-line restatement of the reference's FeatureManager (estimator/feature_manager.cpp) and of the visual-table
loop of Estimator::optimization() (estimator.cpp:1585-1638) on Python lists that keep the reference's order.  The checks hold the resident
FeatureManager of the library (viwb_features_*) to it, and it to the reference's compiled FeatureManager (oracle/viw_ref_features.py).

An observation is what FeaturePerFrame holds: obs = 12 float32 {x, y, p_u, p_v, v_x, v_y} of the left camera, then of the right one (zeros
without one), the double cur_td and is_stereo; point = (x, y, 1) as every featureFrame producer of the reference sets z = 1."""
import math

import numpy as np

import feedback_oracle as fbo
import viw_oracle as vo

WINDOW_SIZE = 10


class FeaturePerId:
    def __init__(self, feature_id, start_frame):
        self.feature_id, self.start_frame = int(feature_id), int(start_frame)
        self.frames = []                 # [(obs float32[12], cur_td, is_stereo)]
        self.estimated_depth, self.solve_flag = -1.0, 0

    def end_frame(self):
        return self.start_frame + len(self.frames) - 1


def _point(obs, cam=0):
    return np.array([float(obs[6 * cam]), float(obs[6 * cam + 1]), 1.0])


class FeatureManagerRef:
    def __init__(self, stereo, min_parallax, focal_length=460.0, init_depth=5.0):
        self.stereo, self.min_parallax, self.focal, self.init_depth = bool(stereo), float(min_parallax), float(focal_length), float(init_depth)
        self.feature = []
        self.last_track_num = self.new_feature_num = self.long_track_num = 0
        self.last_average_parallax = 0.0
        self.reason = None               # which clause of :95-118 decided the last add (for the coverage checks)

    # ---- addFeatureCheckParallax (:52-119)
    def add_feature_check_parallax(self, frame_count, image, td):
        """image: {id: (left float32[6], right float32[6] or None)}, iterated in ascending id order as std::map does -> keyframe"""
        parallax_sum, parallax_num = 0.0, 0
        self.last_track_num = self.new_feature_num = self.long_track_num = 0
        self.last_average_parallax = 0.0
        by_id = {f.feature_id: f for f in self.feature}
        for fid in sorted(image):
            left, right = image[fid]
            obs = np.zeros(12, np.float32)
            obs[:6] = left
            if right is not None:
                obs[6:] = right
            fpf = (obs, float(td), right is not None)
            it = by_id.get(int(fid))
            if it is None:
                f = FeaturePerId(fid, frame_count)
                f.frames.append(fpf)
                self.feature.append(f)
                by_id[f.feature_id] = f
                self.new_feature_num += 1
            else:
                it.frames.append(fpf)
                self.last_track_num += 1
                if len(it.frames) >= 4:
                    self.long_track_num += 1
        for cond, why in ((frame_count < 2, "frame_count"), (self.last_track_num < 20, "last_track"), (self.long_track_num < 40, "long_track"),
                          (self.new_feature_num > 0.5 * self.last_track_num, "new_features")):
            if cond:
                self.reason = why
                return True
        for f in self.feature:
            if f.start_frame <= frame_count - 2 and f.start_frame + len(f.frames) - 1 >= frame_count - 1:
                parallax_sum += self.compensated_parallax2(f, frame_count)
                parallax_num += 1
        if parallax_num == 0:
            self.reason = "no_eligible"
            return True
        self.last_average_parallax = parallax_sum / parallax_num * self.focal
        keyframe = parallax_sum / parallax_num >= self.min_parallax
        self.reason = "parallax" if keyframe else "non_keyframe"
        return keyframe

    @staticmethod
    def compensated_parallax2(f, frame_count):
        p_i = _point(f.frames[frame_count - 2 - f.start_frame][0])
        p_j = _point(f.frames[frame_count - 1 - f.start_frame][0])
        u_j, v_j = p_j[0], p_j[1]
        dep_i = p_i[2]
        u_i, v_i = p_i[0] / dep_i, p_i[1] / dep_i
        du, dv = u_i - u_j, v_i - v_j
        s = math.sqrt(min(du * du + dv * dv, du * du + dv * dv))
        return s if 0.0 < s else 0.0

    # ---- triangulate (:309-389): the two live branches, depths from the C oracle's triangulatePoint
    def triangulate(self, state):
        rows = []
        for f in self.feature:
            if f.estimated_depth > 0:
                continue
            if self.stereo and f.frames[0][2]:
                rows.append((f, 1, _point(f.frames[0][0])[:2], _point(f.frames[0][0], 1)[:2]))
            elif len(f.frames) > 1:
                rows.append((f, 0, _point(f.frames[0][0])[:2], _point(f.frames[1][0])[:2]))
        if rows:
            dep = vo.triangulate(np.asarray(state, np.float64)[:207], np.array([r[1] for r in rows], np.int32), np.array([r[0].start_frame for r in rows], np.int32),
                                 np.array([r[2] for r in rows]), np.array([r[3] for r in rows]), self.init_depth)
            for r, d in zip(rows, dep):
                r[0].estimated_depth = float(d)
        return [r[0] for r in rows]

    # ---- the numbering of optimization() / setDepth / getDepthVector
    def landmarks(self):
        return [f for f in self.feature if len(f.frames) >= 4]

    def window(self):
        """estimator.cpp:1585-1638: (table dict for abi.WindowProblem, inverse depths, ids)"""
        vt, vl, vi, vj, vobs = [], [], [], [], []
        lms = self.landmarks()
        for k, f in enumerate(lms):
            imu_i = f.start_frame
            o0, td0 = f.frames[0][0], f.frames[0][1]
            pts_i = _point(o0)
            for j, (o, td, ster) in enumerate(f.frames):
                imu_j = imu_i + j
                rows = []
                if imu_i != imu_j:
                    rows.append((0, imu_j, 0))
                if self.stereo and ster:
                    rows.append((1 if imu_i != imu_j else 2, imu_j if imu_i != imu_j else imu_i, 1))
                for typ, fj, cam in rows:
                    vt.append(typ); vl.append(k); vi.append(imu_i); vj.append(fj)
                    vobs.append(np.concatenate([pts_i, _point(o, cam), [float(o0[4]), float(o0[5]), float(o[6 * cam + 4]), float(o[6 * cam + 5]), td0, td]]))
        table = dict(num_landmarks=len(lms), vis_type=np.array(vt, np.int32), vis_landmark=np.array(vl, np.int32), vis_frame_i=np.array(vi, np.int32),
                     vis_frame_j=np.array(vj, np.int32), vis_obs=np.array(vobs, np.float64).reshape(-1, 12))
        return table, np.array([1.0 / f.estimated_depth for f in lms]), np.array([f.feature_id for f in lms], np.int32)

    # ---- setDepth (:142-160)
    def set_depth(self, x):
        for f, v in zip(self.landmarks(), x):
            f.estimated_depth = 1.0 / float(v)
            f.solve_flag = 2 if f.estimated_depth < 0 else 1

    # ---- removeOutlier (:440-455)
    def remove_outlier(self, ids):
        ids = set(int(i) for i in ids)
        self.feature = [f for f in self.feature if f.feature_id not in ids]

    def outlier_ids(self, verdicts):
        return sorted(f.feature_id for f, v in zip(self.landmarks(), verdicts) if v)

    # ---- predictPtsInNextFrame (:2080-2113) through feedback_oracle's restatement
    def predict(self, state, frame_count):
        if frame_count < 2:
            return None
        n = len(self.feature)
        pts, valid = fbo.predict_pts_in_next_frame(np.asarray(state, np.float64)[:207], frame_count, np.array([f.start_frame for f in self.feature], np.int32),
                                                   np.array([len(f.frames) for f in self.feature], np.int32),
                                                   np.array([_point(f.frames[0][0]) for f in self.feature]).reshape(n, 3),
                                                   np.array([f.estimated_depth for f in self.feature]))
        keep = np.asarray(valid, bool)
        return np.array([f.feature_id for f in self.feature], np.int32)[keep], np.asarray(pts).reshape(-1, 3)[keep]

    # ---- slideWindow's FeatureManager part (estimator.cpp:1898-2063; :457-536)
    def remove_back_shift_depth(self, marg_R, marg_P, new_R, new_P):
        out, shifted = [], []
        for f in self.feature:
            if f.start_frame != 0:
                f.start_frame -= 1
            else:
                uv_i = _point(f.frames[0][0])
                del f.frames[0]
                if len(f.frames) < 2:
                    continue
                shifted.append((f, uv_i))
            out.append(f)
        if shifted:
            dep = vo.shift_depth(np.array([u for _, u in shifted]), np.array([f.estimated_depth for f, _ in shifted]), marg_R, marg_P, new_R, new_P, self.init_depth)
            for (f, _), d in zip(shifted, dep):
                f.estimated_depth = float(d)
        self.feature = out
        return [f for f, _ in shifted]

    def remove_back(self):
        out = []
        for f in self.feature:
            if f.start_frame != 0:
                f.start_frame -= 1
            else:
                del f.frames[0]
                if len(f.frames) == 0:
                    continue
            out.append(f)
        self.feature = out

    def remove_front(self, frame_count):
        out = []
        for f in self.feature:
            if f.start_frame == frame_count:
                f.start_frame -= 1
            else:
                j = WINDOW_SIZE - 1 - f.start_frame
                if f.end_frame() >= frame_count - 1:
                    del f.frames[j]
                    if len(f.frames) == 0:
                        continue
            out.append(f)
        self.feature = out

    def slide(self, frame_count, keyframe, shift_depth, mats=None):
        if frame_count != WINDOW_SIZE:
            return []
        if keyframe:
            if shift_depth:
                return self.remove_back_shift_depth(*mats)
            self.remove_back()
        else:
            self.remove_front(frame_count)
        return []

    # ---- removeFailures (:162-171)
    def remove_failures(self):
        self.feature = [f for f in self.feature if f.solve_flag != 2]

    def as_arrays(self):
        """the list in viwb_features_download's form (one stream)"""
        n = len(self.feature)
        obs, td, ster = np.zeros((n, 11, 12), np.float32), np.zeros((n, 11)), np.zeros((n, 11), np.uint8)
        for k, f in enumerate(self.feature):
            for j, (o, t, s) in enumerate(f.frames):
                obs[k, j], td[k, j], ster[k, j] = o, t, s
        return dict(ids=np.array([f.feature_id for f in self.feature], np.int32), start_frame=np.array([f.start_frame for f in self.feature], np.int32),
                    num_obs=np.array([len(f.frames) for f in self.feature], np.int32), depth=np.array([f.estimated_depth for f in self.feature]),
                    solve_flag=np.array([f.solve_flag for f in self.feature], np.int32), obs=obs, cur_td=td, is_stereo=ster)
