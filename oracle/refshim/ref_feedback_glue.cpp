// ref_feedback_glue.cpp -- TEST INFRASTRUCTURE ONLY.  C entry points over the reference's OWN Estimator::predictPtsInNextFrame
// (estimator/estimator.cpp:2080-2113), FeatureTracker::removeOutliers and FeatureTracker::setPrediction (featureTracker/feature_tracker.cpp:
// 715-755), compiled unmodified from VIW-Fusion.  Built by oracle/feedback.mk into _ref/libviw_ref_feedback.so, which links against
// _ref/libviw_ref.so (the reference's translation units and the globals they read live there); nothing of the reference is restated here.
// Compiled with -fno-access-control, as the estimator glue is.
#include "estimator/estimator.h"
#include "camodocal/camera_models/PinholeCamera.h"
#include <cmath>
#include <cstdlib>
#include <map>
#include <new>
#include <set>

extern int ROW, COL;

namespace {
// m_camera[0] of the tracker predictPtsInNextFrame hands its map to: the reference's pinhole camera, which also notes the camera-frame point
// each spaceToPlane call receives -- the only place where the entries of the local predictPts map can be seen from outside
struct NotingCamera : public camodocal::PinholeCamera {
    using camodocal::PinholeCamera::PinholeCamera;
    mutable std::vector<Eigen::Vector3d> seen;
    void spaceToPlane(const Eigen::Vector3d &P, Eigen::Vector2d &p) const override { seen.push_back(P); camodocal::PinholeCamera::spaceToPlane(P, p); }
};
Eigen::Quaterniond quat_at(const double *q) { return Eigen::Quaterniond(q[3], q[0], q[1], q[2]); }
camodocal::PinholeCamera *make_camera(const double *c, int width, int height) { return new camodocal::PinholeCamera("cam", width, height, c[4], c[5], c[6], c[7], c[0], c[1], c[2], c[3]); }
}  // namespace

// state: the window of include/viwb.h (poses 7 x 11, extrinsics of camera 0 at 176); features as in viwb_predict_pts, ids = 0..n-1.
// valid[k] = 1 and pts_cam[k] = the map entry where predictPtsInNextFrame inserted feature k; has_prediction = featureTracker.hasPrediction.
extern "C" int ref_predict_pts(const double *state, int frame_count, int n, const int32_t *start_frame, const int32_t *num_obs, const double *pt0, const double *depth,
                               double *pts_cam, uint8_t *valid, int32_t *has_prediction) {
    void *mem = calloc(1, sizeof(Estimator));
    Estimator *e = new (mem) Estimator();                               // never destroyed, as in the estimator glue
    e->frame_count = frame_count;
    for (int i = 0; i <= WINDOW_SIZE; i++) { e->Ps[i] = Eigen::Vector3d(state[7 * i], state[7 * i + 1], state[7 * i + 2]); e->Rs[i] = quat_at(state + 7 * i + 3).toRotationMatrix(); }
    e->tic[0] = Eigen::Vector3d(state[176], state[177], state[178]); e->ric[0] = quat_at(state + 179).toRotationMatrix();
    Eigen::Matrix<double, 7, 1> obs;
    for (int k = 0; k < n; k++) {
        FeaturePerId f(k, start_frame[k]);
        for (int j = 0; j < num_obs[k]; j++) {
            if (j == 0) obs << pt0[3 * k], pt0[3 * k + 1], pt0[3 * k + 2], 0.0, 0.0, 0.0, 0.0; else obs.setZero();
            f.feature_per_frame.push_back(FeaturePerFrame(obs, 0.0));
        }
        f.estimated_depth = depth[k];
        e->f_manager.feature.push_back(f);
    }
    const double ident[8] = {1.0, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    NotingCamera *cam = new NotingCamera("cam", 640, 480, ident[4], ident[5], ident[6], ident[7], ident[0], ident[1], ident[2], ident[3]);
    FeatureTracker &t = e->featureTracker;
    t.m_camera.push_back(camodocal::CameraPtr(cam));
    for (int k = 0; k < n; k++) { t.ids.push_back(k); t.prev_pts.push_back(cv::Point2f(std::nanf(""), std::nanf(""))); }
    t.hasPrediction = false;
    e->predictPtsInNextFrame();
    *has_prediction = t.hasPrediction ? 1 : 0;
    for (int k = 0; k < n; k++) { valid[k] = 0; pts_cam[3 * k] = pts_cam[3 * k + 1] = pts_cam[3 * k + 2] = 0.0; }
    if (!t.hasPrediction) return cam->seen.empty() ? 0 : 1;
    // setPrediction walks ids in order and calls spaceToPlane for exactly the ids found in the map; a row without an entry receives its
    // prev_pts, which were set to NaN above: the k-th row that is not NaN belongs to the k-th noted point
    if ((int)t.predict_pts.size() != n) return 2;
    size_t s = 0;
    for (int k = 0; k < n; k++) {
        if (t.predict_pts[k].x != t.predict_pts[k].x) continue;
        if (s >= cam->seen.size()) return 3;
        valid[k] = 1; for (int c = 0; c < 3; c++) pts_cam[3 * k + c] = cam->seen[s](c);
        s++;
    }
    return s == cam->seen.size() ? 0 : 4;
}

// FeatureTracker::removeOutliers, then (when has_prediction) FeatureTracker::setPrediction, on a tracker whose prev_pts / ids / track_cnt are given.
// Outputs: the reduced rows and predict_pts (one per remaining row).  *n_out = remaining rows.
extern "C" int ref_tracker_feedback(const double *cam, int width, int height, int n, const float *prev_pts, const int32_t *ids, const int32_t *track_cnt,
                                    int n_remove, const int32_t *remove_ids, int has_prediction, int n_pred, const int32_t *pred_ids, const double *pred_pts_cam,
                                    int32_t *n_out, float *prev_out, int32_t *ids_out, int32_t *cnt_out, float *predict_out, int32_t *has_pred_out) {
    ROW = height; COL = width;
    FeatureTracker *t = new FeatureTracker();
    t->m_camera.push_back(camodocal::CameraPtr(make_camera(cam, width, height)));
    for (int i = 0; i < n; i++) { t->prev_pts.push_back(cv::Point2f(prev_pts[2 * i], prev_pts[2 * i + 1])); t->ids.push_back(ids[i]); t->track_cnt.push_back(track_cnt[i]); }
    t->hasPrediction = false;
    std::set<int> removeIndex(remove_ids, remove_ids + n_remove);
    t->removeOutliers(removeIndex);
    if (has_prediction) {
        std::map<int, Eigen::Vector3d> predictPts;
        for (int k = 0; k < n_pred; k++) predictPts[pred_ids[k]] = Eigen::Vector3d(pred_pts_cam[3 * k], pred_pts_cam[3 * k + 1], pred_pts_cam[3 * k + 2]);
        t->setPrediction(predictPts);
    }
    const int m = (int)t->ids.size();
    if ((int)t->prev_pts.size() != m || (int)t->track_cnt.size() != m || (has_prediction && (int)t->predict_pts.size() != m)) return 1;
    *n_out = m; *has_pred_out = t->hasPrediction ? 1 : 0;
    for (int i = 0; i < m; i++) {
        prev_out[2 * i] = t->prev_pts[i].x; prev_out[2 * i + 1] = t->prev_pts[i].y; ids_out[i] = t->ids[i]; cnt_out[i] = t->track_cnt[i];
        if (has_prediction) { predict_out[2 * i] = t->predict_pts[i].x; predict_out[2 * i + 1] = t->predict_pts[i].y; }
    }
    delete t;
    return 0;
}

// the same two calls on a live tracker handle of ref_tracker_create (libviw_ref.so), between two ref_tracker_track calls
extern "C" void ref_tracker_remove_outliers(void *h, int n, const int32_t *ids) {
    std::set<int> removeIndex(ids, ids + n);
    ((FeatureTracker *)h)->removeOutliers(removeIndex);
}
extern "C" void ref_tracker_set_prediction_map(void *h, int n, const int32_t *ids, const double *pts_cam) {
    std::map<int, Eigen::Vector3d> predictPts;
    for (int k = 0; k < n; k++) predictPts[ids[k]] = Eigen::Vector3d(pts_cam[3 * k], pts_cam[3 * k + 1], pts_cam[3 * k + 2]);
    ((FeatureTracker *)h)->setPrediction(predictPts);
}
