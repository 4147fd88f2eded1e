// ref_camera_glue.cpp -- TEST INFRASTRUCTURE ONLY.  C entry points over the reference's OWN camodocal::CataCamera (camera_models/src/
// camera_models/CataCamera.cc, the MEI model of the shipped EuRoC / mynteye / vi_car configurations), compiled unmodified, and over the
// FeatureTracker members that call a camera model: undistortedPts (featureTracker/feature_tracker.cpp:606-617), setPrediction (:715-736)
// after removeOutliers (:739-755), and the live trackImage() handle of libviw_ref.so with its m_camera entries exchanged.  Built by
// oracle/camera.mk into _ref/libviw_ref_camera.so, which links against _ref/libviw_ref.so (FeatureTracker, Camera.cc, PinholeCamera.cc live
// there); nothing of the reference is restated here.  Compiled with -fno-access-control, as the estimator glue is.
//
// A camera is (model, p[9]) as viwb_camera lays it out: model 0 = PinholeCamera, p = fx fy cx cy k1 k2 p1 p2; model 1 = CataCamera,
// p = xi k1 k2 p1 p2 gamma1 gamma2 u0 v0 (CataCamera's constructor order, CataCamera.cc:300-303).
#include "featureTracker/feature_tracker.h"
#include "camodocal/camera_models/CataCamera.h"
#include "camodocal/camera_models/PinholeCamera.h"
#include <map>
#include <set>

extern int ROW, COL;

namespace {
camodocal::CameraPtr make_camera(int model, const double *p, int width, int height) {
    if (model == 1) return camodocal::CameraPtr(new camodocal::CataCamera("cam", width, height, p[0], p[1], p[2], p[3], p[4], p[5], p[6], p[7], p[8]));
    if (model == 0) return camodocal::CameraPtr(new camodocal::PinholeCamera("cam", width, height, p[4], p[5], p[6], p[7], p[0], p[1], p[2], p[3]));
    return camodocal::CameraPtr();
}
}  // namespace

// FeatureTracker::undistortedPts(pts, camera): pts / un n x 2 floats
extern "C" int ref_camera_undistorted_pts(int model, const double *p, int width, int height, int n, const float *pts, float *un) {
    camodocal::CameraPtr cam = make_camera(model, p, width, height);
    if (!cam) return 1;
    FeatureTracker t;
    std::vector<cv::Point2f> v;
    for (int i = 0; i < n; i++) v.push_back(cv::Point2f(pts[2 * i], pts[2 * i + 1]));
    std::vector<cv::Point2f> out = t.undistortedPts(v, cam);
    if ((int)out.size() != n) return 2;
    for (int i = 0; i < n; i++) { un[2 * i] = out[i].x; un[2 * i + 1] = out[i].y; }
    return 0;
}

// camera->spaceToPlane: P n x 3 doubles -> pixel n x 2 doubles
extern "C" int ref_camera_space_to_plane(int model, const double *p, int width, int height, int n, const double *P, double *uv) {
    camodocal::CameraPtr cam = make_camera(model, p, width, height);
    if (!cam) return 1;
    for (int i = 0; i < n; i++) { Eigen::Vector2d q; cam->spaceToPlane(Eigen::Vector3d(P[3 * i], P[3 * i + 1], P[3 * i + 2]), q); uv[2 * i] = q.x(); uv[2 * i + 1] = q.y(); }
    return 0;
}

// FeatureTracker::removeOutliers, then (when has_prediction) FeatureTracker::setPrediction, on a tracker whose m_camera[0] is the given camera
// and whose prev_pts / ids / track_cnt are given.  Outputs as ref_tracker_feedback (ref_feedback_glue.cpp).
extern "C" int ref_camera_tracker_feedback(int model, const double *p, int width, int height, int n, const float *prev_pts, const int32_t *ids, const int32_t *track_cnt,
                                           int n_remove, const int32_t *remove_ids, int has_prediction, int n_pred, const int32_t *pred_ids, const double *pred_pts_cam,
                                           int32_t *n_out, float *prev_out, int32_t *ids_out, int32_t *cnt_out, float *predict_out, int32_t *has_pred_out) {
    ROW = height; COL = width;
    camodocal::CameraPtr cam = make_camera(model, p, width, height);
    if (!cam) return 1;
    FeatureTracker *t = new FeatureTracker();
    t->m_camera.push_back(cam);
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
    if ((int)t->prev_pts.size() != m || (int)t->track_cnt.size() != m || (has_prediction && (int)t->predict_pts.size() != m)) return 2;
    *n_out = m; *has_pred_out = t->hasPrediction ? 1 : 0;
    for (int i = 0; i < m; i++) {
        prev_out[2 * i] = t->prev_pts[i].x; prev_out[2 * i + 1] = t->prev_pts[i].y; ids_out[i] = t->ids[i]; cnt_out[i] = t->track_cnt[i];
        if (has_prediction) { predict_out[2 * i] = t->predict_pts[i].x; predict_out[2 * i + 1] = t->predict_pts[i].y; }
    }
    delete t;
    return 0;
}

// m_camera[c] of a live tracker handle of ref_tracker_create (libviw_ref.so) exchanged for the given camera
extern "C" int ref_tracker_set_camera(void *h, int c, int model, const double *p, int width, int height) {
    FeatureTracker *t = (FeatureTracker *)h;
    camodocal::CameraPtr cam = make_camera(model, p, width, height);
    if (!cam || c < 0 || c >= (int)t->m_camera.size()) return 1;
    t->m_camera[c] = cam;
    return 0;
}
