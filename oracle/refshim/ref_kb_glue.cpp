// ref_kb_glue.cpp -- TEST INFRASTRUCTURE ONLY.  C entry points over the reference's OWN camodocal::EquidistantCamera (camera_models/src/
// camera_models/EquidistantCamera.cc, the Kannala-Brandt model), compiled unmodified, under FeatureTracker::undistortedPts
// (featureTracker/feature_tracker.cpp:606-617) and spaceToPlane.  Built by oracle/kb.mk into _ref/libviw_ref_kb.so, which links against
// _ref/libviw_ref.so (FeatureTracker, Camera.cc live there); nothing of the reference is restated here.
//
// A camera is p[8] = k2 k3 k4 k5 mu mv u0 v0 (EquidistantCamera's constructor order).
#include "featureTracker/feature_tracker.h"
#include "camodocal/camera_models/EquidistantCamera.h"

namespace {
camodocal::CameraPtr make_camera(const double *p, int width, int height) {
    return camodocal::CameraPtr(new camodocal::EquidistantCamera("cam", width, height, p[0], p[1], p[2], p[3], p[4], p[5], p[6], p[7]));
}
}  // namespace

// FeatureTracker::undistortedPts(pts, camera): pts / un n x 2 floats
extern "C" int ref_kb_undistorted_pts(const double *p, int width, int height, int n, const float *pts, float *un) {
    camodocal::CameraPtr cam = make_camera(p, width, height);
    FeatureTracker t;
    std::vector<cv::Point2f> v;
    for (int i = 0; i < n; i++) v.push_back(cv::Point2f(pts[2 * i], pts[2 * i + 1]));
    std::vector<cv::Point2f> out = t.undistortedPts(v, cam);
    if ((int)out.size() != n) return 2;
    for (int i = 0; i < n; i++) { un[2 * i] = out[i].x; un[2 * i + 1] = out[i].y; }
    return 0;
}

// camera->spaceToPlane: P n x 3 doubles -> pixel n x 2 doubles
extern "C" int ref_kb_space_to_plane(const double *p, int width, int height, int n, const double *P, double *uv) {
    camodocal::CameraPtr cam = make_camera(p, width, height);
    for (int i = 0; i < n; i++) { Eigen::Vector2d q; cam->spaceToPlane(Eigen::Vector3d(P[3 * i], P[3 * i + 1], P[3 * i + 2]), q); uv[2 * i] = q.x(); uv[2 * i + 1] = q.y(); }
    return 0;
}
