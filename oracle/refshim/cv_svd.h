// TEST INFRASTRUCTURE ONLY.  Forced in front of camera_models/src/camera_models/CataCamera.cc by oracle/camera.mk: the one OpenCV name that
// file needs beyond the stand-ins of refshim/opencv2, cv::SVD::solveZ, used by CataCamera::estimateIntrinsics (:418) -- calibration, never
// called by the tracker.  Only declared: the link turns it into an aborting stub (refshim/gen_stubs.py).
#pragma once
namespace cv {
class Mat;
struct SVD { static void solveZ(const Mat &src, Mat &dst); };
}  // namespace cv
