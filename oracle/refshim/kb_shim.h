// TEST INFRASTRUCTURE ONLY.  Forced in front of camera_models/src/camera_models/EquidistantCamera.cc by oracle/kb.mk (beside cv_svd.h): the
// two things that file needs beyond the stand-ins of mini_eigen.h and opencv2/, supplied here so that those stand-ins stay as they are.
//  * Eigen::EigenSolver<MatrixXd>(A).eigenvalues() and MatrixXcd, as backprojectSymmetric (:784-785) calls them on a companion matrix.  The
//    arithmetic is vo_kb_eigenvalues (oracle/vo_kb.c, linked into the same library): a restatement of Eigen 3.3's RealSchur + EigenSolver
//    for upper Hessenberg matrices up to 9 x 9, which that file describes.  Eigenvalues Eigen would leave unset are 0.  No eigenvectors.
//  * cv::Point2d built from a cv::Point2f, which estimateIntrinsics (:351) asks for: an explicit specialisation of the stand-in's
//    cv::Point_<double>, the same two doubles with the converting constructor added.  estimateIntrinsics is calibration, never called.
#pragma once
#include <complex>
#include "opencv2/opencv.hpp"
#include "mini_eigen.h"

namespace cv {
template <> struct Point_<double> {
    double x, y;
    Point_() : x(0), y(0) {}
    Point_(double x_, double y_) : x(x_), y(y_) {}
    template <typename U> Point_(const Point_<U> &o) : x(double(o.x)), y(double(o.y)) {}
};
}  // namespace cv

extern "C" int vo_kb_eigenvalues(const double *A, int n, double *wr, double *wi);

namespace Eigen {
typedef Matrix<std::complex<double>, Dynamic, Dynamic> MatrixXcd;
template <typename MatrixType> class EigenSolver {
    MatrixXcd ev;
  public:
    template <typename O> explicit EigenSolver(const MatrixBase<O> &m, bool = true) {
        const int n = m.rows();
        assert(n == m.cols() && n >= 1 && n <= 9);
        double a[81], wr[9], wi[9];
        for (int j = 0; j < n; j++) for (int i = 0; i < n; i++) a[j * n + i] = m.coeff(i, j);
        vo_kb_eigenvalues(a, n, wr, wi);
        ev.resize(n, 1);
        for (int i = 0; i < n; i++) ev.coeffRef(i, 0) = std::complex<double>(wr[i], wi[i]);
    }
    const MatrixXcd &eigenvalues() const { return ev; }
};
}  // namespace Eigen
