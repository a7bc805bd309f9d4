// oracle/refshim/refshim_cv_undistort.h — TEST INFRASTRUCTURE ONLY.
// refshim_cv.h with a working cv::undistortPoints, for oracle/_ref/libref_frame_undistort.so (oracle/undistort.mk): the
// reference's monocular and RGB-D Frame constructors reach it through Frame::UndistortKeyPoints and ComputeImageBounds
// when k1 != 0.  refshim_cv.h's own undistortPoints (an abort(): the stereo libraries never undistort) is renamed while
// it is included, and this file defines the real one on the oracle's restatement of OpenCV 4 (oracle/orb_undistort.cpp,
// pinned to cv2 by tests/test_undistort_oracle.py).  Pre-include it before slam_stubs.h.
#pragma once
#define undistortPoints undistortPoints_abort_stand_in
#include "refshim_cv.h"
#undef undistortPoints
#include "../undistort_oracle.h"

namespace cv {
// cv::undistortPoints(src, dst, K, D, R = Mat(), P = K) on an N x 2 CV_32F matrix
inline void undistortPoints(const Mat& src, Mat& dst, const Mat& K, const Mat& D, const Mat& R, const Mat& P) {
  assert(R.empty() && P.data && P.rows == 3 && P.cols == 3 && K.rows == 3 && K.cols == 3);
  (void)R; (void)P;
  const float K4[4] = {K.at<float>(0, 0), K.at<float>(1, 1), K.at<float>(0, 2), K.at<float>(1, 2)};
  std::vector<float> d((size_t)D.rows * D.cols), xy((size_t)src.rows * 2);
  for (int i = 0; i < (int)d.size(); i++) d[i] = D.at<float>(i);
  for (int i = 0; i < src.rows; i++) {
    xy[2 * i] = src.at<float>(i, 0);
    xy[2 * i + 1] = src.at<float>(i, 1);
  }
  orc_undistort_points(xy.data(), src.rows, K4, d.data(), (int)d.size(), xy.data());
  if (dst.rows != src.rows || dst.cols != 2 || !dst.data) dst.create(src.rows, 2, CV_32F);
  for (int i = 0; i < src.rows; i++) {
    dst.at<float>(i, 0) = xy[2 * i];
    dst.at<float>(i, 1) = xy[2 * i + 1];
  }
}
}  // namespace cv
