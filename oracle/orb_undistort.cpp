/*
 * oracle/orb_undistort.cpp — cv::undistortPoints(src, dst, K, D, noArray(), K) of OpenCV 4 (cvUndistortPointsInternal
 * with its default criteria: COUNT, 5 iterations) restated on the CPU (TEST INFRASTRUCTURE, see orb_oracle.h).
 * K and the coefficients are the float values widened to double, missing coefficients are 0, and every operation is
 * rounded on its own (built with -ffp-contract=off); tests/test_undistort_oracle.py pins it bit for bit against cv2.
 * refshim/refshim_cv_undistort.h makes it the cv::undistortPoints of oracle/_ref/libref_frame_undistort.so, so the
 * reference's own Frame::UndistortKeyPoints / ComputeImageBounds run on it there.
 */
#include "undistort_oracle.h"

extern "C" void orc_undistort_points(const float* xy, int n, const float* K4, const float* dist, int n_dist, float* out) {
  double k[14] = {0};
  for (int i = 0; i < n_dist && i < 14; i++) k[i] = dist[i];
  const double fx = K4[0], fy = K4[1], cx = K4[2], cy = K4[3];
  const double ifx = 1. / fx, ify = 1. / fy;
  for (int i = 0; i < n; i++) {
    const double u = xy[2 * i], v = xy[2 * i + 1];
    double x = (u - cx) * ifx, y = (v - cy) * ify;
    const double x0 = x, y0 = y;  // the tilt model is the identity here
    for (int j = 0; j < 5; j++) {
      const double r2 = x * x + y * y;
      const double icdist = (1 + ((k[7] * r2 + k[6]) * r2 + k[5]) * r2) / (1 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2);
      if (icdist < 0) {  // OpenCV 4 (not 3.2): give up and keep the first normalised point
        x = (u - cx) * ifx;
        y = (v - cy) * ify;
        break;
      }
      const double deltaX = 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x) + k[8] * r2 + k[9] * r2 * r2;
      const double deltaY = k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y + k[10] * r2 + k[11] * r2 * r2;
      x = (x0 - deltaX) * icdist;
      y = (y0 - deltaY) * icdist;
    }
    // P = K, R = I: RR = K, so ww = 1
    out[2 * i] = (float)(fx * x + 0 * y + cx);
    out[2 * i + 1] = (float)(0 * x + fy * y + cy);
  }
}
