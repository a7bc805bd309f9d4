/*
 * oracle/undistort_oracle.h — C API of the undistortion restatement (TEST INFRASTRUCTURE, see orb_oracle.h):
 * cv::undistortPoints(src, dst, K, D, noArray(), K) of OpenCV 4 on n points, in oracle/orb_undistort.cpp, built into
 * liborb_undistort.so and into oracle/_ref/libref_frame_undistort.so (oracle/undistort.mk).
 */
#ifndef UNDISTORT_ORACLE_H
#define UNDISTORT_ORACLE_H
#ifdef __cplusplus
extern "C" {
#endif
/* xy: n x 2 floats (out may equal xy); K4 = fx, fy, cx, cy; dist: n_dist coefficients k1 k2 p1 p2 [k3 ..] */
void orc_undistort_points(const float* xy, int n, const float* K4, const float* dist, int n_dist, float* out);
#ifdef __cplusplus
}
#endif
#endif
