// TEST INFRASTRUCTURE — CPU restatement of PnPsolver (src/PnPsolver.cc) with the minimal sets as input, and the OpenCV
// C API operations EPnP calls, as OpenCV 4 computes them for CV_64F (cvMulTransposed -> MulTransposedR, cvSVD ->
// JacobiSVDImpl_<double>, cvInvert / cvSolve with CV_SVD -> SVBkSb).  The problem and result are the C ABI's
// (include/b200slam.h).  Built by `make -f pnpsolver.mk` into liborb_pnpsolver.so.
#pragma once
#include <stdint.h>

#include "../include/b200slam.h"

#ifdef __cplusplus
extern "C" {
#endif

// cvMulTransposed(A, D, 1): A rows x cols (row-major), D = A^T A (cols x cols), each entry a serial double sum over the
// rows in row order
void orc_pnp_mul_transposed(const double* A, int rows, int cols, double* D);
// SVD::compute(A, w, u, vt) of a square n x n CV_64F matrix (n <= 12): JacobiSVDImpl_<double>, u = U (n x n)
void orc_pnp_svd(const double* A, int n, double* w, double* u, double* vt);
// cv::invert(A, D, DECOMP_SVD) of a square n x n CV_64F matrix (n <= 12)
void orc_pnp_invert_svd(const double* A, int n, double* D);
// cv::solve(A, b, x, DECOMP_SVD): A rows x cols (rows >= cols, cols <= 12), b rows x 1, x cols x 1
void orc_pnp_solve_svd(const double* A, int rows, int cols, const double* b, double* x);
// SetRansacParameters(probability, minInliers, maxIterations, minSet, epsilon, th2) with N correspondences: the
// resulting mRansacMinInliers and mRansacMaxIts
void orc_pnp_ransac_parameters(int N, double probability, int min_inliers, int max_iterations, int min_set,
                               float epsilon, int* min_inliers_out, int* max_its_out);
// compute_pose on the m correspondences idx[0..m) of P3Dw (n x 3) / P2D (n x 2) with cam = fu, fv, uc, vc: R (9, row-
// major) and t (3) in double as the reference leaves mRi / mti; returns the chosen model's reprojection error
double orc_pnp_compute_pose(const float* P3Dw, const float* P2D, const int* idx, int m, const float* cam, double* R,
                            double* t);
// iterate(nIterations) as the reference runs it on a solver whose state is p (mnIterations, mnBestInliers, mBestTcw,
// mvbBestInliers) and whose draws are p->sets (k = max(nIterations, max_its - iterations_done) of them).  The caller
// validates the problem (b2s_pnpsolver_iterate's rules).  margin (optional): the smallest |error2 - max_error| /
// max_error over every CheckInliers comparison of the call.  hyp (optional, k x 15): each iteration's R, t,
// reprojection error, inlier count and the count of the Refine it ran (-1 for none).
void orc_pnp_iterate(const b2s_pnpsolver_problem* p, b2s_pnpsolver_result* r, double* margin, double* hyp);

#ifdef __cplusplus
}
#endif
