// TEST INFRASTRUCTURE — CPU restatement of Sim3Solver (src/Sim3Solver.cc) with the minimal sets as input, and the
// OpenCV operations ComputeSim3 needs (cv::reduce, cv::eigen of a symmetric float matrix, cv::Rodrigues, cv::norm,
// Mat::dot, cv::pow, gemm with the second operand transposed).  The problem and result are the C ABI's
// (include/b200slam.h).  Built by `make -f sim3solver.mk` into liborb_sim3solver.so, with init.cpp's orc_gemm.
#pragma once
#include <stdint.h>

#include "../include/b200slam.h"

#ifdef __cplusplus
extern "C" {
#endif

// cv::reduce(P, C, 1, REDUCE_SUM) of a rows x cols CV_32F matrix (row-major): C has rows entries
void orc_s3s_reduce_sum_cols(const float* P, int rows, int cols, float* C);
// cv::eigen(A, eval, evec) of a symmetric n x n CV_32F matrix (n <= 8): the float Jacobi of lapack.cpp, eigenvalues
// sorted descending, eigenvectors as rows of evec (n x n)
void orc_s3s_eigen(const float* A, int n, float* eval, float* evec);
// cv::Rodrigues(v, R) of a CV_32F rotation vector (3 entries) into a 3 x 3 CV_32F matrix: double arithmetic, one rounding
void orc_s3s_rodrigues(const float* v, float* R);
// cv::norm(a) (NORM_L2) and Mat::dot of len CV_32F entries: double accumulators
double orc_s3s_norm(const float* a, int len);
double orc_s3s_dot(const float* a, const float* b, int len);
// cv::pow(a, 2, out) of len CV_32F entries
void orc_s3s_pow2(const float* a, int len, float* out);
// cv::gemm(A, B, 1, noArray(), 0, D, GEMM_2_T): A m x k, B n x k, D m x n (double sums, one rounding)
void orc_s3s_gemm_bt(const float* A, const float* B, int m, int k, int n, float* D);
// SetRansacParameters(probability, minInliers, maxIterations) with N correspondences: the resulting mRansacMaxIts
int orc_s3s_ransac_max_its(int N, double probability, int min_inliers, int max_iterations);
// ComputeSim3(P1, P2) of two 3 x 3 matrices whose columns are the three points: hyp = R12 (9), t12 (3), s12, T12 (16),
// T21 (16) as the reference leaves mR12i, mt12i, ms12i, mT12i, mT21i
void orc_s3s_compute_sim3(const float* P1, const float* P2, int fix_scale, float* hyp);
// iterate(k) as the reference runs it on a solver whose state is p (mnIterations, mnBestInliers) and whose draws are
// p->sets.  The caller validates the problem (b2s_sim3solver_iterate's rules).  margin (optional): the smallest
// |err - threshold| / threshold over every error the call compared.
void orc_s3s_iterate(const b2s_sim3solver_problem* p, b2s_sim3solver_result* r, double* margin);

#ifdef __cplusplus
}
#endif
