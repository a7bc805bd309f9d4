// TEST INFRASTRUCTURE — CPU restatement of Initializer::Initialize (src/Initializer.cc) with the minimal sets as input,
// and the OpenCV linear algebra it needs (SVD::compute / SVDecomp by one-sided Jacobi, Mat::inv and cv::determinant of
// a 3 x 3 matrix, gemm).  The problem and result are the C ABI's (include/b200slam.h).
// Built by `make -f init.mk` into liborb_init.so.
#pragma once
#include <stdint.h>

#include "../include/b200slam.h"

#ifdef __cplusplus
extern "C" {
#endif

// cv::SVD::compute(A, w, u, vt, flags) of a rows x cols CV_32F matrix (row-major).  full_uv: SVD::FULL_UV.  With
// m = max(rows, cols), n = min(rows, cols) and urows = full_uv ? m : n: w has n entries; rows >= cols: u is rows x urows
// and vt n x n; rows < cols: u is n x n and vt urows x cols.
void orc_svd(const float* A, int rows, int cols, int full_uv, float* w, float* u, float* vt);
// Mat::inv() (DECOMP_LU, closed form for 3 x 3): returns 0 and writes zeros when the double determinant is 0
int orc_inv3(const float* A, float* out);
double orc_det3(const float* A);
// cv::gemm(A, B, alpha, C, 1, D, tA ? GEMM_1_T : 0): A is m x k (k x m when tA), B k x n, C (optional) m x n; float
// sums for the small untransposed products, double otherwise (init.cpp)
void orc_gemm(const float* A, const float* B, const float* C, int m, int k, int n, double alpha, int tA, float* D);

// Initialize(CurrentFrame, vMatches12, R21, t21, vP3D, vbTriangulated) of an Initializer built on the reference frame
// with (sigma, iterations) whose mvSets are p->sets.  The caller validates the problem (b2s_initialize's rules).
int orc_initialize(const b2s_init_problem* p, b2s_init_result* r);
// FindHomography / FindFundamental with mvSets = p->sets: returns the best iteration (-1: none scored above 0); score,
// the best matrix (zeros when none) and n_matches inlier flags
int orc_find(const b2s_init_problem* p, int homography, float* score, float* X, uint8_t* inl);
// ReconstructH / ReconstructF(inl, X, mK, ..., 1.0, 50): fills ret, rt_state, R21, t21, p3d / triangulated (when ret),
// n_hyp, n_good, parallax
int orc_reconstruct(const b2s_init_problem* p, int homography, const uint8_t* inl, const float* X, b2s_init_result* r);

#ifdef __cplusplus
}
#endif
