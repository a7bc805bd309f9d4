// pnpsolver.cu — EPnP RANSAC for relocalisation candidates: PnPsolver::iterate (src/PnPsolver.cc:240-363) with the
// minimal sets drawn by the caller, on the GPU.  The device restates oracle/pnpsolver.cpp operation by operation: double
// precision throughout EPnP with OpenCV's C API as OpenCV computes it on CV_64F (MulTransposedR's serial sums,
// JacobiSVDImpl_<double> with lapack.cpp's hypot template, SVBkSb for cvInvert / cvSolve), CheckInliers' float / double
// mix, and no libm call on the path (only + - * / sqrt fabs).  Compiled without FMA contraction, so it is bit-identical
// to the restatement in every output, the double R and t included (DESIGN §7).
//
// EPnP runs on a team of threads (a CTA): the per-correspondence loops are strided over the team, every sum the
// reference accumulates stays one serial sum in the reference's order on one thread, and the small solves run on thread
// 0.  So the result does not depend on the team's size, and the 4-point hypotheses and Refine share one code path.
//
// A call is three launches on one stream, no host synchronisation between them; every launch covers the whole batch:
//   k_pnp_hypothesis  one warp per (problem, set): compute_pose on the set's 4 correspondences; R, t (double) and the
//                     reprojection error per hypothesis
//   k_pnp_inliers     one CTA per (problem, set): CheckInliers over every correspondence, the flags as warp ballots into
//                     a bitmask, the count by popc (an integer: no order dependence)
//   k_pnp_scan        one CTA per problem: the reference's serial scan in set order (best on >, an iteration qualifies on
//                     >= min_inliers); a qualifying iteration runs Refine on the CTA: the best mask compacted in index
//                     order, compute_pose over it, CheckInliers over all n; the call returns on more than min_inliers
//                     refined inliers.  Refine depends only on the best mask, so a failed Refine is not repeated until
//                     the mask changes.
// Hypotheses after an early return are computed and discarded.
#include <float.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "jacobi.cuh"

namespace b2s {
namespace pnp {

constexpr int MAX_MATCHES = 65536;
constexpr int MAX_BATCH = 65535;  // gridDim.y of k_pnp_hypothesis / k_pnp_inliers
constexpr int HT = 32;   // threads of a hypothesis team (one warp)
constexpr int CT = 256;  // threads of the per-hypothesis inlier CTAs and of the per-problem scan / Refine CTAs
constexpr int HYP = 13;  // doubles per hypothesis: R 9 (row-major), t 3, reprojection error
constexpr int SCR = 13;  // scratch doubles per correspondence for Refine: pws 3, us 2, alphas 4, pcs 3, one term

struct Prob {
  int n, off, k, offSet, words, offMask, offWords, minInl, maxIts, done, best;
  float fu, fv, uc, vc, th2;
};

struct St {
  int returned, used, doneAfter, bestAfter, noMore, nInl, bestChanged, pad;
  float Tcw[16], bestTcw[16];
};

struct Ptrs {
  const Prob* prob;
  const float *P3Dw, *P2D, *sig, *bestTcwIn;
  const int* sets;
  const uint8_t* bestIn;
  double* hyp;
  int* cnt;
  uint32_t* mask;     // per (problem, set): words
  uint32_t* carried;  // per problem: words, the best mask on entry as bits
  uint32_t* refined;  // per problem: words, the last Refine's inliers
  double* scratch;    // per correspondence: SCR
  int* idx;           // per correspondence: the compacted best mask
  St* st;
  uint8_t *inl, *bestOut;  // out: per correspondence
};

// The team's per-correspondence arrays (the reference's pws, us, alphas, pcs) and one term per correspondence
struct Pts {
  double *pws, *us, *alphas, *pcs, *term;
};

// The team's shared state of one compute_pose (the reference's members and locals)
struct PoseSh {
  double cws[4][3], ccs[4][3];
  double pw0tpw0[9], cc_inv[9], abt[9], pc0[3], pw0[3];
  double mtm[144], ut[144], vt[144], d[12];
  double l[60], rho[6];
  double Betas[4][4], rep[4], Rs[4][9], ts[4][3];
  double R[9], t[3], err;
  int neg;
};

// ------------------------------------------------------------------------------------------------ OpenCV's C API
// SVD::compute of a square N x N matrix: At = rows of U^T (the transposed input, rotated), w, Vt
template <int N>
__device__ void svd_at(const double* A, double* At, double* w, double* Vt) {
  for (int i = 0; i < N; i++)
    for (int k = 0; k < N; k++) At[i * N + k] = A[k * N + i];
  jacobi_svd<N>(At, N, w, Vt, N, N, N);
}

// cvInvert(A, D, CV_SVD) of a 3 x 3: SVD::compute, then SVBkSb with b = null
__device__ void invert3_svd(const double* A, double* D) {
  double At[9], w[3], Vt[9];
  svd_at<3>(A, At, w, Vt);
  double threshold = 0;
  for (int i = 0; i < 3; i++) threshold += w[i];
  threshold *= DBL_EPSILON * 2;
  for (int i = 0; i < 9; i++) D[i] = 0;
  for (int i = 0; i < 3; i++) {
    double wi = w[i];
    if (fabs(wi) <= threshold) continue;
    wi = 1 / wi;
    double buf[3];
    for (int j = 0; j < 3; j++) buf[j] = At[i * 3 + j] * wi;
    for (int r = 0; r < 3; r++) {
      const double s = Vt[i * 3 + r];
      for (int j = 0; j < 3; j++) D[r * 3 + j] = D[r * 3 + j] + s * buf[j];
    }
  }
}

// cvSolve(A, b, x, CV_SVD) of a 6 x N system: JacobiSVD of A^T, then SVBkSb with u transposed and one right-hand side
template <int N>
__device__ void solve6_svd(const double* A, const double* b, double* x) {
  double At[N * 6], w[N], Vt[N * N];
  for (int i = 0; i < N; i++)
    for (int k = 0; k < 6; k++) At[i * 6 + k] = A[k * N + i];
  jacobi_svd<N>(At, 6, w, Vt, 6, N, N);
  double threshold = 0;
  for (int i = 0; i < N; i++) threshold += w[i];
  threshold *= DBL_EPSILON * 2;
  for (int j = 0; j < N; j++) x[j] = 0;
  for (int i = 0; i < N; i++) {
    double wi = w[i];
    if (fabs(wi) <= threshold) continue;
    wi = 1 / wi;
    double s = 0;
    for (int j = 0; j < 6; j++) s += At[i * 6 + j] * b[j];
    s *= wi;
    for (int j = 0; j < N; j++) x[j] = x[j] + s * Vt[i * N + j];
  }
}

// ------------------------------------------------------------------------------------------------ EPnP (one thread)
__device__ __forceinline__ double dot3(const double* v1, const double* v2) {
  return v1[0] * v2[0] + v1[1] * v2[1] + v1[2] * v2[2];
}
__device__ __forceinline__ double dist2(const double* p1, const double* p2) {
  return (p1[0] - p2[0]) * (p1[0] - p2[0]) + (p1[1] - p2[1]) * (p1[1] - p2[1]) + (p1[2] - p2[2]) * (p1[2] - p2[2]);
}

__device__ void find_betas_approx_1(const double* L, const double* rho, double* betas) {
  double l_6x4[24], b4[4];
  for (int i = 0; i < 6; i++) {
    l_6x4[4 * i] = L[10 * i];
    l_6x4[4 * i + 1] = L[10 * i + 1];
    l_6x4[4 * i + 2] = L[10 * i + 3];
    l_6x4[4 * i + 3] = L[10 * i + 6];
  }
  solve6_svd<4>(l_6x4, rho, b4);
  if (b4[0] < 0) {
    betas[0] = sqrt(-b4[0]);
    betas[1] = -b4[1] / betas[0];
    betas[2] = -b4[2] / betas[0];
    betas[3] = -b4[3] / betas[0];
  } else {
    betas[0] = sqrt(b4[0]);
    betas[1] = b4[1] / betas[0];
    betas[2] = b4[2] / betas[0];
    betas[3] = b4[3] / betas[0];
  }
}

__device__ void find_betas_approx_2(const double* L, const double* rho, double* betas) {
  double l_6x3[18], b3[3];
  for (int i = 0; i < 6; i++)
    for (int j = 0; j < 3; j++) l_6x3[3 * i + j] = L[10 * i + j];
  solve6_svd<3>(l_6x3, rho, b3);
  if (b3[0] < 0) {
    betas[0] = sqrt(-b3[0]);
    betas[1] = (b3[2] < 0) ? sqrt(-b3[2]) : 0.0;
  } else {
    betas[0] = sqrt(b3[0]);
    betas[1] = (b3[2] > 0) ? sqrt(b3[2]) : 0.0;
  }
  if (b3[1] < 0) betas[0] = -betas[0];
  betas[2] = 0.0;
  betas[3] = 0.0;
}

__device__ void find_betas_approx_3(const double* L, const double* rho, double* betas) {
  double l_6x5[30], b5[5];
  for (int i = 0; i < 6; i++)
    for (int j = 0; j < 5; j++) l_6x5[5 * i + j] = L[10 * i + j];
  solve6_svd<5>(l_6x5, rho, b5);
  if (b5[0] < 0) {
    betas[0] = sqrt(-b5[0]);
    betas[1] = (b5[2] < 0) ? sqrt(-b5[2]) : 0.0;
  } else {
    betas[0] = sqrt(b5[0]);
    betas[1] = (b5[2] > 0) ? sqrt(b5[2]) : 0.0;
  }
  if (b5[1] < 0) betas[0] = -betas[0];
  betas[2] = b5[3] / betas[0];
  betas[3] = 0.0;
}

__device__ void compute_L_6x10(const double* ut, double* l_6x10) {
  const double* v[4] = {ut + 12 * 11, ut + 12 * 10, ut + 12 * 9, ut + 12 * 8};
  double dv[4][6][3];
  for (int i = 0; i < 4; i++) {
    int a = 0, b = 1;
    for (int j = 0; j < 6; j++) {
      dv[i][j][0] = v[i][3 * a] - v[i][3 * b];
      dv[i][j][1] = v[i][3 * a + 1] - v[i][3 * b + 1];
      dv[i][j][2] = v[i][3 * a + 2] - v[i][3 * b + 2];
      b++;
      if (b > 3) {
        a++;
        b = a + 1;
      }
    }
  }
  for (int i = 0; i < 6; i++) {
    double* row = l_6x10 + 10 * i;
    row[0] = dot3(dv[0][i], dv[0][i]);
    row[1] = 2.0f * dot3(dv[0][i], dv[1][i]);
    row[2] = dot3(dv[1][i], dv[1][i]);
    row[3] = 2.0f * dot3(dv[0][i], dv[2][i]);
    row[4] = 2.0f * dot3(dv[1][i], dv[2][i]);
    row[5] = dot3(dv[2][i], dv[2][i]);
    row[6] = 2.0f * dot3(dv[0][i], dv[3][i]);
    row[7] = 2.0f * dot3(dv[1][i], dv[3][i]);
    row[8] = 2.0f * dot3(dv[2][i], dv[3][i]);
    row[9] = dot3(dv[3][i], dv[3][i]);
  }
}

// qr_solve (:1251-1385) for the 6 x 4 Gauss-Newton system.  The eta scan reads rows k..4 (not the last); where a
// column's eta is 0 the reference returns with X unwritten, so X keeps the previous step's increment (0 at the first)
__device__ void qr_solve(double* pA, double* b, double* pX) {
  const int nr = 6, nc = 4;
  double A1[4], A2[4];
  double* ppAkk = pA;
  for (int k = 0; k < nc; k++) {
    double* ppAik = ppAkk;
    double eta = fabs(*ppAik);
    for (int i = k + 1; i < nr; i++) {
      const double elt = fabs(*ppAik);
      if (eta < elt) eta = elt;
      ppAik += nc;
    }
    if (eta == 0) return;
    double sum = 0.0;
    const double inv_eta = 1. / eta;
    ppAik = ppAkk;
    for (int i = k; i < nr; i++) {
      *ppAik *= inv_eta;
      sum += *ppAik * *ppAik;
      ppAik += nc;
    }
    double sigma = sqrt(sum);
    if (*ppAkk < 0) sigma = -sigma;
    *ppAkk += sigma;
    A1[k] = sigma * *ppAkk;
    A2[k] = -eta * sigma;
    for (int j = k + 1; j < nc; j++) {
      double* q = ppAkk;
      double s = 0;
      for (int i = k; i < nr; i++) {
        s += *q * q[j - k];
        q += nc;
      }
      const double tau = s / A1[k];
      q = ppAkk;
      for (int i = k; i < nr; i++) {
        q[j - k] -= tau * *q;
        q += nc;
      }
    }
    ppAkk += nc + 1;
  }
  double* ppAjj = pA;
  for (int j = 0; j < nc; j++) {
    double* ppAij = ppAjj;
    double tau = 0;
    for (int i = j; i < nr; i++) {
      tau += *ppAij * b[i];
      ppAij += nc;
    }
    tau /= A1[j];
    ppAij = ppAjj;
    for (int i = j; i < nr; i++) {
      b[i] -= tau * *ppAij;
      ppAij += nc;
    }
    ppAjj += nc + 1;
  }
  pX[nc - 1] = b[nc - 1] / A2[nc - 1];
  for (int i = nc - 2; i >= 0; i--) {
    const double* ppAij = pA + i * nc + (i + 1);
    double sum = 0;
    for (int j = i + 1; j < nc; j++) {
      sum += *ppAij * pX[j];
      ppAij++;
    }
    pX[i] = (b[i] - sum) / A2[i];
  }
}

__device__ void gauss_newton(const double* L, const double* rho, double* betas) {
  double a[24], b[6], x[4] = {0, 0, 0, 0};
  for (int k = 0; k < 5; k++) {
    for (int i = 0; i < 6; i++) {  // compute_A_and_b_gauss_newton
      const double* rowL = L + i * 10;
      double* rowA = a + i * 4;
      rowA[0] = 2 * rowL[0] * betas[0] + rowL[1] * betas[1] + rowL[3] * betas[2] + rowL[6] * betas[3];
      rowA[1] = rowL[1] * betas[0] + 2 * rowL[2] * betas[1] + rowL[4] * betas[2] + rowL[7] * betas[3];
      rowA[2] = rowL[3] * betas[0] + rowL[4] * betas[1] + 2 * rowL[5] * betas[2] + rowL[8] * betas[3];
      rowA[3] = rowL[6] * betas[0] + rowL[7] * betas[1] + rowL[8] * betas[2] + 2 * rowL[9] * betas[3];
      b[i] = rho[i] - (rowL[0] * betas[0] * betas[0] + rowL[1] * betas[0] * betas[1] + rowL[2] * betas[1] * betas[1] +
                       rowL[3] * betas[0] * betas[2] + rowL[4] * betas[1] * betas[2] + rowL[5] * betas[2] * betas[2] +
                       rowL[6] * betas[0] * betas[3] + rowL[7] * betas[1] * betas[3] + rowL[8] * betas[2] * betas[3] +
                       rowL[9] * betas[3] * betas[3]);
    }
    qr_solve(a, b, x);
    for (int i = 0; i < 4; i++) betas[i] += x[i];
  }
}

// ------------------------------------------------------------------------------------------------ EPnP (a team)
// Entry e of the upper triangle of a c x c matrix, row by row
__device__ __forceinline__ void upper(int e, int c, int& a, int& b) {
  a = 0;
  while (e >= c - a) e -= c - a, a++;
  b = a + e;
}

// Entry (r, c) of fill_M's M (2n x 12)
__device__ __forceinline__ double m_entry(const Pts& p, double fu, double fv, double uc, double vc, int r, int c) {
  const int i = r >> 1, j = c / 3, q = c - 3 * j;
  const double as = p.alphas[4 * i + j];
  if ((r & 1) == 0) return q == 0 ? as * fu : q == 1 ? 0.0 : as * (uc - p.us[2 * i]);
  return q == 0 ? 0.0 : q == 1 ? as * fv : as * (vc - p.us[2 * i + 1]);
}

// compute_R_and_t (:917-932) for Betas[x]; leaves Rs[x], ts[x], rep[x]
__device__ void compute_R_and_t(int n, const Pts& p, PoseSh& S, int x, double fu, double fv, double uc, double vc) {
  const int tid = threadIdx.x, nt = blockDim.x;
  if (tid == 0) {  // compute_ccs
    for (int i = 0; i < 4; i++) S.ccs[i][0] = S.ccs[i][1] = S.ccs[i][2] = 0.0f;
    for (int i = 0; i < 4; i++) {
      const double* v = S.ut + 12 * (11 - i);
      for (int j = 0; j < 4; j++)
        for (int k = 0; k < 3; k++) S.ccs[j][k] += S.Betas[x][i] * v[3 * j + k];
    }
  }
  __syncthreads();
  for (int i = tid; i < n; i += nt) {  // compute_pcs
    const double* a = p.alphas + 4 * i;
    for (int j = 0; j < 3; j++)
      p.pcs[3 * i + j] = a[0] * S.ccs[0][j] + a[1] * S.ccs[1][j] + a[2] * S.ccs[2][j] + a[3] * S.ccs[3][j];
  }
  __syncthreads();
  // solve_for_sign: the first correspondence's depth decides (ccs is negated too but read no more)
  const bool neg = p.pcs[2] < 0.0;
  __syncthreads();
  if (neg)
    for (int i = tid; i < 3 * n; i += nt) p.pcs[i] = -p.pcs[i];
  __syncthreads();
  // estimate_R_and_t: the centroids, then ABt, each a serial sum in correspondence order
  if (tid < 6) {
    const double* src = tid < 3 ? p.pcs : p.pws;
    const int j = tid % 3;
    double s = 0.0;
    for (int i = 0; i < n; i++) s += src[3 * i + j];
    (tid < 3 ? S.pc0 : S.pw0)[j] = s / n;
  }
  __syncthreads();
  if (tid < 9) {
    const int j = tid / 3, c = tid % 3;
    double s = 0;
    for (int i = 0; i < n; i++) s += (p.pcs[3 * i + j] - S.pc0[j]) * (p.pws[3 * i + c] - S.pw0[c]);
    S.abt[tid] = s;
  }
  __syncthreads();
  if (tid == 0) {
    double At[9], d[3], Vt[9], u[9], v[9];
    svd_at<3>(S.abt, At, d, Vt);  // cvSVD(ABt, D, U, V, CV_SVD_MODIFY_A): U = At^T, V = Vt^T
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) {
        u[3 * i + j] = At[3 * j + i];
        v[3 * i + j] = Vt[3 * j + i];
      }
    double* R = S.Rs[x];
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) R[3 * i + j] = dot3(u + 3 * i, v + 3 * j);
    const double det = R[0] * R[4] * R[8] + R[1] * R[5] * R[6] + R[2] * R[3] * R[7] - R[2] * R[4] * R[6] -
                       R[1] * R[3] * R[8] - R[0] * R[5] * R[7];
    if (det < 0) {
      R[6] = -R[6];
      R[7] = -R[7];
      R[8] = -R[8];
    }
    for (int i = 0; i < 3; i++) S.ts[x][i] = S.pc0[i] - dot3(R + 3 * i, S.pw0);
  }
  __syncthreads();
  // reprojection_error: the terms in parallel, their sum serial in correspondence order
  const double* R = S.Rs[x];
  const double* t = S.ts[x];
  for (int i = tid; i < n; i += nt) {
    const double* pw = p.pws + 3 * i;
    const double Xc = dot3(R, pw) + t[0];
    const double Yc = dot3(R + 3, pw) + t[1];
    const double inv_Zc = 1.0 / (dot3(R + 6, pw) + t[2]);
    const double ue = uc + fu * Xc * inv_Zc;
    const double ve = vc + fv * Yc * inv_Zc;
    const double u = p.us[2 * i], v = p.us[2 * i + 1];
    p.term[i] = sqrt((u - ue) * (u - ue) + (v - ve) * (v - ve));
  }
  __syncthreads();
  if (tid == 0) {
    double sum2 = 0.0;
    for (int i = 0; i < n; i++) sum2 += p.term[i];
    S.rep[x] = sum2 / n;
  }
  __syncthreads();
}

// compute_pose (:684-759) of the n correspondences in p.pws / p.us; leaves S.R, S.t, S.err
__device__ void compute_pose(int n, const Pts& p, PoseSh& S, float fuf, float fvf, float ucf, float vcf) {
  const double fu = fuf, fv = fvf, uc = ucf, vc = vcf;
  const int tid = threadIdx.x, nt = blockDim.x;
  // choose_control_points: the centroid, then PW0^T PW0 (cvMulTransposed), each entry a serial sum
  if (tid < 3) {
    double s = 0;
    for (int i = 0; i < n; i++) s += p.pws[3 * i + tid];
    S.cws[0][tid] = s / n;
  }
  __syncthreads();
  if (tid < 6) {
    int a, b;
    upper(tid, 3, a, b);
    double s = 0;
    for (int i = 0; i < n; i++) s += (p.pws[3 * i + a] - S.cws[0][a]) * (p.pws[3 * i + b] - S.cws[0][b]);
    S.pw0tpw0[3 * a + b] = S.pw0tpw0[3 * b + a] = s;
  }
  __syncthreads();
  if (tid == 0) {
    double uct[9], dc[3], vt[9];
    svd_at<3>(S.pw0tpw0, uct, dc, vt);  // cvSVD(.., CV_SVD_MODIFY_A | CV_SVD_U_T): UCt = the rows of At
    for (int i = 1; i < 4; i++) {
      const double k = sqrt(dc[i - 1] / n);
      for (int j = 0; j < 3; j++) S.cws[i][j] = S.cws[0][j] + k * uct[3 * (i - 1) + j];
    }
    double cc[9];  // compute_barycentric_coordinates
    for (int i = 0; i < 3; i++)
      for (int j = 1; j < 4; j++) cc[3 * i + j - 1] = S.cws[j][i] - S.cws[0][i];
    invert3_svd(cc, S.cc_inv);
  }
  __syncthreads();
  for (int i = tid; i < n; i += nt) {
    const double* pi = p.pws + 3 * i;
    double* a = p.alphas + 4 * i;
    const double* ci = S.cc_inv;
    for (int j = 0; j < 3; j++)
      a[1 + j] = ci[3 * j] * (pi[0] - S.cws[0][0]) + ci[3 * j + 1] * (pi[1] - S.cws[0][1]) +
                 ci[3 * j + 2] * (pi[2] - S.cws[0][2]);
    a[0] = 1.0f - a[1] - a[2] - a[3];
  }
  __syncthreads();
  // M^T M (cvMulTransposed of fill_M's 2n x 12 M): the 78 entries of the upper triangle, each a serial sum over rows
  for (int e = tid; e < 78; e += nt) {
    int a, b;
    upper(e, 12, a, b);
    double s = 0;
    for (int r = 0; r < 2 * n; r++) s += m_entry(p, fu, fv, uc, vc, r, a) * m_entry(p, fu, fv, uc, vc, r, b);
    S.mtm[12 * a + b] = S.mtm[12 * b + a] = s;
  }
  __syncthreads();
  if (tid == 0) {
    svd_at<12>(S.mtm, S.ut, S.d, S.vt);  // cvSVD(MtM, D, Ut, 0, CV_SVD_MODIFY_A | CV_SVD_U_T)
    compute_L_6x10(S.ut, S.l);
    S.rho[0] = dist2(S.cws[0], S.cws[1]);
    S.rho[1] = dist2(S.cws[0], S.cws[2]);
    S.rho[2] = dist2(S.cws[0], S.cws[3]);
    S.rho[3] = dist2(S.cws[1], S.cws[2]);
    S.rho[4] = dist2(S.cws[1], S.cws[3]);
    S.rho[5] = dist2(S.cws[2], S.cws[3]);
    find_betas_approx_1(S.l, S.rho, S.Betas[1]);
    gauss_newton(S.l, S.rho, S.Betas[1]);
    find_betas_approx_2(S.l, S.rho, S.Betas[2]);
    gauss_newton(S.l, S.rho, S.Betas[2]);
    find_betas_approx_3(S.l, S.rho, S.Betas[3]);
    gauss_newton(S.l, S.rho, S.Betas[3]);
  }
  __syncthreads();
  for (int x = 1; x <= 3; x++) compute_R_and_t(n, p, S, x, fu, fv, uc, vc);
  if (tid == 0) {
    int N = 1;
    if (S.rep[2] < S.rep[1]) N = 2;
    if (S.rep[3] < S.rep[N]) N = 3;
    for (int i = 0; i < 9; i++) S.R[i] = S.Rs[N][i];
    for (int i = 0; i < 3; i++) S.t[i] = S.ts[N][i];
    S.err = S.rep[N];
  }
  __syncthreads();
}

// CheckInliers (:421-458) of (R, t) over the problem's n correspondences: bits into mask (words), returns the count
// (every thread)
__device__ int check_inliers(const Ptrs& a, const Prob& P, const double* R, const double* t, uint32_t* mask,
                             int* count) {
  const int tid = threadIdx.x, lane = tid & 31;
  if (tid == 0) *count = 0;
  __syncthreads();
  const double uc = P.uc, vc = P.vc, fu = P.fu, fv = P.fv;
  int mine = 0;
  for (int base = 0; base < P.n; base += blockDim.x) {
    const int i = base + tid;
    bool in = false;
    if (i < P.n) {
      const size_t q = (size_t)P.off + i;
      const float x = a.P3Dw[3 * q], y = a.P3Dw[3 * q + 1], z = a.P3Dw[3 * q + 2];
      const float Xc = R[0] * x + R[1] * y + R[2] * z + t[0];
      const float Yc = R[3] * x + R[4] * y + R[5] * z + t[1];
      const float invZc = 1 / (R[6] * x + R[7] * y + R[8] * z + t[2]);
      const double ue = uc + fu * Xc * invZc;
      const double ve = vc + fv * Yc * invZc;
      const float distX = a.P2D[2 * q] - ue;
      const float distY = a.P2D[2 * q + 1] - ve;
      const float error2 = distX * distX + distY * distY;
      in = error2 < a.sig[q] * P.th2;
    }
    const uint32_t b = __ballot_sync(0xffffffffu, in);
    if (lane == 0 && i < P.n) mask[i >> 5] = b;
    mine += lane == 0 ? __popc(b) : 0;
  }
  if (lane == 0) atomicAdd(count, mine);
  __syncthreads();
  const int c = *count;
  __syncthreads();
  return c;
}

__device__ __forceinline__ void to_Tcw(const double* R, const double* t, float* T) {
  for (int i = 0; i < 16; i++) T[i] = (i % 5 == 0) ? 1.f : 0.f;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) T[4 * r + c] = (float)R[3 * r + c];
    T[4 * r + 3] = (float)t[r];
  }
}

__device__ __forceinline__ bool runs(const Prob& P) { return P.n >= P.minInl; }

// ------------------------------------------------------------------------------------------------ kernels
__global__ void __launch_bounds__(HT) k_pnp_hypothesis(Ptrs a) {
  const Prob P = a.prob[blockIdx.y];
  const int j = blockIdx.x;
  if (j >= P.k || !runs(P)) return;
  __shared__ PoseSh S;
  __shared__ double arr[4 * SCR];
  const Pts p = {arr, arr + 12, arr + 20, arr + 36, arr + 48};
  const int* set = a.sets + 4 * (size_t)(P.offSet + j);
  if (threadIdx.x < 4) {  // add_correspondence in draw order
    const size_t q = (size_t)P.off + set[threadIdx.x];
    for (int c = 0; c < 3; c++) p.pws[3 * threadIdx.x + c] = a.P3Dw[3 * q + c];
    for (int c = 0; c < 2; c++) p.us[2 * threadIdx.x + c] = a.P2D[2 * q + c];
  }
  __syncthreads();
  compute_pose(4, p, S, P.fu, P.fv, P.uc, P.vc);
  double* out = a.hyp + (size_t)HYP * (P.offSet + j);
  if (threadIdx.x < 9) out[threadIdx.x] = S.R[threadIdx.x];
  if (threadIdx.x < 3) out[9 + threadIdx.x] = S.t[threadIdx.x];
  if (threadIdx.x == 0) out[12] = S.err;
}

__global__ void __launch_bounds__(CT) k_pnp_inliers(Ptrs a) {
  const Prob P = a.prob[blockIdx.y];
  const int j = blockIdx.x;
  if (j >= P.k || !runs(P)) return;
  __shared__ double Rt[12];
  __shared__ int count;
  const double* h = a.hyp + (size_t)HYP * (P.offSet + j);
  if (threadIdx.x < 12) Rt[threadIdx.x] = h[threadIdx.x];
  __syncthreads();
  const int c = check_inliers(a, P, Rt, Rt + 9, a.mask + P.offMask + (size_t)j * P.words, &count);
  if (threadIdx.x == 0) a.cnt[P.offSet + j] = c;
}

__global__ void __launch_bounds__(CT) k_pnp_scan(Ptrs a) {
  const Prob P = a.prob[blockIdx.x];
  __shared__ PoseSh S;
  __shared__ int count, part[CT + 1];
  __shared__ St out;
  const int tid = threadIdx.x;
  uint32_t* carried = a.carried + P.offWords;
  uint32_t* refined = a.refined + P.offWords;
  // the best mask on entry, as bits
  for (int w = tid; w < P.words; w += CT) {
    uint32_t b = 0;
    for (int l = 0; l < 32 && 32 * w + l < P.n; l++) b |= (a.bestIn[(size_t)P.off + 32 * w + l] != 0 ? 1u : 0u) << l;
    carried[w] = b;
  }
  if (tid == 0) {
    out.returned = out.used = out.noMore = out.nInl = out.bestChanged = 0;
    for (int i = 0; i < 16; i++) out.bestTcw[i] = a.bestTcwIn[16 * (size_t)blockIdx.x + i];
  }
  __syncthreads();
  // the scan: every thread keeps the same copy of the state (it reads only the counts), so Refine runs on the CTA
  int it = P.done, best = P.best, cur = 0, bestIdx = -1, version = 0, failedVersion = -1, nRef = 0;
  const uint32_t* bestMask = carried;
  bool returned = false;
  if (runs(P)) {
    while (cur < P.k) {  // k = max(nIterations, max_its - iterations_done): the reference's || condition
      const int j = cur;
      cur++;
      it++;
      const int ni = a.cnt[P.offSet + j];
      if (ni < P.minInl) continue;
      if (ni > best) {
        best = ni;
        bestIdx = j;
        bestMask = a.mask + P.offMask + (size_t)j * P.words;
        version++;
      }
      if (failedVersion == version) continue;  // Refine of this mask already failed: it would fail again
      // Refine (:366-418): the best mask compacted in index order
      {
        const int w0 = (int)((long long)P.words * tid / CT), w1 = (int)((long long)P.words * (tid + 1) / CT);
        int c = 0;
        for (int w = w0; w < w1; w++) c += __popc(bestMask[w]);
        part[tid + 1] = c;
        __syncthreads();
        if (tid == 0) {
          part[0] = 0;
          for (int i = 1; i <= CT; i++) part[i] += part[i - 1];
        }
        __syncthreads();
        int o = part[tid];
        for (int w = w0; w < w1; w++)
          for (uint32_t b = bestMask[w]; b; b &= b - 1) a.idx[(size_t)P.off + o++] = 32 * w + __ffs(b) - 1;
        __syncthreads();
      }
      const int m = part[CT];
      double* scr = a.scratch + (size_t)SCR * P.off;
      const Pts p = {scr, scr + 3 * (size_t)m, scr + 5 * (size_t)m, scr + 9 * (size_t)m, scr + 12 * (size_t)m};
      for (int i = tid; i < m; i += CT) {
        const size_t q = (size_t)P.off + a.idx[(size_t)P.off + i];
        for (int c = 0; c < 3; c++) p.pws[3 * i + c] = a.P3Dw[3 * q + c];
        for (int c = 0; c < 2; c++) p.us[2 * i + c] = a.P2D[2 * q + c];
      }
      __syncthreads();
      compute_pose(m, p, S, P.fu, P.fv, P.uc, P.vc);
      nRef = check_inliers(a, P, S.R, S.t, refined, &count);
      if (nRef > P.minInl) {
        returned = true;
        break;
      }
      failedVersion = version;
    }
  }
  const bool noMore = !runs(P) || (!returned && it >= P.maxIts);
  const bool retBest = runs(P) && noMore && best >= P.minInl;
  const uint32_t* retMask = returned ? refined : retBest ? bestMask : nullptr;
  if (tid == 0) {
    out.returned = returned || retBest;
    out.used = cur;
    out.doneAfter = it;
    out.bestAfter = best;
    out.noMore = noMore;
    out.bestChanged = bestIdx >= 0;
    if (bestIdx >= 0) {
      const double* h = a.hyp + (size_t)HYP * (P.offSet + bestIdx);
      to_Tcw(h, h + 9, out.bestTcw);
    }
    if (returned) {
      out.nInl = nRef;
      to_Tcw(S.R, S.t, out.Tcw);
    } else if (retBest) {
      out.nInl = best;
      for (int i = 0; i < 16; i++) out.Tcw[i] = out.bestTcw[i];
    }
  }
  __syncthreads();
  if (tid == 0) a.st[blockIdx.x] = out;
  for (int i = tid; i < P.n; i += CT) {
    const size_t q = (size_t)P.off + i;
    a.inl[q] = retMask ? (uint8_t)((retMask[i >> 5] >> (i & 31)) & 1u) : 0;
    a.bestOut[q] = (uint8_t)((bestMask[i >> 5] >> (i & 31)) & 1u);
  }
}

}  // namespace pnp
}  // namespace b2s

using namespace b2s;
using namespace b2s::pnp;

// ================================================================================================ host side
struct b2s_pnpsolver {
  int maxMatches, maxSets, maxBatch, device;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  float lastMs = 0.f;
  Prob* prob = nullptr;
  float *P3Dw = nullptr, *P2D = nullptr, *sig = nullptr, *bestTcw = nullptr;
  int *sets = nullptr, *cnt = nullptr, *idx = nullptr;
  uint8_t *bestIn = nullptr, *inl = nullptr, *bestOut = nullptr;
  double *hyp = nullptr, *scratch = nullptr;
  uint32_t *mask = nullptr, *carried = nullptr, *refined = nullptr;
  St* st = nullptr;
  std::vector<Prob> hProb;
  std::vector<float> hP3Dw, hP2D, hSig, hBestTcw;
  std::vector<int> hSets;
  std::vector<uint8_t> hBestIn, hInl, hBestOut;
  std::vector<St> hSt;
};

extern "C" int b2s_pnpsolver_create(int max_matches, int max_sets, int max_batch, int device, b2s_pnpsolver** out) {
  // the per-set launches put the batch on grid y, and the sets of a problem on grid x
  if (!out || max_matches < 4 || max_matches > MAX_MATCHES || max_sets < 1 || max_batch < 1 || max_batch > MAX_BATCH) {
    set_error("b2s_pnpsolver_create: bad argument (4 <= max_matches <= %d, max_sets >= 1, 1 <= max_batch <= %d)",
              MAX_MATCHES, MAX_BATCH);
    return B2S_ERR_BAD_ARG;
  }
  *out = nullptr;
  int rc = select_device(device);
  if (rc != B2S_OK) return rc;
  b2s_pnpsolver* h = new b2s_pnpsolver();
  h->maxMatches = max_matches;
  h->maxSets = max_sets;
  h->maxBatch = max_batch;
  h->device = device;
  const size_t B = max_batch, NM = (size_t)max_matches * B, NS = (size_t)max_sets * B;
  const size_t WPB = (size_t)((max_matches + 31) / 32) * B, W = (size_t)((max_matches + 31) / 32) * NS;
  cudaError_t e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreate(&h->ev[0]);
  if (e == cudaSuccess) e = cudaEventCreate(&h->ev[1]);
  if (e == cudaSuccess) e = cudaMalloc(&h->prob, B * sizeof(Prob));
  if (e == cudaSuccess) e = cudaMalloc(&h->P3Dw, NM * 3 * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->P2D, NM * 2 * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->sig, NM * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->bestTcw, B * 16 * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->bestIn, NM);
  if (e == cudaSuccess) e = cudaMalloc(&h->sets, NS * 4 * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc(&h->hyp, NS * HYP * sizeof(double));
  if (e == cudaSuccess) e = cudaMalloc(&h->cnt, NS * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc(&h->mask, W * sizeof(uint32_t));
  if (e == cudaSuccess) e = cudaMalloc(&h->carried, WPB * sizeof(uint32_t));
  if (e == cudaSuccess) e = cudaMalloc(&h->refined, WPB * sizeof(uint32_t));
  if (e == cudaSuccess) e = cudaMalloc(&h->scratch, NM * SCR * sizeof(double));
  if (e == cudaSuccess) e = cudaMalloc(&h->idx, NM * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc(&h->st, B * sizeof(St));
  if (e == cudaSuccess) e = cudaMalloc(&h->inl, NM);
  if (e == cudaSuccess) e = cudaMalloc(&h->bestOut, NM);
  if (e != cudaSuccess) {
    set_error("b2s_pnpsolver_create: %s", cudaGetErrorString(e));
    b2s_pnpsolver_destroy(h);
    return B2S_ERR_CUDA;
  }
  *out = h;
  return B2S_OK;
}

extern "C" void b2s_pnpsolver_destroy(b2s_pnpsolver* h) {
  if (!h) return;
  if (h->stream) cudaStreamSynchronize(h->stream);
  for (void* q : {(void*)h->prob, (void*)h->P3Dw, (void*)h->P2D, (void*)h->sig, (void*)h->bestTcw, (void*)h->bestIn,
                  (void*)h->sets, (void*)h->hyp, (void*)h->cnt, (void*)h->mask, (void*)h->carried, (void*)h->refined,
                  (void*)h->scratch, (void*)h->idx, (void*)h->st, (void*)h->inl, (void*)h->bestOut})
    if (q) cudaFree(q);
  for (cudaEvent_t ev : h->ev)
    if (ev) cudaEventDestroy(ev);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

extern "C" float b2s_pnpsolver_last_ms(const b2s_pnpsolver* h) { return h ? h->lastMs : 0.f; }

static int pnp_bad(int i, const char* what) {
  set_error("b2s_pnpsolver_iterate: problem %d: %s", i, what);
  return B2S_ERR_BAD_ARG;
}

extern "C" int b2s_pnpsolver_iterate(b2s_pnpsolver* h, int batch, const b2s_pnpsolver_problem* p,
                                     b2s_pnpsolver_result* r) {
  if (!h || !p || !r || batch < 1) {
    set_error("b2s_pnpsolver_iterate: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  if (batch > h->maxBatch) {
    set_error("b2s_pnpsolver_iterate: batch %d exceeds the handle's capacity %d", batch, h->maxBatch);
    return B2S_ERR_CAPACITY;
  }
  for (int i = 0; i < batch; i++) {
    const b2s_pnpsolver_problem& q = p[i];
    if (q.n > h->maxMatches || q.k > h->maxSets) {
      set_error("b2s_pnpsolver_iterate: problem %d (n = %d, k = %d) exceeds the handle's capacity", i, q.n, q.k);
      return B2S_ERR_CAPACITY;
    }
    if (q.n < 0 || q.max_its < 1 || q.min_set != 4 || q.min_inliers < q.min_set || q.iterations_done < 0 ||
        q.best_inliers < 0 || q.best_inliers > q.n || q.k < 0)
      return pnp_bad(i, "bad argument");
    const bool run = q.n >= q.min_inliers;
    if (run && q.k < std::max(0, q.max_its - q.iterations_done))
      return pnp_bad(i, "k is below max_its - iterations_done (the loop cannot stop before max_its)");
    if (!q.best_Tcw || (q.n > 0 && !r[i].best_mask) ||
        (q.n > 0 && (!q.P3Dw || !q.P2D || !q.sigma2 || !q.best_mask || !r[i].inliers)) || (run && q.k > 0 && !q.sets))
      return pnp_bad(i, "null array");
    int nb = 0;
    for (int c = 0; c < q.n; c++) {
      if (!(q.sigma2[c] >= 0.f && q.sigma2[c] <= FLT_MAX)) return pnp_bad(i, "a sigma2 is negative or not finite");
      nb += q.best_mask[c] != 0;
    }
    if (q.best_inliers > 0 && nb != q.best_inliers) return pnp_bad(i, "best_mask does not hold best_inliers entries");
    if (run)
      for (int j = 0; j < q.k; j++)
        for (int l = 0; l < 4; l++) {
          const int s = q.sets[4 * j + l];
          bool dup = false;
          for (int m = 0; m < l; m++) dup |= q.sets[4 * j + m] == s;
          if (s < 0 || s >= q.n || dup) {
            set_error("b2s_pnpsolver_iterate: problem %d: set %d entry %d = %d (n = %d)", i, j, l, s, q.n);
            return B2S_ERR_BAD_ARG;
          }
        }
  }
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;

  h->hProb.resize((size_t)batch);
  size_t on = 0, os = 0, om = 0, ow = 0;
  int maxK = 0;
  for (int i = 0; i < batch; i++) {
    const b2s_pnpsolver_problem& q = p[i];
    Prob& P = h->hProb[(size_t)i];
    P.n = q.n;
    P.off = (int)on;
    P.k = q.n >= q.min_inliers ? q.k : 0;
    P.offSet = (int)os;
    P.words = (q.n + 31) / 32;
    P.offMask = (int)om;
    P.offWords = (int)ow;
    P.minInl = q.min_inliers;
    P.maxIts = q.max_its;
    P.done = q.iterations_done;
    P.best = q.best_inliers;
    P.fu = q.fu;
    P.fv = q.fv;
    P.uc = q.uc;
    P.vc = q.vc;
    P.th2 = q.th2;
    on += (size_t)q.n;
    os += (size_t)P.k;
    om += (size_t)P.k * P.words;
    ow += (size_t)P.words;
    maxK = std::max(maxK, P.k);
  }
  h->hP3Dw.resize(on * 3);
  h->hP2D.resize(on * 2);
  h->hSig.resize(on);
  h->hBestIn.resize(on);
  h->hBestTcw.resize((size_t)batch * 16);
  h->hSets.resize(os * 4);
  for (int i = 0; i < batch; i++) {
    const b2s_pnpsolver_problem& q = p[i];
    const Prob& P = h->hProb[(size_t)i];
    if (q.n > 0) {
      memcpy(&h->hP3Dw[3 * (size_t)P.off], q.P3Dw, 3 * sizeof(float) * q.n);
      memcpy(&h->hP2D[2 * (size_t)P.off], q.P2D, 2 * sizeof(float) * q.n);
      memcpy(&h->hSig[(size_t)P.off], q.sigma2, sizeof(float) * q.n);
      memcpy(&h->hBestIn[(size_t)P.off], q.best_mask, (size_t)q.n);
    }
    memcpy(&h->hBestTcw[16 * (size_t)i], q.best_Tcw, 16 * sizeof(float));
    if (P.k > 0) memcpy(&h->hSets[4 * (size_t)P.offSet], q.sets, 4 * sizeof(int) * P.k);
  }
  h->hSt.resize((size_t)batch);
  h->hInl.resize(on);
  h->hBestOut.resize(on);

  B2S_CUDA(cudaEventRecord(h->ev[0], s));
  B2S_CUDA(cudaMemcpyAsync(h->prob, h->hProb.data(), (size_t)batch * sizeof(Prob), cudaMemcpyHostToDevice, s));
  B2S_CUDA(cudaMemcpyAsync(h->bestTcw, h->hBestTcw.data(), (size_t)batch * 16 * sizeof(float), cudaMemcpyHostToDevice,
                           s));
  if (on) {
    B2S_CUDA(cudaMemcpyAsync(h->P3Dw, h->hP3Dw.data(), on * 3 * sizeof(float), cudaMemcpyHostToDevice, s));
    B2S_CUDA(cudaMemcpyAsync(h->P2D, h->hP2D.data(), on * 2 * sizeof(float), cudaMemcpyHostToDevice, s));
    B2S_CUDA(cudaMemcpyAsync(h->sig, h->hSig.data(), on * sizeof(float), cudaMemcpyHostToDevice, s));
    B2S_CUDA(cudaMemcpyAsync(h->bestIn, h->hBestIn.data(), on, cudaMemcpyHostToDevice, s));
  }
  if (os) B2S_CUDA(cudaMemcpyAsync(h->sets, h->hSets.data(), os * 4 * sizeof(int), cudaMemcpyHostToDevice, s));
  Ptrs a = {h->prob, h->P3Dw,    h->P2D,     h->sig,     h->bestTcw, h->sets, h->bestIn, h->hyp, h->cnt,
            h->mask, h->carried, h->refined, h->scratch, h->idx,     h->st,   h->inl,    h->bestOut};
  if (maxK > 0) {
    k_pnp_hypothesis<<<dim3(maxK, batch), HT, 0, s>>>(a);
    k_pnp_inliers<<<dim3(maxK, batch), CT, 0, s>>>(a);
  }
  k_pnp_scan<<<batch, CT, 0, s>>>(a);
  B2S_CUDA(cudaGetLastError());
  B2S_CUDA(cudaMemcpyAsync(h->hSt.data(), h->st, (size_t)batch * sizeof(St), cudaMemcpyDeviceToHost, s));
  if (on) {
    B2S_CUDA(cudaMemcpyAsync(h->hInl.data(), h->inl, on, cudaMemcpyDeviceToHost, s));
    B2S_CUDA(cudaMemcpyAsync(h->hBestOut.data(), h->bestOut, on, cudaMemcpyDeviceToHost, s));
  }
  B2S_CUDA(cudaEventRecord(h->ev[1], s));
  B2S_CUDA(cudaStreamSynchronize(s));
  B2S_CUDA(cudaGetLastError());

  for (int i = 0; i < batch; i++) {
    const St& S = h->hSt[(size_t)i];
    const Prob& P = h->hProb[(size_t)i];
    b2s_pnpsolver_result& R = r[i];
    R.returned = S.returned;
    if (S.returned) memcpy(R.Tcw, S.Tcw, sizeof(R.Tcw));
    if (P.n > 0) {
      memcpy(R.inliers, &h->hInl[(size_t)P.off], (size_t)P.n);
      memcpy(R.best_mask, &h->hBestOut[(size_t)P.off], (size_t)P.n);
    }
    R.n_inliers = S.nInl;
    R.no_more = S.noMore;
    R.iterations_used = S.used;
    R.iterations_done = S.doneAfter;
    R.best_inliers = S.bestAfter;
    R.best_changed = S.bestChanged;
    memcpy(R.best_Tcw, S.bestTcw, sizeof(R.best_Tcw));
  }
  float ms = 0.f;
  B2S_CUDA(cudaEventElapsedTime(&ms, h->ev[0], h->ev[1]));
  h->lastMs = ms;
  return B2S_OK;
}
