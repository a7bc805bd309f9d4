// initializer.cu — monocular initialisation: Initializer::Initialize (src/Initializer.cc:68-231) with the minimal sets
// drawn by the caller, on the GPU.  The device restates oracle/init.cpp operation by operation (float where the reference
// stores CV_32F, double where OpenCV's gemm / dot / norm / SVD accumulate in double) and is compiled without FMA
// contraction, so every output but the parallax is bit-identical to it; the parallax goes through acos in double rounded
// to float where the reference calls glibc's acosf (at most 1 ulp apart).
//
// A call is six launches on one stream, no host synchronisation between them; every launch covers the whole batch:
//   k_init_prepare    one CTA per problem: compact vMatches12 in frame-1 order, Normalize both keypoint sets (the mean
//                     and mean-deviation sums stay serial in keypoint order)
//   k_init_hypothesis one thread per (problem, iteration, model): ComputeH21 (16 x 9 Jacobi SVD) -> T2inv*Hn*T1 and its
//                     inverse, or ComputeF21 (8 x 9 SVD with the basis completion, rank 2 by a 3 x 3 SVD) -> T2t*Fn*T1
//   k_init_score      one CTA per (problem, iteration, model): CheckHomography / CheckFundamental terms in parallel, the
//                     score a serial float sum in match order, inlier flags as bitmasks
//   k_init_select     one thread per problem: the first strict maximum of each model, RH, the chosen model's motion
//                     hypotheses (ReconstructH's 8 or ReconstructF's 4)
//   k_init_checkrt    one CTA per (problem, hypothesis): CheckRT over the inliers in parallel, nGood an integer count, the
//                     parallax from the cos-parallax list sorted in shared memory
//   k_init_decide     one CTA per problem: the reference's winner logic, then vP3D / vbTriangulated of the winner
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
namespace ini {

constexpr int MAX_KEYS = 16384;
constexpr int CT = 256;  // threads of the per-problem / per-hypothesis CTAs

struct Prob {
  int n1, n2, off1, off2, iters, offIt, offInl, w1;  // w1: 32-bit words of one inlier mask
  float K[9];
  float sigma;
};

struct St {
  float T1[9], T2[9];
  int nm;
  float SH, SF, RH;
  int bestH, bestF, model, nhyp, ninl, ret, rtState, chosen;
  float H[9], F[9];
  float R[8][9], t[8][3];
  int ngood[8];
  float par[8];
};

struct Ptrs {
  const Prob* prob;
  const float *kp1, *kp2;
  const int *m12, *sets;
  float *pn1, *pn2;
  int* mt;             // compacted matches (first, second)
  float* hyp;          // per (iteration, model): 18 floats (H21, H12) or 9 (F21)
  float* score;        // per (iteration, model)
  uint32_t* inl;       // per (iteration, model): w1 words
  St* st;
  float* p3dh;         // per (hypothesis, frame-1 keypoint): 3 floats
  uint8_t* goodh;      // per (hypothesis, frame-1 keypoint)
  float* p3d;          // out: per frame-1 keypoint
  uint8_t *tri, *inlH, *inlF;
};

// ------------------------------------------------------------------------------------------------ OpenCV arithmetic
// SVD::compute of a square 3 x 3 (u, w, vt) or, with want_u = false, vt of a 4 x 4 (Triangulate)
template <int N>
__device__ void svd_square(const float* A, float* w, float* u, float* vt, bool want_u) {
  float At[N * N];
  for (int i = 0; i < N; i++)
    for (int k = 0; k < N; k++) At[i * N + k] = A[k * N + i];
  jacobi_svd<N>(At, N, w, vt, N, N, want_u ? N : 0);
  if (want_u)
    for (int k = 0; k < N; k++)
      for (int i = 0; i < N; i++) u[k * N + i] = At[i * N + k];
}

// cv::gemm, flags 0, inner size 3 equal to an outer size: float sums; alpha and C in double
__device__ void mul3(const float* A, const float* B, int m, int n, float* D, double alpha = 1.0,
                     const float* C = nullptr) {
  for (int r = 0; r < m; r++)
    for (int c = 0; c < n; c++) {
      float f = 0;
      for (int q = 0; q < 3; q++) f = f + A[r * 3 + q] * B[q * n + c];
      double v = (double)f * alpha;
      if (C) v += (double)C[r * n + c];
      D[r * n + c] = (float)v;
    }
}
// cv::gemm with GEMM_1_T (3 x 3): double accumulation
__device__ void mul3_t(const float* A, const float* B, int n, float* D, double alpha) {
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < n; c++) {
      double s = 0;
      for (int q = 0; q < 3; q++) s += (double)A[q * 3 + r] * B[q * n + c];
      D[r * n + c] = (float)(s * alpha);
    }
}
__device__ __forceinline__ void scale(float* v, int n, double alpha) {
  const float a = (float)alpha;
  for (int i = 0; i < n; i++) v[i] = v[i] * a;
}
__device__ __forceinline__ double norm3(const float* v) {
  double s = 0;
  for (int i = 0; i < 3; i++) s += (double)v[i] * v[i];
  return sqrt(s);
}
__device__ __forceinline__ double det3(const float* m) {
  return m[0] * ((double)m[4] * m[8] - (double)m[5] * m[7]) - m[1] * ((double)m[3] * m[8] - (double)m[5] * m[6]) +
         m[2] * ((double)m[3] * m[7] - (double)m[4] * m[6]);
}
__device__ void inv3(const float* m, float* o) {
  double d = det3(m);
  if (d == 0.) {
    for (int i = 0; i < 9; i++) o[i] = 0.f;
    return;
  }
  d = 1. / d;
  o[0] = (float)(((double)m[4] * m[8] - (double)m[5] * m[7]) * d);
  o[1] = (float)(((double)m[2] * m[7] - (double)m[1] * m[8]) * d);
  o[2] = (float)(((double)m[1] * m[5] - (double)m[2] * m[4]) * d);
  o[3] = (float)(((double)m[5] * m[6] - (double)m[3] * m[8]) * d);
  o[4] = (float)(((double)m[0] * m[8] - (double)m[2] * m[6]) * d);
  o[5] = (float)(((double)m[2] * m[3] - (double)m[0] * m[5]) * d);
  o[6] = (float)(((double)m[3] * m[7] - (double)m[4] * m[6]) * d);
  o[7] = (float)(((double)m[1] * m[6] - (double)m[0] * m[7]) * d);
  o[8] = (float)(((double)m[0] * m[4] - (double)m[1] * m[3]) * d);
}
__device__ __forceinline__ void eye3(float* T) {
  for (int i = 0; i < 9; i++) T[i] = (i % 4 == 0) ? 1.f : 0.f;
}

// ------------------------------------------------------------------------------------------------ kernels
__global__ void __launch_bounds__(CT) k_init_prepare(Ptrs a) {
  const Prob& P = a.prob[blockIdx.x];
  St& S = a.st[blockIdx.x];
  __shared__ float sm[4];  // meanX, meanY, sX, sY
  for (int f = 0; f < 2; f++) {
    const int N = f ? P.n2 : P.n1;
    const float* kp = f ? a.kp2 + 2 * P.off2 : a.kp1 + 2 * P.off1;
    float* pn = f ? a.pn2 + 2 * P.off2 : a.pn1 + 2 * P.off1;
    if (threadIdx.x == 0) {  // Normalize (:1501-1575): serial float sums in keypoint order
      float meanX = 0, meanY = 0;
      for (int i = 0; i < N; i++) {
        meanX += kp[2 * i];
        meanY += kp[2 * i + 1];
      }
      meanX = meanX / N;
      meanY = meanY / N;
      float meanDevX = 0, meanDevY = 0;
      for (int i = 0; i < N; i++) {
        meanDevX += fabsf(kp[2 * i] - meanX);
        meanDevY += fabsf(kp[2 * i + 1] - meanY);
      }
      meanDevX = meanDevX / N;
      meanDevY = meanDevY / N;
      const float sX = 1.0 / meanDevX;
      const float sY = 1.0 / meanDevY;
      float* T = f ? S.T2 : S.T1;
      eye3(T);
      T[0] = sX;
      T[4] = sY;
      T[2] = -meanX * sX;
      T[5] = -meanY * sY;
      sm[0] = meanX;
      sm[1] = meanY;
      sm[2] = sX;
      sm[3] = sY;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < N; i += CT) {
      pn[2 * i] = (kp[2 * i] - sm[0]) * sm[2];
      pn[2 * i + 1] = (kp[2 * i + 1] - sm[1]) * sm[3];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {  // mvMatches12 in frame-1 order
    int nm = 0;
    const int* m12 = a.m12 + P.off1;
    int* mt = a.mt + 2 * P.off1;
    for (int i = 0; i < P.n1; i++)
      if (m12[i] >= 0) {
        mt[2 * nm] = i;
        mt[2 * nm + 1] = m12[i];
        nm++;
      }
    S.nm = nm;
  }
}

// one thread per (problem, iteration, model); blockIdx.y = problem
__global__ void __launch_bounds__(64) k_init_hypothesis(Ptrs a) {
  const int b = blockIdx.y;
  const Prob& P = a.prob[b];
  const int job = blockIdx.x * blockDim.x + threadIdx.x;
  if (job >= 2 * P.iters) return;
  const int it = job >> 1, model = job & 1;  // 0: H, 1: F
  const St& S = a.st[b];
  const int* mt = a.mt + 2 * P.off1;
  const float *pn1 = a.pn1 + 2 * P.off1, *pn2 = a.pn2 + 2 * P.off2;
  float u1[8], v1[8], u2[8], v2[8];
  for (int j = 0; j < 8; j++) {
    const int idx = a.sets[8 * (P.offIt + it) + j];
    u1[j] = pn1[2 * mt[2 * idx]];
    v1[j] = pn1[2 * mt[2 * idx] + 1];
    u2[j] = pn2[2 * mt[2 * idx + 1]];
    v2[j] = pn2[2 * mt[2 * idx + 1] + 1];
  }
  float* out = a.hyp + 18 * (2 * (size_t)(P.offIt + it) + model);
  float Xn[9], tmp[9], X[9];
  if (model == 0) {
    // ComputeH21: A 16 x 9, At = A^T (9 rows of 16); vt.row(8) = Vt row 8 (u unused: no completion needed)
    float At[9 * 16], w[9], Vt[81];
    for (int i = 0; i < 8; i++) {
      const float r0[9] = {0, 0, 0, -u1[i], -v1[i], -1, v2[i] * u1[i], v2[i] * v1[i], v2[i]};
      const float r1[9] = {u1[i], v1[i], 1, 0, 0, 0, -u2[i] * u1[i], -u2[i] * v1[i], -u2[i]};
      for (int c = 0; c < 9; c++) {
        At[c * 16 + 2 * i] = r0[c];
        At[c * 16 + 2 * i + 1] = r1[c];
      }
    }
    jacobi_svd<9>(At, 16, w, Vt, 16, 9, 0);
    for (int k = 0; k < 9; k++) Xn[k] = Vt[72 + k];
    float T2inv[9];
    inv3(S.T2, T2inv);
    mul3(T2inv, Xn, 3, 3, tmp);
    mul3(tmp, S.T1, 3, 3, X);
    inv3(X, out + 9);
  } else {
    // ComputeF21: A 8 x 9 -> m = 9, n = 8, At = A (8 rows of 9) in a 9-row buffer; vt = At after completing row 8
    float At[9 * 9], w[8], V8[64];
    for (int i = 0; i < 8; i++) {
      const float r[9] = {u2[i] * u1[i], u2[i] * v1[i], u2[i], v2[i] * u1[i], v2[i] * v1[i], v2[i], u1[i], v1[i], 1};
      for (int c = 0; c < 9; c++) At[i * 9 + c] = r[c];
    }
    for (int c = 0; c < 9; c++) At[72 + c] = 0;
    jacobi_svd<8>(At, 9, w, V8, 9, 8, 9);
    float Fpre[9], w3[3], u3[9], vt3[9], UD[9];
    for (int k = 0; k < 9; k++) Fpre[k] = At[72 + k];
    svd_square<3>(Fpre, w3, u3, vt3, true);
    w3[2] = 0;
    const float D[9] = {w3[0], 0, 0, 0, w3[1], 0, 0, 0, w3[2]};
    mul3(u3, D, 3, 3, UD);
    mul3(UD, vt3, 3, 3, Xn);
    float T2t[9];
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) T2t[3 * r + c] = S.T2[3 * c + r];
    mul3(T2t, Xn, 3, 3, tmp);
    mul3(tmp, S.T1, 3, 3, X);
  }
  for (int k = 0; k < 9; k++) out[k] = X[k];
}

// one CTA per (iteration, model) of a problem: blockIdx.x = 2 * it + model, blockIdx.y = problem
__global__ void __launch_bounds__(CT) k_init_score(Ptrs a) {
  const int b = blockIdx.y;
  const Prob& P = a.prob[b];
  const int job = blockIdx.x;
  if (job >= 2 * P.iters) return;
  const int model = job & 1;
  const St& S = a.st[b];
  const int N = S.nm;
  const float* X = a.hyp + 18 * ((size_t)2 * P.offIt + job);
  const int* mt = a.mt + 2 * P.off1;
  const float *kp1 = a.kp1 + 2 * P.off1, *kp2 = a.kp2 + 2 * P.off2;
  uint32_t* inl = a.inl + (size_t)P.offInl + (size_t)job * P.w1;
  __shared__ float terms[2 * CT];
  float score = 0;  // thread 0's
  const float invSigmaSquare = 1.0 / (P.sigma * P.sigma);
  for (int base = 0; base < N; base += CT) {
    const int i = base + threadIdx.x;
    float s1 = 0, s2 = 0;
    bool bIn = false;
    if (i < N) {
      bIn = true;
      const float u1 = kp1[2 * mt[2 * i]], v1 = kp1[2 * mt[2 * i] + 1];
      const float u2 = kp2[2 * mt[2 * i + 1]], v2 = kp2[2 * mt[2 * i + 1] + 1];
      if (model == 0) {  // CheckHomography (:616-809)
        const float th = 5.991;
        const float* Hi = X + 9;
        const float w2in1inv = 1.0 / (Hi[6] * u2 + Hi[7] * v2 + Hi[8]);
        const float u2in1 = (Hi[0] * u2 + Hi[1] * v2 + Hi[2]) * w2in1inv;
        const float v2in1 = (Hi[3] * u2 + Hi[4] * v2 + Hi[5]) * w2in1inv;
        const float chiSquare1 = ((u1 - u2in1) * (u1 - u2in1) + (v1 - v2in1) * (v1 - v2in1)) * invSigmaSquare;
        if (chiSquare1 > th) bIn = false; else s1 = th - chiSquare1;
        const float w1in2inv = 1.0 / (X[6] * u1 + X[7] * v1 + X[8]);
        const float u1in2 = (X[0] * u1 + X[1] * v1 + X[2]) * w1in2inv;
        const float v1in2 = (X[3] * u1 + X[4] * v1 + X[5]) * w1in2inv;
        const float chiSquare2 = ((u2 - u1in2) * (u2 - u1in2) + (v2 - v1in2) * (v2 - v1in2)) * invSigmaSquare;
        if (chiSquare2 > th) bIn = false; else s2 = th - chiSquare2;
      } else {  // CheckFundamental (:813-945)
        const float th = 3.841, thScore = 5.991;
        const float a2 = X[0] * u1 + X[1] * v1 + X[2];
        const float b2 = X[3] * u1 + X[4] * v1 + X[5];
        const float c2 = X[6] * u1 + X[7] * v1 + X[8];
        const float num2 = a2 * u2 + b2 * v2 + c2;
        const float chiSquare1 = num2 * num2 / (a2 * a2 + b2 * b2) * invSigmaSquare;
        if (chiSquare1 > th) bIn = false; else s1 = thScore - chiSquare1;
        const float a1 = X[0] * u2 + X[3] * v2 + X[6];
        const float b1 = X[1] * u2 + X[4] * v2 + X[7];
        const float c1 = X[2] * u2 + X[5] * v2 + X[8];
        const float num1 = a1 * u1 + b1 * v1 + c1;
        const float chiSquare2 = num1 * num1 / (a1 * a1 + b1 * b1) * invSigmaSquare;
        if (chiSquare2 > th) bIn = false; else s2 = thScore - chiSquare2;
      }
    }
    // a term that was not added is 0 here; adding +0.0f to a float sum leaves it unchanged (the sum starts at +0 and
    // terms are >= 0, so it is never -0)
    terms[2 * threadIdx.x] = s1;
    terms[2 * threadIdx.x + 1] = s2;
    const unsigned bits = __ballot_sync(0xffffffffu, bIn);
    if ((threadIdx.x & 31) == 0 && base + (int)threadIdx.x < N) inl[(base + threadIdx.x) >> 5] = bits;
    __syncthreads();
    if (threadIdx.x == 0) {
      const int cnt = min(CT, N - base);
      for (int k = 0; k < 2 * cnt; k++) score += terms[k];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) a.score[(size_t)2 * P.offIt + job] = score;
}

// one thread per problem: FindHomography / FindFundamental's selection, RH, the chosen model's motion hypotheses
__global__ void k_init_select(Ptrs a, int batch) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  const Prob& P = a.prob[b];
  St& S = a.st[b];
  float SH = 0, SF = 0;
  int bh = -1, bf = -1;
  for (int it = 0; it < P.iters; it++) {
    const float sh = a.score[(size_t)2 * (P.offIt + it)], sf = a.score[(size_t)2 * (P.offIt + it) + 1];
    if (sh > SH) { SH = sh; bh = it; }
    if (sf > SF) { SF = sf; bf = it; }
  }
  S.SH = SH;
  S.SF = SF;
  S.bestH = bh;
  S.bestF = bf;
  for (int k = 0; k < 9; k++) {
    S.H[k] = bh >= 0 ? a.hyp[18 * ((size_t)2 * (P.offIt + bh)) + k] : 0.f;
    S.F[k] = bf >= 0 ? a.hyp[18 * ((size_t)2 * (P.offIt + bf) + 1) + k] : 0.f;
  }
  const float RH = SH / (SH + SF);
  S.RH = RH;
  S.model = RH > 0.40 ? 1 : 2;
  S.nhyp = 0;
  S.ret = 0;
  S.rtState = 0;
  S.chosen = -1;
  for (int h = 0; h < 8; h++) {
    S.ngood[h] = 0;
    S.par[h] = 0.f;
  }
  const int best = S.model == 1 ? bh : bf;
  if (best < 0) return;
  const uint32_t* m = a.inl + (size_t)P.offInl + (size_t)(2 * best + (S.model - 1)) * P.w1;
  int N = 0;
  for (int w = 0; w < (S.nm + 31) / 32; w++) N += __popc(m[w]);  // k_init_score writes the words of the nm matches only
  S.ninl = N;
  const float* K = P.K;
  if (S.model == 1) {  // ReconstructH (:1135-1344)
    float invK[9], tmp[9], A[9], w[3], U[9], Vt[9];
    inv3(K, invK);
    mul3(invK, S.H, 3, 3, tmp);
    mul3(tmp, K, 3, 3, A);
    svd_square<3>(A, w, U, Vt, true);
    const float s = det3(U) * det3(Vt);
    const float d1 = w[0], d2 = w[1], d3 = w[2];
    if (d1 / d2 < 1.00001 || d2 / d3 < 1.00001) return;
    const float aux1 = sqrtf((d1 * d1 - d2 * d2) / (d1 * d1 - d3 * d3));
    const float aux3 = sqrtf((d2 * d2 - d3 * d3) / (d1 * d1 - d3 * d3));
    const float x1[] = {aux1, aux1, -aux1, -aux1};
    const float x3[] = {aux3, -aux3, aux3, -aux3};
    const float aux_stheta = sqrtf((d1 * d1 - d2 * d2) * (d2 * d2 - d3 * d3)) / ((d1 + d3) * d2);
    const float ctheta = (d2 * d2 + d1 * d3) / ((d1 + d3) * d2);
    const float stheta[] = {aux_stheta, -aux_stheta, -aux_stheta, aux_stheta};
    const float aux_sphi = sqrtf((d1 * d1 - d2 * d2) * (d2 * d2 - d3 * d3)) / ((d1 - d3) * d2);
    const float cphi = (d1 * d3 - d2 * d2) / ((d1 - d3) * d2);
    const float sphi[] = {aux_sphi, -aux_sphi, -aux_sphi, aux_sphi};
    for (int h = 0; h < 8; h++) {
      const int i = h & 3;
      float Rp[9], URp[9];
      eye3(Rp);
      float tp[3];
      if (h < 4) {
        Rp[0] = ctheta; Rp[2] = -stheta[i]; Rp[6] = stheta[i]; Rp[8] = ctheta;
        tp[0] = x1[i]; tp[1] = 0; tp[2] = -x3[i];
      } else {
        Rp[0] = cphi; Rp[2] = sphi[i]; Rp[4] = -1; Rp[6] = sphi[i]; Rp[8] = -cphi;
        tp[0] = x1[i]; tp[1] = 0; tp[2] = x3[i];
      }
      mul3(U, Rp, 3, 3, URp, (double)s);
      mul3(URp, Vt, 3, 3, S.R[h]);
      scale(tp, 3, h < 4 ? d1 - d3 : d1 + d3);
      mul3(U, tp, 3, 1, S.t[h]);
      scale(S.t[h], 3, 1. / norm3(S.t[h]));
    }
    S.nhyp = 8;
  } else {  // ReconstructF (:956-1033) with DecomposeE (:1798-1843)
    float KtF[9], E[9], w[3], u[9], vt[9], uW[9], R1[9], R2[9];
    mul3_t(K, S.F, 3, KtF, 1.0);
    mul3(KtF, K, 3, 3, E);
    svd_square<3>(E, w, u, vt, true);
    float t[3] = {u[2], u[5], u[8]};
    scale(t, 3, 1. / norm3(t));
    const float W[9] = {0, -1, 0, 1, 0, 0, 0, 0, 1};
    const float Wt[9] = {0, 1, 0, -1, 0, 0, 0, 0, 1};
    mul3(u, W, 3, 3, uW);
    mul3(uW, vt, 3, 3, R1);
    if (det3(R1) < 0) scale(R1, 9, -1.0);
    mul3(u, Wt, 3, 3, uW);
    mul3(uW, vt, 3, 3, R2);
    if (det3(R2) < 0) scale(R2, 9, -1.0);
    for (int h = 0; h < 4; h++) {
      const float* R = (h & 1) ? R2 : R1;
      for (int k = 0; k < 9; k++) S.R[h][k] = R[k];
      for (int k = 0; k < 3; k++) S.t[h][k] = h < 2 ? t[k] : t[k] * -1.0f;
    }
    S.nhyp = 4;
  }
}

// one CTA per (hypothesis, problem): CheckRT (:1578-1785)
__global__ void __launch_bounds__(CT) k_init_checkrt(Ptrs a) {
  extern __shared__ float cosv[];  // the cos-parallax list, padded to a power of two for the sort
  __shared__ int nGood;
  const int h = blockIdx.x, b = blockIdx.y;
  const Prob& P = a.prob[b];
  St& S = a.st[b];
  if (h >= S.nhyp) return;
  const float* R = S.R[h];
  const float* t = S.t[h];
  const float* K = P.K;
  const float fx = K[0], fy = K[4], cx = K[2], cy = K[5];
  const float th2 = 4.0 * (P.sigma * P.sigma);
  float* p3d = a.p3dh + 3 * ((size_t)8 * P.off1 + (size_t)h * P.n1);
  uint8_t* good = a.goodh + (size_t)8 * P.off1 + (size_t)h * P.n1;
  for (int i = threadIdx.x; i < P.n1; i += CT) {
    p3d[3 * i] = p3d[3 * i + 1] = p3d[3 * i + 2] = 0.f;
    good[i] = 0;
  }
  if (threadIdx.x == 0) nGood = 0;
  float P1[12] = {0}, Rt[12], P2[12], O2[3];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) P1[4 * r + c] = K[3 * r + c];
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) Rt[4 * r + c] = R[3 * r + c];
    Rt[4 * r + 3] = t[r];
  }
  mul3(K, Rt, 3, 4, P2);
  mul3_t(R, t, 1, O2, -1.0);
  __syncthreads();
  const int N = S.nm;
  const uint32_t* inl = a.inl + (size_t)P.offInl + (size_t)(2 * (S.model == 1 ? S.bestH : S.bestF) + (S.model - 1)) * P.w1;
  const int* mt = a.mt + 2 * P.off1;
  const float *kp1 = a.kp1 + 2 * P.off1, *kp2 = a.kp2 + 2 * P.off2;
  for (int i = threadIdx.x; i < N; i += CT) {
    if (!((inl[i >> 5] >> (i & 31)) & 1u)) continue;
    const int i1 = mt[2 * i];
    const float* k1 = kp1 + 2 * i1;
    const float* k2 = kp2 + 2 * mt[2 * i + 1];
    float A[16], w[4], vt[16], X[3];
    for (int c = 0; c < 4; c++) {  // Triangulate (:1461-1498)
      A[c] = (float)((double)k1[0] * P1[8 + c] - P1[c]);
      A[4 + c] = (float)((double)k1[1] * P1[8 + c] - P1[4 + c]);
      A[8 + c] = (float)((double)k2[0] * P2[8 + c] - P2[c]);
      A[12 + c] = (float)((double)k2[1] * P2[8 + c] - P2[4 + c]);
    }
    svd_square<4>(A, w, nullptr, vt, false);
    for (int k = 0; k < 3; k++) X[k] = vt[12 + k];
    scale(X, 3, 1. / vt[15]);
    if (!isfinite(X[0]) || !isfinite(X[1]) || !isfinite(X[2])) continue;
    const float n2[3] = {X[0] - O2[0], X[1] - O2[1], X[2] - O2[2]};
    const float dist1 = norm3(X);
    const float dist2 = norm3(n2);
    const double dot = (double)X[0] * n2[0] + (double)X[1] * n2[1] + (double)X[2] * n2[2];
    const float cosParallax = dot / (dist1 * dist2);
    if (X[2] <= 0 && cosParallax < 0.99998) continue;
    float X2[3];
    mul3(R, X, 3, 1, X2, 1.0, t);
    if (X2[2] <= 0 && cosParallax < 0.99998) continue;
    const float invZ1 = 1.0 / X[2];
    const float im1x = fx * X[0] * invZ1 + cx;
    const float im1y = fy * X[1] * invZ1 + cy;
    const float squareError1 = (im1x - k1[0]) * (im1x - k1[0]) + (im1y - k1[1]) * (im1y - k1[1]);
    if (squareError1 > th2) continue;
    const float invZ2 = 1.0 / X2[2];
    const float im2x = fx * X2[0] * invZ2 + cx;
    const float im2y = fy * X2[1] * invZ2 + cy;
    const float squareError2 = (im2x - k2[0]) * (im2x - k2[0]) + (im2y - k2[1]) * (im2y - k2[1]);
    if (squareError2 > th2) continue;
    cosv[atomicAdd(&nGood, 1)] = cosParallax;
    for (int k = 0; k < 3; k++) p3d[3 * i1 + k] = X[k];
    if (cosParallax < 0.99998) good[i1] = 1;
  }
  __syncthreads();
  const int n = nGood;
  int L = 1;
  while (L < n) L <<= 1;
  for (int i = n + threadIdx.x; i < L; i += CT) cosv[i] = INFINITY;
  __syncthreads();
  for (int k = 2; k <= L; k <<= 1)  // bitonic sort, ascending
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < L; i += CT) {
        const int l = i ^ j;
        if (l > i) {
          const float x = cosv[i], y = cosv[l];
          if (((i & k) == 0) == (x > y)) {
            cosv[i] = y;
            cosv[l] = x;
          }
        }
      }
      __syncthreads();
    }
  if (threadIdx.x == 0) {
    S.ngood[h] = n;
    // parallax = acos(vCosParallax[idx])*180/CV_PI with glibc's acosf: acos in double rounded to float (<= 1 ulp)
    S.par[h] = n > 0 ? (float)((float)acos((double)cosv[min(50, n - 1)]) * 180 / 3.1415926535897932384626433832795) : 0.f;
  }
}

// one CTA per problem: the winner logic of ReconstructH (:1347-1431) / ReconstructF (:1029-1125), then the outputs
__global__ void __launch_bounds__(CT) k_init_decide(Ptrs a) {
  const int b = blockIdx.x;
  const Prob& P = a.prob[b];
  St& S = a.st[b];
  __shared__ int chosen;
  if (threadIdx.x == 0) {
    chosen = -1;
    const float minParallax = 1.0;
    const int minTriangulated = 50;
    const int N = S.ninl;
    if (S.nhyp == 8) {
      int bestGood = 0, secondBestGood = 0, bestSolutionIdx = -1;
      float bestParallax = -1;
      for (int i = 0; i < 8; i++) {
        const int nGood = S.ngood[i];
        if (nGood > bestGood) {
          secondBestGood = bestGood;
          bestGood = nGood;
          bestSolutionIdx = i;
          bestParallax = S.par[i];
        } else if (nGood > secondBestGood) {
          secondBestGood = nGood;
        }
      }
      if (secondBestGood < 0.75 * bestGood && bestParallax >= minParallax && bestGood > minTriangulated &&
          bestGood > 0.9 * N)
        chosen = bestSolutionIdx;
    } else if (S.nhyp == 4) {
      S.rtState = -1;
      const int maxGood = max(S.ngood[0], max(S.ngood[1], max(S.ngood[2], S.ngood[3])));
      const int nMinGood = max(static_cast<int>(0.9 * N), minTriangulated);
      int nsimilar = 0;
      for (int i = 0; i < 4; i++)
        if (S.ngood[i] > 0.7 * maxGood) nsimilar++;
      if (!(maxGood < nMinGood || nsimilar > 1))
        for (int i = 0; i < 4; i++)
          if (maxGood == S.ngood[i]) {
            if (S.par[i] > minParallax) chosen = i;
            break;
          }
    }
    if (chosen >= 0) {
      S.ret = 1;
      S.rtState = 1;
    }
    S.chosen = chosen;
  }
  __syncthreads();
  // inlier flags of the best hypotheses
  for (int model = 0; model < 2; model++) {
    const int best = model ? S.bestF : S.bestH;
    uint8_t* o = (model ? a.inlF : a.inlH) + P.off1;
    const uint32_t* m = a.inl + (size_t)P.offInl + (size_t)(2 * best + model) * P.w1;
    for (int i = threadIdx.x; i < S.nm; i += CT) o[i] = best >= 0 ? (uint8_t)((m[i >> 5] >> (i & 31)) & 1u) : 0;
  }
  const int c = chosen;
  if (c < 0) return;
  const float* src = a.p3dh + 3 * ((size_t)8 * P.off1 + (size_t)c * P.n1);
  const uint8_t* g = a.goodh + (size_t)8 * P.off1 + (size_t)c * P.n1;
  for (int i = threadIdx.x; i < P.n1; i += CT) {
    for (int k = 0; k < 3; k++) a.p3d[3 * ((size_t)P.off1 + i) + k] = src[3 * i + k];
    a.tri[P.off1 + i] = g[i];
  }
}

}  // namespace ini
}  // namespace b2s

using namespace b2s;
using namespace b2s::ini;

// ================================================================================================ host side
struct b2s_init_solver {
  int maxKeys, maxIters, maxBatch, device;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  float lastMs = 0.f;
  Prob* prob = nullptr;
  float *kp1 = nullptr, *kp2 = nullptr, *pn1 = nullptr, *pn2 = nullptr, *hyp = nullptr, *score = nullptr;
  int *m12 = nullptr, *sets = nullptr, *mt = nullptr;
  uint32_t* inl = nullptr;
  St* st = nullptr;
  float *p3dh = nullptr, *p3d = nullptr;
  uint8_t *goodh = nullptr, *tri = nullptr, *inlH = nullptr, *inlF = nullptr;
  std::vector<Prob> hProb;
  std::vector<float> hKp1, hKp2, hP3d;
  std::vector<int> hM12, hSets;
  std::vector<St> hSt;
  std::vector<uint8_t> hTri, hInlH, hInlF;
};

extern "C" int b2s_init_create(int max_keys, int max_iterations, int max_batch, int device, b2s_init_solver** out) {
  if (!out || max_keys < 8 || max_keys > MAX_KEYS || max_iterations < 1 || max_batch < 1) {
    set_error("b2s_init_create: bad argument (8 <= max_keys <= %d, max_iterations >= 1, max_batch >= 1)", MAX_KEYS);
    return B2S_ERR_BAD_ARG;
  }
  *out = nullptr;
  int rc = select_device(device);
  if (rc != B2S_OK) return rc;
  b2s_init_solver* h = new b2s_init_solver();
  h->maxKeys = max_keys;
  h->maxIters = max_iterations;
  h->maxBatch = max_batch;
  h->device = device;
  const size_t B = max_batch, NK = (size_t)max_keys * B, IT = (size_t)max_iterations * B;
  const size_t W = (size_t)((max_keys + 31) / 32) * 2 * IT;
  cudaError_t e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreate(&h->ev[0]);
  if (e == cudaSuccess) e = cudaEventCreate(&h->ev[1]);
  if (e == cudaSuccess) e = cudaMalloc(&h->prob, B * sizeof(Prob));
  if (e == cudaSuccess) e = cudaMalloc(&h->kp1, NK * 2 * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->kp2, NK * 2 * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->pn1, NK * 2 * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->pn2, NK * 2 * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->m12, NK * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc(&h->mt, NK * 2 * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc(&h->sets, IT * 8 * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc(&h->hyp, IT * 2 * 18 * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->score, IT * 2 * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->inl, W * sizeof(uint32_t));
  if (e == cudaSuccess) e = cudaMalloc(&h->st, B * sizeof(St));
  if (e == cudaSuccess) e = cudaMalloc(&h->p3dh, NK * 8 * 3 * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->goodh, NK * 8);
  if (e == cudaSuccess) e = cudaMalloc(&h->p3d, NK * 3 * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->tri, NK);
  if (e == cudaSuccess) e = cudaMalloc(&h->inlH, NK);
  if (e == cudaSuccess) e = cudaMalloc(&h->inlF, NK);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(k_init_checkrt, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_KEYS * sizeof(float));
  if (e != cudaSuccess) {
    set_error("b2s_init_create: %s", cudaGetErrorString(e));
    b2s_init_destroy(h);
    return B2S_ERR_CUDA;
  }
  *out = h;
  return B2S_OK;
}

extern "C" void b2s_init_destroy(b2s_init_solver* h) {
  if (!h) return;
  if (h->stream) cudaStreamSynchronize(h->stream);
  for (void* q : {(void*)h->prob, (void*)h->kp1, (void*)h->kp2, (void*)h->pn1, (void*)h->pn2, (void*)h->m12,
                  (void*)h->mt, (void*)h->sets, (void*)h->hyp, (void*)h->score, (void*)h->inl, (void*)h->st,
                  (void*)h->p3dh, (void*)h->goodh, (void*)h->p3d, (void*)h->tri, (void*)h->inlH, (void*)h->inlF})
    if (q) cudaFree(q);
  for (cudaEvent_t ev : h->ev)
    if (ev) cudaEventDestroy(ev);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

extern "C" float b2s_init_last_ms(const b2s_init_solver* h) { return h ? h->lastMs : 0.f; }

extern "C" int b2s_initialize(b2s_init_solver* h, int batch, const b2s_init_problem* p, b2s_init_result* r) {
  if (!h || !p || !r || batch < 1) {
    set_error("b2s_initialize: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  if (batch > h->maxBatch) {
    set_error("b2s_initialize: batch %d exceeds the handle's capacity %d", batch, h->maxBatch);
    return B2S_ERR_CAPACITY;
  }
  std::vector<int> nm((size_t)batch);
  for (int i = 0; i < batch; i++) {
    const b2s_init_problem& q = p[i];
    if (q.n1 > h->maxKeys || q.n2 > h->maxKeys || q.iterations > h->maxIters) {
      set_error("b2s_initialize: problem %d (n1 = %d, n2 = %d, iterations = %d) exceeds the handle's capacity", i, q.n1,
                q.n2, q.iterations);
      return B2S_ERR_CAPACITY;
    }
    if (q.n1 < 1 || q.n2 < 1 || q.iterations < 1 || !(q.sigma > 0.f) || !q.kp1 || !q.kp2 || !q.matches12 || !q.sets ||
        !r[i].p3d || !r[i].triangulated) {
      set_error("b2s_initialize: problem %d: bad argument", i);
      return B2S_ERR_BAD_ARG;
    }
    int n = 0;
    for (int k = 0; k < q.n1; k++) {
      if (q.matches12[k] >= q.n2) {
        set_error("b2s_initialize: problem %d: match %d -> %d outside [0, %d)", i, k, q.matches12[k], q.n2);
        return B2S_ERR_BAD_ARG;
      }
      n += q.matches12[k] >= 0;
    }
    if (n < 8) {
      set_error("b2s_initialize: problem %d has %d matches (at least 8)", i, n);
      return B2S_ERR_BAD_ARG;
    }
    for (int it = 0; it < q.iterations; it++)
      for (int j = 0; j < 8; j++) {
        const int s = q.sets[8 * it + j];
        bool dup = false;
        for (int l = 0; l < j; l++) dup |= q.sets[8 * it + l] == s;
        if (s < 0 || s >= n || dup) {
          set_error("b2s_initialize: problem %d: set %d entry %d = %d (n_matches = %d)", i, it, j, s, n);
          return B2S_ERR_BAD_ARG;
        }
      }
    nm[(size_t)i] = n;
  }
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;

  h->hProb.resize((size_t)batch);
  size_t o1 = 0, o2 = 0, oit = 0, oinl = 0;
  int maxIt = 0, maxNm = 0;
  for (int i = 0; i < batch; i++) {
    const b2s_init_problem& q = p[i];
    Prob& P = h->hProb[(size_t)i];
    P.n1 = q.n1;
    P.n2 = q.n2;
    P.off1 = (int)o1;
    P.off2 = (int)o2;
    P.iters = q.iterations;
    P.offIt = (int)oit;
    P.w1 = (q.n1 + 31) / 32;
    P.offInl = (int)oinl;
    memcpy(P.K, q.K, sizeof(P.K));
    P.sigma = q.sigma;
    o1 += (size_t)q.n1;
    o2 += (size_t)q.n2;
    oit += (size_t)q.iterations;
    oinl += (size_t)2 * q.iterations * P.w1;
    maxIt = std::max(maxIt, q.iterations);
    maxNm = std::max(maxNm, nm[(size_t)i]);
  }
  h->hKp1.resize(o1 * 2);
  h->hKp2.resize(o2 * 2);
  h->hM12.resize(o1);
  h->hSets.resize(oit * 8);
  for (int i = 0; i < batch; i++) {
    const b2s_init_problem& q = p[i];
    const Prob& P = h->hProb[(size_t)i];
    memcpy(&h->hKp1[2 * (size_t)P.off1], q.kp1, 2 * sizeof(float) * q.n1);
    memcpy(&h->hKp2[2 * (size_t)P.off2], q.kp2, 2 * sizeof(float) * q.n2);
    memcpy(&h->hM12[(size_t)P.off1], q.matches12, sizeof(int) * q.n1);
    memcpy(&h->hSets[8 * (size_t)P.offIt], q.sets, 8 * sizeof(int) * q.iterations);
  }
  h->hSt.resize((size_t)batch);
  h->hP3d.resize(o1 * 3);
  h->hTri.resize(o1);
  h->hInlH.resize(o1);
  h->hInlF.resize(o1);

  B2S_CUDA(cudaEventRecord(h->ev[0], s));
  B2S_CUDA(cudaMemcpyAsync(h->prob, h->hProb.data(), (size_t)batch * sizeof(Prob), cudaMemcpyHostToDevice, s));
  B2S_CUDA(cudaMemcpyAsync(h->kp1, h->hKp1.data(), o1 * 2 * sizeof(float), cudaMemcpyHostToDevice, s));
  B2S_CUDA(cudaMemcpyAsync(h->kp2, h->hKp2.data(), o2 * 2 * sizeof(float), cudaMemcpyHostToDevice, s));
  B2S_CUDA(cudaMemcpyAsync(h->m12, h->hM12.data(), o1 * sizeof(int), cudaMemcpyHostToDevice, s));
  B2S_CUDA(cudaMemcpyAsync(h->sets, h->hSets.data(), oit * 8 * sizeof(int), cudaMemcpyHostToDevice, s));
  Ptrs a = {h->prob, h->kp1, h->kp2, h->m12, h->sets, h->pn1, h->pn2, h->mt, h->hyp, h->score, h->inl, h->st,
            h->p3dh, h->goodh, h->p3d, h->tri, h->inlH, h->inlF};
  k_init_prepare<<<batch, CT, 0, s>>>(a);
  k_init_hypothesis<<<dim3((2 * maxIt + 63) / 64, batch), 64, 0, s>>>(a);
  k_init_score<<<dim3(2 * maxIt, batch), CT, 0, s>>>(a);
  k_init_select<<<(batch + 63) / 64, 64, 0, s>>>(a, batch);
  int L = 1;
  while (L < maxNm) L <<= 1;
  k_init_checkrt<<<dim3(8, batch), CT, (size_t)L * sizeof(float), s>>>(a);
  k_init_decide<<<batch, CT, 0, s>>>(a);
  B2S_CUDA(cudaGetLastError());
  B2S_CUDA(cudaMemcpyAsync(h->hSt.data(), h->st, (size_t)batch * sizeof(St), cudaMemcpyDeviceToHost, s));
  B2S_CUDA(cudaMemcpyAsync(h->hP3d.data(), h->p3d, o1 * 3 * sizeof(float), cudaMemcpyDeviceToHost, s));
  B2S_CUDA(cudaMemcpyAsync(h->hTri.data(), h->tri, o1, cudaMemcpyDeviceToHost, s));
  B2S_CUDA(cudaMemcpyAsync(h->hInlH.data(), h->inlH, o1, cudaMemcpyDeviceToHost, s));
  B2S_CUDA(cudaMemcpyAsync(h->hInlF.data(), h->inlF, o1, cudaMemcpyDeviceToHost, s));
  B2S_CUDA(cudaEventRecord(h->ev[1], s));
  B2S_CUDA(cudaStreamSynchronize(s));
  B2S_CUDA(cudaGetLastError());

  for (int i = 0; i < batch; i++) {
    const St& S = h->hSt[(size_t)i];
    const Prob& P = h->hProb[(size_t)i];
    b2s_init_result& R = r[i];
    R.ret = S.ret;
    R.model = S.model;
    R.rt_state = S.rtState;
    if (S.ret) {
      memcpy(R.R21, S.R[S.chosen], sizeof(R.R21));
      memcpy(R.t21, S.t[S.chosen], sizeof(R.t21));
      memcpy(R.p3d, &h->hP3d[3 * (size_t)P.off1], 3 * sizeof(float) * P.n1);
      memcpy(R.triangulated, &h->hTri[(size_t)P.off1], (size_t)P.n1);
    }
    if (R.inliers_h) memcpy(R.inliers_h, &h->hInlH[(size_t)P.off1], (size_t)S.nm);
    if (R.inliers_f) memcpy(R.inliers_f, &h->hInlF[(size_t)P.off1], (size_t)S.nm);
    R.n_matches = S.nm;
    R.best_h_iter = S.bestH;
    R.best_f_iter = S.bestF;
    R.SH = S.SH;
    R.SF = S.SF;
    R.RH = S.RH;
    memcpy(R.H21, S.H, sizeof(R.H21));
    memcpy(R.F21, S.F, sizeof(R.F21));
    R.n_hyp = S.nhyp;
    for (int k = 0; k < 8; k++) {
      R.n_good[k] = S.ngood[k];
      R.parallax[k] = S.par[k];
    }
  }
  float ms = 0.f;
  B2S_CUDA(cudaEventElapsedTime(&ms, h->ev[0], h->ev[1]));
  h->lastMs = ms;
  return B2S_OK;
}
