// sim3solver.cu — Sim3 RANSAC for loop-closure candidates: Sim3Solver::iterate (src/Sim3Solver.cc:199-285) with the
// minimal sets drawn by the caller, on the GPU.  The device restates oracle/sim3solver.cpp operation by operation (float
// where the reference stores CV_32F, double where OpenCV's gemm / dot / norm / Rodrigues compute in double) and is
// compiled without FMA contraction, so it is bit-identical to it except where CUDA's double atan2 / sin / cos differ
// from glibc's in the last bit (DESIGN §7).
//
// A call is three launches on one stream, no host synchronisation between them; every launch covers the whole batch:
//   k_s3s_hypothesis  one thread per (problem, set): ComputeSim3 (centroids, M, the 4 x 4 float Jacobi eigen, Rodrigues,
//                     scale, T12 and T21)
//   k_s3s_inliers     one CTA per (problem, set): CheckInliers over every correspondence in both directions, the flags
//                     as warp ballots into a bitmask, the count by popc (an integer: no order dependence)
//   k_s3s_scan        one CTA per problem: the reference's serial scan in set order (best on >=, the return on more
//                     than min_inliers inliers), then vbInliers of the returned hypothesis expanded from its bitmask
// Hypotheses after an early return are computed and discarded.
#include <float.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>

#include "common.cuh"

namespace b2s {
namespace s3s {

constexpr int MAX_MATCHES = 65536;
constexpr int CT = 128;  // threads of the per-hypothesis and per-problem CTAs
constexpr int HYP = 48;  // floats per hypothesis: R 9, t 3, s 1, T12 16, T21 16 (45 used)

struct Prob {
  int n, off, k, offSet, words, offMask, fix, minInl, maxIts, done, best;
  float K1[4], K2[4];
};

struct St {
  int returned, retIdx, changedIdx, used, doneAfter, bestAfter, noMore, nInl;
  float hyp[HYP];  // the hypothesis at changedIdx
};

struct Ptrs {
  const Prob* prob;
  const float *X1, *X2, *sig1, *sig2;
  const int* sets;
  float* hyp;
  int* cnt;
  uint32_t* mask;
  St* st;
  uint8_t* inl;  // out: per correspondence
};

// ------------------------------------------------------------------------------------------------ OpenCV arithmetic
// lapack.cpp's hypot template in float
__device__ __forceinline__ float cv_hypot(float a, float b) {
  a = fabsf(a);
  b = fabsf(b);
  if (a > b) {
    b /= a;
    return a * sqrtf(1 + b * b);
  }
  if (b > 0) {
    a /= b;
    return b * sqrtf(1 + a * a);
  }
  return 0;
}

// JacobiImpl_<float> of a symmetric 4 x 4 matrix with eigenvectors, then the descending sort (oracle orc_s3s_eigen)
__device__ void eigen4(float* A, float* W, float* V) {
  constexpr int n = 4;
  int indR[n], indC[n];
  for (int i = 0; i < n; i++)
    for (int j = 0; j < n; j++) V[i * n + j] = i == j ? 1.f : 0.f;
  int k, m, i;
  float mv;
  for (k = 0; k < n; k++) {
    W[k] = A[(n + 1) * k];
    if (k < n - 1) {
      for (m = k + 1, mv = fabsf(A[n * k + m]), i = k + 2; i < n; i++) {
        const float val = fabsf(A[n * k + i]);
        if (mv < val) mv = val, m = i;
      }
      indR[k] = m;
    }
    if (k > 0) {
      for (m = 0, mv = fabsf(A[k]), i = 1; i < k; i++) {
        const float val = fabsf(A[n * i + k]);
        if (mv < val) mv = val, m = i;
      }
      indC[k] = m;
    }
  }
  for (int iters = 0; iters < n * n * 30; iters++) {
    for (k = 0, mv = fabsf(A[indR[0]]), i = 1; i < n - 1; i++) {
      const float val = fabsf(A[n * i + indR[i]]);
      if (mv < val) mv = val, k = i;
    }
    int l = indR[k];
    for (i = 1; i < n; i++) {
      const float val = fabsf(A[n * indC[i] + i]);
      if (mv < val) mv = val, k = indC[i], l = i;
    }
    const float p = A[n * k + l];
    if (fabsf(p) <= FLT_EPSILON) break;
    const float y = (float)((double)(W[l] - W[k]) * 0.5);
    float t = fabsf(y) + cv_hypot(p, y);
    float s = cv_hypot(p, t);
    const float c = t / s;
    s = p / s;
    t = (p / t) * p;
    if (y < 0) s = -s, t = -t;
    A[n * k + l] = 0;
    W[k] -= t;
    W[l] += t;
    float a0, b0;
#define S3S_ROTATE(v0, v1) a0 = v0, b0 = v1, v0 = a0 * c - b0 * s, v1 = a0 * s + b0 * c
    for (i = 0; i < k; i++) S3S_ROTATE(A[n * i + k], A[n * i + l]);
    for (i = k + 1; i < l; i++) S3S_ROTATE(A[n * k + i], A[n * i + l]);
    for (i = l + 1; i < n; i++) S3S_ROTATE(A[n * k + i], A[n * l + i]);
    for (i = 0; i < n; i++) S3S_ROTATE(V[n * k + i], V[n * l + i]);
#undef S3S_ROTATE
    for (int j = 0; j < 2; j++) {
      const int idx = j == 0 ? k : l;
      if (idx < n - 1) {
        for (m = idx + 1, mv = fabsf(A[n * idx + m]), i = idx + 2; i < n; i++) {
          const float val = fabsf(A[n * idx + i]);
          if (mv < val) mv = val, m = i;
        }
        indR[idx] = m;
      }
      if (idx > 0) {
        for (m = 0, mv = fabsf(A[idx]), i = 1; i < idx; i++) {
          const float val = fabsf(A[n * i + idx]);
          if (mv < val) mv = val, m = i;
        }
        indC[idx] = m;
      }
    }
  }
  for (k = 0; k < n - 1; k++) {
    m = k;
    for (i = k + 1; i < n; i++)
      if (W[m] < W[i]) m = i;
    if (k != m) {
      float tmp = W[m];
      W[m] = W[k];
      W[k] = tmp;
      for (i = 0; i < n; i++) {
        tmp = V[n * m + i];
        V[n * m + i] = V[n * k + i];
        V[n * k + i] = tmp;
      }
    }
  }
}

// cvRodrigues2, vector to matrix (oracle orc_s3s_rodrigues)
__device__ void rodrigues(const float* v, float* R) {
  double rx = v[0], ry = v[1], rz = v[2];
  const double theta = sqrt(rx * rx + ry * ry + rz * rz);
  if (theta < DBL_EPSILON) {
    for (int i = 0; i < 9; i++) R[i] = (i % 4 == 0) ? 1.f : 0.f;
    return;
  }
  const double c = cos(theta), s = sin(theta), c1 = 1. - c;
  const double itheta = theta ? 1. / theta : 0.;
  rx *= itheta;
  ry *= itheta;
  rz *= itheta;
  const double rrt[9] = {rx * rx, rx * ry, rx * rz, rx * ry, ry * ry, ry * rz, rx * rz, ry * rz, rz * rz};
  const double r_x[9] = {0, -rz, ry, rz, 0, -rx, -ry, rx, 0};
  for (int i = 0; i < 9; i++) {
    const double e = (i % 4 == 0) ? 1. : 0.;
    R[i] = (float)((c * e + c1 * rrt[i]) + s * r_x[i]);
  }
}

// gemm's float path for an inner size of 3 (A 3 x 3 row-major, x 3): products summed in float, in k order, from 0 as
// the restatement's orc_gemm does
__device__ __forceinline__ float dot3f(const float* a, float x0, float x1, float x2) {
  return ((0.f + a[0] * x0) + a[1] * x1) + a[2] * x2;
}

// ComputeCentroid: reduce (float, left to right), times (float)(1./3), then Pr = P - C
__device__ __forceinline__ void centroid(const float* P, float* Pr, float* C) {
  const float sc = (float)(1. / 3);
  for (int r = 0; r < 3; r++) {
    C[r] = ((P[r * 3] + P[r * 3 + 1]) + P[r * 3 + 2]) * sc;
    for (int i = 0; i < 3; i++) Pr[r * 3 + i] = P[r * 3 + i] - C[r];
  }
}

// ComputeSim3 (oracle compute_sim3); h: R 9, t 3, s, T12 16, T21 16
__device__ void compute_sim3(const float* P1, const float* P2, bool fix, float* h) {
  float Pr1[9], Pr2[9], O1[3], O2[3], M[9];
  centroid(P1, Pr1, O1);
  centroid(P2, Pr2, O2);
  for (int r = 0; r < 3; r++)  // M = Pr2*Pr1.t(): gemm with the second operand transposed, double sums
    for (int c = 0; c < 3; c++) {
      double s = 0;
      for (int q = 0; q < 3; q++) s += (double)Pr2[r * 3 + q] * Pr1[c * 3 + q];
      M[r * 3 + c] = (float)s;
    }
#define m(r, c) M[(r) * 3 + (c)]
  const float N11 = m(0, 0) + m(1, 1) + m(2, 2), N12 = m(1, 2) - m(2, 1), N13 = m(2, 0) - m(0, 2),
              N14 = m(0, 1) - m(1, 0), N22 = m(0, 0) - m(1, 1) - m(2, 2), N23 = m(0, 1) + m(1, 0),
              N24 = m(2, 0) + m(0, 2), N33 = -m(0, 0) + m(1, 1) - m(2, 2), N34 = m(1, 2) + m(2, 1),
              N44 = -m(0, 0) - m(1, 1) + m(2, 2);
#undef m
  float N[16] = {N11, N12, N13, N14, N12, N22, N23, N24, N13, N23, N33, N34, N14, N24, N34, N44};
  float eval[4], evec[16];
  eigen4(N, eval, evec);
  float vec[3] = {evec[1], evec[2], evec[3]};
  // cv::norm: two double lanes (even, odd entries)
  const double nv = sqrt(((double)vec[0] * vec[0] + (double)vec[2] * vec[2]) + (double)vec[1] * vec[1]);
  const double ang = atan2(nv, (double)evec[0]);
  const float alpha = (float)((2 * ang) * (1. / nv));
  for (int i = 0; i < 3; i++) vec[i] = vec[i] * alpha;
  float* R = h;
  rodrigues(vec, R);
  float s;
  if (!fix) {
    float P3[9];
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) P3[r * 3 + c] = dot3f(R + 3 * r, Pr2[c], Pr2[3 + c], Pr2[6 + c]);
    // Mat::dot: dotProd_ unrolled by 4 in double
    double nom = 0;
    nom += (double)Pr1[0] * P3[0] + (double)Pr1[1] * P3[1] + (double)Pr1[2] * P3[2] + (double)Pr1[3] * P3[3];
    nom += (double)Pr1[4] * P3[4] + (double)Pr1[5] * P3[5] + (double)Pr1[6] * P3[6] + (double)Pr1[7] * P3[7];
    nom += (double)Pr1[8] * P3[8];
    double den = 0;
    for (int i = 0; i < 9; i++) den += (double)(P3[i] * P3[i]);
    s = (float)(nom / den);
  } else {
    s = 1.0f;
  }
  float* t = h + 9;
  for (int r = 0; r < 3; r++) t[r] = (float)((double)dot3f(R + 3 * r, O2[0], O2[1], O2[2]) * -(double)s + (double)O1[r]);
  h[12] = s;
  float* T12 = h + 13;
  float* T21 = h + 29;
  const float si = (float)(1.0 / (double)s);
  float sRinv[9];
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) {
      T12[r * 4 + c] = R[r * 3 + c] * s;
      sRinv[r * 3 + c] = R[c * 3 + r] * si;
      T21[r * 4 + c] = sRinv[r * 3 + c];
    }
    T12[r * 4 + 3] = t[r];
    T12[12 + r] = T21[12 + r] = 0.f;
  }
  T12[15] = T21[15] = 1.f;
  for (int r = 0; r < 3; r++) T21[r * 4 + 3] = (float)((double)dot3f(sRinv + 3 * r, t[0], t[1], t[2]) * -1.0);
}

__device__ __forceinline__ void to_image(float X0, float X1, float X2, const float* K, float& u, float& v) {
  const float invz = 1 / X2;
  const float x = X0 * invz, y = X1 * invz;
  u = K[0] * x + K[2];
  v = K[1] * y + K[3];
}

// Project: Rcw*X + tcw as gemm(Rcw, X, 1, tcw, 1) (float sum, then the double addition rounded once = a float add)
__device__ __forceinline__ void project(const float* T, float X0, float X1, float X2, const float* K, float& u,
                                        float& v) {
  const float R0[3] = {T[0], T[1], T[2]}, R1[3] = {T[4], T[5], T[6]}, R2[3] = {T[8], T[9], T[10]};
  const float P0 = dot3f(R0, X0, X1, X2) + T[3], P1 = dot3f(R1, X0, X1, X2) + T[7], P2 = dot3f(R2, X0, X1, X2) + T[11];
  to_image(P0, P1, P2, K, u, v);
}

__device__ __forceinline__ float threshold(float sigma2) {
  return (float)(unsigned long long)(9.210 * (double)sigma2);
}

__device__ __forceinline__ bool runs(const Prob& P) { return P.n >= P.minInl; }

// ------------------------------------------------------------------------------------------------ kernels
__global__ void __launch_bounds__(64) k_s3s_hypothesis(Ptrs a) {
  const Prob P = a.prob[blockIdx.y];
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P.k || !runs(P)) return;
  const int* set = a.sets + 3 * (size_t)(P.offSet + j);
  float P1[9], P2[9];
  for (int i = 0; i < 3; i++) {
    const size_t q = 3 * ((size_t)P.off + set[i]);
    for (int r = 0; r < 3; r++) {
      P1[r * 3 + i] = a.X1[q + r];
      P2[r * 3 + i] = a.X2[q + r];
    }
  }
  float h[HYP];
  compute_sim3(P1, P2, P.fix != 0, h);
  float* out = a.hyp + (size_t)HYP * (P.offSet + j);
  for (int i = 0; i < 45; i++) out[i] = h[i];
}

__global__ void __launch_bounds__(CT) k_s3s_inliers(Ptrs a) {
  const Prob P = a.prob[blockIdx.y];
  const int j = blockIdx.x;
  if (j >= P.k || !runs(P)) return;
  __shared__ float T[32];
  __shared__ int count;
  const float* h = a.hyp + (size_t)HYP * (P.offSet + j);
  if (threadIdx.x < 32) T[threadIdx.x] = h[13 + threadIdx.x];
  if (threadIdx.x == 0) count = 0;
  __syncthreads();
  uint32_t* mask = a.mask + P.offMask + (size_t)j * P.words;
  const int lane = threadIdx.x & 31;
  int mine = 0;
  for (int base = 0; base < P.n; base += CT) {
    const int i = base + threadIdx.x;
    bool in = false;
    if (i < P.n) {
      const size_t q = 3 * ((size_t)P.off + i);
      const float x10 = a.X1[q], x11 = a.X1[q + 1], x12 = a.X1[q + 2];
      const float x20 = a.X2[q], x21 = a.X2[q + 1], x22 = a.X2[q + 2];
      float u11, v11, u22, v22, u21, v21, u12, v12;
      to_image(x10, x11, x12, P.K1, u11, v11);
      to_image(x20, x21, x22, P.K2, u22, v22);
      project(T, x20, x21, x22, P.K1, u21, v21);
      project(T + 16, x10, x11, x12, P.K2, u12, v12);
      const float d10 = u11 - u21, d11 = v11 - v21, d20 = u12 - u22, d21 = v12 - v22;
      const float err1 = (float)((double)d10 * d10 + (double)d11 * d11);
      const float err2 = (float)((double)d20 * d20 + (double)d21 * d21);
      in = err1 < threshold(a.sig1[P.off + i]) && err2 < threshold(a.sig2[P.off + i]);
    }
    const uint32_t b = __ballot_sync(0xffffffffu, in);
    if (lane == 0 && i < P.n) mask[i >> 5] = b;
    mine += lane == 0 ? __popc(b) : 0;
  }
  if (lane == 0) atomicAdd(&count, mine);
  __syncthreads();
  if (threadIdx.x == 0) a.cnt[P.offSet + j] = count;
}

__global__ void __launch_bounds__(CT) k_s3s_scan(Ptrs a) {
  const Prob P = a.prob[blockIdx.x];
  __shared__ St S;
  if (threadIdx.x == 0) {
    St s;
    s.returned = s.used = s.noMore = s.nInl = 0;
    s.retIdx = s.changedIdx = -1;
    s.doneAfter = P.done;
    s.bestAfter = P.best;
    if (!runs(P)) {
      s.noMore = 1;
    } else {
      int it = P.done, best = P.best, cur = 0;
      while (it < P.maxIts && cur < P.k) {
        const int ni = a.cnt[P.offSet + cur];
        cur++;
        it++;
        if (ni >= best) {
          best = ni;
          s.changedIdx = cur - 1;
          if (ni > P.minInl) {
            s.returned = 1;
            s.retIdx = cur - 1;
            s.nInl = ni;
            break;
          }
        }
      }
      s.used = cur;
      s.doneAfter = it;
      s.bestAfter = best;
      s.noMore = !s.returned && it >= P.maxIts;
    }
    S = s;
  }
  __syncthreads();
  St& out = a.st[blockIdx.x];
  if (threadIdx.x < 8) (&out.returned)[threadIdx.x] = (&S.returned)[threadIdx.x];
  if (S.changedIdx >= 0 && threadIdx.x < 45)
    out.hyp[threadIdx.x] = a.hyp[(size_t)HYP * (P.offSet + S.changedIdx) + threadIdx.x];
  const uint32_t* mask = S.returned ? a.mask + P.offMask + (size_t)S.retIdx * P.words : nullptr;
  for (int i = threadIdx.x; i < P.n; i += CT) a.inl[P.off + i] = mask ? (uint8_t)((mask[i >> 5] >> (i & 31)) & 1u) : 0;
}

}  // namespace s3s
}  // namespace b2s

using namespace b2s;
using namespace b2s::s3s;

// ================================================================================================ host side
struct b2s_sim3solver : b2s::Stage {
  int maxMatches, maxSets, maxBatch;
  float* hyp = nullptr;
  int* cnt = nullptr;
  uint32_t* mask = nullptr;
  // a call's inputs and outputs, laid out by lay() for its problems, correspondences and sets
  Packed in, out;
  Seg<Prob> prob;
  Seg<float> X1, X2, sig1, sig2;
  Seg<int> sets;
  Seg<St> st;
  Seg<uint8_t> inl;
  void lay(size_t batch, size_t nm, size_t ns) {
    in.clear();
    prob = in.add<Prob>(batch);
    X1 = in.add<float>(nm * 3);
    X2 = in.add<float>(nm * 3);
    sig1 = in.add<float>(nm);
    sig2 = in.add<float>(nm);
    sets = in.add<int>(ns * 3);
    out.clear();
    st = out.add<St>(batch);
    inl = out.add<uint8_t>(nm);
  }
};

extern "C" int b2s_sim3solver_create(int max_matches, int max_sets, int max_batch, int device, b2s_sim3solver** out) {
  if (!out || max_matches < 3 || max_matches > MAX_MATCHES || max_sets < 1 || max_batch < 1) {
    set_error("b2s_sim3solver_create: bad argument (3 <= max_matches <= %d, max_sets >= 1, max_batch >= 1)",
              MAX_MATCHES);
    return B2S_ERR_BAD_ARG;
  }
  *out = nullptr;
  int rc = select_device(device);
  if (rc != B2S_OK) return rc;
  b2s_sim3solver* h = new b2s_sim3solver();
  h->maxMatches = max_matches;
  h->maxSets = max_sets;
  h->maxBatch = max_batch;
  const size_t B = max_batch, NM = (size_t)max_matches * B, NS = (size_t)max_sets * B;
  const size_t W = (size_t)((max_matches + 31) / 32) * NS;
  h->open(device);
  h->lay(B, NM, NS);
  h->in.reserve(h->error);
  h->out.reserve(h->error);
  h->alloc(h->hyp, NS * HYP * sizeof(float));
  h->alloc(h->cnt, NS * sizeof(int));
  h->alloc(h->mask, W * sizeof(uint32_t));
  if (h->error != cudaSuccess) {
    set_error("b2s_sim3solver_create: %s", cudaGetErrorString(h->error));
    b2s_sim3solver_destroy(h);
    return B2S_ERR_CUDA;
  }
  *out = h;
  return B2S_OK;
}

extern "C" void b2s_sim3solver_destroy(b2s_sim3solver* h) {
  if (!h) return;
  h->close();
  delete h;
}

extern "C" float b2s_sim3solver_last_ms(const b2s_sim3solver* h) { return h ? h->lastMs : 0.f; }

extern "C" int b2s_sim3solver_iterate(b2s_sim3solver* h, int batch, const b2s_sim3solver_problem* p,
                                      b2s_sim3solver_result* r) {
  if (!h || !p || !r || batch < 1) {
    set_error("b2s_sim3solver_iterate: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  if (batch > h->maxBatch) {
    set_error("b2s_sim3solver_iterate: batch %d exceeds the handle's capacity %d", batch, h->maxBatch);
    return B2S_ERR_CAPACITY;
  }
  size_t on = 0, os = 0, om = 0;  // correspondences, sets and mask words of the batch
  for (int i = 0; i < batch; i++) {
    const b2s_sim3solver_problem& q = p[i];
    if (q.n > h->maxMatches || q.k > h->maxSets) {
      set_error("b2s_sim3solver_iterate: problem %d (n = %d, k = %d) exceeds the handle's capacity", i, q.n, q.k);
      return B2S_ERR_CAPACITY;
    }
    const bool run = q.n >= q.min_inliers && q.k > 0;
    if (q.n < 0 || q.max_its < 1 || q.iterations_done < 0 || q.best_inliers < 0 || q.k < 0 ||
        q.k > q.max_its - q.iterations_done || (q.n > 0 && (!q.X1c || !q.X2c || !q.sigma2_1 || !q.sigma2_2 ||
                                                             !r[i].inliers)) ||
        (run && (q.n < 3 || !q.sets))) {
      set_error("b2s_sim3solver_iterate: problem %d: bad argument", i);
      return B2S_ERR_BAD_ARG;
    }
    for (int c = 0; c < q.n; c++)
      if (!(q.sigma2_1[c] >= 0.f && q.sigma2_1[c] <= FLT_MAX && q.sigma2_2[c] >= 0.f && q.sigma2_2[c] <= FLT_MAX)) {
        set_error("b2s_sim3solver_iterate: problem %d: sigma2 of correspondence %d is negative or not finite", i, c);
        return B2S_ERR_BAD_ARG;
      }
    int j, l;
    if (run && !sets_ok(q.sets, q.k, 3, q.n, &j, &l)) {
      set_error("b2s_sim3solver_iterate: problem %d: set %d entry %d = %d (n = %d)", i, j, l, q.sets[3 * j + l], q.n);
      return B2S_ERR_BAD_ARG;
    }
    on += (size_t)q.n;
    os += (size_t)(run ? q.k : 0);
  }
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;

  h->lay((size_t)batch, on, os);
  int rc = h->in.fit("b2s_sim3solver_iterate");
  if (rc == B2S_OK) rc = h->out.fit("b2s_sim3solver_iterate");
  if (rc != B2S_OK) return rc;
  Prob* prob = h->in.host(h->prob);
  float *X1 = h->in.host(h->X1), *X2 = h->in.host(h->X2), *sig1 = h->in.host(h->sig1), *sig2 = h->in.host(h->sig2);
  int* sets = h->in.host(h->sets);
  on = os = 0;
  int maxK = 0;
  for (int i = 0; i < batch; i++) {
    const b2s_sim3solver_problem& q = p[i];
    Prob& P = prob[i];
    P.n = q.n;
    P.off = (int)on;
    P.k = q.n >= q.min_inliers ? q.k : 0;
    P.offSet = (int)os;
    P.words = (q.n + 31) / 32;
    P.offMask = (int)om;
    P.fix = q.fix_scale != 0;
    P.minInl = q.min_inliers;
    P.maxIts = q.max_its;
    P.done = q.iterations_done;
    P.best = q.best_inliers;
    memcpy(P.K1, q.K1, sizeof(P.K1));
    memcpy(P.K2, q.K2, sizeof(P.K2));
    if (q.n > 0) {
      memcpy(X1 + 3 * on, q.X1c, 3 * sizeof(float) * q.n);
      memcpy(X2 + 3 * on, q.X2c, 3 * sizeof(float) * q.n);
      memcpy(sig1 + on, q.sigma2_1, sizeof(float) * q.n);
      memcpy(sig2 + on, q.sigma2_2, sizeof(float) * q.n);
    }
    if (P.k > 0) memcpy(sets + 3 * os, q.sets, 3 * sizeof(int) * P.k);
    on += (size_t)q.n;
    os += (size_t)P.k;
    om += (size_t)P.k * P.words;
    maxK = std::max(maxK, P.k);
  }

  if ((rc = h->begin()) != B2S_OK) return rc;
  if ((rc = h->in.upload(s)) != B2S_OK) return rc;
  const Packed &in = h->in, &out = h->out;
  Ptrs a = {in.dev(h->prob), in.dev(h->X1), in.dev(h->X2), in.dev(h->sig1), in.dev(h->sig2), in.dev(h->sets),
            h->hyp,          h->cnt,        h->mask,       out.dev(h->st),  out.dev(h->inl)};
  if (maxK > 0) {
    k_s3s_hypothesis<<<dim3((maxK + 63) / 64, batch), 64, 0, s>>>(a);
    k_s3s_inliers<<<dim3(maxK, batch), CT, 0, s>>>(a);
  }
  k_s3s_scan<<<batch, CT, 0, s>>>(a);
  B2S_CUDA(cudaGetLastError());
  if ((rc = out.download(s)) != B2S_OK) return rc;
  if ((rc = h->finish()) != B2S_OK) return rc;

  const St* st = out.host(h->st);
  const uint8_t* inl = out.host(h->inl);
  for (int i = 0; i < batch; i++) {
    const St& S = st[i];
    const Prob& P = prob[i];
    b2s_sim3solver_result& R = r[i];
    R.returned = S.returned;
    R.best_changed = S.changedIdx >= 0;
    if (S.changedIdx >= 0) {
      const float* hy = S.hyp;
      memcpy(R.R, hy, sizeof(R.R));
      memcpy(R.t, hy + 9, sizeof(R.t));
      R.s = hy[12];
      if (S.returned) memcpy(R.T12, hy + 13, sizeof(R.T12));
    }
    if (P.n > 0) memcpy(R.inliers, inl + P.off, (size_t)P.n);
    R.n_inliers = S.nInl;
    R.no_more = S.noMore;
    R.iterations_used = S.used;
    R.iterations_done = S.doneAfter;
    R.best_inliers = S.bestAfter;
  }
  return B2S_OK;
}
