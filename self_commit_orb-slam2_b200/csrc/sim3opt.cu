// sim3opt.cu — the Sim3 refinement of loop-closure verification: Optimizer::OptimizeSim3 (src/Optimizer.cc:1364-1590)
// from the point where the graph is built, on the GPU.
//
// One free VertexSim3Expmap (oplus = Sim3(update) * estimate, update[6] = 0 under fix_scale, written through to the
// solver's x), fixed points in the two cameras' frames, and per correspondence two edges in insertion order:
//   e12 = obs1 - cam_map1(project(S12 X2c))          (EdgeSim3ProjectXYZ)
//   e21 = obs2 - cam_map2(project(S12^-1 X1c))       (EdgeInverseSim3ProjectXYZ)
// with information I * invSigma2 of the edge's keyframe and Huber (delta = (float)sqrt(th2)).  The edges have no
// analytic Jacobian, so g2o differentiates numerically (core/base_binary_edge.hpp:131-200, central differences with
// delta = 1e-9, only for the Sim3 vertex); this file does the same and is compiled without FMA contraction.  The 7 x 7
// system is built as constructQuadraticForm does for a robust edge (:91-113, rho' weighting of the `to` block only) and
// solved by Levenberg-Marquardt (levenberg.cuh, lambda from computeLambdaInit with tau = 1e-5 at each optimize()).
//
// The whole function runs in one launch, one CTA per problem (problems of a batch are independent):
//   optimize(5); an edge pair with e12.chi2() > th2 or e21.chi2() > th2 (the last evaluated state, which is the
//   rejected trial's when the last trial was rejected) loses its match and both edges; fewer than 10 pairs left: return
//   0 with S12 untouched; optimize(nBad ? 10 : 5) over the rest; the same test counts the inliers and nulls matches.
// Per linearisation the 14 perturbed estimates Sim3(+-delta e_d) S and their inverses are computed once into shared
// memory (the same arithmetic on the same operands as g2o's per-edge recomputation).  Every sum (chi2, H, b) is a
// serial loop in edge order, as g2o accumulates them: no floating-point atomics, and two calls give bit-identical
// outputs.
#include <float.h>
#include <math.h>
#include <stddef.h>

#include <algorithm>
#include <vector>

#include "ba_math.cuh"
#include "common.cuh"
#include "levenberg.cuh"
#include "sim3.cuh"

namespace b2s {
namespace s3o {

constexpr int T = 128;        // threads per problem
constexpr int MAX_N = 65536;  // correspondences per problem (the edge flags live in shared memory)
constexpr int IN = 12;        // floats per correspondence: X1c, X2c, obs1, obs2, invSigma2 of pKF1, of pKF2
constexpr int OUT_I = 258;    // ints per problem: n_inliers, n_trials, trace[256]
// doubles per edge in the scratch: J (2 x 7, row = error component), error, chi2 = e^T Omega e, Huber rho(chi2),
// rho' * information, -rho' * information * error
constexpr int ES = 21, OJ = 0, OE = 14, OCHI = 16, ORHO = 17, OW = 18, OR = 19;

struct Prob {
  int n, off, fixScale;
  double th2, delta, dsqr;  // th2 and Huber's delta / delta^2 as the reference's float deltaHuber gives them
  double K[8];              // fx1 fy1 cx1 cy1 fx2 fy2 cx2 cy2
  double S[8];              // g2oS12 on entry
};

struct Ptrs {
  const Prob* prob;
  const float* in;  // IN per correspondence, problems packed at Prob::off
  double* scr;      // 2 * ES per correspondence
  uint8_t* keep;    // per correspondence
  double* Sout;     // 8 per problem
  int* outI;        // OUT_I per problem
};

// EdgeSim3ProjectXYZ / EdgeInverseSim3ProjectXYZ::computeError: obs - cam_map(project(S.map(X)))
__device__ __forceinline__ void proj_error(const double* S, const float* X, const float* obs, const double* K, double* e) {
  const double x[3] = {X[0], X[1], X[2]};
  double y[3];
  s3_map(S, x, y);
  const double u = y[0] / y[2], v = y[1] / y[2];
  e[0] = (double)obs[0] - (u * K[0] + K[2]);
  e[1] = (double)obs[1] - (v * K[1] + K[3]);
}

struct Smem {
  double S[8], Si[8], ST[8], STi[8];  // estimate, its inverse, trial estimate, its inverse
  double P[14][8], Pi[14][8];         // Sim3(+-delta e_d) S (row 2d: +, 2d + 1: -) and their inverses
  double H[49], A[49], b[7], x[7];
  double chi, scale;
  int solved, stop;
  Levenberg lm;
};

// errors, chi2 and Huber rho of every active edge at (S, S^-1); thread 0 returns their sum in edge order
// (activeRobustChi2)
__device__ double evaluate(const Ptrs& p, const Prob& pr, const uint8_t* active, const double* S, const double* Si,
                           Smem& sm) {
  const float* in = p.in + (size_t)pr.off * IN;
  double* scr = p.scr + (size_t)pr.off * 2 * ES;
  for (int m = threadIdx.x; m < pr.n; m += T) {
    if (!active[m]) continue;
    const float* c = in + (size_t)m * IN;
    for (int side = 0; side < 2; side++) {
      double* E = scr + ((size_t)m * 2 + side) * ES;
      const double w = (double)c[10 + side];
      double e[2];
      if (side == 0) proj_error(S, c + 3, c + 6, pr.K, e);
      else proj_error(Si, c, c + 8, pr.K + 4, e);
      const double chi = e[0] * (w * e[0]) + e[1] * (w * e[1]);
      E[OE] = e[0];
      E[OE + 1] = e[1];
      E[OCHI] = chi;
      E[ORHO] = chi <= pr.dsqr ? chi : 2 * sqrt(chi) * pr.delta - pr.dsqr;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0;
    for (int m = 0; m < pr.n; m++) {
      if (!active[m]) continue;
      s += scr[(size_t)m * 2 * ES + ORHO];
      s += scr[((size_t)m * 2 + 1) * ES + ORHO];
    }
    sm.chi = s;
  }
  __syncthreads();
  return sm.chi;
}

// linearizeOplus of every active edge at sm.S, then H (upper triangle, mirrored) and b summed in edge order
__device__ void build_system(const Ptrs& p, const Prob& pr, const uint8_t* active, Smem& sm) {
  const double delta = 1e-9, scalar = 1.0 / (2 * delta);
  if (threadIdx.x < 14) {
    const int d = threadIdx.x >> 1;
    double u[7] = {0, 0, 0, 0, 0, 0, 0}, E[8];
    u[d] = (threadIdx.x & 1) ? -delta : delta;
    if (pr.fixScale) u[6] = 0;
    s3_exp(u, E);
    s3_mul(E, sm.S, sm.P[threadIdx.x]);
    s3_inv(sm.P[threadIdx.x], sm.Pi[threadIdx.x]);
  }
  __syncthreads();
  const float* in = p.in + (size_t)pr.off * IN;
  double* scr = p.scr + (size_t)pr.off * 2 * ES;
  for (int m = threadIdx.x; m < pr.n; m += T) {
    if (!active[m]) continue;
    const float* c = in + (size_t)m * IN;
    for (int side = 0; side < 2; side++) {
      double* E = scr + ((size_t)m * 2 + side) * ES;
      for (int d = 0; d < 7; d++) {
        double ep[2], em[2];
        if (side == 0) {
          proj_error(sm.P[2 * d], c + 3, c + 6, pr.K, ep);
          proj_error(sm.P[2 * d + 1], c + 3, c + 6, pr.K, em);
        } else {
          proj_error(sm.Pi[2 * d], c, c + 8, pr.K + 4, ep);
          proj_error(sm.Pi[2 * d + 1], c, c + 8, pr.K + 4, em);
        }
        E[OJ + d] = scalar * (ep[0] - em[0]);
        E[OJ + 7 + d] = scalar * (ep[1] - em[1]);
      }
      // RobustKernelHuber::robustify, robustInformation = rho' * Omega, omega_r = -Omega e * rho'
      const double w = (double)c[10 + side], chi = E[OCHI];
      const double rho1 = chi <= pr.dsqr ? 1. : pr.delta / sqrt(chi);
      E[OW] = rho1 * w;
      E[OR] = -(w * E[OE]) * rho1;
      E[OR + 1] = -(w * E[OE + 1]) * rho1;
    }
  }
  __syncthreads();
  const int t = threadIdx.x;
  if (t < 35) {
    int r = 0, cc = 0;
    if (t < 28) {  // upper-triangle entry t, row-major
      int k = t;
      while (k >= 7 - r) {
        k -= 7 - r;
        r++;
      }
      cc = r + k;
    } else {
      r = t - 28;
    }
    double acc = 0;
    for (int m = 0; m < pr.n; m++) {
      if (!active[m]) continue;
      for (int side = 0; side < 2; side++) {
        const double* E = scr + ((size_t)m * 2 + side) * ES;
        const double* J = E + OJ;
        double h;
        if (t < 28) h = (J[r] * E[OW]) * J[cc] + (J[7 + r] * E[OW]) * J[7 + cc];
        else h = J[r] * E[OR] + J[7 + r] * E[OR + 1];
        acc += h;
      }
    }
    if (t < 28) {
      sm.H[r * 7 + cc] = acc;
      sm.H[cc * 7 + r] = acc;
    } else {
      sm.b[r] = acc;
    }
  }
  __syncthreads();
}

// (H + lambda I) x = b: Cholesky on warp 0 (column k: lane 0 the pivot, lanes k+1..6 the column), substitutions on lane
// 0; the trial estimate Sim3(x) S and computeScale
__device__ void solve_update(const Prob& pr, Smem& sm) {
  const int lane = threadIdx.x;
  if (lane < 32) {
    const double lambda = sm.lm.lambda;
    for (int i = lane; i < 49; i += 32) sm.A[i] = (i % 8 == 0) ? sm.H[i] + lambda : sm.H[i];
    __syncwarp();
    bool ok = true;
    for (int k = 0; k < 7 && ok; k++) {
      if (lane == 0) {
        double s = sm.A[k * 7 + k];
        for (int j = 0; j < k; j++) s -= sm.A[k * 7 + j] * sm.A[k * 7 + j];
        sm.A[k * 7 + k] = (s > 0.0 && isfinite(s)) ? sqrt(s) : -1.0;
      }
      __syncwarp();
      ok = sm.A[k * 7 + k] > 0.0;
      if (ok && lane > k && lane < 7) {
        double s = sm.A[lane * 7 + k];
        for (int j = 0; j < k; j++) s -= sm.A[lane * 7 + j] * sm.A[k * 7 + j];
        sm.A[lane * 7 + k] = s / sm.A[k * 7 + k];
      }
      __syncwarp();
    }
    if (lane == 0) {
      sm.solved = ok;
      if (ok) {
        double y[7];
        for (int i = 0; i < 7; i++) {
          double s = sm.b[i];
          for (int k = 0; k < i; k++) s -= sm.A[i * 7 + k] * y[k];
          y[i] = s / sm.A[i * 7 + i];
        }
        for (int i = 6; i >= 0; i--) {
          double s = y[i];
          for (int k = i + 1; k < 7; k++) s -= sm.A[k * 7 + i] * sm.x[k];
          sm.x[i] = s / sm.A[i * 7 + i];
        }
        if (pr.fixScale) sm.x[6] = 0;
        double E[8];
        s3_exp(sm.x, E);
        s3_mul(E, sm.S, sm.ST);
        s3_inv(sm.ST, sm.STi);
        double sc = 0;
        for (int j = 0; j < 7; j++) sc += sm.x[j] * (lambda * sm.x[j] + sm.b[j]);
        sm.scale = sc;
      }
    }
  }
  __syncthreads();
}

// SparseOptimizer::optimize(iterations) with OptimizationAlgorithmLevenberg::solve
__device__ void optimize(const Ptrs& p, const Prob& pr, const uint8_t* active, int iterations, int* trace, Smem& sm) {
  for (int it = 0; it < iterations; it++) {
    const double chi = evaluate(p, pr, active, sm.S, sm.Si, sm);
    build_system(p, pr, active, sm);
    if (threadIdx.x == 0) {
      sm.lm.begin(chi);
      if (it == 0) {  // computeLambdaInit
        double maxDiag = 0;
        for (int j = 0; j < 7; j++) maxDiag = fmax(fabs(sm.H[j * 7 + j]), maxDiag);
        sm.lm.init_lambda(1e-5 * maxDiag);
      }
    }
    __syncthreads();
    bool again;
    do {
      solve_update(pr, sm);
      // a failed solve leaves the state and the edges' errors as they were; the trial is rejected
      const double tempChi = sm.solved ? evaluate(p, pr, active, sm.ST, sm.STi, sm) : DBL_MAX;
      if (threadIdx.x == 0 && sm.lm.trial(sm.solved != 0, tempChi, sm.scale, trace))
        for (int i = 0; i < 8; i++) {
          sm.S[i] = sm.ST[i];
          sm.Si[i] = sm.STi[i];
        }
      __syncthreads();
      again = sm.lm.retry(false);
      __syncthreads();
    } while (again);
    if (threadIdx.x == 0) sm.stop = sm.lm.end_iteration();
    __syncthreads();
    if (sm.stop) break;
  }
}

// the edge-pair test of both classifications: chi2 of the last evaluated state above th2 on either edge
__device__ __forceinline__ bool pair_bad(const double* scr, int m, double th2) {
  return scr[(size_t)m * 2 * ES + OCHI] > th2 || scr[((size_t)m * 2 + 1) * ES + OCHI] > th2;
}

__global__ void __launch_bounds__(T) k_optimize_sim3(Ptrs p) {
  extern __shared__ uint8_t active[];  // the edge pairs still in the graph
  __shared__ Smem sm;
  __shared__ Prob pr;
  const int pb = blockIdx.x;
  if (threadIdx.x == 0) {
    pr = p.prob[pb];
    for (int i = 0; i < 8; i++) sm.S[i] = pr.S[i];
    s3_inv(sm.S, sm.Si);
    sm.lm = Levenberg{};
  }
  __syncthreads();
  const int n = pr.n;
  uint8_t* keep = p.keep + pr.off;
  int* outI = p.outI + (size_t)pb * OUT_I;
  int* trace = outI + 2;
  const double* scr = p.scr + (size_t)pr.off * 2 * ES;
  for (int m = threadIdx.x; m < n; m += T) active[m] = 1;
  __syncthreads();

  // round 1 (an empty graph is not optimised: initializeOptimization refuses it)
  if (n > 0) optimize(p, pr, active, 5, trace, sm);
  int nBad = 0;
  for (int m0 = 0; m0 < n; m0 += T) {
    const int m = m0 + threadIdx.x;
    const bool bad = m < n && pair_bad(scr, m, pr.th2);
    if (m < n) active[m] = !bad;
    nBad += __syncthreads_count(bad);
  }
  int nIn = 0;
  const bool early = n - nBad < 10;
  if (!early) {
    optimize(p, pr, active, nBad > 0 ? 10 : 5, trace, sm);
    for (int m0 = 0; m0 < n; m0 += T) {
      const int m = m0 + threadIdx.x;
      const bool in = m < n && active[m] && !pair_bad(scr, m, pr.th2);
      if (m < n) active[m] = in;
      nIn += __syncthreads_count(in);
    }
  }
  for (int m = threadIdx.x; m < n; m += T) keep[m] = active[m];
  if (threadIdx.x == 0) {
    for (int i = 0; i < 8; i++) p.Sout[(size_t)pb * 8 + i] = early ? pr.S[i] : sm.S[i];
    outI[0] = early ? 0 : nIn;
    outI[1] = sm.lm.nTrials;
    trace[sm.lm.nTrials < 255 ? sm.lm.nTrials : 255] = -1;
  }
}

}  // namespace s3o
}  // namespace b2s

using namespace b2s;
using namespace b2s::s3o;

// ================================================================================================ host side
struct b2s_sim3opt_solver {
  int maxN, maxBatch, device;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  float lastMs = 0.f;
  long long lastTrials = 0;
  Prob* prob = nullptr;
  float* in = nullptr;
  double *scr = nullptr, *Sout = nullptr;
  uint8_t* keep = nullptr;
  int* outI = nullptr;
  std::vector<Prob> hProb;
  std::vector<float> hIn;
  std::vector<double> hSout;
  std::vector<int> hOutI;
  std::vector<uint8_t> hKeep;
};

extern "C" int b2s_sim3opt_create(int max_matches, int max_batch, int device, b2s_sim3opt_solver** out) {
  if (!out || max_matches < 1 || max_matches > MAX_N || max_batch < 1) {
    set_error("b2s_sim3opt_create: bad argument (1 <= max_matches <= %d, max_batch >= 1)", MAX_N);
    return B2S_ERR_BAD_ARG;
  }
  *out = nullptr;
  int rc = select_device(device);
  if (rc != B2S_OK) return rc;
  b2s_sim3opt_solver* h = new b2s_sim3opt_solver();
  h->maxN = max_matches;
  h->maxBatch = max_batch;
  h->device = device;
  const size_t M = (size_t)max_matches * max_batch, B = max_batch;
  cudaError_t e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreate(&h->ev[0]);
  if (e == cudaSuccess) e = cudaEventCreate(&h->ev[1]);
  if (e == cudaSuccess) e = cudaMalloc(&h->prob, B * sizeof(Prob));
  if (e == cudaSuccess) e = cudaMalloc(&h->in, M * IN * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->scr, M * 2 * ES * sizeof(double));
  if (e == cudaSuccess) e = cudaMalloc(&h->keep, M);
  if (e == cudaSuccess) e = cudaMalloc(&h->Sout, B * 8 * sizeof(double));
  if (e == cudaSuccess) e = cudaMalloc(&h->outI, B * OUT_I * sizeof(int));
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(k_optimize_sim3, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_N);
  if (e != cudaSuccess) {
    set_error("b2s_sim3opt_create: %s", cudaGetErrorString(e));
    b2s_sim3opt_destroy(h);
    return B2S_ERR_CUDA;
  }
  *out = h;
  return B2S_OK;
}

extern "C" void b2s_sim3opt_destroy(b2s_sim3opt_solver* h) {
  if (!h) return;
  if (h->stream) cudaStreamSynchronize(h->stream);
  for (void* q : {(void*)h->prob, (void*)h->in, (void*)h->scr, (void*)h->keep, (void*)h->Sout, (void*)h->outI})
    if (q) cudaFree(q);
  for (cudaEvent_t ev : h->ev)
    if (ev) cudaEventDestroy(ev);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

extern "C" float b2s_sim3opt_last_ms(const b2s_sim3opt_solver* h, long long* lm_trials) {
  if (!h) return 0.f;
  if (lm_trials) *lm_trials = h->lastTrials;
  return h->lastMs;
}

extern "C" int b2s_optimize_sim3(b2s_sim3opt_solver* h, int batch, const b2s_sim3_problem* p, b2s_sim3_result* r) {
  if (!h || !p || !r || batch < 1) {
    set_error("b2s_optimize_sim3: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  if (batch > h->maxBatch) {
    set_error("b2s_optimize_sim3: batch %d exceeds the handle's capacity %d", batch, h->maxBatch);
    return B2S_ERR_CAPACITY;
  }
  size_t total = 0;
  for (int i = 0; i < batch; i++) {
    const b2s_sim3_problem& q = p[i];
    if (q.n < 0 || !(q.th2 > 0.f) ||
        (q.n > 0 && (!q.X1c || !q.X2c || !q.obs1 || !q.obs2 || !q.inv_sigma2_1 || !q.inv_sigma2_2 || !r[i].keep))) {
      set_error("b2s_optimize_sim3: problem %d: bad argument (n = %d, th2 = %g)", i, q.n, (double)q.th2);
      return B2S_ERR_BAD_ARG;
    }
    if (q.n > h->maxN) {
      set_error("b2s_optimize_sim3: problem %d has %d correspondences, the handle's capacity is %d", i, q.n, h->maxN);
      return B2S_ERR_CAPACITY;
    }
    total += (size_t)q.n;
  }
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;

  // ---- pack: one Prob per problem, IN floats per correspondence, problems back to back
  h->hProb.resize((size_t)batch);
  h->hIn.resize(std::max<size_t>(total, 1) * IN);
  int maxN = 0;
  size_t off = 0;
  for (int i = 0; i < batch; i++) {
    const b2s_sim3_problem& q = p[i];
    Prob& P = h->hProb[(size_t)i];
    P.n = q.n;
    P.off = (int)off;
    P.fixScale = q.fix_scale != 0;
    P.th2 = (double)q.th2;
    const float deltaHuber = sqrtf(q.th2);  // const float deltaHuber = sqrt(th2) (:1421)
    P.delta = (double)deltaHuber;
    P.dsqr = P.delta * P.delta;
    const float K[8] = {q.fx1, q.fy1, q.cx1, q.cy1, q.fx2, q.fy2, q.cx2, q.cy2};
    for (int k = 0; k < 8; k++) P.K[k] = (double)K[k];
    memcpy(P.S, &q.S12, sizeof(P.S));
    for (int m = 0; m < q.n; m++) {
      float* c = &h->hIn[(off + (size_t)m) * IN];
      for (int k = 0; k < 3; k++) {
        c[k] = q.X1c[3 * m + k];
        c[3 + k] = q.X2c[3 * m + k];
      }
      for (int k = 0; k < 2; k++) {
        c[6 + k] = q.obs1[2 * m + k];
        c[8 + k] = q.obs2[2 * m + k];
      }
      c[10] = q.inv_sigma2_1[m];
      c[11] = q.inv_sigma2_2[m];
    }
    off += (size_t)q.n;
    maxN = std::max(maxN, q.n);
  }
  h->hSout.resize((size_t)batch * 8);
  h->hOutI.resize((size_t)batch * OUT_I);
  h->hKeep.resize(std::max<size_t>(total, 1));

  B2S_CUDA(cudaEventRecord(h->ev[0], s));
  B2S_CUDA(cudaMemcpyAsync(h->prob, h->hProb.data(), (size_t)batch * sizeof(Prob), cudaMemcpyHostToDevice, s));
  if (total) B2S_CUDA(cudaMemcpyAsync(h->in, h->hIn.data(), total * IN * sizeof(float), cudaMemcpyHostToDevice, s));
  Ptrs a = {h->prob, h->in, h->scr, h->keep, h->Sout, h->outI};
  const size_t smem = (size_t)((maxN + 15) / 16 * 16);
  k_optimize_sim3<<<batch, T, smem, s>>>(a);
  B2S_CUDA(cudaGetLastError());
  B2S_CUDA(cudaMemcpyAsync(h->hSout.data(), h->Sout, (size_t)batch * 8 * sizeof(double), cudaMemcpyDeviceToHost, s));
  B2S_CUDA(cudaMemcpyAsync(h->hOutI.data(), h->outI, (size_t)batch * OUT_I * sizeof(int), cudaMemcpyDeviceToHost, s));
  if (total) B2S_CUDA(cudaMemcpyAsync(h->hKeep.data(), h->keep, total, cudaMemcpyDeviceToHost, s));
  B2S_CUDA(cudaEventRecord(h->ev[1], s));
  B2S_CUDA(cudaStreamSynchronize(s));
  B2S_CUDA(cudaGetLastError());

  long long trials = 0;
  for (int i = 0; i < batch; i++) {
    b2s_sim3_result& R = r[i];
    const int* o = &h->hOutI[(size_t)i * OUT_I];
    memcpy(&R.S12_out, &h->hSout[(size_t)i * 8], 8 * sizeof(double));
    if (p[i].n) memcpy(R.keep, &h->hKeep[(size_t)h->hProb[(size_t)i].off], (size_t)p[i].n);
    R.n_inliers = o[0];
    R.n_trials = o[1];
    if (R.trace) {
      const int nt = std::min(o[1], 255);
      for (int k = 0; k < nt; k++) R.trace[k] = o[2 + k];
      R.trace[nt] = -1;
    }
    trials += o[1];
  }
  float ms = 0.f;
  B2S_CUDA(cudaEventElapsedTime(&ms, h->ev[0], h->ev[1]));
  h->lastMs = ms;
  h->lastTrials = trials;
  return B2S_OK;
}
