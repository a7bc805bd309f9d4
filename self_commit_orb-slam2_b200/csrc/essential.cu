// essential.cu — the essential-graph optimisation of loop closing: Optimizer::OptimizeEssentialGraph
// (src/Optimizer.cc:1017-1339) from the point where the graph is built, on the GPU.
//
// A Sim3 pose graph over every keyframe of the map: 7-DoF vertices (VertexSim3Expmap, oplus = Sim3(update) * estimate,
// update[6] = 0 under fix_scale), EdgeSim3 edges with identity information, one fixed vertex (the loop keyframe), 20
// Levenberg iterations from a user lambda of 1e-16.  EdgeSim3 has no analytic Jacobian, so g2o differentiates
// numerically (core/base_binary_edge.hpp:131-199, central differences with delta = 1e-9); this file does the same, which
// is why it is compiled without FMA contraction: the difference quotient amplifies last-bit differences of the error
// about 5e8 times.
//
// The LM loop (core/optimization_algorithm_levenberg.cpp:61-164) runs on the host with one synchronisation per trial.
// Per iteration / trial, on the device, FP64, no floating-point atomics (two calls give bit-identical outputs):
//   errors      one thread per edge: log(S_ji * S_i * S_j^-1), chi2 = e^T e, summed by the fixed two-level tree
//   linearise   one thread per (edge, endpoint, dimension): oplus(+delta), error, oplus(-delta), error, difference
//   assemble    one warp per free vertex (H_ii + lambda I, b_i over its edges in edge order) and one warp per lower
//               off-diagonal block (H_ij over the edges joining the pair, in edge order), written into the envelope tiles
//   solve       the tiled envelope Cholesky and substitutions of chol.cuh (7-scalar blocks)
//   update      Sim3(x_i) * S_i into a trial copy, trial chi2 and scale = x^T (lambda x + b)
// The write-back recovers [R t/s; 0 1] of every keyframe and moves every point with its reference keyframe:
// S_r,corrected^-1 (S_r,initial X).
#include <float.h>
#include <math.h>
#include <stddef.h>
#include <stdlib.h>

#include <algorithm>
#include <cmath>
#include <utility>
#include <vector>

#include "ba_math.cuh"
#include "chol.cuh"
#include "common.cuh"
#include "levenberg.cuh"
#include "sim3.cuh"

namespace b2s {
namespace eg {

using namespace chol;
constexpr int SD = 8;  // doubles per Sim3: q (x, y, z, w), t, s -- the layout of b2s_sim3
constexpr int JD = 98; // doubles per edge: the 7 x 7 Jacobians of both endpoints (row = error component)

// EdgeSim3::computeError (types_seven_dof_expmap.h:106-114): log(C * v1 * v2^-1)
__device__ __forceinline__ void edge_error(const double* C, const double* Si, const double* Sj, double* e) {
  double CS[SD], Sji[SD], E[SD];
  s3_mul(C, Si, CS);
  s3_inv(Sj, Sji);
  s3_mul(CS, Sji, E);
  s3_log(E, e);
}

struct Args {
  int nKf, nE, nFree, np, fixScale;
  const int* ei;          // vertex 0 of every edge
  const int* ej;          // vertex 1
  const double* meas;     // SD per edge
  const int* pidx;        // per keyframe: free-vertex index or -1 (the fixed keyframe, keyframes without an edge)
  const int* vOff;        // nFree + 1: incidence lists (edge << 1 | endpoint), edge order
  const int* vList;
  const int2* blk;        // lower off-diagonal blocks (row vertex, column vertex), by row then column
  const int* bOff;        // nBlk + 1: edges of each block, edge order
  const int* bList;
  double* err;            // 7 per edge
  double* chi2;           // per edge
  double* J;              // JD per edge
  double* b;              // npPad
  double* x;              // npPad
  double* tmp;            // max(nE, np)
  const int* envT;
  const long long* tileOff;
  double* tiles;
};

__global__ void k_errors(Args a, const double* __restrict__ est) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= a.nE) return;
  double er[7];
  edge_error(a.meas + (size_t)e * SD, est + (size_t)a.ei[e] * SD, est + (size_t)a.ej[e] * SD, er);
  double c = 0;
  for (int k = 0; k < 7; k++) {
    a.err[(size_t)e * 7 + k] = er[k];
    c += er[k] * er[k];
  }
  a.chi2[e] = c;
}

// VertexSim3Expmap::oplusImpl: Sim3(update) * estimate, update[6] = 0 under fix_scale
__device__ __forceinline__ void oplus(const double* est, const double* upd, int fixScale, double* o) {
  double u[7];
  for (int k = 0; k < 7; k++) u[k] = upd[k];
  if (fixScale) u[6] = 0;
  double S[SD];
  s3_exp(u, S);
  s3_mul(S, est, o);
}

// BaseBinaryEdge::linearizeOplus: thread (edge, endpoint, dimension) -> column d of that endpoint's Jacobian
__global__ void k_linearize(Args a, const double* __restrict__ est) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)a.nE * 14) return;
  const int e = (int)(t / 14), side = (int)(t % 14) / 7, d = (int)(t % 7);
  const int vi = a.ei[e], vj = a.ej[e];
  if (a.pidx[side ? vj : vi] < 0) return;  // fixed endpoint: no Jacobian
  const double delta = 1e-9;
  const double scalar = 1.0 / (2 * delta);
  const double* C = a.meas + (size_t)e * SD;
  double upd[7] = {0, 0, 0, 0, 0, 0, 0}, P[SD], ep[7], em[7];
  upd[d] = delta;
  oplus(est + (size_t)(side ? vj : vi) * SD, upd, a.fixScale, P);
  edge_error(C, side ? est + (size_t)vi * SD : P, side ? P : est + (size_t)vj * SD, ep);
  upd[d] = -delta;
  oplus(est + (size_t)(side ? vj : vi) * SD, upd, a.fixScale, P);
  edge_error(C, side ? est + (size_t)vi * SD : P, side ? P : est + (size_t)vj * SD, em);
  double* J = a.J + (size_t)e * JD + side * 49;
  for (int k = 0; k < 7; k++) J[k * 7 + d] = scalar * (ep[k] - em[k]);
}

// one warp per free vertex, over its edges in edge order: H_ii = sum J^T J (+ lambda on the diagonal) into the tiles,
// or (B_ONLY, once per iteration) b_i = -sum J^T e
template <bool B_ONLY>
__global__ void __launch_bounds__(256) k_assemble_diag(Args a, double lambda) {
  const int v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (v >= a.nFree) return;
  for (int ent = B_ONLY ? 49 + lane : lane; ent < (B_ONLY ? 56 : 49); ent += 32) {
    const int r = ent < 49 ? ent / 7 : ent - 49, c = ent % 7;
    if (ent < 49 && c > r) continue;
    double acc = 0;
    for (int q = a.vOff[v]; q < a.vOff[v + 1]; q++) {
      const int ev = a.vList[q], e = ev >> 1;
      const double* J = a.J + (size_t)e * JD + (ev & 1) * 49;
      double h = 0;
      if (ent < 49) {
        for (int k = 0; k < 7; k++) h += J[k * 7 + r] * J[k * 7 + c];
      } else {
        for (int k = 0; k < 7; k++) h += J[k * 7 + r] * -a.err[(size_t)e * 7 + k];
      }
      acc += h;
    }
    const int R = v * 7 + r;
    if (ent < 49) {
      const int Cc = v * 7 + c;
      tile_ptr(a, R / TS, Cc / TS)[(R % TS) * TS + (Cc % TS)] = r == c ? acc + lambda : acc;
    } else {
      a.b[R] = acc;
    }
  }
}

// one warp per lower off-diagonal block (R, C): sum over the edges joining the pair of J_R^T J_C, in edge order
__global__ void __launch_bounds__(256) k_assemble_off(Args a, int nBlk) {
  const int bk = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (bk >= nBlk) return;
  const int2 rc = a.blk[bk];
  for (int ent = lane; ent < 49; ent += 32) {
    const int r = ent / 7, c = ent % 7;
    double acc = 0;
    for (int q = a.bOff[bk]; q < a.bOff[bk + 1]; q++) {
      const int e = a.bList[q];
      const bool iRow = a.pidx[a.ei[e]] == rc.x;
      const double* JR = a.J + (size_t)e * JD + (iRow ? 0 : 49);
      const double* JC = a.J + (size_t)e * JD + (iRow ? 49 : 0);
      double h = 0;
      for (int k = 0; k < 7; k++) h += JR[k * 7 + r] * JC[k * 7 + c];
      acc += h;
    }
    const int R = rc.x * 7 + r, Cc = rc.y * 7 + c;
    tile_ptr(a, R / TS, Cc / TS)[(R % TS) * TS + (Cc % TS)] = acc;
  }
}

// SparseOptimizer::update into the trial copy (fix_scale zeroes x's scale entry, as oplusImpl does through its
// argument); tmp = x (lambda x + b) for computeScale
__global__ void k_update(Args a, const double* __restrict__ est, double* estT, double lambda) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= a.nKf) return;
  const int p = a.pidx[k];
  const double* S = est + (size_t)k * SD;
  double* o = estT + (size_t)k * SD;
  if (p < 0) {
    for (int i = 0; i < SD; i++) o[i] = S[i];
    return;
  }
  double* x = a.x + (size_t)p * 7;
  if (a.fixScale) x[6] = 0;
  oplus(S, x, 0, o);
  for (int i = 0; i < 7; i++) a.tmp[(size_t)p * 7 + i] = x[i] * (lambda * x[i] + a.b[(size_t)p * 7 + i]);
}

// SetPose([R t/s; 0 1]) of every keyframe; every point through its reference keyframe: correctedSwr.map(Srw.map(P))
__global__ void k_writeback(int nKf, int nMp, const double* __restrict__ est, const double* __restrict__ est0,
                            const float* __restrict__ P, const int* __restrict__ ref, float* Tcw, float* Pout) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nKf) {
    const double* S = est + (size_t)i * SD;
    double R[3][3];
    quat_to_R(S, R);
    const double is = 1. / S[7];
    float* T = Tcw + (size_t)i * 16;
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) T[r * 4 + c] = (float)R[r][c];
      T[r * 4 + 3] = (float)(S[4 + r] * is);
    }
    T[12] = 0.f; T[13] = 0.f; T[14] = 0.f; T[15] = 1.f;
  }
  if (i < nMp) {
    const int r = ref[i];
    if (r < 0) {
      for (int c = 0; c < 3; c++) Pout[(size_t)i * 3 + c] = P[(size_t)i * 3 + c];
      return;
    }
    const double X[3] = {P[(size_t)i * 3], P[(size_t)i * 3 + 1], P[(size_t)i * 3 + 2]};
    double Swr[SD], Y[3], Z[3];
    s3_inv(est + (size_t)r * SD, Swr);
    s3_map(est0 + (size_t)r * SD, X, Y);
    s3_map(Swr, Y, Z);
    for (int c = 0; c < 3; c++) Pout[(size_t)i * 3 + c] = (float)Z[c];
  }
}

}  // namespace eg
}  // namespace b2s

using namespace b2s;
using namespace b2s::eg;

// ================================================================================================ host side
struct b2s_eg_solver : b2s::Stage {
  int maxKf, maxE, maxMp;
  long long lastTrials = 0;
  // capacity-sized
  int *ei = nullptr, *ej = nullptr, *pidx = nullptr, *vOff = nullptr, *vList = nullptr, *bOff = nullptr, *bList = nullptr,
      *envT = nullptr, *ref = nullptr, *fail = nullptr;
  int2* blk = nullptr;
  long long* tileOff = nullptr;
  float *P = nullptr, *Pout = nullptr, *Tcw = nullptr;
  double *meas = nullptr, *est0 = nullptr, *est = nullptr, *estT = nullptr, *err = nullptr, *chi2 = nullptr, *J = nullptr,
         *b = nullptr, *rhs = nullptr, *ybuf = nullptr, *x = nullptr, *tmp = nullptr, *linv = nullptr, *part = nullptr,
         *scal = nullptr;
  double* hScal = nullptr;  // pinned
  int* hFail = nullptr;
  DevBuf tiles, rows;  // grown on demand
};

namespace {

inline int blocks(long long n, int t) { return (int)((n + t - 1) / t); }

int validate(const b2s_eg_solver* h, const b2s_eg_problem* p) {
  if (!p || p->n_kf < 1 || p->n_edges < 0 || p->n_mp < 0 || !p->Siw || (p->n_edges && !p->edges) ||
      (p->n_mp && (!p->points || !p->ref_kf))) {
    set_error("b2s_optimize_essential_graph: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  if (p->n_kf > h->maxKf || p->n_edges > h->maxE || p->n_mp > h->maxMp) {
    set_error("b2s_optimize_essential_graph: problem (%d keyframes, %d edges, %d points) exceeds the handle's capacity "
              "(%d, %d, %d)", p->n_kf, p->n_edges, p->n_mp, h->maxKf, h->maxE, h->maxMp);
    return B2S_ERR_CAPACITY;
  }
  if (p->fixed_kf < 0 || p->fixed_kf >= p->n_kf) {
    set_error("b2s_optimize_essential_graph: fixed_kf %d out of range", p->fixed_kf);
    return B2S_ERR_BAD_ARG;
  }
  for (int e = 0; e < p->n_edges; e++) {
    const b2s_sim3_edge& E = p->edges[e];
    if (E.i < 0 || E.i >= p->n_kf || E.j < 0 || E.j >= p->n_kf || E.i == E.j) {
      set_error("b2s_optimize_essential_graph: edge %d (%d, %d): bad vertex index", e, E.i, E.j);
      return B2S_ERR_BAD_ARG;
    }
  }
  for (int m = 0; m < p->n_mp; m++)
    if (p->ref_kf[m] < -1 || p->ref_kf[m] >= p->n_kf) {
      set_error("b2s_optimize_essential_graph: point %d: ref_kf %d out of range", m, p->ref_kf[m]);
      return B2S_ERR_BAD_ARG;
    }
  return B2S_OK;
}

}  // namespace

extern "C" int b2s_eg_create(int max_kf, int max_edges, int max_mp, int device, b2s_eg_solver** out) {
  if (!out || max_kf < 1 || max_edges < 1 || max_mp < 1 || max_kf > 16384) {
    set_error("b2s_eg_create: bad argument (capacities must be >= 1, max_kf <= 16384)");
    return B2S_ERR_BAD_ARG;
  }
  *out = nullptr;
  int rc = select_device(device);
  if (rc != B2S_OK) return rc;
  b2s_eg_solver* h = new b2s_eg_solver();
  h->maxKf = max_kf; h->maxE = max_edges; h->maxMp = max_mp;
  h->open(device);
  auto A = [h](auto* p, size_t bytes) { h->alloc(*p, bytes); };
  const size_t K = max_kf, E = max_edges, M = max_mp;
  const size_t npPad = ((K * 7 + TS - 1) / TS) * TS, nT = npPad / TS;
  A(&h->ei, E * 4); A(&h->ej, E * 4); A(&h->meas, E * SD * 8); A(&h->err, E * 7 * 8); A(&h->chi2, E * 8);
  A(&h->J, E * JD * 8); A(&h->vList, E * 2 * 4); A(&h->blk, E * 8); A(&h->bOff, (E + 1) * 4); A(&h->bList, E * 4);
  A(&h->pidx, K * 4); A(&h->vOff, (K + 1) * 4); A(&h->est0, K * SD * 8); A(&h->est, K * SD * 8);
  A(&h->estT, K * SD * 8); A(&h->Tcw, K * 64); A(&h->envT, nT * 4 + 4); A(&h->tileOff, (nT + 1) * 8);
  A(&h->b, npPad * 8); A(&h->rhs, npPad * 8); A(&h->ybuf, npPad * 8); A(&h->x, npPad * 8);
  A(&h->tmp, std::max(E, npPad) * 8); A(&h->linv, nT * TT * 8);
  A(&h->P, M * 12); A(&h->Pout, M * 12); A(&h->ref, M * 4);
  A(&h->part, RED_BLOCKS * 8); A(&h->scal, 4 * 8); A(&h->fail, 4);
  h->alloc_pinned(h->hScal, 4 * 8);
  h->alloc_pinned(h->hFail, 4);
  cudaError_t e = h->error;
  if (e == cudaSuccess) e = set_smem_limits();
  if (e != cudaSuccess) {
    set_error("b2s_eg_create: %s", cudaGetErrorString(e));
    b2s_eg_destroy(h);
    return B2S_ERR_CUDA;
  }
  *out = h;
  return B2S_OK;
}

extern "C" void b2s_eg_destroy(b2s_eg_solver* h) {
  if (!h) return;
  h->close();
  delete h;
}

extern "C" float b2s_eg_last_ms(const b2s_eg_solver* h, long long* lm_trials) {
  if (!h) return 0.f;
  if (lm_trials) *lm_trials = h->lastTrials;
  return h->lastMs;
}

extern "C" int b2s_optimize_essential_graph(b2s_eg_solver* h, const b2s_eg_problem* p, b2s_eg_result* r) {
  if (!h || !r || !r->Tcw_out || (p && p->n_mp > 0 && !r->points_out)) {
    set_error("b2s_optimize_essential_graph: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  int rc = validate(h, p);
  if (rc != B2S_OK) return rc;
  B2S_CUDA(cudaSetDevice(h->device));
  const int nKf = p->n_kf, nE = p->n_edges, nMp = p->n_mp;
  cudaStream_t s = h->stream;

  // ---- host: free vertices (not fixed, with an edge) in keyframe order, incidence lists, lower off-diagonal blocks
  std::vector<int> pidx((size_t)nKf, -1);
  std::vector<uint8_t> active((size_t)nKf, 0);
  for (int e = 0; e < nE; e++) active[(size_t)p->edges[e].i] = active[(size_t)p->edges[e].j] = 1;
  int nFree = 0;
  for (int k = 0; k < nKf; k++)
    if (active[(size_t)k] && k != p->fixed_kf) pidx[(size_t)k] = nFree++;
  std::vector<int> vOff((size_t)nFree + 1, 0), vList, bOff(1, 0), bList, ei((size_t)nE), ej((size_t)nE);
  std::vector<int2> blk;
  std::vector<double> meas((size_t)nE * SD);
  std::vector<std::pair<long long, int>> pairs;  // (row * nFree + column, edge), sorted stably by block
  for (int e = 0; e < nE; e++) {
    const b2s_sim3_edge& E = p->edges[e];
    ei[(size_t)e] = E.i;
    ej[(size_t)e] = E.j;
    memcpy(&meas[(size_t)e * SD], &E.meas, SD * 8);
    const int pi = pidx[(size_t)E.i], pj = pidx[(size_t)E.j];
    if (pi >= 0) vOff[(size_t)pi + 1]++;
    if (pj >= 0) vOff[(size_t)pj + 1]++;
    if (pi >= 0 && pj >= 0) pairs.push_back({(long long)std::max(pi, pj) * nFree + std::min(pi, pj), e});
  }
  for (int v = 0; v < nFree; v++) vOff[(size_t)v + 1] += vOff[(size_t)v];
  vList.resize((size_t)vOff[(size_t)nFree]);
  {
    std::vector<int> fill(vOff.begin(), vOff.end() - 1);
    for (int e = 0; e < nE; e++) {
      const int pi = pidx[(size_t)ei[(size_t)e]], pj = pidx[(size_t)ej[(size_t)e]];
      if (pi >= 0) vList[(size_t)fill[(size_t)pi]++] = e << 1;
      if (pj >= 0) vList[(size_t)fill[(size_t)pj]++] = e << 1 | 1;
    }
  }
  std::stable_sort(pairs.begin(), pairs.end(),
                   [](const std::pair<long long, int>& x, const std::pair<long long, int>& y) { return x.first < y.first; });
  std::vector<int> envBlk((size_t)nFree);
  for (int v = 0; v < nFree; v++) envBlk[(size_t)v] = v;
  for (size_t q = 0; q < pairs.size(); q++) {
    if (q == 0 || pairs[q].first != pairs[q - 1].first) {
      const int R = (int)(pairs[q].first / nFree), C = (int)(pairs[q].first % nFree);
      blk.push_back(make_int2(R, C));
      if (q) bOff.push_back((int)q);
      envBlk[(size_t)R] = std::min(envBlk[(size_t)R], C);
    }
    bList.push_back(pairs[q].second);
  }
  if (!pairs.empty()) bOff.push_back((int)pairs.size());
  const int nBlk = (int)blk.size();
  std::vector<int> envT, rowOff, rows;
  std::vector<long long> off;
  const long long nTiles = tile_envelope(envBlk, nFree, 7, envT, off, rowOff, rows);
  const int np = nFree * 7, nT = (int)envT.size(), npPad = nT * TS;
  rc = grow(h->tiles, (size_t)nTiles * TT * 8);
  if (rc == B2S_OK) rc = grow(h->rows, rows.size() * 4);
  if (rc != B2S_OK) return rc;

  HostSync sync = {s, h->ev, h->hScal, h->scal, h->hFail, h->fail, 0.f};
  rc = sync.start();
  if (rc != B2S_OK) return rc;
  // ---- upload
  B2S_CUDA(cudaMemcpyAsync(h->est0, p->Siw, (size_t)nKf * SD * 8, cudaMemcpyHostToDevice, s));
  B2S_CUDA(cudaMemcpyAsync(h->est, p->Siw, (size_t)nKf * SD * 8, cudaMemcpyHostToDevice, s));
  B2S_CUDA(cudaMemcpyAsync(h->pidx, pidx.data(), (size_t)nKf * 4, cudaMemcpyHostToDevice, s));
  if (nE) {
    B2S_CUDA(cudaMemcpyAsync(h->ei, ei.data(), (size_t)nE * 4, cudaMemcpyHostToDevice, s));
    B2S_CUDA(cudaMemcpyAsync(h->ej, ej.data(), (size_t)nE * 4, cudaMemcpyHostToDevice, s));
    B2S_CUDA(cudaMemcpyAsync(h->meas, meas.data(), (size_t)nE * SD * 8, cudaMemcpyHostToDevice, s));
    B2S_CUDA(cudaMemcpyAsync(h->vOff, vOff.data(), vOff.size() * 4, cudaMemcpyHostToDevice, s));
    B2S_CUDA(cudaMemcpyAsync(h->vList, vList.data(), vList.size() * 4, cudaMemcpyHostToDevice, s));
  }
  if (nBlk) {
    B2S_CUDA(cudaMemcpyAsync(h->blk, blk.data(), (size_t)nBlk * 8, cudaMemcpyHostToDevice, s));
    B2S_CUDA(cudaMemcpyAsync(h->bOff, bOff.data(), bOff.size() * 4, cudaMemcpyHostToDevice, s));
    B2S_CUDA(cudaMemcpyAsync(h->bList, bList.data(), bList.size() * 4, cudaMemcpyHostToDevice, s));
  }
  if (nT) {
    B2S_CUDA(cudaMemcpyAsync(h->envT, envT.data(), (size_t)nT * 4, cudaMemcpyHostToDevice, s));
    B2S_CUDA(cudaMemcpyAsync(h->tileOff, off.data(), (size_t)(nT + 1) * 8, cudaMemcpyHostToDevice, s));
    B2S_CUDA(cudaMemsetAsync(h->b, 0, (size_t)npPad * 8, s));
    B2S_CUDA(cudaMemsetAsync(h->x, 0, (size_t)npPad * 8, s));
  }
  if (!rows.empty()) B2S_CUDA(cudaMemcpyAsync(h->rows.p, rows.data(), rows.size() * 4, cudaMemcpyHostToDevice, s));
  if (nMp) {
    B2S_CUDA(cudaMemcpyAsync(h->P, p->points, (size_t)nMp * 12, cudaMemcpyHostToDevice, s));
    B2S_CUDA(cudaMemcpyAsync(h->ref, p->ref_kf, (size_t)nMp * 4, cudaMemcpyHostToDevice, s));
  }

  Args a;
  memset(&a, 0, sizeof(a));
  a.nKf = nKf; a.nE = nE; a.nFree = nFree; a.np = np; a.fixScale = p->fix_scale != 0;
  a.ei = h->ei; a.ej = h->ej; a.meas = h->meas; a.pidx = h->pidx; a.vOff = h->vOff; a.vList = h->vList; a.blk = h->blk;
  a.bOff = h->bOff; a.bList = h->bList; a.err = h->err; a.chi2 = h->chi2; a.J = h->J; a.b = h->b;
  a.x = h->x; a.tmp = h->tmp; a.envT = h->envT; a.tileOff = h->tileOff; a.tiles = (double*)h->tiles.p;
  const TileSys ts = {np, h->envT, h->tileOff, (double*)h->tiles.p, h->linv, h->rhs, h->ybuf, h->x, h->fail};
  const size_t tileBytes = (size_t)nTiles * TT * 8;

  double* est = h->est;
  double* estT = h->estT;
  auto chi2_of = [&](const double* S, double* out) {
    k_errors<<<blocks(nE, 128), 128, 0, s>>>(a, S);
    chol::reduce<0>(h->chi2, nE, h->part, out, s);
  };

  // ---- SparseOptimizer::optimize(20) + OptimizationAlgorithmLevenberg::solve (an empty graph optimises nothing)
  Levenberg lm = {};
  int32_t trace[256];
  double chi2Initial = 0;
  lm.init_lambda(1e-16);  // computeLambdaInit returns the user lambda (setUserLambdaInit(1e-16), :1035)
  bool ok = nE > 0;
  for (int it = 0; it < 20 && ok; it++) {
    chi2_of(est, h->scal);
    k_linearize<<<blocks((long long)nE * 14, 128), 128, 0, s>>>(a, est);
    k_assemble_diag<true><<<blocks((long long)nFree * 32, 256), 256, 0, s>>>(a, 0.0);
    rc = sync.scalars(1);
    if (rc != B2S_OK) return rc;
    lm.begin(h->hScal[0]);
    if (it == 0) chi2Initial = lm.currentChi;
    do {
      B2S_CUDA(cudaMemsetAsync(h->fail, 0, 4, s));
      B2S_CUDA(cudaMemsetAsync(h->tiles.p, 0, tileBytes, s));
      B2S_CUDA(cudaMemcpyAsync(h->rhs, h->b, (size_t)npPad * 8, cudaMemcpyDeviceToDevice, s));
      k_assemble_diag<false><<<blocks((long long)nFree * 32, 256), 256, 0, s>>>(a, lm.lambda);
      if (nBlk) k_assemble_off<<<blocks((long long)nBlk * 32, 256), 256, 0, s>>>(a, nBlk);
      factor_solve(ts, nT, envT, rowOff, (const int*)h->rows.p, s);
      k_update<<<blocks(nKf, 128), 128, 0, s>>>(a, est, estT, lm.lambda);
      chi2_of(estT, h->scal);
      chol::reduce<0>(h->tmp, np, h->part, h->scal + 1, s);
      rc = sync.scalars(2);
      if (rc != B2S_OK) return rc;
      if (lm.trial(*h->hFail == 0, h->hScal[0], h->hScal[1], trace)) std::swap(est, estT);
    } while (lm.retry(false));
    if (lm.end_iteration()) break;
  }

  // ---- write-back and the chi2 of the returned estimate
  if (nE) chi2_of(est, h->scal);
  else B2S_CUDA(cudaMemsetAsync(h->scal, 0, 8, s));
  k_writeback<<<blocks(std::max(nKf, nMp), 256), 256, 0, s>>>(nKf, nMp, est, h->est0, h->P, h->ref, h->Tcw, h->Pout);
  B2S_CUDA(cudaMemcpyAsync(r->Tcw_out, h->Tcw, (size_t)nKf * 64, cudaMemcpyDeviceToHost, s));
  if (nMp) B2S_CUDA(cudaMemcpyAsync(r->points_out, h->Pout, (size_t)nMp * 12, cudaMemcpyDeviceToHost, s));
  B2S_CUDA(cudaMemcpyAsync(h->hScal, h->scal, 8, cudaMemcpyDeviceToHost, s));
  rc = sync.stream();
  if (rc != B2S_OK) return rc;
  B2S_CUDA(cudaGetLastError());
  r->chi2_initial = nE ? chi2Initial : 0.0;
  r->chi2_final = h->hScal[0];
  r->n_trials = lm.nTrials;
  if (r->trace) {
    const int n = std::min(lm.nTrials, 255);
    for (int i = 0; i < n; i++) r->trace[i] = trace[i];
    r->trace[n] = -1;
  }
  h->lastMs = sync.busyMs;
  h->lastTrials = lm.nTrials;
  return B2S_OK;
}
