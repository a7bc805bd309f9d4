// gba.cu — global bundle adjustment: Optimizer::BundleAdjustment (src/Optimizer.cc:86-341), the body of
// GlobalBundleAdjustemnt, for whole maps (thousands of keyframes, hundreds of thousands of points) on the whole GPU.
//
// The Levenberg loop of g2o (core/optimization_algorithm_levenberg.cpp:61-189, sparse_optimizer.cpp:354-435) runs on the
// host; each LM trial is a sequence of kernels and ends in one synchronisation that returns the trial chi2, the
// predicted gain and the factorisation status.  Per call, on the device:
//   structure   CSR of the edges by point (they arrive grouped by point) and by free keyframe (stable radix sort), the
//               covisibility pair records {row edge, column edge, point} of every lower 6x6 block of the reduced camera
//               system S, sorted by block (stable radix sort: points ascending inside a block), the unique blocks and the
//               block envelope (first non-zero block column of every block row); the host turns the envelope into
//               64 x 64 tiles and sizes the tile storage from it.
// Per iteration / trial:
//   errors      one thread per edge; the robust chi2 is summed by a fixed two-level tree (no atomics in this file)
//   linearise   one thread per point (Hll, b_l and the W_e blocks of its edges, in edge order), one warp per free
//               keyframe (Hpp, b_p over its CSR list: lane-strided, then a fixed butterfly)
//   Schur       Dinv per point; S = Hpp + lambda I - sum W Dinv W^T: one warp per lower block over its pair list in order,
//               written straight into the envelope tiles
//   Cholesky    tiled right-looking over the tile envelope: the diagonal tile is factorised and inverted by one CTA, the
//               panel (L_IK = A_IK Linv_KK^T) and the trailing update (A_IJ -= L_IK L_JK^T) run on many CTAs with
//               mma.sync.m8n8k4.f64 (DMMA); tiles left of a row's envelope are never touched (skyline fill-in stays
//               inside the envelope, so skipping them is exact)
//   solve       blocked forward / backward substitution with the inverted diagonal tiles, then x_l = Dinv (b_l - W^T x_p)
//   update      SE3 exp update and point step into a trial copy, trial chi2 and scale = x^T (lambda x + b)
// Keyframes without an edge are inactive vertices (no block, estimate kept); points without an edge are excluded (inert
// here, not written back).  A non-positive pivot is a rejected LM step (tempChi = DBL_MAX), as in the LocalBA path.
#include <float.h>
#include <math.h>
#include <stddef.h>
#include <stdlib.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include <cub/cub.cuh>

#include "ba_math.cuh"
#include "chol.cuh"
#include "common.cuh"
#include "levenberg.cuh"

namespace b2s {
namespace gba {

using namespace chol;  // tiles, deterministic sums, the tiled Cholesky (chol.cuh)

struct Cam {
  float fx, fy, cx, cy, bf;
};

// computeError (types_six_dof_expmap.h:90-95 mono, :122-127 stereo; cam_project .cpp:141-157) from camera coordinates
__device__ __forceinline__ double edge_error(const double* Xc, bool stereo, const float* ob, double wgt, const Cam& C,
                                             double* e) {
  if (stereo) {
    const float invz = (float)(1.0 / Xc[2]);  // const float invz = 1.0f/trans_xyz[2]  (.cpp:151)
    const double u = Xc[0] * invz * (double)C.fx + (double)C.cx;
    const double v = Xc[1] * invz * (double)C.fy + (double)C.cy;
    const double ur = u - (double)__fmul_rn(C.bf, invz);
    e[0] = (double)ob[0] - u;
    e[1] = (double)ob[1] - v;
    e[2] = (double)ob[2] - ur;
    return e[0] * (wgt * e[0]) + e[1] * (wgt * e[1]) + e[2] * (wgt * e[2]);
  }
  const double u = Xc[0] / Xc[2] * (double)C.fx + (double)C.cx;
  const double v = Xc[1] / Xc[2] * (double)C.fy + (double)C.cy;
  e[0] = (double)ob[0] - u;
  e[1] = (double)ob[1] - v;
  e[2] = 0;
  return e[0] * (wgt * e[0]) + e[1] * (wgt * e[1]);
}

// const float thHuber2D = sqrt(5.99), thHuber3D = sqrt(7.815)  (src/Optimizer.cc:141-142).  BundleAdjustment's own
// constants: its monocular threshold is sqrt(5.99), not LocalBA / PoseOptimization's sqrt(5.991) (delta_of, localba.cu).
__device__ __forceinline__ double gba_delta(bool stereo) {
  return stereo ? (double)(float)2.795532150593156 : (double)(float)2.4474476501040834;
}

struct Edges {
  const int* kf;
  const int* mp;
  const float* obs;  // 3 per edge
  const float* w;    // inv_sigma2
};

// ================================================================================================ set-up and structure
// Converter::toSE3Quat (src/Converter.cc:57-66) / toVector3d
__global__ void k_pose_init(const float* __restrict__ Tcw, int nKf, double* pose) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nKf) return;
  se3quat_from_Tcw(Tcw + (size_t)k * 16, pose + (size_t)k * POSE_STRIDE);
}
__global__ void k_point_init(const float* __restrict__ X, int n, double* pts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) pts[i] = X[i];
}
// point CSR: [ptBeg, ptEnd) of every point (0, 0 for a point without an edge)
__global__ void k_point_csr(const int* __restrict__ eMp, int nE, int* ptBeg, int* ptEnd) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= nE) return;
  const int m = eMp[e];
  if (e == 0 || eMp[e - 1] != m) ptBeg[m] = e;
  if (e == nE - 1 || eMp[e + 1] != m) ptEnd[m] = e + 1;
}
// sort key of an edge for the keyframe CSR: its free-pose index, nFree for an edge of a fixed / inactive keyframe
__global__ void k_kf_keys(const int* __restrict__ eKf, const int* __restrict__ pidx, int nE, int nFree, unsigned* key,
                          int* val) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= nE) return;
  const int p = pidx[eKf[e]];
  key[e] = p >= 0 ? (unsigned)p : (unsigned)nFree;
  val[e] = e;
}
__global__ void k_kf_csr(const unsigned* __restrict__ key, int nE, int nFree, int* kfBeg, int* kfEnd) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= nE) return;
  const unsigned k = key[e];
  if (k >= (unsigned)nFree) return;
  if (e == 0 || key[e - 1] != k) kfBeg[k] = e;
  if (e == nE - 1 || key[e + 1] != k) kfEnd[k] = e + 1;
}
// pairs per point: f (f + 1) / 2 over its f edges with a free keyframe
__global__ void k_pair_count(const int* __restrict__ ptBeg, const int* __restrict__ ptEnd, const int* __restrict__ eKf,
                             const int* __restrict__ pidx, int nMp, long long* cnt) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m > nMp) return;
  if (m == nMp) {
    cnt[m] = 0;
    return;
  }
  long long f = 0;
  for (int e = ptBeg[m]; e < ptEnd[m]; e++) f += pidx[eKf[e]] >= 0;
  cnt[m] = f * (f + 1) / 2;
}
// pair records of point m in (a, c) edge order; oriented so that the row edge has the larger pose index (lower block)
__global__ void k_pair_emit(const int* __restrict__ ptBeg, const int* __restrict__ ptEnd, const int* __restrict__ eKf,
                            const int* __restrict__ pidx, const long long* __restrict__ off, int nMp, int nFree,
                            unsigned* key, unsigned* val, int4* rec) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= nMp) return;
  long long o = off[m];
  for (int a = ptBeg[m]; a < ptEnd[m]; a++) {
    const int pa = pidx[eKf[a]];
    if (pa < 0) continue;
    for (int c = a; c < ptEnd[m]; c++) {
      const int pc = pidx[eKf[c]];
      if (pc < 0) continue;
      const bool aRow = pa >= pc;
      key[o] = (unsigned)(aRow ? pa : pc) * (unsigned)nFree + (unsigned)(aRow ? pc : pa);
      val[o] = (unsigned)o;
      rec[o] = make_int4(aRow ? a : c, aRow ? c : a, m, 0);
      o++;
    }
  }
}
__global__ void k_pair_gather(const unsigned* __restrict__ order, const int4* __restrict__ rec, long long n, int4* out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = rec[order[i]];
}
// first block column of every block row (the diagonal block always exists: a free keyframe has an edge)
__global__ void k_envelope(const unsigned* __restrict__ ukey, int nBlk, int nFree, int* envBlk) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nBlk) return;
  const unsigned i = ukey[b] / (unsigned)nFree;
  if (b == 0 || ukey[b - 1] / (unsigned)nFree != i) envBlk[i] = (int)(ukey[b] % (unsigned)nFree);
}

// ================================================================================================ LM stages
struct LmArgs {
  Edges E;
  Cam C;
  int nKf, nMp, nE, nFree, np, npPad;
  int robust;
  const int* pidx;   // per keyframe: free-pose index or -1
  const int *ptBeg, *ptEnd, *kfBeg, *kfEnd, *kfEdge;
  double* err;       // 3 per edge
  double* chi2;      // per edge
  double* rho;       // per edge: robustified chi2
  double* Hpp;       // nFree x 36
  double* Hll;       // nMp x 9
  double* b;         // [npPad | nMp x 3]
  double* W;         // 18 per edge (edges of free keyframes)
  double* Dinv;      // nMp x 9
  double* db;        // nMp x 3: Dinv b_l
  double* x;         // [npPad | nMp x 3]
  double* rhs;       // npPad
  double* ybuf;      // npPad
  double* tmp;       // max(nE, npPad + 3 nMp): per-element terms of the sums
  const int* envT;   // per tile row
  const long long* tileOff;
  double* tiles;
  double* linv;      // nT x TT
  int* fail;
};

__global__ void k_errors(LmArgs a, const double* __restrict__ pose, const double* __restrict__ pts) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= a.nE) return;
  const double* X = pts + (size_t)a.E.mp[e] * 3;
  double Xc[3];
  pose_map(pose + (size_t)a.E.kf[e] * POSE_STRIDE, X, Xc);
  const float* ob = a.E.obs + (size_t)e * 3;
  const bool st = !(ob[2] < 0);
  double er[3];
  const double c = edge_error(Xc, st, ob, (double)a.E.w[e], a.C, er);
  a.err[(size_t)e * 3] = er[0];
  a.err[(size_t)e * 3 + 1] = er[1];
  a.err[(size_t)e * 3 + 2] = er[2];
  a.chi2[e] = c;
  double r0 = c, r1;
  if (a.robust) huber(c, gba_delta(st), r0, r1);
  a.rho[e] = r0;
}

struct EdgeLin {
  EdgeJac J;
  double omega[3];  // -(w0 e_r) rho1
  double w;         // rho1 w0
  int D;
};
__device__ __forceinline__ void edge_lin(const LmArgs& a, const double* pose, const double* pts, int e, EdgeLin& L) {
  const float* ob = a.E.obs + (size_t)e * 3;
  const bool st = !(ob[2] < 0);
  edge_jacobians(pose + (size_t)a.E.kf[e] * POSE_STRIDE, pts + (size_t)a.E.mp[e] * 3, st, (double)a.C.fx, (double)a.C.fy,
                 (double)a.C.bf, L.J);
  const double w0 = (double)a.E.w[e];
  double rho1 = 1.0;
  if (a.robust) {
    double r0;
    huber(a.chi2[e], gba_delta(st), r0, rho1);
  }
  for (int r = 0; r < 3; r++) L.omega[r] = -(w0 * a.err[(size_t)e * 3 + r]) * rho1;
  L.w = rho1 * w0;
  L.D = st ? 3 : 2;
}

// one thread per point: Hll, b_l and W_e = B^T w A of its edges, in edge order (constructQuadraticForm)
__global__ void k_build_points(LmArgs a, const double* __restrict__ pose, const double* __restrict__ pts) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= a.nMp) return;
  double H[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, bl[3] = {0, 0, 0};
  for (int e = a.ptBeg[m]; e < a.ptEnd[m]; e++) {
    EdgeLin L;
    edge_lin(a, pose, pts, e, L);
    for (int i = 0; i < 3; i++) {
      double s = 0;
      for (int r = 0; r < L.D; r++) s += L.J.A[r][i] * L.omega[r];
      bl[i] += s;
      for (int j = 0; j < 3; j++) {
        double h = 0;
        for (int r = 0; r < L.D; r++) h += L.J.A[r][i] * L.w * L.J.A[r][j];
        H[i * 3 + j] += h;
      }
    }
    if (a.pidx[a.E.kf[e]] >= 0) {
      double* W = a.W + (size_t)e * 18;
      for (int i = 0; i < 6; i++)
        for (int j = 0; j < 3; j++) {
          double h = 0;
          for (int r = 0; r < L.D; r++) h += L.J.B[r][i] * L.w * L.J.A[r][j];
          W[i * 3 + j] = h;
        }
    }
  }
  for (int k = 0; k < 9; k++) a.Hll[(size_t)m * 9 + k] = H[k];
  for (int k = 0; k < 3; k++) a.b[(size_t)a.npPad + (size_t)m * 3 + k] = bl[k];
}

// one warp per free keyframe: Hpp and b_p over its CSR edge list (lane-strided partial sums, fixed butterfly)
__global__ void __launch_bounds__(256) k_build_poses(LmArgs a, const double* __restrict__ pose,
                                                     const double* __restrict__ pts) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= a.nFree) return;
  double H[21], bp[6];
#pragma unroll
  for (int k = 0; k < 21; k++) H[k] = 0;
#pragma unroll
  for (int k = 0; k < 6; k++) bp[k] = 0;
  for (int q = a.kfBeg[i] + lane; q < a.kfEnd[i]; q += 32) {
    const int e = a.kfEdge[q];
    EdgeLin L;
    edge_lin(a, pose, pts, e, L);
    int k = 0;
#pragma unroll
    for (int r1 = 0; r1 < 6; r1++) {
      double s = 0;
      for (int r = 0; r < L.D; r++) s += L.J.B[r][r1] * L.omega[r];
      bp[r1] += s;
#pragma unroll
      for (int c1 = 0; c1 <= r1; c1++) {
        double h = 0;
        for (int r = 0; r < L.D; r++) h += L.J.B[r][r1] * L.w * L.J.B[r][c1];
        H[k++] += h;
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 21; k++) H[k] = warp_sum(H[k]);
#pragma unroll
  for (int k = 0; k < 6; k++) bp[k] = warp_sum(bp[k]);
  if (lane == 0) {
    double* Hp = a.Hpp + (size_t)i * 36;
    int k = 0;
    for (int r1 = 0; r1 < 6; r1++)
      for (int c1 = 0; c1 <= r1; c1++, k++) {
        Hp[r1 * 6 + c1] = H[k];
        Hp[c1 * 6 + r1] = H[k];
      }
    for (int r1 = 0; r1 < 6; r1++) a.b[(size_t)i * 6 + r1] = bp[r1];
  }
}

// diagonals of all active free vertices, for lambda_0 (computeLambdaInit)
__global__ void k_diag(LmArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int nP = a.nFree * 6;
  if (i < nP) a.tmp[i] = a.Hpp[(size_t)(i / 6) * 36 + (i % 6) * 7];
  else if (i < nP + a.nMp * 3) {
    const int m = (i - nP) / 3, c = (i - nP) % 3;
    a.tmp[i] = a.Hll[(size_t)m * 9 + c * 4];
  }
}

// Dinv = (Hll + lambda I)^-1 (Eigen 3x3 cofactor inverse), db = Dinv b_l
__global__ void k_dinv(LmArgs a, double lambda) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= a.nMp) return;
  double D[9];
  for (int k = 0; k < 9; k++) D[k] = a.Hll[(size_t)m * 9 + k];
  D[0] += lambda; D[4] += lambda; D[8] += lambda;
  const double c00 = D[4] * D[8] - D[5] * D[7];
  const double c01 = D[5] * D[6] - D[3] * D[8];
  const double c02 = D[3] * D[7] - D[4] * D[6];
  const double id = 1.0 / (D[0] * c00 + D[1] * c01 + D[2] * c02);
  double Di[9];
  Di[0] = c00 * id; Di[1] = (D[2] * D[7] - D[1] * D[8]) * id; Di[2] = (D[1] * D[5] - D[2] * D[4]) * id;
  Di[3] = c01 * id; Di[4] = (D[0] * D[8] - D[2] * D[6]) * id; Di[5] = (D[2] * D[3] - D[0] * D[5]) * id;
  Di[6] = c02 * id; Di[7] = (D[1] * D[6] - D[0] * D[7]) * id; Di[8] = (D[0] * D[4] - D[1] * D[3]) * id;
  for (int k = 0; k < 9; k++) a.Dinv[(size_t)m * 9 + k] = Di[k];
  const double* bl = a.b + (size_t)a.npPad + (size_t)m * 3;
  for (int i = 0; i < 3; i++) a.db[(size_t)m * 3 + i] = Di[i * 3] * bl[0] + Di[i * 3 + 1] * bl[1] + Di[i * 3 + 2] * bl[2];
}

// reduced right-hand side: rhs_i = b_i - sum_e W_e Dinv b_l (one warp per free keyframe)
__global__ void __launch_bounds__(256) k_rhs(LmArgs a) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= a.nFree) return;
  double s[6] = {0, 0, 0, 0, 0, 0};
  for (int q = a.kfBeg[i] + lane; q < a.kfEnd[i]; q += 32) {
    const int e = a.kfEdge[q];
    const double* W = a.W + (size_t)e * 18;
    const double* d = a.db + (size_t)a.E.mp[e] * 3;
#pragma unroll
    for (int r = 0; r < 6; r++) s[r] += W[r * 3] * d[0] + W[r * 3 + 1] * d[1] + W[r * 3 + 2] * d[2];
  }
#pragma unroll
  for (int r = 0; r < 6; r++) s[r] = warp_sum(s[r]);
  if (lane < 6) {
    double v = s[0];
#pragma unroll
    for (int r = 1; r < 6; r++)
      if (lane == r) v = s[r];
    a.rhs[(size_t)i * 6 + lane] = a.b[(size_t)i * 6 + lane] - v;
  }
}

// one warp per lower 6x6 block (i, j) of S, summed over its pair records in order, written into the envelope tiles
__global__ void __launch_bounds__(256) k_schur(LmArgs a, const unsigned* __restrict__ ukey, const int* __restrict__ blkBeg,
                                               int nBlk, const int4* __restrict__ rec, double lambda) {
  const int blk = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (blk >= nBlk) return;
  const int i = (int)(ukey[blk] / (unsigned)a.nFree), j = (int)(ukey[blk] % (unsigned)a.nFree);
  const int q0 = blkBeg[blk], q1 = blkBeg[blk + 1];
  for (int ent = lane; ent < 36; ent += 32) {
    const int r = ent / 6, c = ent % 6;
    if (i == j && c > r) continue;
    double acc = 0;
    for (int q = q0; q < q1; q++) {
      const int4 p = rec[q];
      const double* Wa = a.W + (size_t)p.x * 18 + r * 3;
      const double* Wc = a.W + (size_t)p.y * 18 + c * 3;
      const double* Di = a.Dinv + (size_t)p.z * 9;
      const double t0 = Wa[0] * Di[0] + Wa[1] * Di[3] + Wa[2] * Di[6];
      const double t1 = Wa[0] * Di[1] + Wa[1] * Di[4] + Wa[2] * Di[7];
      const double t2 = Wa[0] * Di[2] + Wa[1] * Di[5] + Wa[2] * Di[8];
      acc += t0 * Wc[0] + t1 * Wc[1] + t2 * Wc[2];
    }
    double v = -acc;
    if (i == j) v = (a.Hpp[(size_t)i * 36 + r * 6 + c] + (r == c ? lambda : 0.0)) - acc;
    const int R = i * 6 + r, Cc = j * 6 + c;
    tile_ptr(a, R / TS, Cc / TS)[(R % TS) * TS + (Cc % TS)] = v;
  }
}

// x_l = Dinv (b_l - sum_e W_e^T x_p)
__global__ void k_backsub_points(LmArgs a) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= a.nMp) return;
  const double* bl = a.b + (size_t)a.npPad + (size_t)m * 3;
  double cl[3] = {bl[0], bl[1], bl[2]};
  for (int e = a.ptBeg[m]; e < a.ptEnd[m]; e++) {
    const int p = a.pidx[a.E.kf[e]];
    if (p < 0) continue;
    const double* W = a.W + (size_t)e * 18;
    const double* xp = a.x + (size_t)p * 6;
    for (int c = 0; c < 3; c++)
      for (int r = 0; r < 6; r++) cl[c] -= W[r * 3 + c] * xp[r];
  }
  const double* Di = a.Dinv + (size_t)m * 9;
  for (int i = 0; i < 3; i++)
    a.x[(size_t)a.npPad + (size_t)m * 3 + i] = Di[i * 3] * cl[0] + Di[i * 3 + 1] * cl[1] + Di[i * 3 + 2] * cl[2];
}

// trial estimate: SE3Quat::exp(x) * T for free keyframes (the others are copied), X + x_l for points;
// tmp = x (lambda x + b) for computeScale
__global__ void k_update(LmArgs a, const double* __restrict__ pose, const double* __restrict__ pts, double* poseT,
                         double* ptsT, double lambda) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < a.nKf) {
    double P[POSE_STRIDE];
    for (int k = 0; k < POSE_STRIDE; k++) P[k] = pose[(size_t)i * POSE_STRIDE + k];
    const int p = a.pidx[i];
    if (p >= 0) pose_oplus(P, a.x + (size_t)p * 6);
    for (int k = 0; k < POSE_STRIDE; k++) poseT[(size_t)i * POSE_STRIDE + k] = P[k];
  }
  if (i < a.nMp * 3) ptsT[i] = pts[i] + a.x[(size_t)a.npPad + i];
  if (i < a.npPad + a.nMp * 3) a.tmp[i] = a.x[i] * (lambda * a.x[i] + a.b[i]);
}

// Converter::toCvMat(SE3Quat) of every keyframe; points with an edge
__global__ void k_writeback(LmArgs a, const double* __restrict__ pose, const double* __restrict__ pts, float* Tcw,
                            float* X) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < a.nKf) se3quat_to_Tcw(pose + (size_t)i * POSE_STRIDE, Tcw + (size_t)i * 16);
  if (i < a.nMp * 3) X[i] = (float)pts[i];
}

}  // namespace gba
}  // namespace b2s

using namespace b2s;
using namespace b2s::gba;

// ================================================================================================ host side
struct b2s_gba_solver : b2s::Stage {
  int maxKf, maxMp, maxE;
  long long lastTrials = 0;
  // capacity-sized
  int *eKf = nullptr, *eMp = nullptr, *pidx = nullptr, *ptBeg = nullptr, *ptEnd = nullptr, *kfBeg = nullptr,
      *kfEnd = nullptr, *kfEdge = nullptr, *kfVal = nullptr, *envBlk = nullptr, *envT = nullptr;
  unsigned *kfKey = nullptr, *kfKeyS = nullptr;
  float *eObs = nullptr, *eW = nullptr, *Tcw = nullptr, *X = nullptr;
  double *pose = nullptr, *poseT = nullptr, *pts = nullptr, *ptsT = nullptr, *err = nullptr, *chi2 = nullptr,
         *rho = nullptr, *Hpp = nullptr, *Hll = nullptr, *W = nullptr, *Dinv = nullptr, *db = nullptr, *part = nullptr,
         *scal = nullptr;
  long long *pairCnt = nullptr, *pairOff = nullptr, *tileOff = nullptr;
  uint8_t* fixedD = nullptr;
  int* fail = nullptr;
  double* hScal = nullptr;  // pinned: [0] sum, [1] second sum; fail read separately
  int* hFail = nullptr;
  // grown on demand
  DevBuf pairKey, pairKeyS, pairVal, pairValS, pairRec, pairRecS, uKey, runLen, blkBeg, nRuns, cubTmp, tiles, linv, bvec, xvec,
      rhs, ybuf, tmp, rows;
};

namespace {

inline int blocks(long long n, int t) { return (int)((n + t - 1) / t); }

// deterministic sum (OP 0) or max |.| (OP 1) of v[0, n) into *out (device)
template <int OP>
void reduce(b2s_gba_solver* h, const double* v, long long n, double* out) {
  chol::reduce<OP>(v, n, h->part, out, h->stream);
}

int validate(const b2s_gba_solver* h, const b2s_gba_problem* p) {
  if (!p || p->n_kf < 0 || p->n_mp < 0 || p->n_edges < 0 || p->iterations < 0 || (p->n_kf && (!p->Tcw || !p->fixed)) ||
      (p->n_mp && !p->points) || (p->n_edges && !p->edges)) {
    set_error("b2s_global_ba: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  if (p->n_kf > h->maxKf || p->n_mp > h->maxMp || p->n_edges > h->maxE) {
    set_error("b2s_global_ba: problem (%d keyframes, %d points, %d edges) exceeds the handle's capacity (%d, %d, %d)",
              p->n_kf, p->n_mp, p->n_edges, h->maxKf, h->maxMp, h->maxE);
    return B2S_ERR_CAPACITY;
  }
  std::vector<int> lastPt((size_t)p->n_kf, -1);
  for (int e = 0; e < p->n_edges; e++) {
    const b2s_ba_edge& ed = p->edges[e];
    if (ed.kf < 0 || ed.kf >= p->n_kf || ed.mp < 0 || ed.mp >= p->n_mp) {
      set_error("b2s_global_ba: edge %d: index out of range", e);
      return B2S_ERR_BAD_ARG;
    }
    if (e > 0 && ed.mp < p->edges[e - 1].mp) {
      set_error("b2s_global_ba: edge %d: points are not ascending", e);
      return B2S_ERR_BAD_ARG;
    }
    if (lastPt[(size_t)ed.kf] == ed.mp) {
      set_error("b2s_global_ba: edge %d: duplicate (keyframe %d, point %d)", e, ed.kf, ed.mp);
      return B2S_ERR_BAD_ARG;
    }
    lastPt[(size_t)ed.kf] = ed.mp;
  }
  return B2S_OK;
}

}  // namespace

extern "C" int b2s_gba_create(int max_kf, int max_mp, int max_edges, int device, b2s_gba_solver** out) {
  if (!out || max_kf < 1 || max_mp < 1 || max_edges < 1 || max_kf > 16384) {
    set_error("b2s_gba_create: bad argument (capacities must be >= 1, max_kf <= 16384)");
    return B2S_ERR_BAD_ARG;
  }
  *out = nullptr;
  int rc = select_device(device);
  if (rc != B2S_OK) return rc;
  b2s_gba_solver* h = new b2s_gba_solver();
  h->maxKf = max_kf; h->maxMp = max_mp; h->maxE = max_edges;
  h->open(device);
  auto A = [h](auto* p, size_t bytes) { h->alloc(*p, bytes); };
  const size_t K = max_kf, M = max_mp, E = max_edges;
  A(&h->eKf, E * 4); A(&h->eMp, E * 4); A(&h->eObs, E * 12); A(&h->eW, E * 4);
  A(&h->kfKey, E * 4); A(&h->kfKeyS, E * 4); A(&h->kfVal, E * 4); A(&h->kfEdge, E * 4);
  A(&h->err, E * 24); A(&h->chi2, E * 8); A(&h->rho, E * 8); A(&h->W, E * 18 * 8);
  A(&h->pidx, K * 4); A(&h->fixedD, K); A(&h->Tcw, K * 64); A(&h->kfBeg, K * 4); A(&h->kfEnd, K * 4);
  A(&h->envBlk, K * 4); A(&h->envT, K * 4 + 4); A(&h->tileOff, (K + 1) * 8);
  A(&h->pose, K * POSE_STRIDE * 8); A(&h->poseT, K * POSE_STRIDE * 8); A(&h->Hpp, K * 36 * 8);
  A(&h->X, M * 12); A(&h->pts, M * 24); A(&h->ptsT, M * 24); A(&h->ptBeg, M * 4); A(&h->ptEnd, M * 4);
  A(&h->Hll, M * 72); A(&h->Dinv, M * 72); A(&h->db, M * 24); A(&h->pairCnt, (M + 1) * 8); A(&h->pairOff, (M + 1) * 8);
  A(&h->part, RED_BLOCKS * 8); A(&h->scal, 4 * 8); A(&h->fail, 4);
  h->alloc_pinned(h->hScal, 4 * 8);
  h->alloc_pinned(h->hFail, 4);
  cudaError_t e = h->error;
  if (e == cudaSuccess) e = set_smem_limits();
  if (e != cudaSuccess) {
    set_error("b2s_gba_create: %s", cudaGetErrorString(e));
    b2s_gba_destroy(h);
    return B2S_ERR_CUDA;
  }
  *out = h;
  return B2S_OK;
}

extern "C" void b2s_gba_destroy(b2s_gba_solver* h) {
  if (!h) return;
  h->close();
  delete h;
}

extern "C" float b2s_gba_last_ms(const b2s_gba_solver* h, long long* lm_trials) {
  if (!h) return 0.f;
  if (lm_trials) *lm_trials = h->lastTrials;
  return h->lastMs;
}

extern "C" int b2s_global_ba(b2s_gba_solver* h, const b2s_gba_problem* p, const volatile uint8_t* stop, b2s_gba_result* r) {
  if (!h || !r || !r->Tcw_out || !r->point_included || (p && p->n_mp && !r->points_out)) {
    set_error("b2s_global_ba: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  int rc = validate(h, p);
  if (rc != B2S_OK) return rc;
  B2S_CUDA(cudaSetDevice(h->device));
  const int nKf = p->n_kf, nMp = p->n_mp, nE = p->n_edges;
  cudaStream_t s = h->stream;
  auto terminate = [&]() { return stop && *stop; };

  // ---- host: pose indices (free = not fixed and with an edge), included points
  std::vector<int> pidx((size_t)nKf, -1);
  std::vector<uint8_t> active((size_t)nKf, 0);
  for (int k = 0; k < nMp; k++) r->point_included[k] = 0;
  for (int e = 0; e < nE; e++) {
    active[(size_t)p->edges[e].kf] = 1;
    r->point_included[p->edges[e].mp] = 1;
  }
  int nFree = 0;
  for (int k = 0; k < nKf; k++)
    if (active[(size_t)k] && !p->fixed[k]) pidx[(size_t)k] = nFree++;
  const int np = nFree * 6, nT = (np + TS - 1) / TS, npPad = nT * TS;

  HostSync sync = {s, h->ev, h->hScal, h->scal, h->hFail, h->fail, 0.f};
  rc = sync.start();
  if (rc != B2S_OK) return rc;
  // ---- upload
  std::vector<int> ek((size_t)nE), em((size_t)nE);
  std::vector<float> eo((size_t)nE * 3), ew((size_t)nE);
  for (int e = 0; e < nE; e++) {
    ek[(size_t)e] = p->edges[e].kf;
    em[(size_t)e] = p->edges[e].mp;
    for (int c = 0; c < 3; c++) eo[(size_t)e * 3 + c] = p->edges[e].obs[c];
    ew[(size_t)e] = p->edges[e].inv_sigma2;
  }
  if (nE) {
    B2S_CUDA(cudaMemcpyAsync(h->eKf, ek.data(), (size_t)nE * 4, cudaMemcpyHostToDevice, s));
    B2S_CUDA(cudaMemcpyAsync(h->eMp, em.data(), (size_t)nE * 4, cudaMemcpyHostToDevice, s));
    B2S_CUDA(cudaMemcpyAsync(h->eObs, eo.data(), (size_t)nE * 12, cudaMemcpyHostToDevice, s));
    B2S_CUDA(cudaMemcpyAsync(h->eW, ew.data(), (size_t)nE * 4, cudaMemcpyHostToDevice, s));
  }
  if (nKf) {
    B2S_CUDA(cudaMemcpyAsync(h->Tcw, p->Tcw, (size_t)nKf * 64, cudaMemcpyHostToDevice, s));
    B2S_CUDA(cudaMemcpyAsync(h->pidx, pidx.data(), (size_t)nKf * 4, cudaMemcpyHostToDevice, s));
    k_pose_init<<<blocks(nKf, 128), 128, 0, s>>>(h->Tcw, nKf, h->pose);
  }
  if (nMp) {
    B2S_CUDA(cudaMemcpyAsync(h->X, p->points, (size_t)nMp * 12, cudaMemcpyHostToDevice, s));
    k_point_init<<<blocks((long long)nMp * 3, 256), 256, 0, s>>>(h->X, nMp * 3, h->pts);
  }
  LmArgs a;
  memset(&a, 0, sizeof(a));
  a.E.kf = h->eKf; a.E.mp = h->eMp; a.E.obs = h->eObs; a.E.w = h->eW;
  a.C.fx = p->fx; a.C.fy = p->fy; a.C.cx = p->cx; a.C.cy = p->cy; a.C.bf = p->bf;
  a.nKf = nKf; a.nMp = nMp; a.nE = nE; a.nFree = nFree; a.np = np; a.npPad = npPad;
  a.robust = p->robust != 0;
  a.pidx = h->pidx; a.ptBeg = h->ptBeg; a.ptEnd = h->ptEnd; a.kfBeg = h->kfBeg; a.kfEnd = h->kfEnd; a.kfEdge = h->kfEdge;
  a.err = h->err; a.chi2 = h->chi2; a.rho = h->rho; a.Hpp = h->Hpp; a.Hll = h->Hll; a.W = h->W; a.Dinv = h->Dinv;
  a.db = h->db; a.envT = h->envT; a.tileOff = h->tileOff; a.fail = h->fail;
  const long long nx = (long long)npPad + 3LL * nMp;
  rc = grow(h->bvec, (size_t)nx * 8);
  if (rc == B2S_OK) rc = grow(h->xvec, (size_t)nx * 8);
  if (rc == B2S_OK) rc = grow(h->rhs, (size_t)npPad * 8);
  if (rc == B2S_OK) rc = grow(h->ybuf, (size_t)npPad * 8);
  if (rc == B2S_OK) rc = grow(h->tmp, (size_t)std::max<long long>(nx, nE) * 8);
  if (rc == B2S_OK) rc = grow(h->linv, (size_t)nT * TT * 8);
  if (rc != B2S_OK) return rc;
  a.b = (double*)h->bvec.p; a.x = (double*)h->xvec.p; a.rhs = (double*)h->rhs.p; a.ybuf = (double*)h->ybuf.p;
  a.tmp = (double*)h->tmp.p; a.linv = (double*)h->linv.p;

  int nBlk = 0;
  long long nPairs = 0, nTiles = 0;
  std::vector<int> envT((size_t)nT), rowOff;
  if (nE > 0) {
    // ---- structure: CSR by point and by free keyframe, pair records by lower block, block envelope
    B2S_CUDA(cudaMemsetAsync(h->ptBeg, 0, (size_t)nMp * 4, s));
    B2S_CUDA(cudaMemsetAsync(h->ptEnd, 0, (size_t)nMp * 4, s));
    k_point_csr<<<blocks(nE, 256), 256, 0, s>>>(h->eMp, nE, h->ptBeg, h->ptEnd);
    k_kf_keys<<<blocks(nE, 256), 256, 0, s>>>(h->eKf, h->pidx, nE, nFree, h->kfKey, h->kfVal);
    int keyBits = 1;
    while ((1LL << keyBits) <= (long long)nFree) keyBits++;
    size_t tb = 0;
    B2S_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, h->kfKey, h->kfKeyS, h->kfVal, h->kfEdge, nE, 0, keyBits, s));
    rc = grow(h->cubTmp, tb);
    if (rc != B2S_OK) return rc;
    B2S_CUDA(cub::DeviceRadixSort::SortPairs(h->cubTmp.p, tb, h->kfKey, h->kfKeyS, h->kfVal, h->kfEdge, nE, 0, keyBits, s));
    if (nFree) {
      B2S_CUDA(cudaMemsetAsync(h->kfBeg, 0, (size_t)nFree * 4, s));
      B2S_CUDA(cudaMemsetAsync(h->kfEnd, 0, (size_t)nFree * 4, s));
    }
    k_kf_csr<<<blocks(nE, 256), 256, 0, s>>>(h->kfKeyS, nE, nFree, h->kfBeg, h->kfEnd);
    k_pair_count<<<blocks(nMp + 1, 256), 256, 0, s>>>(h->ptBeg, h->ptEnd, h->eKf, h->pidx, nMp, h->pairCnt);
    tb = 0;
    B2S_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, h->pairCnt, h->pairOff, nMp + 1, s));
    rc = grow(h->cubTmp, tb);
    if (rc != B2S_OK) return rc;
    B2S_CUDA(cub::DeviceScan::ExclusiveSum(h->cubTmp.p, tb, h->pairCnt, h->pairOff, nMp + 1, s));
    B2S_CUDA(cudaMemcpyAsync(h->hScal, h->pairOff + nMp, 8, cudaMemcpyDeviceToHost, s));
    rc = sync.stream();
    if (rc != B2S_OK) return rc;
    memcpy(&nPairs, h->hScal, 8);
    if (nPairs > 0x7fffffffLL) {
      set_error("b2s_global_ba: %lld covisibility pairs exceed 2^31", nPairs);
      return B2S_ERR_CAPACITY;
    }
    if (nPairs > 0) {
      const int keyBits2 = std::min(32, 2 * keyBits);
      rc = grow(h->pairKey, (size_t)nPairs * 4);
      if (rc == B2S_OK) rc = grow(h->pairKeyS, (size_t)nPairs * 4);
      if (rc == B2S_OK) rc = grow(h->pairVal, (size_t)nPairs * 4);
      if (rc == B2S_OK) rc = grow(h->pairValS, (size_t)nPairs * 4);
      if (rc == B2S_OK) rc = grow(h->pairRec, (size_t)nPairs * 16);
      if (rc == B2S_OK) rc = grow(h->pairRecS, (size_t)nPairs * 16);
      if (rc == B2S_OK) rc = grow(h->uKey, (size_t)nPairs * 4);
      if (rc == B2S_OK) rc = grow(h->runLen, (size_t)(nPairs + 1) * 4);
      if (rc == B2S_OK) rc = grow(h->blkBeg, (size_t)(nPairs + 1) * 4);
      if (rc == B2S_OK) rc = grow(h->nRuns, 8);
      if (rc != B2S_OK) return rc;
      unsigned *pk = (unsigned*)h->pairKey.p, *pkS = (unsigned*)h->pairKeyS.p, *pv = (unsigned*)h->pairVal.p,
               *pvS = (unsigned*)h->pairValS.p, *uk = (unsigned*)h->uKey.p;
      int *rl = (int*)h->runLen.p, *bb = (int*)h->blkBeg.p, *nr = (int*)h->nRuns.p;
      k_pair_emit<<<blocks(nMp, 128), 128, 0, s>>>(h->ptBeg, h->ptEnd, h->eKf, h->pidx, h->pairOff, nMp, nFree, pk, pv,
                                                   (int4*)h->pairRec.p);
      const int nP = (int)nPairs;
      size_t t1 = 0, t2 = 0, t3 = 0;
      B2S_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t1, pk, pkS, pv, pvS, nP, 0, keyBits2, s));
      B2S_CUDA(cub::DeviceRunLengthEncode::Encode(nullptr, t2, pkS, uk, rl, nr, nP, s));
      B2S_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, t3, rl, bb, nP + 1, s));
      rc = grow(h->cubTmp, std::max(t1, std::max(t2, t3)));
      if (rc != B2S_OK) return rc;
      B2S_CUDA(cub::DeviceRadixSort::SortPairs(h->cubTmp.p, t1, pk, pkS, pv, pvS, nP, 0, keyBits2, s));
      k_pair_gather<<<blocks(nPairs, 256), 256, 0, s>>>(pvS, (const int4*)h->pairRec.p, nPairs, (int4*)h->pairRecS.p);
      B2S_CUDA(cub::DeviceRunLengthEncode::Encode(h->cubTmp.p, t2, pkS, uk, rl, nr, nP, s));
      B2S_CUDA(cudaMemcpyAsync(h->hFail, nr, 4, cudaMemcpyDeviceToHost, s));
      rc = sync.stream();
      if (rc != B2S_OK) return rc;
      nBlk = *h->hFail;
      B2S_CUDA(cudaMemsetAsync(rl + nBlk, 0, 4, s));
      B2S_CUDA(cub::DeviceScan::ExclusiveSum(h->cubTmp.p, t3, rl, bb, nBlk + 1, s));
      k_envelope<<<blocks(nBlk, 256), 256, 0, s>>>(uk, nBlk, nFree, h->envBlk);
    }
    if (nFree) {
      // tile envelope: first tile column any scalar row of the tile row reaches; tile storage sized from it
      std::vector<int> envBlk((size_t)nFree);
      B2S_CUDA(cudaMemcpyAsync(envBlk.data(), h->envBlk, (size_t)nFree * 4, cudaMemcpyDeviceToHost, s));
      rc = sync.stream();
      if (rc != B2S_OK) return rc;
      std::vector<long long> off;
      std::vector<int> rows;
      nTiles = tile_envelope(envBlk, nFree, 6, envT, off, rowOff, rows);
      rc = grow(h->tiles, (size_t)nTiles * TT * 8);
      if (rc == B2S_OK) rc = grow(h->rows, rows.size() * 4);
      if (rc != B2S_OK) return rc;
      a.tiles = (double*)h->tiles.p;
      if (!rows.empty())
        B2S_CUDA(cudaMemcpyAsync(h->rows.p, rows.data(), rows.size() * 4, cudaMemcpyHostToDevice, s));
      B2S_CUDA(cudaMemcpyAsync(h->envT, envT.data(), (size_t)nT * 4, cudaMemcpyHostToDevice, s));
      B2S_CUDA(cudaMemcpyAsync(h->tileOff, off.data(), (size_t)(nT + 1) * 8, cudaMemcpyHostToDevice, s));
    }
  }
  const size_t tileBytes = (size_t)nTiles * TT * 8;
  const TileSys ts = {np, h->envT, h->tileOff, a.tiles, a.linv, a.rhs, a.ybuf, a.x, h->fail};
  B2S_CUDA(cudaMemsetAsync(a.b, 0, (size_t)nx * 8, s));
  B2S_CUDA(cudaMemsetAsync(a.x, 0, (size_t)nx * 8, s));

  double* pose = h->pose;
  double* poseT = h->poseT;
  double* pts = h->pts;
  double* ptsT = h->ptsT;
  const int nUpd = std::max(nKf, std::max(nMp * 3, (int)nx));
  auto chi2_of = [&](const double* P, const double* X, double* out) {
    k_errors<<<blocks(nE, 256), 256, 0, s>>>(a, P, X);
    reduce<0>(h, h->rho, nE, out);
  };

  // ---- SparseOptimizer::optimize + OptimizationAlgorithmLevenberg::solve ("empty graph": nothing to optimise)
  Levenberg lm = {};
  int32_t trace[256];
  bool ok = nE > 0;
  for (int it = 0; it < p->iterations && !terminate() && ok; it++) {
    chi2_of(pose, pts, h->scal);
    if (nMp) k_build_points<<<blocks(nMp, 128), 128, 0, s>>>(a, pose, pts);
    if (nFree) k_build_poses<<<blocks((long long)nFree * 32, 256), 256, 0, s>>>(a, pose, pts);
    if (it == 0) {
      const long long nd = (long long)nFree * 6 + 3LL * nMp;
      k_diag<<<blocks(nd, 256), 256, 0, s>>>(a);
      reduce<1>(h, a.tmp, nd, h->scal + 1);
    }
    rc = sync.scalars(2);
    if (rc != B2S_OK) return rc;
    lm.begin(h->hScal[0]);
    if (it == 0) lm.init_lambda(1e-5 * h->hScal[1]);
    do {
      // ---- BlockSolver::solve: Schur complement, tiled Cholesky, substitutions, point back-substitution
      B2S_CUDA(cudaMemsetAsync(h->fail, 0, 4, s));
      if (nMp) k_dinv<<<blocks(nMp, 128), 128, 0, s>>>(a, lm.lambda);
      if (nFree) {
        B2S_CUDA(cudaMemsetAsync(a.rhs, 0, (size_t)npPad * 8, s));
        k_rhs<<<blocks((long long)nFree * 32, 256), 256, 0, s>>>(a);
        B2S_CUDA(cudaMemsetAsync(a.tiles, 0, tileBytes, s));
        k_schur<<<blocks((long long)nBlk * 32, 256), 256, 0, s>>>(a, (const unsigned*)h->uKey.p, (const int*)h->blkBeg.p,
                                                                   nBlk, (const int4*)h->pairRecS.p, lm.lambda);
        factor_solve(ts, nT, envT, rowOff, (const int*)h->rows.p, s);
      }
      if (nMp) k_backsub_points<<<blocks(nMp, 128), 128, 0, s>>>(a);
      // ---- SparseOptimizer::update into the trial copy, trial chi2, computeScale
      k_update<<<blocks(nUpd, 256), 256, 0, s>>>(a, pose, pts, poseT, ptsT, lm.lambda);
      chi2_of(poseT, ptsT, h->scal);
      reduce<0>(h, a.tmp, nx, h->scal + 1);
      rc = sync.scalars(2);
      if (rc != B2S_OK) return rc;
      if (lm.trial(*h->hFail == 0, h->hScal[0], h->hScal[1], trace)) {
        std::swap(pose, poseT);
        std::swap(pts, ptsT);
      }
    } while (lm.retry(terminate()));
    ok = !lm.end_iteration();
  }

  // ---- write-back (every keyframe through Converter; points with an edge) and the chi2 of the returned estimate
  if (nE) chi2_of(pose, pts, h->scal);
  else B2S_CUDA(cudaMemsetAsync(h->scal, 0, 8, s));
  if (nKf || nMp) k_writeback<<<blocks(std::max(nKf, nMp * 3), 256), 256, 0, s>>>(a, pose, pts, h->Tcw, h->X);
  std::vector<float> Xout((size_t)nMp * 3);
  if (nKf) B2S_CUDA(cudaMemcpyAsync(r->Tcw_out, h->Tcw, (size_t)nKf * 64, cudaMemcpyDeviceToHost, s));
  if (nMp) B2S_CUDA(cudaMemcpyAsync(Xout.data(), h->X, (size_t)nMp * 12, cudaMemcpyDeviceToHost, s));
  B2S_CUDA(cudaMemcpyAsync(h->hScal, h->scal, 8, cudaMemcpyDeviceToHost, s));
  rc = sync.stream();
  if (rc != B2S_OK) return rc;
  B2S_CUDA(cudaGetLastError());
  for (int m = 0; m < nMp; m++)
    if (r->point_included[m])
      for (int c = 0; c < 3; c++) r->points_out[(size_t)m * 3 + c] = Xout[(size_t)m * 3 + c];
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
