// localba.cu — H100 (sm_90a) Optimizer::LocalBundleAdjustment numerics (FP64), batched over independent windows.
//
// Replaces /root/reference/src/Optimizer.cc:698-996 from graph construction to the write-back values, i.e. the g2o
// functions it executes (Thirdparty/g2o/g2o/...):
//   types/types_six_dof_expmap.{h,cpp}   computeError / linearizeOplus of EdgeSE3ProjectXYZ, EdgeStereoSE3ProjectXYZ
//   core/base_binary_edge.hpp:55-120     constructQuadraticForm (Huber weighted)      -> k_build_landmarks / k_build_poses
//   core/block_solver.hpp:354-486        Schur complement + back substitution         -> k_schur / k_chol / k_backsub
//   core/optimization_algorithm_levenberg.cpp:61-189   LM control                     -> control_begin / control_end
//                                                      (the step policy itself: Levenberg, levenberg.cuh)
//   types/se3quat.h:223-257, types_sba.h:52-56         oplus updates                  -> k_update_poses / k_backsub
// The whole Levenberg-Marquardt loop of a window runs inside ONE persistent kernel: a window owns `nCta` thread blocks
// that move through the phases (linearise -> Schur -> Cholesky -> back-substitute -> evaluate -> accept/reject) separated
// by a per-window barrier in global memory; the LM state machine is a device record per window, so a batch of windows
// needs a single launch and no host round trips.  All reductions have a fixed order (no floating-point atomics).
#include <float.h>
#include <limits.h>
#include <stddef.h>
#include <stdlib.h>
#include <math.h>

#include <algorithm>
#include <thread>
#include <vector>

#include "common.cuh"
#include "ba_math.cuh"  // quat / pose helpers, huber, edge_jacobians
#include "levenberg.cuh"

namespace b2s {

constexpr int CHOL_BS = 32;

struct BaState {
  int active, round, it, needBuild, restore, doOutlier, solveOk, stop, robust, finishedRound0;
  int errBuf, errCurrent;  // which err / eWq buffer describes the linearisation state; it is up to date
  int nLive;               // edges left at level 0 by the outlier pass between the rounds (0: round 2 has nothing to optimise)
  int pairsOverflow;       // the covisibility pair list did not fit capPairs: the window was not run
  int its[2];
  Levenberg lm;
  double chi2Final;
  unsigned long long maxDiagBits;
  int trace[256];
};

struct BaWin {  // per-window sizes (device copy)
  int nKf, nLocal, nMp, nEdges, nFree;
  float fx, fy, cx, cy, bf;
};

struct BaPtrs {  // strided per-window arrays
  int capKf, capMp, capE, ldS, nPartE, nPartM;
  BaWin* win;
  BaState* st;
  double *pose, *poseBak, *pts, *ptsBak;
  int* poseIndex;
  int *eKf, *eMp;
  float *eObs, *eW;
  uint8_t *eStereo, *eLevel, *eOutlier;
  double* chi2;
  // per edge: error vector and rho' * invSigma2 of the linearisation state (0: edge excluded), from which the Schur and
  // back-substitution phases recompute W_e; double-buffered (phase_errors fills the other one, an accepted step swaps)
  double *errB[2], *eWqB[2];
  int *mpStart, *mpEdges, *kfStart, *kfEdges;
  double *Hpp, *Hll, *b, *x, *Dinv, *S;
  double* db;          // Dinv*b_l per landmark
  double* DinvP;       // per landmark, 16-byte items: {d00,d01,d02,d11,d12,d22, db0,db1,db2, pad} (Schur gather record)
  int *lmEdge, *freeKf;  // [landmark][free pose] -> edge id or -1 ; free pose index -> keyframe index
  int* blkOff;             // covisibility pair lists per lower block (built once per window): offsets
  int4* pairRec;           // pair record {edge of pose i1, edge of pose i2, landmark, stereo flags}, capPairs per window
  int2* lmRec;             // landmark-CSR order: {edge, free pose index of its keyframe or -1}
  int* blkFirst;           // per block row: first non-empty block column (envelope of the reduced system)
  int *blkOrder, *blkNZ;   // lower blocks sorted by descending pair count; number of non-empty blocks
  int capPairs, capBlk;
  double *partChi, *partScale;   // per-CTA partial sums [window][nCta]
  unsigned int* bar;             // per-window barrier counters
  // launch plan (ba_run): CTA of the launch -> (window << 8 | index inside the window), and CTAs per window
  int *ctaMap, *winCtas;
};

__device__ __forceinline__ double delta_of(bool stereo) {
  // const float thHuberMono = sqrt(5.991), thHuberStereo = sqrt(7.815)  (src/Optimizer.cc:764-765)
  return stereo ? (double)(float)2.795532150593156 : (double)(float)2.4476519360399226;
}

__device__ double block_sum(double v, double* sm) {  // deterministic block reduction (blockDim multiple of 32, <=1024)
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  __syncthreads();
  if (lane == 0) sm[wid] = v;
  __syncthreads();
  double r = 0;
  if (threadIdx.x == 0) {
    const int nw = (blockDim.x + 31) >> 5;
    for (int i = 0; i < nw; i++) r += sm[i];
  }
  return r;  // valid in thread 0
}


// ---------------------------------------------------------------- per-window barrier
__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// All CTAs of a window call this the same number of times; `epoch` counts arrivals expected so far.
// A bounded spin: if the CTAs of a window ever fail to meet (which would mean they are not co-resident), the window is
// flagged `hung`, every CTA leaves, and the host reports an error instead of hanging the GPU.
__device__ __forceinline__ void win_barrier(unsigned int* bar, unsigned int& epoch, int nCta, volatile int* hung) {
  __syncthreads();
  epoch += (unsigned int)nCta;
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(bar, 1u);
    // the CTAs of a cooperative launch are co-resident, so the wait always ends; the timeout only guards against a
    // wedged partner and is generous (20 s of wall time on %globaltimer, checked every 1024 polls): preemption,
    // time-slicing with another process or a profiler replay must not turn a slow barrier into a failed batch
    unsigned int spins = 0;
    unsigned long long t0 = 0;
    while (ld_acquire_u32(bar) < epoch) {
      __nanosleep(20);
      if (*hung) break;
      if ((++spins & 1023u) == 0u) {
        unsigned long long now;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
        if (t0 == 0)
          t0 = now;
        else if (now - t0 > 20000000000ull) {
          *hung = 1;
          break;
        }
      }
    }
    __threadfence();
  }
  __syncthreads();
}


// computeError (types_six_dof_expmap.h:90-95 mono, :122-127 stereo; cam_project .cpp:141-157) from camera coordinates
__device__ __forceinline__ double edge_error(const double* Xc, bool stereo, const float* ob, double wgt, const BaWin& W,
                                             double* e) {
  if (stereo) {
    const float invz = (float)(1.0 / Xc[2]);  // const float invz = 1.0f/trans_xyz[2]  (.cpp:151)
    const double u = Xc[0] * invz * (double)W.fx + (double)W.cx;
    const double v = Xc[1] * invz * (double)W.fy + (double)W.cy;
    const double ur = u - (double)__fmul_rn(W.bf, invz);
    e[0] = (double)ob[0] - u;
    e[1] = (double)ob[1] - v;
    e[2] = (double)ob[2] - ur;
    return e[0] * (wgt * e[0]) + e[1] * (wgt * e[1]) + e[2] * (wgt * e[2]);
  }
  const double u = Xc[0] / Xc[2] * (double)W.fx + (double)W.cx;
  const double v = Xc[1] / Xc[2] * (double)W.fy + (double)W.cy;
  e[0] = (double)ob[0] - u;
  e[1] = (double)ob[1] - v;
  e[2] = 0;
  return e[0] * (wgt * e[0]) + e[1] * (wgt * e[1]);
}

__device__ __forceinline__ void atomic_max_pos_double(unsigned long long* addr, double v) {
  atomicMax(addr, (unsigned long long)__double_as_longlong(fabs(v)));  // |v| >= 0: IEEE order == integer order
}

struct WinCtx {
  int w, cta, nCta, gtid, gthreads;  // window id, CTA index inside the window, threads of the window
};

// Branch-free operand loads of one edge in two waves (everything indexed by the edge id, then the gathered pose and
// landmark): callers issue the waves of several edges back to back so that the memory latencies overlap.  With 8 warps
// per SM and three dependent loads per edge (level -> indices -> operands) these phases were bound by that chain.
struct EdgeIdx {
  int kf, mp;
  float ob[3], wgt;
  bool stereo, live;
};
struct EdgeOps {
  double P[7], X[3];
};
__device__ __forceinline__ void load_edge_idx(const BaPtrs& p, int w, int e, int nE, EdgeIdx& x) {
  const bool ok = e < nE;
  const size_t eo = (size_t)w * p.capE + (ok ? e : 0);
  x.live = ok & (p.eLevel[eo] == 0);
  x.kf = p.eKf[eo];
  x.mp = p.eMp[eo];
#pragma unroll
  for (int k = 0; k < 3; k++) x.ob[k] = p.eObs[eo * 3 + k];
  x.wgt = p.eW[eo];
  x.stereo = p.eStereo[eo] != 0;
}
__device__ __forceinline__ void load_edge_ops(const BaPtrs& p, int w, const EdgeIdx& x, EdgeOps& o) {
  const double* P = p.pose + ((size_t)w * p.capKf + x.kf) * POSE_STRIDE;
  const double* X = p.pts + ((size_t)w * p.capMp + x.mp) * 3;
#pragma unroll
  for (int k = 0; k < 7; k++) o.P[k] = P[k];
#pragma unroll
  for (int k = 0; k < 3; k++) o.X[k] = X[k];
}

// ---------------------------------------------------------------- phases (device functions, strided over the window's threads)
// The landmark side of buildSystem straight from the stored errors and weights — per edge
// A = d e / d X (from R|t of its keyframe and the landmark), H_ll += A^T (rho' Omega) A, b_l -= A^T (rho' Omega) e, in list order.
__device__ void phase_reduce_landmarks(const BaPtrs& p, const WinCtx& c, const BaWin& W, int cur, double* RtTab) {
  const int w = c.w;
  for (int k = threadIdx.x; k < W.nKf; k += blockDim.x) {
    const double* P = p.pose + ((size_t)w * p.capKf + k) * POSE_STRIDE;
    double R[3][3];
    quat_to_R(P, R);
    double* o = RtTab + (size_t)k * 12;
#pragma unroll
    for (int a = 0; a < 3; a++)
#pragma unroll
      for (int b2 = 0; b2 < 3; b2++) o[a * 3 + b2] = R[a][b2];
    o[9] = P[4]; o[10] = P[5]; o[11] = P[6];
  }
  __syncthreads();
  const int* ms = p.mpStart + (size_t)w * (p.capMp + 1);
  const int* me = p.mpEdges + (size_t)w * p.capE;
  const int* eKf = p.eKf + (size_t)w * p.capE;
  const uint8_t* eSt = p.eStereo + (size_t)w * p.capE;
  const double* wqW = p.eWqB[cur] + (size_t)w * p.capE;
  const double* erW = p.errB[cur] + (size_t)w * p.capE * 3;
  const double fx = W.fx, fy = W.fy, bf = W.bf;
  double md = 0;
  for (int l = c.gtid; l < W.nMp; l += c.gthreads) {
    const size_t mo = (size_t)w * p.capMp + l;
    const double* Xp = p.pts + mo * 3;
    const double X0 = Xp[0], X1 = Xp[1], X2 = Xp[2];
    double h[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    const int kBeg = ms[l], kEnd = ms[l + 1];
    for (int k0 = kBeg; k0 < kEnd; k0 += 4) {
      int ee[4], kf[4];
      double wq[4], er[4][3];
      bool st[4];
#pragma unroll
      for (int j = 0; j < 4; j++) ee[j] = me[min(k0 + j, kEnd - 1)];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        kf[j] = eKf[ee[j]];
        wq[j] = wqW[ee[j]];
        st[j] = eSt[ee[j]] != 0;
#pragma unroll
        for (int r = 0; r < 3; r++) er[j][r] = erW[(size_t)ee[j] * 3 + r];
      }
#pragma unroll
      for (int j = 0; j < 4; j++) {
        if (k0 + j >= kEnd || !(wq[j] > 0.0)) continue;
        const double* Rt = RtTab + (size_t)kf[j] * 12;
        const double x = Rt[0] * X0 + Rt[1] * X1 + Rt[2] * X2 + Rt[9];
        const double y = Rt[3] * X0 + Rt[4] * X1 + Rt[5] * X2 + Rt[10];
        const double z = Rt[6] * X0 + Rt[7] * X1 + Rt[8] * X2 + Rt[11];
        const double iz = 1.0 / z, iz2 = iz * iz;
        const double fxz = fx * iz, fyz = fy * iz, fxx = fx * x * iz2, fyy = fy * y * iz2;
        const double bz = st[j] ? bf * iz2 : 0.0;
        double A[3][3];
#pragma unroll
        for (int cc = 0; cc < 3; cc++) {
          A[0][cc] = -fxz * Rt[cc] + fxx * Rt[6 + cc];
          A[1][cc] = -fyz * Rt[3 + cc] + fyy * Rt[6 + cc];
          A[2][cc] = st[j] ? (A[0][cc] - bz * Rt[6 + cc]) : 0.0;
        }
        const double wv = wq[j];
        int t = 0;
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
          for (int jj = i; jj < 3; jj++) {
            double hh = 0;
#pragma unroll
            for (int r = 0; r < 3; r++) hh += A[r][i] * wv * A[r][jj];
            h[t++] += hh;
          }
#pragma unroll
        for (int i = 0; i < 3; i++) {
          double s2 = 0;
#pragma unroll
          for (int r = 0; r < 3; r++) s2 += A[r][i] * (-(wv * er[j][r]));
          h[6 + i] += s2;
        }
      }
    }
    double* H = p.Hll + mo * 9;
    H[0] = h[0]; H[1] = h[1]; H[2] = h[2];
    H[3] = h[1]; H[4] = h[3]; H[5] = h[4];
    H[6] = h[2]; H[7] = h[4]; H[8] = h[5];
    double* bb = p.b + (size_t)w * (p.capKf * 6 + p.capMp * 3) + (size_t)W.nFree * 6 + (size_t)l * 3;
    bb[0] = h[6]; bb[1] = h[7]; bb[2] = h[8];
    md = fmax(md, fmax(fabs(h[0]), fmax(fabs(h[3]), fabs(h[5]))));
  }
  atomic_max_pos_double(&p.st[w].maxDiagBits, md);
}

// buildSystem (pose side): one warp per free pose, lanes stride over the pose's edges, ordered shuffle reduction
__device__ void phase_build_poses(const BaPtrs& p, const WinCtx& c, const BaWin& W, int robust, int cur) {
  const int w = c.w;
  const int lane = threadIdx.x & 31;
  const int nWarps = c.gthreads >> 5, gw = c.gtid >> 5;
  const int* ks = p.kfStart + (size_t)w * (p.capKf + 1);
  const int* ke = p.kfEdges + (size_t)w * p.capE;
  for (int pi = gw; pi < W.nFree; pi += nWarps) {
    const int kf = p.freeKf[(size_t)w * p.capKf + pi];
    double acc[27];
#pragma unroll
    for (int k = 0; k < 27; k++) acc[k] = 0;
    const double* P = p.pose + ((size_t)w * p.capKf + kf) * POSE_STRIDE;
    double Pv[7];
#pragma unroll
    for (int k = 0; k < 7; k++) Pv[k] = P[k];
    const int kBeg = ks[kf], kEnd = ks[kf + 1];
    for (int k0 = kBeg; k0 < kEnd; k0 += 64) {  // two edges per lane and iteration, loads in three waves up front
      int ee[2], mp[2];
      bool live[2], stereo[2];
      float wgt[2];
      double c2v[2], er[2][3], X[2][3];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int kk = k0 + h * 32 + lane;
        live[h] = kk < kEnd;
        ee[h] = ke[live[h] ? kk : kBeg];
      }
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const size_t eo = (size_t)w * p.capE + ee[h];
        live[h] = live[h] & (p.eLevel[eo] == 0);
        stereo[h] = p.eStereo[eo] != 0;
        mp[h] = p.eMp[eo];
        wgt[h] = p.eW[eo];
        c2v[h] = p.chi2[eo];
#pragma unroll
        for (int r = 0; r < 3; r++) er[h][r] = p.errB[cur][eo * 3 + r];  // phase_errors
      }
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const double* Xp = p.pts + ((size_t)w * p.capMp + mp[h]) * 3;
#pragma unroll
        for (int r = 0; r < 3; r++) X[h][r] = Xp[r];
      }
#pragma unroll
      for (int h = 0; h < 2; h++) {
        if (!live[h]) continue;
        EdgeJac J;
        edge_jacobians(Pv, X[h], stereo[h], W.fx, W.fy, W.bf, J);
        const double w0 = (double)wgt[h];
        double rho1 = 1.0;
        if (robust) {
          double r0;
          huber(c2v[h], delta_of(stereo[h]), r0, rho1);
        }
        double omr[3];
#pragma unroll
        for (int r = 0; r < 3; r++) omr[r] = -(w0 * er[h][r]) * rho1;
        const double wq = rho1 * w0;
        int t = 0;
#pragma unroll
        for (int i = 0; i < 6; i++) {
#pragma unroll
          for (int j = i; j < 6; j++) {
            double hh = 0;
#pragma unroll
            for (int r = 0; r < 3; r++) hh += J.B[r][i] * wq * J.B[r][j];
            acc[t++] += hh;
          }
        }
#pragma unroll
        for (int i = 0; i < 6; i++) {
          double s2 = 0;
#pragma unroll
          for (int r = 0; r < 3; r++) s2 += J.B[r][i] * omr[r];
          acc[21 + i] += s2;
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 27; k++) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_down_sync(0xffffffffu, acc[k], o);
    }
    if (lane == 0) {
      double* Hp = p.Hpp + ((size_t)w * p.capKf + pi) * 36;
      int t = 0;
      double md = 0;
#pragma unroll
      for (int i = 0; i < 6; i++)
#pragma unroll
        for (int j = i; j < 6; j++) {
          Hp[i * 6 + j] = acc[t];
          Hp[j * 6 + i] = acc[t];
          if (i == j) md = fmax(md, fabs(acc[t]));
          t++;
        }
      double* bp = p.b + (size_t)w * (p.capKf * 6 + p.capMp * 3) + (size_t)pi * 6;
#pragma unroll
      for (int i = 0; i < 6; i++) bp[i] = acc[21 + i];
      atomic_max_pos_double(&p.st[w].maxDiagBits, md);
    }
  }
}

// iteration begin (levenberg.cpp:83-100): chi2 of the current state, lambda init on the first iteration
__device__ void control_begin(const BaPtrs& p, int w, int nCta) {
  BaState& st = p.st[w];
  if (st.needBuild) {
    double chi = 0;
    for (int k = 0; k < nCta; k++) chi += p.partChi[(size_t)w * p.nPartE + k];
    st.lm.begin(chi);
    if (st.it == 0) st.lm.init_lambda(1e-5 * __longlong_as_double((long long)st.maxDiagBits));
    st.needBuild = 0;
  }
  st.maxDiagBits = 0ull;
}

// Schur complement (block_solver.hpp:381-439), atomic-free:
//   phase_dinv         per landmark:  Dinv = (Hll + lambda I)^-1,  db = Dinv b_l
//   phase_schur_blocks per lower block (i1 >= i2): S(i1,i2) = [Hpp + lambda I] - sum_{l seen by both} Y_a W_c^T
__device__ void phase_dinv(const BaPtrs& p, const WinCtx& c, const BaWin& W, double lambda) {
  const int w = c.w;
  for (int l = c.gtid; l < W.nMp; l += c.gthreads) {
    const size_t mo = (size_t)w * p.capMp + l;
    double D[9];
#pragma unroll
    for (int k = 0; k < 9; k++) D[k] = p.Hll[mo * 9 + k];
    D[0] += lambda; D[4] += lambda; D[8] += lambda;
    double Di[9];
    const double c00 = D[4] * D[8] - D[5] * D[7], c01 = D[5] * D[6] - D[3] * D[8], c02 = D[3] * D[7] - D[4] * D[6];
    const double id = 1.0 / (D[0] * c00 + D[1] * c01 + D[2] * c02);
    Di[0] = c00 * id; Di[1] = (D[2] * D[7] - D[1] * D[8]) * id; Di[2] = (D[1] * D[5] - D[2] * D[4]) * id;
    Di[3] = c01 * id; Di[4] = (D[0] * D[8] - D[2] * D[6]) * id; Di[5] = (D[2] * D[3] - D[0] * D[5]) * id;
    Di[6] = c02 * id; Di[7] = (D[1] * D[6] - D[0] * D[7]) * id; Di[8] = (D[0] * D[4] - D[1] * D[3]) * id;
#pragma unroll
    for (int k = 0; k < 9; k++) p.Dinv[mo * 9 + k] = Di[k];
    const double* bl = p.b + (size_t)w * (p.capKf * 6 + p.capMp * 3) + (size_t)W.nFree * 6 + (size_t)l * 3;
    p.db[mo * 3 + 0] = Di[0] * bl[0] + Di[1] * bl[1] + Di[2] * bl[2];
    p.db[mo * 3 + 1] = Di[3] * bl[0] + Di[4] * bl[1] + Di[5] * bl[2];
    p.db[mo * 3 + 2] = Di[6] * bl[0] + Di[7] * bl[1] + Di[8] * bl[2];
    double2* rec = reinterpret_cast<double2*>(p.DinvP + mo * 10);  // Hll is exactly symmetric, so is the cofactor inverse
    rec[0] = make_double2(Di[0], Di[1]);
    rec[1] = make_double2(Di[2], Di[4]);
    rec[2] = make_double2(Di[5], Di[8]);
    rec[3] = make_double2(p.db[mo * 3 + 0], p.db[mo * 3 + 1]);
    rec[4] = make_double2(p.db[mo * 3 + 2], 0.0);
  }
}

__device__ __forceinline__ void decode_block(int t, int& i1, int& i2) {
  i1 = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
  while ((i1 + 1) * (i1 + 2) / 2 <= t) i1++;
  while (i1 * (i1 + 1) / 2 > t) i1--;
  i2 = t - i1 * (i1 + 1) / 2;
}

// Butterfly reduce-scatter of 32 per-lane values across the warp: lane L ends with the warp-wide sum of element L
// (31 double shuffles instead of 32 x 5; fixed summation tree => deterministic).
__device__ __forceinline__ double warp_reduce_scatter32(double (&v)[32], int lane) {
  double a16[16];
  const bool h16 = lane & 16;
#pragma unroll
  for (int k = 0; k < 16; k++) {
    const double keep = h16 ? v[k + 16] : v[k], send = h16 ? v[k] : v[k + 16];
    a16[k] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
  }
  double a8[8];
  const bool h8 = lane & 8;
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const double keep = h8 ? a16[k + 8] : a16[k], send = h8 ? a16[k] : a16[k + 8];
    a8[k] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
  double a4[4];
  const bool h4 = lane & 4;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const double keep = h4 ? a8[k + 4] : a8[k], send = h4 ? a8[k] : a8[k + 4];
    a4[k] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  }
  double a2[2];
  const bool h2 = lane & 2;
#pragma unroll
  for (int k = 0; k < 2; k++) {
    const double keep = h2 ? a4[k + 2] : a4[k], send = h2 ? a4[k] : a4[k + 2];
    a2[k] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
  }
  const bool h1 = lane & 1;
  const double keep = h1 ? a2[1] : a2[0], send = h1 ? a2[0] : a2[1];
  return keep + __shfl_xor_sync(0xffffffffu, send, 1);
}


__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  const unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
// Warp-cooperative asynchronous gather of one record per lane (REC16 16-byte items each, record index `rec` held by the
// lane) into a shared-memory tile laid out [lane][N16]: consecutive lanes fetch consecutive 16-byte items, so one copy
// instruction touches ~32*16/128 lines per record run instead of 32 lines, and no registers are held across the memory
// latency.  Only the first N16 items of each record are fetched.  Tile reads by the owning lane (stride N16*16 B, N16
// odd) are bank-conflict free for 128-bit accesses.
template <int N16, int REC16>
__device__ __forceinline__ void warp_gather16_async(double2* tile, const double2* base, int rec, int lane) {
#pragma unroll
  for (int r = 0; r < N16; r++) {
    const int idx = lane + 32 * r;
    const int pr = idx / N16, el = idx - pr * N16;
    const int src = __shfl_sync(0xffffffffu, rec, pr);
    cp_async16(tile + idx, base + (size_t)src * REC16 + el);
  }
}

// One covisibility pair per lane out of the staged records: acc += (W_a Dinv_l) W_c^T (36 entries: 32 in acc, 4 in
// tail[0..3]); diagonal blocks also accumulate W_a (Dinv_l b_l) into tail[4..9].
template <bool DIAG>
__device__ __forceinline__ void schur_accumulate(const double2* tA, const double2* tC, const double2* tD, int lane,
                                                 double (&acc)[32], double (&tail)[10]) {
  const double2* ra = tA + lane * 9;
  const double2* rc = DIAG ? ra : tC + lane * 9;
  const double2* rd = tD + lane * (DIAG ? 5 : 3);
  double wc[18];
#pragma unroll
  for (int z = 0; z < 9; z++) {
    const double2 v = rc[z];
    wc[2 * z] = v.x;
    wc[2 * z + 1] = v.y;
  }
  const double2 dA = rd[0], dB = rd[1], dC = rd[2];
  const double d00 = dA.x, d01 = dA.y, d02 = dB.x, d11 = dB.y, d12 = dC.x, d22 = dC.y;
  double b0 = 0, b1 = 0, b2 = 0;
  if (DIAG) {
    const double2 e0 = rd[3], e1 = rd[4];
    b0 = e0.x; b1 = e0.y; b2 = e1.x;
  }
#pragma unroll
  for (int r2 = 0; r2 < 3; r2++) {  // two rows of W_a at a time (register budget)
    const double2 u0 = ra[3 * r2], u1 = ra[3 * r2 + 1], u2 = ra[3 * r2 + 2];
    const double wr[2][3] = {{u0.x, u0.y, u1.x}, {u1.y, u2.x, u2.y}};
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int r = 2 * r2 + h;
      const double w0 = wr[h][0], w1 = wr[h][1], w2 = wr[h][2];
      const double y0 = w0 * d00 + w1 * d01 + w2 * d02;
      const double y1 = w0 * d01 + w1 * d11 + w2 * d12;
      const double y2 = w0 * d02 + w1 * d12 + w2 * d22;
#pragma unroll
      for (int cc = 0; cc < 6; cc++) {
        const double v = y0 * wc[cc * 3] + y1 * wc[cc * 3 + 1] + y2 * wc[cc * 3 + 2];
        const int en = r * 6 + cc;
        if (en < 32) acc[en] += v;
        else tail[en - 32] += v;
      }
      if (DIAG) tail[4 + r] += w0 * b0 + w1 * b1 + w2 * b2;
    }
  }
}

// W_e = B^T (rho' Omega) A of one edge from the camera's rotation / translation (Rt: R row-major, then t), the landmark and
// the edge weight — the same closed forms as edge_jacobians; wq == 0 (excluded edge) gives an exact zero block.
__device__ __forceinline__ void edge_W_regs(const double* __restrict__ Rt, const double X0, const double X1, const double X2,
                                            bool st, double wq, double fx, double fy, double bf, double (&wv)[18]) {
  const double x = Rt[0] * X0 + Rt[1] * X1 + Rt[2] * X2 + Rt[9];
  const double y = Rt[3] * X0 + Rt[4] * X1 + Rt[5] * X2 + Rt[10];
  const double z = Rt[6] * X0 + Rt[7] * X1 + Rt[8] * X2 + Rt[11];
  const double iz = 1.0 / z, iz2 = iz * iz;
  const double fxz = fx * iz, fyz = fy * iz, fxx = fx * x * iz2, fyy = fy * y * iz2;
  const double bz = st ? bf * iz2 : 0.0;
  double A[3][3];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    A[0][c] = wq * (-fxz * Rt[c] + fxx * Rt[6 + c]);
    A[1][c] = wq * (-fyz * Rt[3 + c] + fyy * Rt[6 + c]);
    A[2][c] = st ? (A[0][c] - wq * bz * Rt[6 + c]) : 0.0;
  }
  double B[3][6];
  B[0][0] = x * y * iz2 * fx;
  B[0][1] = -(1 + (x * x * iz2)) * fx;
  B[0][2] = y * iz * fx;
  B[0][3] = -iz * fx;
  B[0][4] = 0;
  B[0][5] = x * iz2 * fx;
  B[1][0] = (1 + y * y * iz2) * fy;
  B[1][1] = -x * y * iz2 * fy;
  B[1][2] = -x * iz * fy;
  B[1][3] = 0;
  B[1][4] = -iz * fy;
  B[1][5] = y * iz2 * fy;
  B[2][0] = st ? (B[0][0] - bz * y) : 0.0;
  B[2][1] = st ? (B[0][1] + bz * x) : 0.0;
  B[2][2] = st ? B[0][2] : 0.0;
  B[2][3] = st ? B[0][3] : 0.0;
  B[2][4] = 0;
  B[2][5] = st ? (B[0][5] - bz) : 0.0;
  const bool zero = !(wq > 0.0);
#pragma unroll
  for (int i = 0; i < 6; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) {
      const double v = B[0][i] * A[0][j] + B[1][i] * A[1][j] + B[2][i] * A[2][j];
      wv[i * 3 + j] = zero ? 0.0 : v;
    }
}
__device__ __forceinline__ void edge_W_from_Rt(const double* __restrict__ Rt, const double X0, const double X1, const double X2,
                                               bool st, double wq, double fx, double fy, double bf, double2* __restrict__ out) {
  double wv[18];
  edge_W_regs(Rt, X0, X1, X2, st, wq, fx, fy, bf, wv);
#pragma unroll
  for (int k = 0; k < 9; k++) out[k] = make_double2(wv[2 * k], wv[2 * k + 1]);
}

__device__ __forceinline__ void cp_async8(void* smem, const void* gmem) {
  const unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(sa), "l"(gmem) : "memory");
}

// per-warp staging of the Schur loop (double2 units): W_a | W_c tiles (one 9-double2 record per lane each), two Dinv
// tiles (5 per lane) and two operand tiles (3 per lane: X0 X1 | X2 wq_a | wq_c -), then R|t of the block's two poses
constexpr int RC_W = 0, RC_D = 32 * 18, RC_OP = RC_D + 2 * 32 * 5, RC_RT = RC_OP + 2 * 32 * 3, RC_TOTAL = RC_RT + 12;

// Pair-list Schur accumulation of one block, software pipelined: while the lanes multiply the pairs of iteration i, the
// cp.async copies of iteration i+1 are in flight and the pair records of iteration i+2 are being loaded.  W_a / W_c are
// recomputed per pair from 40 bytes of operands that stay resident in L2 (landmark position, two edge weights) instead
// of being stored per edge and gathered (144 bytes each from an array that 32 concurrent windows push out of L2).
// Edges excluded from the optimisation (level 1) have weight 0 and so an exact zero W_e: they need no test here.
template <bool DIAG>
__device__ __forceinline__ void schur_block_pairs(const int4* prs, int qBeg, int qEnd, const double* __restrict__ pts,
                                                     const double* __restrict__ eWq, const double2* Db, double2* buf, int lane,
                                                     double fx, double fy, double bf, double (&acc)[32], double (&tail)[10]) {
  const int nIt = (qEnd - qBeg + 31) >> 5;
  double2* tW = buf + RC_W;
  const double* Rt = reinterpret_cast<const double*>(buf + RC_RT);
  auto issue = [&](int slot, const int4& r, bool v) {
    double2* op = buf + RC_OP + slot * (32 * 3) + lane * 3;
    if (v) {
      const double* X = pts + (size_t)r.z * 3;
      double* o = reinterpret_cast<double*>(op);
      cp_async8(o, X);
      cp_async8(o + 1, X + 1);
      cp_async8(o + 2, X + 2);
      cp_async8(o + 3, eWq + r.x);
      if (!DIAG) cp_async8(o + 4, eWq + r.y);
    }
    warp_gather16_async<DIAG ? 5 : 3, 5>(buf + RC_D + slot * (32 * 5), Db, r.z, lane);
  };
  auto loadRec = [&](int it, int4& r, bool& v) {
    const int q = qBeg + it * 32 + lane;
    v = q < qEnd;
    r = v ? prs[q] : make_int4(0, 0, 0, 0);
  };
  int4 r0, r1 = make_int4(0, 0, 0, 0);
  bool v0, v1 = false;
  loadRec(0, r0, v0);
  issue(0, r0, v0);
  cp_async_commit();
  if (nIt > 1) loadRec(1, r1, v1);
  for (int it = 0; it < nIt; it++) {
    const int slot = it & 1;
    if (it + 1 < nIt) issue(slot ^ 1, r1, v1);
    cp_async_commit();
    int4 r2 = make_int4(0, 0, 0, 0);
    bool v2 = false;
    if (it + 2 < nIt) loadRec(it + 2, r2, v2);
    cp_async_wait<1>();
    __syncwarp();
    if (v0) {
      const double* o = reinterpret_cast<const double*>(buf + RC_OP + slot * (32 * 3) + lane * 3);
      const double X0 = o[0], X1 = o[1], X2 = o[2];
      edge_W_from_Rt(Rt, X0, X1, X2, (r0.w & 1) != 0, o[3], fx, fy, bf, tW + lane * 9);
      if (!DIAG) edge_W_from_Rt(Rt + 12, X0, X1, X2, (r0.w & 2) != 0, o[4], fx, fy, bf, tW + 32 * 9 + lane * 9);
      schur_accumulate<DIAG>(tW, tW + 32 * 9, buf + RC_D + slot * (32 * 5), lane, acc, tail);
    }
    __syncwarp();
    r0 = r1; v0 = v1;
    r1 = r2; v1 = v2;
  }
  cp_async_wait<0>();
}

// Schur complement (block_solver.hpp:381-439): one warp per lower block (i1 >= i2); lanes stride over the block's
// covisibility pairs (edge a of pose i1, edge c of pose i2, same landmark l) and accumulate (W_a Dinv_l) W_c^T; the
// diagonal blocks also accumulate W_a (Dinv_l b_l) for the right-hand side.  S(i1,i2) = [Hpp + lambda I] - sum.
// Blocks are dealt to the warps of the window in snake order over the list sorted by descending pair count.
__device__ void phase_schur_blocks(const BaPtrs& p, const WinCtx& c, const BaWin& W, double lambda, double* stage, int cur) {
  const int w = c.w;
  const int lane = threadIdx.x & 31;
  const int nWarps = c.gthreads >> 5, gw = c.gtid >> 5;
  const int nb = W.nFree * (W.nFree + 1) / 2;
  const int n = W.nFree * 6;
  const int* off = p.blkOff + (size_t)w * (p.capBlk + 1);
  const int* order = p.blkOrder + (size_t)w * p.capBlk;
  const int4* prs = p.pairRec + (size_t)w * p.capPairs;
  const double2* Db = reinterpret_cast<const double2*>(p.DinvP + (size_t)w * p.capMp * 10);
  const double* ptsW = p.pts + (size_t)w * p.capMp * 3;
  const double* wqW = p.eWqB[cur] + (size_t)w * p.capE;
  double2* buf = reinterpret_cast<double2*>(stage) + (size_t)(threadIdx.x >> 5) * RC_TOTAL;
  for (int k0 = 0; k0 < nb; k0 += nWarps) {
    const int k = k0 + (((k0 / nWarps) & 1) ? nWarps - 1 - gw : gw);
    if (k >= nb) continue;
    const int t = order[k];
    int i1, i2;
    decode_block(t, i1, i2);
    const bool diag = (i1 == i2);
    double acc[32], tail[10];  // entries 0..31, entries 32..35 + the 6 right-hand-side sums
#pragma unroll
    for (int z = 0; z < 32; z++) acc[z] = 0;
#pragma unroll
    for (int z = 0; z < 10; z++) tail[z] = 0;
    const int qBeg = off[t], qEnd = off[t + 1];
    const bool any = qEnd > qBeg;
    if (any) {
      // rotation / translation of the block's two cameras, staged once per block for the whole warp
      __syncwarp();
      if (lane < 2) {
        const int kf = p.freeKf[(size_t)w * p.capKf + (lane ? i2 : i1)];
        const double* P = p.pose + ((size_t)w * p.capKf + kf) * POSE_STRIDE;
        double R[3][3];
        quat_to_R(P, R);
        double* o = reinterpret_cast<double*>(buf + RC_RT) + lane * 12;
#pragma unroll
        for (int a = 0; a < 3; a++)
#pragma unroll
          for (int b2 = 0; b2 < 3; b2++) o[a * 3 + b2] = R[a][b2];
        o[9] = P[4]; o[10] = P[5]; o[11] = P[6];
      }
      __syncwarp();
      if (diag) schur_block_pairs<true>(prs, qBeg, qEnd, ptsW, wqW, Db, buf, lane, W.fx, W.fy, W.bf, acc, tail);
      else schur_block_pairs<false>(prs, qBeg, qEnd, ptsW, wqW, Db, buf, lane, W.fx, W.fy, W.bf, acc, tail);
    }
    double mine = 0;
    if (any) {  // (warp-uniform) a block without pairs is just its Hpp part
      mine = warp_reduce_scatter32(acc, lane);
#pragma unroll
      for (int z = 0; z < 10; z++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) tail[z] += __shfl_xor_sync(0xffffffffu, tail[z], o);
      }
    }
    double* Sb = p.S + (size_t)w * p.ldS * p.ldS + (size_t)(i1 * 6) * p.ldS + i2 * 6;
    const double* Hp = p.Hpp + ((size_t)w * p.capKf + i1) * 36;
    {
      const int r = lane / 6, cc = lane - r * 6;
      double base = 0;
      if (diag) {
        base = Hp[lane];
        if (r == cc) base += lambda;
      }
      Sb[(size_t)r * p.ldS + cc] = base - mine;
    }
    if (lane < 4) {  // entries 32..35 = row 5, columns 2..5
      const int cc = 2 + lane;
      double base = 0;
      if (diag) {
        base = Hp[32 + lane];
        if (cc == 5) base += lambda;
      }
      double tv = tail[0];
      if (lane == 1) tv = tail[1];
      if (lane == 2) tv = tail[2];
      if (lane == 3) tv = tail[3];
      Sb[(size_t)5 * p.ldS + cc] = base - tv;
    }
    if (diag && lane >= 8 && lane < 14) {  // augmented row: b_p - sum_e W_e (Dinv b_l)
      const int r = lane - 8;
      double tv = tail[4];
      if (r == 1) tv = tail[5];
      if (r == 2) tv = tail[6];
      if (r == 3) tv = tail[7];
      if (r == 4) tv = tail[8];
      if (r == 5) tv = tail[9];
      const double* bp = p.b + (size_t)w * (p.capKf * 6 + p.capMp * 3) + (size_t)i1 * 6;
      p.S[(size_t)w * p.ldS * p.ldS + (size_t)n * p.ldS + i1 * 6 + r] = bp[r] - tv;
    }
  }
}

// LinearSolver on the reduced camera system: blocked right-looking Cholesky (lower) by ONE CTA of the window.
// The augmented last row carries b and ends up holding y = L^-1 b; then L^T x = y by blocked back substitution.
// Diagonal 32x32 blocks are factored by one warp with a row per lane in registers (shuffle broadcast), the panel solve
// keeps each row in registers, the trailing update is 4x4 register tiled out of the shared-memory panel.
constexpr int CHOL_PP = CHOL_BS + 1;
__device__ void phase_chol(const BaPtrs& p, int w, const BaWin& W, double* dsm) {
  BaState& st = p.st[w];
  const int n = W.nFree * 6, ld = p.ldS;
  double* S = p.S + (size_t)w * ld * ld;
  double* Dblk = dsm;                                // 33 x 33 (last row: reciprocal diagonal)
  double* panel = dsm + (CHOL_BS + 1) * CHOL_PP;     // (ld+8) x 33
  double* xs = panel + (size_t)(ld + 8) * CHOL_PP;   // ld
  double* rdiag = xs + ld;                           // ld: 1 / L[i][i], kept for the back substitution
  int* rowList = reinterpret_cast<int*>(rdiag + ld);  // ld + 4 ints: compacted row list of the current block column
  int* bfirst = rowList + ld + 4;                     // nFree ints: first non-empty block of every block row (envelope)
  __shared__ int fail, mRows;
  for (int i = threadIdx.x; i < W.nFree; i += blockDim.x) bfirst[i] = p.blkFirst[(size_t)w * p.capKf + i];
  const int tid = threadIdx.x, T = blockDim.x, lane = tid & 31;
  if (tid == 0) fail = 0;
  __syncthreads();
  for (int kb = 0; kb < n; kb += CHOL_BS) {
    const int wd = min(CHOL_BS, n - kb);
    for (int idx = tid; idx < CHOL_BS * CHOL_BS; idx += T) {
      const int r = idx >> 5, cc = idx & 31;
      double v = (r == cc) ? 1.0 : 0.0;  // identity padding for a short last block
      if (r < wd && cc < wd) v = (cc <= r) ? S[(size_t)(kb + r) * ld + kb + cc] : 0.0;
      Dblk[r * CHOL_PP + cc] = v;
    }
    __syncthreads();
    if (tid < 32) {
      double row[CHOL_BS];
#pragma unroll
      for (int cc = 0; cc < CHOL_BS; cc++) row[cc] = Dblk[lane * CHOL_PP + cc];
      bool bad = false;
      double mydinv = 1.0;
#pragma unroll
      for (int j = 0; j < CHOL_BS; j++) {
        double djj = __shfl_sync(0xffffffffu, row[j], j);
        if (!(djj > 0.0) || !isfinite(djj)) {
          bad = true;
          djj = 1.0;
        }
        const double rinv = rsqrt(djj);
        const double ljj = djj * rinv;
        mydinv = (lane == j) ? rinv : mydinv;  // 1 / L[j][j]
        // branch-free on purpose: entries above the diagonal (k > lane) hold don't-care values that are never read;
        // lane-dependent control flow here makes the compiler index `row` dynamically and spill it to local memory
        row[j] = (lane == j) ? ljj : row[j] * rinv;
#pragma unroll
        for (int k = j + 1; k < CHOL_BS; k++) {
          const double lkj = __shfl_sync(0xffffffffu, row[j], k);  // L[k][j]
          row[k] = fma(-row[j], lkj, row[k]);
        }
      }
      if (bad && lane == 0) fail = 1;
#pragma unroll
      for (int cc = 0; cc < CHOL_BS; cc++) Dblk[lane * CHOL_PP + cc] = (cc <= lane) ? row[cc] : 0.0;
      Dblk[CHOL_BS * CHOL_PP + lane] = mydinv;
      if (lane < wd) rdiag[kb + lane] = mydinv;
    } else if (tid == 32) {  // meanwhile: the rows this block column reaches (envelope), in ascending order
      int cnt = 0;
      const int rEnd = kb + wd;
      for (int pr = rEnd / 6; pr < W.nFree; pr++) {
        if (bfirst[pr] * 6 >= rEnd) continue;
        for (int i = max(pr * 6, rEnd); i < pr * 6 + 6; i++) rowList[cnt++] = i;
      }
      rowList[cnt++] = n;
      mRows = cnt;
    }
    __syncthreads();
    for (int idx = tid; idx < wd * wd; idx += T) {
      const int r = idx / wd, cc = idx - r * wd;
      if (cc <= r) S[(size_t)(kb + r) * ld + kb + cc] = Dblk[r * CHOL_PP + cc];
    }
    // rows below the diagonal block whose envelope reaches into this block column (rowList, built during the factor
    // step; the augmented row n is always among them); all other rows hold zeros here and stay untouched
    const int m = mRows;
    for (int rowi = tid; rowi < m; rowi += T) {
      const int i = rowList[rowi];
      double v[CHOL_BS];
      const double* dinv = Dblk + CHOL_BS * CHOL_PP;
#pragma unroll
      for (int cc = 0; cc < CHOL_BS; cc++) v[cc] = (cc < wd) ? S[(size_t)i * ld + kb + cc] : 0.0;
#pragma unroll
      for (int cc = 0; cc < CHOL_BS; cc++) {
        double a = v[cc];
#pragma unroll
        for (int k = 0; k < cc; k++) a -= v[k] * Dblk[cc * CHOL_PP + k];
        v[cc] = a * dinv[cc];
      }
#pragma unroll
      for (int cc = 0; cc < CHOL_BS; cc++) {
        panel[rowi * CHOL_PP + cc] = v[cc];
        if (cc < wd) S[(size_t)i * ld + kb + cc] = v[cc];
      }
    }
    for (int idx = tid; idx < 8 * CHOL_PP; idx += T) panel[(m + idx / CHOL_PP) * CHOL_PP + idx % CHOL_PP] = 0.0;  // pad to a multiple of 8 rows
    __syncthreads();
    // trailing update S[i][j] -= sum_k panel[i][k] * panel[j][k] on the FP64 tensor pipe: one warp per 8 x 8 tile of the
    // (compacted) row list, eight DMMA.8x8x4 per tile (k = 32), fragments loaded straight from the panel in shared memory.
    // mma.m8n8k4 f64 fragments: A[g][t] and B[t][g] one value per lane (g = lane / 4, t = lane % 4), C[g][2t], C[g][2t+1].
    {
      const int mt = (m + 7) >> 3;
      const int ntile = mt * (mt + 1) / 2;
      const int warp = tid >> 5, nwarp = T >> 5;
      const int g = lane >> 2, t4 = lane & 3;
      for (int t = warp; t < ntile; t += nwarp) {
        int ti, tj;
        decode_block(t, ti, tj);
        const double* pa = panel + (size_t)(8 * ti + g) * CHOL_PP + t4;
        const double* pb = panel + (size_t)(8 * tj + g) * CHOL_PP + t4;
        double c0 = 0.0, c1 = 0.0;
#pragma unroll
        for (int k0 = 0; k0 < CHOL_BS; k0 += 4) {
          const double av = pa[k0], bv = pb[k0];
          asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                       : "+d"(c0), "+d"(c1)
                       : "d"(av), "d"(bv));
        }
        const int ia = 8 * ti + g;
        if (ia < m) {
          const int i = rowList[ia];
          const int jb0 = 8 * tj + 2 * t4;
          if (jb0 <= ia) {  // lower triangle only (the list is ascending); column n is never needed
            const int j = rowList[jb0];
            if (j < n) S[(size_t)i * ld + j] -= c0;
          }
          if (jb0 + 1 <= ia) {
            const int j = rowList[jb0 + 1];
            if (j < n) S[(size_t)i * ld + j] -= c1;
          }
        }
      }
    }
    __syncthreads();
  }
  // back substitution L^T x = y
  for (int i = tid; i < n; i += T) xs[i] = S[(size_t)n * ld + i];
  __syncthreads();
  const int nblk = (n + CHOL_BS - 1) / CHOL_BS;
  for (int bk = nblk - 1; bk >= 0; bk--) {
    const int kb = bk * CHOL_BS, wd = min(CHOL_BS, n - kb);
    for (int idx = tid; idx < CHOL_BS * CHOL_BS; idx += T) {
      const int r = idx >> 5, cc = idx & 31;
      double v = (r == cc) ? 1.0 : 0.0;
      if (r < wd && cc < wd) v = (cc <= r) ? S[(size_t)(kb + r) * ld + kb + cc] : 0.0;
      Dblk[r * CHOL_PP + cc] = v;
    }
    __syncthreads();
    if (tid < 32) {
      double col[CHOL_BS];  // column `lane` of L_D == row `lane` of L_D^T
#pragma unroll
      for (int r = 0; r < CHOL_BS; r++) col[r] = Dblk[r * CHOL_PP + lane];
      double tv = (lane < wd) ? xs[kb + lane] : 0.0;
      const double myrcp = (lane < wd) ? rdiag[kb + lane] : 1.0;  // 1 / L[lane][lane] from the factorisation
#pragma unroll
      for (int j = CHOL_BS - 1; j >= 0; j--) {
        double xj = tv * myrcp;  // meaningful on lane j
        xj = __shfl_sync(0xffffffffu, xj, j);
        tv = (lane == j) ? xj : ((lane < j) ? fma(-col[j], xj, tv) : tv);
      }
      if (lane < wd) xs[kb + lane] = tv;
    }
    __syncthreads();
    int cmin = kb;  // leftmost column any row of this block reaches
    for (int pr = kb / 6; pr <= min((kb + wd - 1) / 6, W.nFree - 1); pr++) cmin = min(cmin, bfirst[pr] * 6);
    for (int cc = cmin + tid; cc < kb; cc += T) {
      double sacc = xs[cc];
#pragma unroll 8
      for (int r = 0; r < CHOL_BS; r++)
        if (r < wd) sacc -= S[(size_t)(kb + r) * ld + cc] * xs[kb + r];
      xs[cc] = sacc;
    }
    __syncthreads();
  }
  double* x = p.x + (size_t)w * (p.capKf * 6 + p.capMp * 3);
  for (int i = tid; i < n; i += T) x[i] = xs[i];
  if (tid == 0) st.solveOk = fail ? 0 : 1;
  __syncthreads();
}

// landmark back-substitution (block_solver.hpp:461-481) + updates (types_sba.h:52-56, se3quat oplus) + computeScale
__device__ void phase_backsub_update(const BaPtrs& p, const WinCtx& c, const BaWin& W, double lambda, int solveOk,
                                     double* sm, double* stage, int cur) {
  const int w = c.w;
  const int* ms = p.mpStart + (size_t)w * (p.capMp + 1);
  const size_t xo = (size_t)w * (p.capKf * 6 + p.capMp * 3);
  double sc = 0;
  const int lane = threadIdx.x & 31;
  const int2* lrec = p.lmRec + (size_t)w * p.capE;
  double* RtTab = stage + (size_t)(blockDim.x >> 5) * RC_TOTAL * 2;  // R | t of every free pose (behind the Schur staging)
  if (solveOk) {
    for (int i = threadIdx.x; i < W.nFree; i += blockDim.x) {
      const double* P = p.pose + ((size_t)w * p.capKf + p.freeKf[(size_t)w * p.capKf + i]) * POSE_STRIDE;
      double R[3][3];
      quat_to_R(P, R);
      double* o = RtTab + (size_t)i * 12;
#pragma unroll
      for (int a = 0; a < 3; a++)
#pragma unroll
        for (int b2 = 0; b2 < 3; b2++) o[a * 3 + b2] = R[a][b2];
      o[9] = P[4]; o[10] = P[5]; o[11] = P[6];
    }
    __syncthreads();
  }
  const double* wqW = p.eWqB[cur] + (size_t)w * p.capE;
  const uint8_t* stW = p.eStereo + (size_t)w * p.capE;
  for (int l0 = c.gtid - lane; l0 < W.nMp; l0 += c.gthreads) {  // 32 consecutive landmarks per warp, one per lane
    const int l = l0 + lane;
    const bool live = l < W.nMp;
    const size_t mo = (size_t)w * p.capMp + (live ? l : 0);
    double* X = p.pts + mo * 3;
    double* Xb = p.ptsBak + mo * 3;
    if (!solveOk) {
      if (live)
        for (int i = 0; i < 3; i++) Xb[i] = X[i];
      continue;
    }
    const double* bl = p.b + xo + (size_t)W.nFree * 6 + (size_t)(live ? l : 0) * 3;
    double cl[3] = {bl[0], bl[1], bl[2]};
    const int kBeg = live ? ms[l] : 0, deg = live ? ms[l + 1] - kBeg : 0;
    // W_e^T x_p with W_e recomputed from (R|t of the pose, this landmark, edge weight): five edges' {edge, pose} records,
    // then their weights and flags, are loaded together, so the five edges share two memory latencies.  Level-1 edges
    // have weight 0 and subtract exact zeros.
    constexpr int NBUF = 5;
    const double X0 = live ? X[0] : 0.0, X1 = live ? X[1] : 0.0, X2 = live ? X[2] : 1.0;
    for (int kb0 = 0; kb0 < deg; kb0 += NBUF) {
      int ee[NBUF], pp[NBUF];
      double wq[NBUF];
      bool st[NBUF];
#pragma unroll
      for (int j = 0; j < NBUF; j++) {
        const int2 r = (kb0 + j < deg) ? lrec[kBeg + kb0 + j] : make_int2(0, -1);
        ee[j] = r.x;
        pp[j] = r.y;
      }
#pragma unroll
      for (int j = 0; j < NBUF; j++) {
        wq[j] = wqW[ee[j]];
        st[j] = stW[ee[j]] != 0;
      }
#pragma unroll
      for (int j = 0; j < NBUF; j++) {
        if (pp[j] < 0) continue;
        double wb[18];
        edge_W_regs(RtTab + (size_t)pp[j] * 12, X0, X1, X2, st[j], wq[j], W.fx, W.fy, W.bf, wb);
        const double* xp = p.x + xo + (size_t)pp[j] * 6;
#pragma unroll
        for (int cc = 0; cc < 3; cc++)
#pragma unroll
          for (int r = 0; r < 6; r++) cl[cc] -= wb[r * 3 + cc] * xp[r];
      }
    }
    if (!live) continue;
    const double* Di = p.Dinv + mo * 9;
    double* xout = p.x + xo + (size_t)W.nFree * 6 + (size_t)l * 3;
    for (int i = 0; i < 3; i++) {
      const double xl = Di[i * 3] * cl[0] + Di[i * 3 + 1] * cl[1] + Di[i * 3 + 2] * cl[2];
      xout[i] = xl;
      Xb[i] = X[i];
      X[i] += xl;
      sc += xl * (lambda * xl + bl[i]);
    }
  }
  // poses: the last CTA of the window also backs up and updates the keyframe poses
  if (c.cta == c.nCta - 1) {
    for (int kf = threadIdx.x; kf < W.nKf; kf += blockDim.x) {
      double* P = p.pose + ((size_t)w * p.capKf + kf) * POSE_STRIDE;
      double* Pb = p.poseBak + ((size_t)w * p.capKf + kf) * POSE_STRIDE;
      for (int k = 0; k < 7; k++) Pb[k] = P[k];
      const int pi = p.poseIndex[(size_t)w * p.capKf + kf];
      if (pi >= 0 && solveOk) {
        const double* xp = p.x + xo + (size_t)pi * 6;
        const double* bp = p.b + xo + (size_t)pi * 6;
        pose_oplus(P, xp);
        for (int i = 0; i < 6; i++) sc += xp[i] * (lambda * xp[i] + bp[i]);
      }
    }
  }
  const double s = block_sum(sc, sm);
  if (threadIdx.x == 0) p.partScale[(size_t)w * p.nPartM + c.cta] = s;
}

// computeActiveErrors + activeRobustChi2 after the update (sparse_optimizer.cpp:61-113), one thread per edge; also keeps
// the error vectors and the edge weights rho' * invSigma2 in buffer storeBuf, so that an accepted step needs no separate
// error pass before the next buildSystem (the values are the same);
// zeroDead: excluded edges get weight 0 (first pass of a round).
__device__ void phase_errors(const BaPtrs& p, const WinCtx& c, const BaWin& W, int robust, double* sm, int storeBuf,
                             bool zeroDead = false) {
  const int w = c.w;
  double chi = 0;
  // four edges per thread and iteration, loaded in two waves ahead of the arithmetic (see load_edge_idx)
  for (int e = c.gtid; e < W.nEdges; e += 4 * c.gthreads) {
    EdgeIdx ix[4];
    EdgeOps op[4];
#pragma unroll
    for (int h = 0; h < 4; h++) load_edge_idx(p, w, e + h * c.gthreads, W.nEdges, ix[h]);
#pragma unroll
    for (int h = 0; h < 4; h++) load_edge_ops(p, w, ix[h], op[h]);
#pragma unroll
    for (int h = 0; h < 4; h++) {
      const size_t eo = (size_t)w * p.capE + e + h * c.gthreads;
      if (!ix[h].live) {
        if (zeroDead && e + h * c.gthreads < W.nEdges) {  // in BOTH buffers: later passes of the round skip excluded edges
          p.eWqB[0][eo] = 0.0;
          p.eWqB[1][eo] = 0.0;
        }
        continue;
      }
      double Xc[3], er[3];
      pose_map(op[h].P, op[h].X, Xc);
      const double c2 = edge_error(Xc, ix[h].stereo, ix[h].ob, (double)ix[h].wgt, W, er);
      p.chi2[eo] = c2;
      double rho0 = c2, rho1 = 1.0;
      if (robust) huber(c2, delta_of(ix[h].stereo), rho0, rho1);
      chi += rho0;
      double* eb = p.errB[storeBuf] + eo * 3;
      eb[0] = er[0]; eb[1] = er[1]; eb[2] = er[2];
      p.eWqB[storeBuf][eo] = rho1 * (double)ix[h].wgt;
    }
  }
  const double s = block_sum(chi, sm);
  if (threadIdx.x == 0) p.partChi[(size_t)w * p.nPartE + c.cta] = s;
}

// LM accept/reject + iteration/round bookkeeping (levenberg.cpp:102-161, sparse_optimizer.cpp:376-412,
// src/Optimizer.cc:863-917)
__device__ void control_end(const BaPtrs& p, int w, int nCta) {
  BaState& st = p.st[w];
  st.restore = 0;
  st.doOutlier = 0;
  double tempChi = 0, scale = 0;
  for (int k = 0; k < nCta; k++) tempChi += p.partChi[(size_t)w * p.nPartE + k];
  for (int k = 0; k < nCta; k++) scale += p.partScale[(size_t)w * p.nPartM + k];
  st.chi2Final = tempChi;  // activeRobustChi2() of the last evaluated state (diagnostic)
  if (st.lm.trial(st.solveOk, tempChi, scale, st.trace)) {
    st.errBuf ^= 1;  // phase_errors just stored this state's errors / weights in the other buffer
    st.errCurrent = 1;
  } else {
    st.restore = 1;
  }
  const int stop = *((volatile int*)&st.stop);
  if (st.lm.retry(stop)) return;  // another trial with the larger lambda
  bool roundEnd = st.lm.end_iteration();
  st.it++;
  if (st.it >= st.its[st.round] || stop) roundEnd = true;
  if (!roundEnd) {
    st.needBuild = 1;
    return;
  }
  if (st.round == 0 && !stop && st.its[1] > 0) {
    st.doOutlier = 1;  // setLevel(1) on outliers, drop the robust kernels, second round
    st.nLive = 0;
    st.round = 1;
    st.it = 0;
    st.robust = 0;
    st.needBuild = 1;
    st.errCurrent = 0;  // levels and kernels change: the stored weights are void
  } else {
    // final outlier test (:921-958); it also runs when round 2 is skipped.  3: skipped because its2 == 0, so ba_run
    // replaces chi2Final by the chi2 of round 2's active set
    st.doOutlier = (st.round == 0 && !stop) ? 3 : 2;
    st.active = 0;
  }
}

__device__ void phase_restore(const BaPtrs& p, const WinCtx& c, const BaWin& W) {
  const int w = c.w;
  for (int i = c.gtid; i < W.nMp * 3; i += c.gthreads) p.pts[(size_t)w * p.capMp * 3 + i] = p.ptsBak[(size_t)w * p.capMp * 3 + i];
  for (int i = c.gtid; i < W.nKf * POSE_STRIDE; i += c.gthreads)
    p.pose[(size_t)w * p.capKf * POSE_STRIDE + i] = p.poseBak[(size_t)w * p.capKf * POSE_STRIDE + i];
}

// chi2 / depth outlier tests (src/Optimizer.cc:880-958)
__device__ void phase_outliers(const BaPtrs& p, const WinCtx& c, const BaWin& W, int mode) {
  const int w = c.w;
  int live = 0;
  for (int e = c.gtid; e < W.nEdges; e += c.gthreads) {
    const size_t eo = (size_t)w * p.capE + e;
    double Xc[3];
    pose_map(p.pose + ((size_t)w * p.capKf + p.eKf[eo]) * POSE_STRIDE, p.pts + ((size_t)w * p.capMp + p.eMp[eo]) * 3, Xc);
    const double th = p.eStereo[eo] ? 7.815 : 5.991;
    const bool out = p.chi2[eo] > th || !(Xc[2] > 0.0);
    if (mode == 1) {
      if (out) p.eLevel[eo] = 1;
      live += out ? 0 : 1;
      p.eOutlier[eo] = out ? 1 : 0;  // final answer already if round 2 turns out to be empty (see k_local_ba)
    } else
      p.eOutlier[eo] = out ? 1 : 0;
  }
  if (mode == 1) {  // level-0 edges that remain: warp sums, one atomic per warp
    for (int o = 16; o > 0; o >>= 1) live += __shfl_down_sync(0xffffffffu, live, o);
    if ((threadIdx.x & 31) == 0 && live) atomicAdd(&p.st[w].nLive, live);
  }
}

// ---------------------------------------------------------------- the persistent kernel: one CTA per entry of p.ctaMap
constexpr int BA_T = 256;
__global__ void __launch_bounds__(BA_T) k_local_ba(BaPtrs p) {
  extern __shared__ __align__(16) double dsm[];
  __shared__ double red[32];
  WinCtx c;
  const int m = p.ctaMap[blockIdx.x];
  c.w = m >> 8;
  c.cta = m & 255;
  const int nCta = p.winCtas[c.w];
  c.nCta = nCta;
  c.gtid = c.cta * blockDim.x + threadIdx.x;
  c.gthreads = nCta * blockDim.x;
  const int w = c.w;
  const BaWin W = p.win[w];
  unsigned int* bar = p.bar + w;
  unsigned int epoch = 0;
  volatile BaState* vst = p.st + w;
  volatile int* hung = &(p.st + w)->finishedRound0;  // (field reused as the barrier-timeout flag)
  for (int guard = 0; guard < 4096; guard++) {
    if (!vst->active || *hung) break;
    const int needBuild = vst->needBuild, robust = vst->robust;
    const int cur = vst->errBuf;
    if (needBuild) {
      // errors + weights: after an accepted step they were stored by that step's phase_errors (same state, same values)
      if (!vst->errCurrent) {
        phase_errors(p, c, W, robust, red, cur, true);
        win_barrier(bar, epoch, nCta, hung);
      }
      phase_reduce_landmarks(p, c, W, cur, dsm);
      phase_build_poses(p, c, W, robust, cur);
      win_barrier(bar, epoch, nCta, hung);
    }
    if (c.cta == 0 && threadIdx.x == 0) control_begin(p, w, nCta);
    win_barrier(bar, epoch, nCta, hung);
    const double lambda = vst->lm.lambda;
    phase_dinv(p, c, W, lambda);
    win_barrier(bar, epoch, nCta, hung);
    phase_schur_blocks(p, c, W, lambda, dsm, cur);
    win_barrier(bar, epoch, nCta, hung);
    if (c.cta == 0) phase_chol(p, w, W, dsm);
    win_barrier(bar, epoch, nCta, hung);
    phase_backsub_update(p, c, W, lambda, vst->solveOk, red, dsm, cur);
    win_barrier(bar, epoch, nCta, hung);
    phase_errors(p, c, W, robust, red, cur ^ 1);
    win_barrier(bar, epoch, nCta, hung);
    if (c.cta == 0 && threadIdx.x == 0) control_end(p, w, nCta);
    win_barrier(bar, epoch, nCta, hung);
    if (vst->restore) phase_restore(p, c, W);
    const int doOutlier = vst->doOutlier;
    if (doOutlier) {
      win_barrier(bar, epoch, nCta, hung);  // the depth test reads the restored state
      phase_outliers(p, c, W, doOutlier);
    }
    win_barrier(bar, epoch, nCta, hung);
    if (doOutlier == 1) {
      // initializeOptimization(0) with every edge at level 1 leaves no active vertex: g2o's optimize() returns at once
      // (sparse_optimizer.cpp:356-359) and src/Optimizer.cc:921-958 flags the edges with the chi2 they already have,
      // which is what the level pass just stored in eOutlier.  Pinned by test_oracle_reference_optimizer (rejections_2).
      if (c.cta == 0 && threadIdx.x == 0 && vst->nLive == 0) {
        (p.st + w)->active = 0;
        (p.st + w)->chi2Final = 0;  // activeRobustChi2() over an empty active set
      }
      win_barrier(bar, epoch, nCta, hung);
    }
  }
}

// ---------------------------------------------------------------- structure kernels (once per window)
__global__ void __launch_bounds__(256) k_lm_edge(BaPtrs p) {
  const int w = blockIdx.y;
  const BaWin W = p.win[w];
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= W.nEdges) return;
  const size_t eo = (size_t)w * p.capE + e;
  const int pi = p.poseIndex[(size_t)w * p.capKf + p.eKf[eo]];
  if (pi >= 0) p.lmEdge[((size_t)w * p.capMp + p.eMp[eo]) * p.capKf + pi] = e;
  const int ek = p.mpEdges[eo];  // position e of the landmark-ordered edge list
  p.lmRec[eo] = make_int2(ek, p.poseIndex[(size_t)w * p.capKf + p.eKf[(size_t)w * p.capE + ek]]);
}

// covisibility pair lists: for every lower block (i1 >= i2) the (edge of pose i1, edge of pose i2) pairs that share a
// landmark, in the order of pose i1's edge list (count -> scan -> ordered fill)
__global__ void __launch_bounds__(64) k_pair_build(BaPtrs p, int fill) {
  __shared__ int wsum[2];
  __shared__ int running;
  const int w = blockIdx.y;
  if (fill && p.st[w].pairsOverflow) return;
  const BaWin W = p.win[w];
  int i1, i2;
  decode_block(blockIdx.x, i1, i2);
  if (i1 >= W.nFree) return;
  const int kf1 = p.freeKf[(size_t)w * p.capKf + i1];
  const int* ks = p.kfStart + (size_t)w * (p.capKf + 1);
  const int* ke = p.kfEdges + (size_t)w * p.capE;
  const int* lm = p.lmEdge + (size_t)w * p.capMp * p.capKf;
  int* off = p.blkOff + (size_t)w * (p.capBlk + 1);
  const int beg = ks[kf1], end = ks[kf1 + 1];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) running = 0;
  __syncthreads();
  int total = 0;
  for (int k0 = beg; k0 < end; k0 += 64) {
    const int k = k0 + threadIdx.x;
    int a = -1, cidx = -1;
    if (k < end) {
      a = ke[k];
      cidx = lm[(size_t)p.eMp[(size_t)w * p.capE + a] * p.capKf + i2];
    }
    const bool hit = cidx >= 0;
    const unsigned bm = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) wsum[wid] = __popc(bm);
    __syncthreads();
    if (fill && hit) {
      const int pos = off[blockIdx.x] + running + (wid ? wsum[0] : 0) + __popc(bm & ((1u << lane) - 1u));
      const int fl = (p.eStereo[(size_t)w * p.capE + a] ? 1 : 0) | (p.eStereo[(size_t)w * p.capE + cidx] ? 2 : 0);
      p.pairRec[(size_t)w * p.capPairs + pos] = make_int4(a, cidx, p.eMp[(size_t)w * p.capE + a], fl);
    }
    total += wsum[0] + wsum[1];
    __syncthreads();
    if (threadIdx.x == 0) running = total;
    __syncthreads();
  }
  if (!fill && threadIdx.x == 0) off[blockIdx.x + 1] = total;  // counts, scanned by k_pair_scan
}

__global__ void k_pair_scan(BaPtrs p, int batch) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= batch) return;
  const BaWin W = p.win[w];
  int* off = p.blkOff + (size_t)w * (p.capBlk + 1);
  const int nb = W.nFree * (W.nFree + 1) / 2;
  off[0] = 0;
  int run = 0;
  for (int t = 0; t < nb; t++) {
    run += off[t + 1];
    off[t + 1] = run;
  }
  if (run > p.capPairs) {  // cannot happen with capPairs >= the host's bound (ba_run); guards the fill pass
    p.st[w].pairsOverflow = 1;
    p.st[w].active = 0;
  }
}

// lower blocks sorted by descending pair count (ties by block id): the Schur phase deals them to its warps in this order
__global__ void __launch_bounds__(256) k_block_order(BaPtrs p) {
  const int w = blockIdx.x;
  const BaWin W = p.win[w];
  const int nb = W.nFree * (W.nFree + 1) / 2;
  const int* off = p.blkOff + (size_t)w * (p.capBlk + 1);
  int* order = p.blkOrder + (size_t)w * p.capBlk;
  int* first = p.blkFirst + (size_t)w * p.capKf;
  for (int i1 = threadIdx.x; i1 < W.nFree; i1 += blockDim.x) {
    int f = i1;
    const int t0 = i1 * (i1 + 1) / 2;
    for (int i2 = 0; i2 < i1; i2++)
      if (off[t0 + i2 + 1] > off[t0 + i2]) {
        f = i2;
        break;
      }
    first[i1] = f;
  }
  int nz = 0;
  for (int t = threadIdx.x; t < nb; t += blockDim.x) {
    const int mine = off[t + 1] - off[t];
    int rank = 0;
    for (int u = 0; u < nb; u++) {
      const int cu = off[u + 1] - off[u];
      rank += (cu > mine) || (cu == mine && u < t);
    }
    order[rank] = t;
    nz += mine > 0;
  }
  if (nz) atomicAdd(&p.blkNZ[w], nz);
}

// ================================================================================================
// Optimizer::PoseOptimization (src/Optimizer.cc:363-605): one CTA per frame.  One free pose, unary edges with fixed map
// points; 4 rounds x 10 Levenberg iterations from the same initial pose, inlier/outlier re-classification after every
// round with the chi2 of the LAST evaluated state (g2o semantics, also after a rejected trial), Huber kernels dropped
// after round 2.  Edge loops are strided over the CTA's threads, sums are fixed-tree block reductions (deterministic),
// the 6x6 solve and the LM bookkeeping run on thread 0.
// ================================================================================================
struct PoFrame {
  int nEdges, edgeOff;        // this frame's edges are [edgeOff, edgeOff+nEdges) of the packed arrays
  float fx, fy, cx, cy, bf;
};
struct PoPtrs {
  const PoFrame* frames;
  const double* poseInit;     // [frame][8]
  const float* Xw;            // [edge][3]
  const float* obs;           // [edge][3] (x, y, uRight; uRight < 0: monocular)
  const float* invSigma2;     // [edge]
  double* err;                // [edge][3] scratch
  double* chi2;               // [edge]
  uint8_t* level;             // [edge]
  uint8_t* outlier;           // [edge] out
  double* poseOut;            // [frame][8]
  int* nInliers;              // [frame]
  int* nTrials;               // [frame]
  int* trace;                 // [frame][256]
};

__device__ __forceinline__ double po_edge_error(const double* P, const float* Xwf, const float* ob, double w,
                                                const PoFrame& F, double* er) {
  const double X[3] = {(double)Xwf[0], (double)Xwf[1], (double)Xwf[2]};
  double Xc[3];
  pose_map(P, X, Xc);
  if (!(ob[2] < 0)) {  // stereo: cam_project with `const float invz` (types_six_dof_expmap.cpp:304-312), double bf
    const float invz = (float)(1.0 / Xc[2]);
    const double u = Xc[0] * invz * (double)F.fx + (double)F.cx;
    const double v = Xc[1] * invz * (double)F.fy + (double)F.cy;
    const double ur = u - (double)F.bf * invz;
    er[0] = (double)ob[0] - u;
    er[1] = (double)ob[1] - v;
    er[2] = (double)ob[2] - ur;
    return er[0] * (w * er[0]) + er[1] * (w * er[1]) + er[2] * (w * er[2]);
  }
  const double u = Xc[0] / Xc[2] * (double)F.fx + (double)F.cx;
  const double v = Xc[1] / Xc[2] * (double)F.fy + (double)F.cy;
  er[0] = (double)ob[0] - u;
  er[1] = (double)ob[1] - v;
  er[2] = 0;
  return er[0] * (w * er[0]) + er[1] * (w * er[1]);
}

// dense 6x6 Cholesky solve (LinearSolverDense uses Eigen LDLT; same solution up to rounding), thread 0 only
__device__ bool po_solve6(const double* H, double lambda, const double* b, double* x) {
  double L[36];
  for (int i = 0; i < 36; i++) L[i] = H[i];
  for (int i = 0; i < 6; i++) L[i * 7] += lambda;
  for (int j = 0; j < 6; j++) {
    double d = L[j * 6 + j];
    for (int k = 0; k < j; k++) d -= L[j * 6 + k] * L[j * 6 + k];
    if (!(d > 0.0) || !isfinite(d)) return false;
    d = sqrt(d);
    L[j * 6 + j] = d;
    for (int i = j + 1; i < 6; i++) {
      double sacc = L[i * 6 + j];
      for (int k = 0; k < j; k++) sacc -= L[i * 6 + k] * L[j * 6 + k];
      L[i * 6 + j] = sacc / d;
    }
  }
  double y[6];
  for (int i = 0; i < 6; i++) {
    double sacc = b[i];
    for (int k = 0; k < i; k++) sacc -= L[i * 6 + k] * y[k];
    y[i] = sacc / L[i * 6 + i];
  }
  for (int i = 5; i >= 0; i--) {
    double sacc = y[i];
    for (int k = i + 1; k < 6; k++) sacc -= L[k * 6 + i] * x[k];
    x[i] = sacc / L[i * 6 + i];
  }
  return true;
}

constexpr int PO_T = 256;
__global__ void __launch_bounds__(PO_T) k_pose_opt(PoPtrs p) {
  __shared__ double sPose[POSE_STRIDE], sInit[POSE_STRIDE], sBackup[POSE_STRIDE], sH[27], sX[6], sRed[32];
  __shared__ double sTemp;
  __shared__ Levenberg lm;
  __shared__ int sOk, sAgain, sRobust, sNActive, sNBad;
  const int fr = blockIdx.x;
  const PoFrame F = p.frames[fr];
  const int tid = threadIdx.x;
  const int nE = F.nEdges, e0 = F.edgeOff;
  if (tid < POSE_STRIDE) {
    sInit[tid] = p.poseInit[(size_t)fr * POSE_STRIDE + tid];
    sPose[tid] = sInit[tid];
  }
  if (tid == 0) {
    sRobust = 1;
    lm.nTrials = 0;
    sNBad = 0;
  }
  for (int e = tid; e < nE; e += PO_T) {
    p.level[e0 + e] = 0;
    p.outlier[e0 + e] = 0;
  }
  __syncthreads();
  if (nE < 3) {  // :492-493: return 0, pose untouched
    if (tid < POSE_STRIDE) p.poseOut[(size_t)fr * POSE_STRIDE + tid] = sInit[tid];
    if (tid == 0) {
      p.nInliers[fr] = 0;
      p.nTrials[fr] = 0;
    }
    return;
  }
  auto eval_errors = [&]() -> void {  // computeActiveErrors + activeRobustChi2 -> sTemp
    double chi = 0;
    const int robust = sRobust;
    for (int e = tid; e < nE; e += PO_T) {
      const int ge = e0 + e;
      if (p.level[ge]) continue;
      double er[3];
      const double c2 = po_edge_error(sPose, p.Xw + (size_t)ge * 3, p.obs + (size_t)ge * 3, (double)p.invSigma2[ge], F, er);
      p.err[(size_t)ge * 3] = er[0];
      p.err[(size_t)ge * 3 + 1] = er[1];
      p.err[(size_t)ge * 3 + 2] = er[2];
      p.chi2[ge] = c2;
      double r0 = c2, r1;
      if (robust) huber(c2, delta_of(!(p.obs[(size_t)ge * 3 + 2] < 0)), r0, r1);
      chi += r0;
    }
    const double tot = block_sum(chi, sRed);
    if (tid == 0) sTemp = tot;
    __syncthreads();
  };
  for (int round = 0; round < 4; round++) {
    if (tid < POSE_STRIDE) sPose[tid] = sInit[tid];  // vSE3->setEstimate(Converter::toSE3Quat(pFrame->mTcw)) (:505)
    int act = 0;
    for (int e = tid; e < nE; e += PO_T) act += p.level[e0 + e] == 0;
    __syncthreads();
    {
      const double a = block_sum((double)act, sRed);
      if (tid == 0) {
        sNActive = (int)a;
        sOk = 1;
      }
      __syncthreads();
    }
    if (sNActive > 0) {
      for (int it = 0; it < 10; it++) {
        if (!sOk) break;
        eval_errors();
        if (tid == 0) lm.begin(sTemp);
        // buildSystem: J^T (rho' Omega) J (upper triangle, 21) and -J^T Omega e rho' (6)
        double acc[27];
#pragma unroll
        for (int k = 0; k < 27; k++) acc[k] = 0;
        const int robust = sRobust;
        for (int e = tid; e < nE; e += PO_T) {
          const int ge = e0 + e;
          if (p.level[ge]) continue;
          const float* Xwf = p.Xw + (size_t)ge * 3;
          const double X[3] = {(double)Xwf[0], (double)Xwf[1], (double)Xwf[2]};
          double Xc[3];
          pose_map(sPose, X, Xc);
          const bool st = !(p.obs[(size_t)ge * 3 + 2] < 0);
          const double fx = F.fx, fy = F.fy, bf = F.bf;
          const double x = Xc[0], y = Xc[1], invz = 1.0 / Xc[2], invz_2 = invz * invz;
          double B[3][6];
          B[0][0] = x * y * invz_2 * fx;
          B[0][1] = -(1 + (x * x * invz_2)) * fx;
          B[0][2] = y * invz * fx;
          B[0][3] = -invz * fx;
          B[0][4] = 0;
          B[0][5] = x * invz_2 * fx;
          B[1][0] = (1 + y * y * invz_2) * fy;
          B[1][1] = -x * y * invz_2 * fy;
          B[1][2] = -x * invz * fy;
          B[1][3] = 0;
          B[1][4] = -invz * fy;
          B[1][5] = y * invz_2 * fy;
          B[2][0] = st ? B[0][0] - bf * y * invz_2 : 0.0;
          B[2][1] = st ? B[0][1] + bf * x * invz_2 : 0.0;
          B[2][2] = st ? B[0][2] : 0.0;
          B[2][3] = st ? B[0][3] : 0.0;
          B[2][4] = 0;
          B[2][5] = st ? B[0][5] - bf * invz_2 : 0.0;
          const double w0 = (double)p.invSigma2[ge];
          double rho1 = 1.0;
          if (robust) {
            double r0;
            huber(p.chi2[ge], delta_of(st), r0, rho1);
          }
          const double* er = p.err + (size_t)ge * 3;
          double omr[3];
#pragma unroll
          for (int r = 0; r < 3; r++) omr[r] = -(w0 * er[r]) * rho1;
          const double wq = rho1 * w0;
          int t = 0;
#pragma unroll
          for (int i = 0; i < 6; i++)
#pragma unroll
            for (int j = i; j < 6; j++) {
              double hh = 0;
#pragma unroll
              for (int r = 0; r < 3; r++) hh += B[r][i] * wq * B[r][j];
              acc[t++] += hh;
            }
#pragma unroll
          for (int i = 0; i < 6; i++) {
            double s2 = 0;
#pragma unroll
            for (int r = 0; r < 3; r++) s2 += B[r][i] * omr[r];
            acc[21 + i] += s2;
          }
        }
#pragma unroll
        for (int k = 0; k < 27; k++) {
          const double tot = block_sum(acc[k], sRed);
          if (tid == 0) sH[k] = tot;
        }
        __syncthreads();
        if (tid == 0) {
          if (it == 0) {  // computeLambdaInit (levenberg.cpp:166-180)
            double mx = 0;
            int t = 0;
            for (int i = 0; i < 6; i++)
              for (int j = i; j < 6; j++) {
                if (i == j) mx = fmax(fabs(sH[t]), mx);
                t++;
              }
            lm.init_lambda(1e-5 * mx);
          }
        }
        __syncthreads();
        do {
          if (tid == 0) {
            for (int k = 0; k < POSE_STRIDE; k++) sBackup[k] = sPose[k];
            double Hf[36], bb[6];
            int t = 0;
            for (int i = 0; i < 6; i++)
              for (int j = i; j < 6; j++) {
                Hf[i * 6 + j] = sH[t];
                Hf[j * 6 + i] = sH[t];
                t++;
              }
            for (int i = 0; i < 6; i++) bb[i] = sH[21 + i];
            double xx[6];
            const bool ok2 = po_solve6(Hf, lm.lambda, bb, xx);
            sAgain = ok2 ? 1 : 0;  // (temporarily: solve status)
            if (ok2) {
              for (int i = 0; i < 6; i++) sX[i] = xx[i];
              pose_oplus(sPose, xx);
            }
          }
          __syncthreads();
          const int ok2 = sAgain;
          eval_errors();
          if (tid == 0) {
            double scale = 0;
            if (ok2)
              for (int j = 0; j < 6; j++) scale += sX[j] * (lm.lambda * sX[j] + sH[21 + j]);
            if (!lm.trial(ok2, sTemp, scale, p.trace + (size_t)fr * 256))
              for (int k = 0; k < POSE_STRIDE; k++) sPose[k] = sBackup[k];
            sAgain = lm.retry(false) ? 1 : 0;
          }
          __syncthreads();
        } while (sAgain);
        if (tid == 0 && lm.end_iteration()) sOk = 0;
        __syncthreads();
      }
    }
    // re-classification (:510-567): chi2 of the last evaluated state for active edges, recomputed for current outliers
    int bad = 0;
    for (int e = tid; e < nE; e += PO_T) {
      const int ge = e0 + e;
      const bool st = !(p.obs[(size_t)ge * 3 + 2] < 0);
      double c2 = p.chi2[ge];
      if (p.outlier[ge]) {
        double er[3];
        c2 = po_edge_error(sPose, p.Xw + (size_t)ge * 3, p.obs + (size_t)ge * 3, (double)p.invSigma2[ge], F, er);
        p.err[(size_t)ge * 3] = er[0];
        p.err[(size_t)ge * 3 + 1] = er[1];
        p.err[(size_t)ge * 3 + 2] = er[2];
        p.chi2[ge] = c2;
      }
      const bool out = (float)c2 > (st ? 7.815f : 5.991f);
      p.outlier[ge] = out ? 1 : 0;
      p.level[ge] = out ? 1 : 0;
      bad += out;
    }
    __syncthreads();
    {
      const double nb = block_sum((double)bad, sRed);
      if (tid == 0) {
        sNBad = (int)nb;
        if (round == 2) sRobust = 0;  // e->setRobustKernel(0)
      }
      __syncthreads();
    }
    if (nE < 10) break;  // optimizer.edges().size() < 10 (:569-570)
  }
  if (tid < POSE_STRIDE) p.poseOut[(size_t)fr * POSE_STRIDE + tid] = sPose[tid];
  if (tid == 0) {
    p.nInliers[fr] = nE - sNBad;
    p.nTrials[fr] = lm.nTrials;
    if (lm.nTrials < 256) p.trace[(size_t)fr * 256 + min(lm.nTrials, 255)] = -1;
  }
}

}  // namespace b2s

using namespace b2s;

// ================================================================================================ host side
struct BaHostStage {  // pinned mirror of the uploaded per-window arrays (same strides as the device arrays)
  double *pose = nullptr, *pts = nullptr;
  int *pidx = nullptr, *freeKf = nullptr, *eKf = nullptr, *eMp = nullptr, *mpStart = nullptr, *kfStart = nullptr,
      *mpEdges = nullptr, *kfEdges = nullptr, *ctaMap = nullptr, *winCtas = nullptr;
  float *eObs = nullptr, *eW = nullptr;
  uint8_t *eSt = nullptr, *eOutlier = nullptr;
  BaWin* win = nullptr;
  BaState* st = nullptr;
};

// Stage::ev / lastMs time the persistent LM kernel of the last LocalBA batch (b2s_ba_last_kernel_ms).
struct b2s_ba_solver : b2s::Stage {
  int maxKf, maxMp, maxE, maxBatch;
  cudaStream_t stream2 = nullptr;  // forwards the abort flag while the LM kernel runs on `stream`
  long long launches = 0;
  BaPtrs d;
  BaHostStage hs;
  size_t smemBytes = 0;
  int numSMs = 0;
  long long lastTrials = 0;
  int smBudget = 0;  // CTAs (= SMs) one LocalBA batch may occupy; 0 = all (b2s_ba_set_sm_budget)
  DevBuf pairRec;    // d.pairRec: batch x d.capPairs records, grown by ba_run when a window needs more
  // PoseOptimization buffers, grown on first use
  DevBuf poFrames, poPoseInit, poPoseOut, poErr, poChi2, poXw, poObs, poInvS, poLevel, poOutlier, poNInl, poNTr, poTrace;
};

extern "C" int b2s_ba_create(int max_kf, int max_mp, int max_edges, int max_batch, int device, b2s_ba_solver** out) {
  if (!out || max_kf < 1 || max_kf > 128 || max_mp < 1 || max_edges < 1 || max_batch < 1) {
    set_error("b2s_ba_create: bad argument (max_kf must be in [1,128])");
    return B2S_ERR_BAD_ARG;
  }
  *out = nullptr;
  int rc = select_device(device);
  if (rc != B2S_OK) return rc;
  b2s_ba_solver* h = new b2s_ba_solver();
  h->maxKf = max_kf; h->maxMp = max_mp; h->maxE = max_edges; h->maxBatch = max_batch;
  cudaDeviceGetAttribute(&h->numSMs, cudaDevAttrMultiProcessorCount, device);
  BaPtrs& d = h->d;
  memset(&d, 0, sizeof(d));
  d.capKf = max_kf; d.capMp = max_mp; d.capE = max_edges;
  d.ldS = max_kf * 6 + 1;
  d.nPartE = 32;  // >= CTAs per window
  d.nPartM = 32;
  d.capBlk = max_kf * (max_kf + 1) / 2;
  d.capPairs = 8 * max_edges;
  const size_t B = max_batch;
  h->open(device);
  cudaError_t& e = h->error;
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&h->stream2, cudaStreamNonBlocking);
  auto A = [h](auto* p, size_t bytes) {  // zero-filled
    h->alloc(*p, bytes);
    if (h->error == cudaSuccess) h->error = cudaMemset(*p, 0, bytes);
  };
  A(&d.win, B * sizeof(BaWin)); A(&d.st, B * sizeof(BaState));
  A(&d.pose, B * max_kf * POSE_STRIDE * 8); A(&d.poseBak, B * max_kf * POSE_STRIDE * 8);
  A(&d.pts, B * max_mp * 3 * 8); A(&d.ptsBak, B * max_mp * 3 * 8);
  A(&d.poseIndex, B * max_kf * 4);
  A(&d.eKf, B * max_edges * 4); A(&d.eMp, B * max_edges * 4);
  A(&d.eObs, B * max_edges * 12); A(&d.eW, B * max_edges * 4);
  A(&d.eStereo, B * max_edges); A(&d.eLevel, B * max_edges); A(&d.eOutlier, B * max_edges);
  A(&d.chi2, B * max_edges * 8);
  A(&d.errB[0], B * max_edges * 24); A(&d.errB[1], B * max_edges * 24);
  A(&d.eWqB[0], B * max_edges * 8); A(&d.eWqB[1], B * max_edges * 8);
  A(&d.mpStart, B * (max_mp + 1) * 4); A(&d.mpEdges, B * max_edges * 4);
  A(&d.kfStart, B * (max_kf + 1) * 4); A(&d.kfEdges, B * max_edges * 4);
  A(&d.Hpp, B * max_kf * 36 * 8); A(&d.Hll, B * max_mp * 9 * 8);
  A(&d.b, B * ((size_t)max_kf * 6 + (size_t)max_mp * 3) * 8); A(&d.x, B * ((size_t)max_kf * 6 + (size_t)max_mp * 3) * 8);
  A(&d.Dinv, B * max_mp * 9 * 8); A(&d.S, B * (size_t)d.ldS * d.ldS * 8);
  A(&d.db, B * max_mp * 3 * 8); A(&d.DinvP, B * max_mp * 10 * 8);
  A(&d.lmEdge, B * (size_t)max_mp * max_kf * 4); A(&d.freeKf, B * max_kf * 4);
  A(&d.blkOff, B * (size_t)(d.capBlk + 1) * 4);
  A(&d.lmRec, B * (size_t)max_edges * 8); A(&d.blkFirst, B * (size_t)max_kf * 4); A(&d.blkOrder, B * (size_t)d.capBlk * 4); A(&d.blkNZ, B * 4);
  A(&d.partChi, B * d.nPartE * 8); A(&d.partScale, B * d.nPartM * 8);
  A(&d.bar, B * 4);
  // launch plan (ba_run): a batch of at most numSMs windows has at most numSMs CTAs, a larger one one CTA per window
  const size_t mapLen = std::max(B, (size_t)h->numSMs);
  A(&d.ctaMap, mapLen * 4); A(&d.winCtas, B * 4);
  BaHostStage& s = h->hs;
  h->alloc_pinned(s.ctaMap, mapLen * 4); h->alloc_pinned(s.winCtas, B * 4);
  h->alloc_pinned(s.pose, B * max_kf * POSE_STRIDE * 8); h->alloc_pinned(s.pts, B * max_mp * 3 * 8);
  h->alloc_pinned(s.pidx, B * max_kf * 4); h->alloc_pinned(s.freeKf, B * max_kf * 4);
  h->alloc_pinned(s.eKf, B * max_edges * 4); h->alloc_pinned(s.eMp, B * max_edges * 4);
  h->alloc_pinned(s.mpStart, B * (max_mp + 1) * 4); h->alloc_pinned(s.kfStart, B * (max_kf + 1) * 4);
  h->alloc_pinned(s.mpEdges, B * max_edges * 4); h->alloc_pinned(s.kfEdges, B * max_edges * 4);
  h->alloc_pinned(s.eObs, B * max_edges * 12); h->alloc_pinned(s.eW, B * max_edges * 4);
  h->alloc_pinned(s.eSt, B * max_edges); h->alloc_pinned(s.eOutlier, B * max_edges);
  h->alloc_pinned(s.win, B * sizeof(BaWin)); h->alloc_pinned(s.st, B * sizeof(BaState));
  if (e == cudaSuccess && grow(h->pairRec, B * (size_t)d.capPairs * 16) != B2S_OK) e = cudaErrorMemoryAllocation;
  d.pairRec = (int4*)h->pairRec.p;
  h->smemBytes = (size_t)((CHOL_BS + 1) * CHOL_PP + (size_t)(d.ldS + 8) * CHOL_PP + 2 * d.ldS) * 8 + (size_t)(d.ldS + 8 + max_kf) * 4;
  h->smemBytes = std::max(h->smemBytes, (size_t)(BA_T / 32) * RC_TOTAL * 16  // per-warp staging of the Schur loop
                                            + (size_t)max_kf * 12 * 8);                  // + R|t table (back-substitution)
  if (e == cudaSuccess && h->smemBytes > 48 * 1024)
    e = cudaFuncSetAttribute(k_local_ba, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smemBytes);
  if (e != cudaSuccess) {
    set_error("b2s_ba_create: %s", cudaGetErrorString(e));
    b2s_ba_destroy(h);
    return B2S_ERR_CUDA;
  }
  *out = h;
  return B2S_OK;
}

extern "C" void b2s_ba_destroy(b2s_ba_solver* h) {
  if (!h) return;
  h->close();
  if (h->stream2) cudaStreamDestroy(h->stream2);
  delete h;
}
extern "C" long long b2s_ba_launch_count(const b2s_ba_solver* h) { return h ? h->launches : 0; }
extern "C" int b2s_ba_set_sm_budget(b2s_ba_solver* h, int sms) {
  if (!h || sms < 0) return B2S_ERR_BAD_ARG;
  h->smBudget = sms;
  return B2S_OK;
}

// host threads for window preparation / write-back: min(batch, 16, cores), or B2S_BA_HOST_THREADS (several ranks per box
// share the host cores)
static int ba_host_threads(int batch) {
  int cap = 16;
  if (const char* ev = getenv("B2S_BA_HOST_THREADS")) cap = std::max(1, atoi(ev));
  return std::max(1, std::min(batch, std::min(cap, (int)std::thread::hardware_concurrency())));
}

template <class F>
static void ba_for_windows(int batch, const F& fn) {  // fn(w) for every window, on ba_host_threads(batch) threads
  const int nth = ba_host_threads(batch);
  auto share = [&](int t) {
    for (int w = t; w < batch; w += nth) fn(w);
  };
  std::vector<std::thread> th;
  for (int t = 1; t < nth; t++) th.emplace_back(share, t);
  share(0);  // the calling thread takes the first share instead of waiting idle (one window: no thread is started)
  for (auto& t : th) t.join();
}

// Converter::toSE3Quat / toVector3d + CSR structure of one window, written into the pinned staging area
static int ba_prepare_window(b2s_ba_solver* h, int w, const b2s_ba_problem& P, int* nFreeOut, long long* pairBoundOut) {
  const BaPtrs& d = h->d;
  BaHostStage& s = h->hs;
  double* pose = s.pose + (size_t)w * d.capKf * POSE_STRIDE;
  int* pidx = s.pidx + (size_t)w * d.capKf;
  int* freeKf = s.freeKf + (size_t)w * d.capKf;
  int nFree = 0;
  for (int k = 0; k < P.n_kf; k++) {
    se3quat_from_Tcw(P.Tcw + (size_t)k * 16, pose + (size_t)k * POSE_STRIDE);
    if (!P.fixed[k]) {
      pidx[k] = nFree;
      freeKf[nFree++] = k;
    } else
      pidx[k] = -1;
  }
  double* pts = s.pts + (size_t)w * d.capMp * 3;
  for (size_t i = 0; i < (size_t)P.n_mp * 3; i++) pts[i] = P.points[i];  // Converter::toVector3d
  int* eKf = s.eKf + (size_t)w * d.capE;
  int* eMp = s.eMp + (size_t)w * d.capE;
  float* eObs = s.eObs + (size_t)w * d.capE * 3;
  float* eW = s.eW + (size_t)w * d.capE;
  uint8_t* eSt = s.eSt + (size_t)w * d.capE;
  int* mpStart = s.mpStart + (size_t)w * (d.capMp + 1);
  int* kfStart = s.kfStart + (size_t)w * (d.capKf + 1);
  int* mpEdges = s.mpEdges + (size_t)w * d.capE;
  int* kfEdges = s.kfEdges + (size_t)w * d.capE;
  for (int i = 0; i <= P.n_mp; i++) mpStart[i] = 0;
  for (int i = 0; i <= P.n_kf; i++) kfStart[i] = 0;
  for (int e = 0; e < P.n_edges; e++) {
    const b2s_ba_edge& E = P.edges[e];
    if (E.kf < 0 || E.kf >= P.n_kf || E.mp < 0 || E.mp >= P.n_mp) return -1;
    eKf[e] = E.kf;
    eMp[e] = E.mp;
    eObs[(size_t)e * 3] = E.obs[0]; eObs[(size_t)e * 3 + 1] = E.obs[1]; eObs[(size_t)e * 3 + 2] = E.obs[2];
    eW[e] = E.inv_sigma2;
    eSt[e] = !(E.obs[2] < 0);  // mvuRight<0 -> monocular edge (src/Optimizer.cc:794)
    mpStart[E.mp + 1]++;
    kfStart[E.kf + 1]++;
  }
  for (int i = 0; i < P.n_mp; i++) mpStart[i + 1] += mpStart[i];
  for (int i = 0; i < P.n_kf; i++) kfStart[i + 1] += kfStart[i];
  {
    std::vector<int> cm(mpStart, mpStart + P.n_mp), ck(kfStart, kfStart + P.n_kf);
    for (int e = 0; e < P.n_edges; e++) {
      mpEdges[cm[eMp[e]]++] = e;
      kfEdges[ck[eKf[e]]++] = e;
    }
  }
  // Upper bound on the window's covisibility pair records (k_pair_build): a landmark with f edges on free keyframes has
  // at most f (f + 1) / 2, because once its free edges are sorted by pose, the k-th of them pairs with at most k distinct
  // poses at or below its own (also when one keyframe observes the landmark twice).
  long long pairs = 0;
  for (int l = 0; l < P.n_mp; l++) {
    long long f = 0;
    for (int k = mpStart[l]; k < mpStart[l + 1]; k++) f += pidx[eKf[mpEdges[k]]] >= 0;
    pairs += f * (f + 1) / 2;
  }
  *nFreeOut = nFree;
  *pairBoundOut = pairs;
  return 0;
}

// Launch plan of k_local_ba: n[w] CTAs for window w, and map[] = (w << 8) | CTA index inside the window, windows in
// order; returns the number of CTAs.  One window takes min(16, numSMs) CTAs (the SM budget does not apply to it).  A batch
// that fits on the GPU deals its budget by estimated cost, because the launch ends with its slowest window.  Cost model
// (per-phase cycle counts measured on 32 windows of 23-51 free keyframes / 16-40 k edges): a serial part (single-CTA
// factorisation, control) that grows with the number of free keyframes, and a part that divides over the window's CTAs
// (linearisation, Schur pairs ~ edges x observations per point, back-substitution, error pass).  Greedy: every window
// starts with one CTA, the currently slowest gets the next.  A batch larger than numSMs runs one CTA per window.
static int ba_launch_plan(const b2s_ba_solver* h, int batch, const b2s_ba_problem* probs, const int* nFree, int* n,
                          int* map) {
  const int numSMs = h->numSMs;
  if (batch == 1) {
    n[0] = std::min(16, numSMs);
  } else if (batch > numSMs) {
    for (int w = 0; w < batch; w++) n[w] = 1;
  } else {
    const int budget = h->smBudget > 0 ? std::max(batch, std::min(numSMs, h->smBudget)) : numSMs;
    std::vector<double> ser(batch), par(batch);
    for (int w = 0; w < batch; w++) {
      const double e = probs[w].n_edges * 1e-3, obs = probs[w].n_mp > 0 ? (double)probs[w].n_edges / probs[w].n_mp : 0.0;
      ser[w] = 0.8 + 0.12 * nFree[w];
      par[w] = 4.0 * (1.65 + 0.127 * e + 0.024 * e * obs);
      n[w] = 1;
    }
    for (int used = batch; used < budget; used++) {
      int worst = -1;
      double tw = -1.0;
      for (int w = 0; w < batch; w++) {
        if (n[w] >= 16) continue;
        const double t = ser[w] + par[w] / n[w];
        if (t > tw) { tw = t; worst = w; }
      }
      if (worst < 0) break;
      n[worst]++;
    }
  }
  int total = 0;
  for (int w = 0; w < batch; w++)
    for (int k = 0; k < n[w]; k++) map[total++] = (w << 8) | k;
  return total;
}

static int ba_run(b2s_ba_solver* h, int batch, const b2s_ba_problem* probs, const volatile uint8_t* stop,
                  b2s_ba_result* res) {
  if (!h || !probs || !res || batch < 1 || batch > h->maxBatch) {
    set_error("b2s_local_ba: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  BaPtrs& d = h->d;
  BaHostStage& s = h->hs;
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->stream;
  if (stop && *stop) return B2S_ERR_ABORTED;  // src/Optimizer.cc:858-860: return without write-back
  for (int w = 0; w < batch; w++) {
    const b2s_ba_problem& P = probs[w];
    if (P.its1 < 1 || P.its2 < 0) {
      set_error("b2s_local_ba: its1 must be >= 1 and its2 >= 0");
      return B2S_ERR_BAD_ARG;
    }
    if (P.n_kf < 1 || P.n_kf > h->maxKf || P.n_mp < 0 || P.n_mp > h->maxMp || P.n_edges < 0 || P.n_edges > h->maxE ||
        P.n_local < 0 || P.n_local > P.n_kf || !P.Tcw || !P.fixed || (P.n_mp && !P.points) || (P.n_edges && !P.edges)) {
      set_error("b2s_local_ba: window %d exceeds the solver's capacity or has null arrays", w);
      return B2S_ERR_BAD_ARG;
    }
  }
  // ---- host preparation of all windows in parallel (pinned staging), then one H2D per array
  std::vector<int> nFree(batch, 0), prc(batch, 0);
  std::vector<long long> pairBound(batch, 0);
  ba_for_windows(batch, [&](int w) { prc[w] = ba_prepare_window(h, w, probs[w], &nFree[w], &pairBound[w]); });
  int maxE = 0, maxMp = 0, maxFree = 0;
  long long maxPairs = 8LL * h->maxE;  // the stride b2s_ba_create allocated for: windows bounded by it never grow the list
  for (int w = 0; w < batch; w++) {
    if (prc[w]) {
      set_error("b2s_local_ba: window %d: an edge references a vertex out of range", w);
      return B2S_ERR_BAD_ARG;
    }
    const b2s_ba_problem& P = probs[w];
    BaWin& Wn = s.win[w];
    Wn.nKf = P.n_kf; Wn.nLocal = P.n_local; Wn.nMp = P.n_mp; Wn.nEdges = P.n_edges; Wn.nFree = nFree[w];
    Wn.fx = P.fx; Wn.fy = P.fy; Wn.cx = P.cx; Wn.cy = P.cy; Wn.bf = P.bf;
    BaState& S0 = s.st[w];
    memset(&S0, 0, sizeof(S0));
    S0.active = 1;
    S0.needBuild = 1;
    S0.robust = 1;
    S0.its[0] = P.its1; S0.its[1] = P.its2;
    S0.lm.ni = 2;
    maxE = std::max(maxE, P.n_edges); maxMp = std::max(maxMp, P.n_mp); maxFree = std::max(maxFree, nFree[w]);
    maxPairs = std::max(maxPairs, pairBound[w]);
  }
  // the pair list of every window fits: grow it before anything is enqueued (a reallocation synchronises the device)
  if (maxPairs > INT_MAX) {
    set_error("b2s_local_ba: a window may have %lld covisibility pairs (at most %d)", maxPairs, INT_MAX);
    return B2S_ERR_CAPACITY;
  }
  d.capPairs = (int)maxPairs;
  {
    const int rc = grow(h->pairRec, (size_t)batch * d.capPairs * 16);
    if (rc != B2S_OK) return rc;
    d.pairRec = (int4*)h->pairRec.p;
  }
  const int nCtas = ba_launch_plan(h, batch, probs, nFree.data(), s.winCtas, s.ctaMap);
  const size_t nb = (size_t)batch;
#define UPALL(dst, src, stride, type) \
  B2S_CUDA(cudaMemcpyAsync((dst), (src), nb * (size_t)(stride) * sizeof(type), cudaMemcpyHostToDevice, st))
  UPALL(d.pose, s.pose, d.capKf * POSE_STRIDE, double);
  UPALL(d.pts, s.pts, (size_t)d.capMp * 3, double);
  UPALL(d.poseIndex, s.pidx, d.capKf, int);
  UPALL(d.freeKf, s.freeKf, d.capKf, int);
  UPALL(d.eKf, s.eKf, d.capE, int);
  UPALL(d.eMp, s.eMp, d.capE, int);
  UPALL(d.eObs, s.eObs, (size_t)d.capE * 3, float);
  UPALL(d.eW, s.eW, d.capE, float);
  UPALL(d.eStereo, s.eSt, d.capE, uint8_t);
  UPALL(d.mpStart, s.mpStart, d.capMp + 1, int);
  UPALL(d.mpEdges, s.mpEdges, d.capE, int);
  UPALL(d.kfStart, s.kfStart, d.capKf + 1, int);
  UPALL(d.kfEdges, s.kfEdges, d.capE, int);
  UPALL(d.win, s.win, 1, BaWin);
  UPALL(d.st, s.st, 1, BaState);
  UPALL(d.winCtas, s.winCtas, 1, int);
#undef UPALL
  B2S_CUDA(cudaMemcpyAsync(d.ctaMap, s.ctaMap, (size_t)nCtas * 4, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemsetAsync(d.eLevel, 0, nb * d.capE, st));
  B2S_CUDA(cudaMemsetAsync(d.chi2, 0, nb * d.capE * 8, st));
  B2S_CUDA(cudaMemsetAsync(d.lmEdge, 0xFF, nb * (size_t)d.capMp * d.capKf * 4, st));
  B2S_CUDA(cudaMemsetAsync(d.bar, 0, nb * 4, st));
  const int gE = std::max(1, div_up(maxE, 256));
  k_lm_edge<<<dim3(gE, batch), 256, 0, st>>>(d);
  const int nblk = std::max(1, maxFree * (maxFree + 1) / 2);
  k_pair_build<<<dim3(nblk, batch), 64, 0, st>>>(d, 0);
  k_pair_scan<<<div_up(batch, 64), 64, 0, st>>>(d, batch);
  k_pair_build<<<dim3(nblk, batch), 64, 0, st>>>(d, 1);
  B2S_CUDA(cudaMemsetAsync(d.blkNZ, 0, nb * 4, st));
  k_block_order<<<batch, 256, 0, st>>>(d);
  // ---- the whole LM loop of every window: persistent cooperative launches, all CTAs of a launch co-resident
  B2S_CUDA(cudaEventRecord(h->ev[0], st));
  // the attribute is per FUNCTION, not per handle: another solver handle (different capacities) may have set a smaller
  // limit since this one was created, which makes the cooperative launch fail with "too many blocks"
  if (h->smemBytes > 48 * 1024)
    B2S_CUDA(cudaFuncSetAttribute(k_local_ba, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smemBytes));
  // consecutive windows share a launch while their CTAs fit on the SMs (the plan gives no window more than numSMs)
  for (int w0 = 0, c0 = 0; w0 < batch;) {
    int grid = 0;
    for (; w0 < batch && grid + s.winCtas[w0] <= h->numSMs; w0++) grid += s.winCtas[w0];
    BaPtrs dl = d;
    dl.ctaMap = d.ctaMap + c0;
    void* args[] = {(void*)&dl};
    B2S_CUDA(cudaLaunchCooperativeKernel((const void*)k_local_ba, dim3(grid), dim3(BA_T), args, h->smemBytes, st));
    h->launches++;
    c0 += grid;
  }
  h->launches += 5;
  B2S_CUDA(cudaEventRecord(h->ev[1], st));
  // asynchronous abort (LocalMapping::InsertKeyFrame sets mbAbortBA): forward the flag while the kernel runs
  if (stop) {
    bool sent = false;
    while (cudaStreamQuery(st) == cudaErrorNotReady) {
      if (*stop && !sent) {
        const int one = 1;
        for (int w = 0; w < batch; w++)
          cudaMemcpyAsync((char*)(d.st + w) + offsetof(BaState, stop), &one, 4, cudaMemcpyHostToDevice, h->stream2);
        cudaStreamSynchronize(h->stream2);
        sent = true;
      }
      std::this_thread::yield();
    }
  }
  // write-back values (src/Optimizer.cc:961-996): SetPose(toCvMat(SE3quat)), SetWorldPos(toCvMat(estimate))
  B2S_CUDA(cudaMemcpyAsync(s.pose, d.pose, nb * d.capKf * POSE_STRIDE * 8, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaMemcpyAsync(s.pts, d.pts, nb * (size_t)d.capMp * 3 * 8, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaMemcpyAsync(s.eOutlier, d.eOutlier, nb * d.capE, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaMemcpyAsync(s.st, d.st, nb * sizeof(BaState), cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaStreamSynchronize(st));
  B2S_CUDA(cudaGetLastError());
  cudaEventElapsedTime(&h->lastMs, h->ev[0], h->ev[1]);
  h->lastTrials = 0;
  for (int w = 0; w < batch; w++) h->lastTrials += s.st[w].lm.nTrials;
  for (int w = 0; w < batch; w++)
    if (s.st[w].finishedRound0) {
      set_error("b2s_local_ba: window %d: LM kernel barrier timed out (CTAs not co-resident?)", w);
      return B2S_ERR_CUDA;
    }
  for (int w = 0; w < batch; w++)
    if (s.st[w].pairsOverflow) {
      set_error("b2s_local_ba: window %d: covisibility pair list exceeds its capacity of %d", w, d.capPairs);
      return B2S_ERR_CAPACITY;
    }
  // round 2 skipped (its2 == 0): the optimiser still ends with round 2's active set, the edges the final test keeps
  // without robust kernels, so chi2_final is their plain chi2 (as when round 2 runs, or has no edge left: k_local_ba)
  for (int w = 0; w < batch; w++)
    if (s.st[w].doOutlier == 3) {
      std::vector<double> c2((size_t)probs[w].n_edges);
      B2S_CUDA(cudaMemcpy(c2.data(), d.chi2 + (size_t)w * d.capE, c2.size() * 8, cudaMemcpyDeviceToHost));
      double chi = 0;
      for (size_t e = 0; e < c2.size(); e++)
        if (!s.eOutlier[(size_t)w * d.capE + e]) chi += c2[e];
      s.st[w].chi2Final = chi;
    }
  ba_for_windows(batch, [&](int w) {
    const b2s_ba_problem& P = probs[w];
    b2s_ba_result& R = res[w];
    const double* pose = s.pose + (size_t)w * d.capKf * POSE_STRIDE;
    const double* pts = s.pts + (size_t)w * d.capMp * 3;
    if (R.Tcw_out)
      for (int k = 0; k < P.n_local; k++) se3quat_to_Tcw(pose + (size_t)k * POSE_STRIDE, R.Tcw_out + (size_t)k * 16);
    if (R.points_out)
      for (size_t i = 0; i < (size_t)P.n_mp * 3; i++) R.points_out[i] = (float)pts[i];
    if (R.edge_outlier && P.n_edges) memcpy(R.edge_outlier, s.eOutlier + (size_t)w * d.capE, P.n_edges);
    R.chi2_final = s.st[w].chi2Final;
    R.n_trials = s.st[w].lm.nTrials;
    if (R.trace) {
      const int n = std::min(s.st[w].lm.nTrials, 255);
      for (int i = 0; i < n; i++) R.trace[i] = s.st[w].trace[i];
      R.trace[n] = -1;
    }
  });
  return B2S_OK;
}

extern "C" float b2s_ba_last_kernel_ms(const b2s_ba_solver* h, long long* lm_trials) {
  if (!h) return 0.f;
  if (lm_trials) *lm_trials = h->lastTrials;
  return h->lastMs;
}

extern "C" int b2s_local_ba(b2s_ba_solver* h, const b2s_ba_problem* p, const volatile uint8_t* stop, b2s_ba_result* r) {
  return ba_run(h, 1, p, stop, r);
}
extern "C" int b2s_local_ba_batch(b2s_ba_solver* h, int batch, const b2s_ba_problem* p, b2s_ba_result* r) {
  return ba_run(h, batch, p, nullptr, r);
}


// ================================================================================================ PoseOptimization host side
extern "C" int b2s_pose_optimization_batch(b2s_ba_solver* h, int batch, const b2s_pose_problem* probs, b2s_pose_result* res) {
  if (!h || !probs || !res || batch < 1) {
    set_error("b2s_pose_optimization_batch: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->stream;
  // pack the edges (features with a MapPoint, ascending feature index = g2o insertion order, :411-487)
  std::vector<PoFrame> frames(batch);
  std::vector<double> poseInit((size_t)batch * POSE_STRIDE);
  size_t totalE = 0;
  for (int f = 0; f < batch; f++) {
    const b2s_pose_problem& P = probs[f];
    if (P.n < 0 || !P.Tcw || !res[f].Tcw_out || (P.n && (!P.has_mp || !P.Xw || !P.kpx || !P.kpy || !P.uright ||
                                                         !P.inv_sigma2 || !res[f].outlier))) {
      set_error("b2s_pose_optimization_batch: frame %d has null arrays", f);
      return B2S_ERR_BAD_ARG;
    }
    int ne = 0;
    for (int i = 0; i < P.n; i++) ne += P.has_mp[i] != 0;
    frames[f].nEdges = ne;
    frames[f].edgeOff = (int)totalE;
    frames[f].fx = P.fx; frames[f].fy = P.fy; frames[f].cx = P.cx; frames[f].cy = P.cy; frames[f].bf = P.bf;
    totalE += ne;
    se3quat_from_Tcw(P.Tcw, &poseInit[(size_t)f * POSE_STRIDE]);
  }
  std::vector<float> Xw(totalE * 3 + 3), obs(totalE * 3 + 3), invS(totalE + 1);
  std::vector<int> featOf(totalE + 1);
  {
    size_t e = 0;
    for (int f = 0; f < batch; f++) {
      const b2s_pose_problem& P = probs[f];
      for (int i = 0; i < P.n; i++) {
        if (!P.has_mp[i]) continue;
        Xw[e * 3] = P.Xw[i * 3]; Xw[e * 3 + 1] = P.Xw[i * 3 + 1]; Xw[e * 3 + 2] = P.Xw[i * 3 + 2];
        obs[e * 3] = P.kpx[i]; obs[e * 3 + 1] = P.kpy[i]; obs[e * 3 + 2] = P.uright[i];
        invS[e] = P.inv_sigma2[i];
        featOf[e] = i;
        e++;
      }
    }
  }
  // a buffer short of this call's need grows to twice it (at least 4096 edges, 16 frames)
  const size_t nE = totalE + 1, nF = batch, capE = std::max<size_t>(nE, 4096) * 2, capF = std::max<size_t>(nF, 16) * 2;
  int rc = B2S_OK;
  auto G = [&](DevBuf& b, size_t n, size_t cap, size_t elem) {
    if (rc == B2S_OK && b.bytes < n * elem) rc = grow(b, cap * elem);
  };
  G(h->poFrames, nF, capF, sizeof(PoFrame)); G(h->poPoseInit, nF, capF, POSE_STRIDE * 8);
  G(h->poPoseOut, nF, capF, POSE_STRIDE * 8);
  G(h->poErr, nE, capE, 24); G(h->poChi2, nE, capE, 8); G(h->poXw, nE, capE, 12); G(h->poObs, nE, capE, 12);
  G(h->poInvS, nE, capE, 4); G(h->poLevel, nE, capE, 1); G(h->poOutlier, nE, capE, 1);
  G(h->poNInl, nF, capF, 4); G(h->poNTr, nF, capF, 4); G(h->poTrace, nF, capF, 256 * 4);
  if (rc != B2S_OK) {
    set_error("b2s_pose_optimization_batch: %s", g_last_error.c_str());
    return rc;
  }
  PoPtrs pp;
  pp.frames = (PoFrame*)h->poFrames.p; pp.poseInit = (double*)h->poPoseInit.p; pp.Xw = (float*)h->poXw.p;
  pp.obs = (float*)h->poObs.p; pp.invSigma2 = (float*)h->poInvS.p; pp.err = (double*)h->poErr.p;
  pp.chi2 = (double*)h->poChi2.p; pp.level = (uint8_t*)h->poLevel.p; pp.outlier = (uint8_t*)h->poOutlier.p;
  pp.poseOut = (double*)h->poPoseOut.p; pp.nInliers = (int*)h->poNInl.p; pp.nTrials = (int*)h->poNTr.p;
  pp.trace = (int*)h->poTrace.p;
  B2S_CUDA(cudaMemcpyAsync(h->poFrames.p, frames.data(), batch * sizeof(PoFrame), cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->poPoseInit.p, poseInit.data(), (size_t)batch * POSE_STRIDE * 8, cudaMemcpyHostToDevice, st));
  if (totalE) {
    B2S_CUDA(cudaMemcpyAsync(h->poXw.p, Xw.data(), totalE * 12, cudaMemcpyHostToDevice, st));
    B2S_CUDA(cudaMemcpyAsync(h->poObs.p, obs.data(), totalE * 12, cudaMemcpyHostToDevice, st));
    B2S_CUDA(cudaMemcpyAsync(h->poInvS.p, invS.data(), totalE * 4, cudaMemcpyHostToDevice, st));
  }
  k_pose_opt<<<batch, PO_T, 0, st>>>(pp);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  std::vector<double> poseOut((size_t)batch * POSE_STRIDE);
  std::vector<uint8_t> outl(totalE + 1);
  std::vector<int> nInl(batch), nTr(batch), trace((size_t)batch * 256);
  B2S_CUDA(cudaMemcpyAsync(poseOut.data(), pp.poseOut, (size_t)batch * POSE_STRIDE * 8, cudaMemcpyDeviceToHost, st));
  if (totalE) B2S_CUDA(cudaMemcpyAsync(outl.data(), pp.outlier, totalE, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaMemcpyAsync(nInl.data(), pp.nInliers, (size_t)batch * 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaMemcpyAsync(nTr.data(), pp.nTrials, (size_t)batch * 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaMemcpyAsync(trace.data(), pp.trace, (size_t)batch * 256 * 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaStreamSynchronize(st));
  for (int f = 0; f < batch; f++) {
    const b2s_pose_problem& P = probs[f];
    b2s_pose_result& R = res[f];
    for (int i = 0; i < P.n; i++) R.outlier[i] = 0;
    for (int e = 0; e < frames[f].nEdges; e++) R.outlier[featOf[frames[f].edgeOff + e]] = outl[frames[f].edgeOff + e];
    R.n_inliers = nInl[f];
    R.n_trials = nTr[f];
    if (frames[f].nEdges < 3) {
      for (int k = 0; k < 16; k++) R.Tcw_out[k] = P.Tcw[k];  // untouched (:492-493)
    } else {
      se3quat_to_Tcw(&poseOut[(size_t)f * POSE_STRIDE], R.Tcw_out);
    }
    if (R.trace) {
      const int n = std::min(nTr[f], 255);
      for (int i = 0; i < n; i++) R.trace[i] = trace[(size_t)f * 256 + i];
      R.trace[n] = -1;
    }
  }
  return B2S_OK;
}

extern "C" int b2s_pose_optimization(b2s_ba_solver* h, const b2s_pose_problem* p, b2s_pose_result* r) {
  return b2s_pose_optimization_batch(h, 1, p, r);
}
