// chol.cuh — the FP64 block-envelope Cholesky and the deterministic sums shared by the global bundle adjustment
// (gba.cu, 6-scalar pose blocks) and the essential graph (essential.cu, 7-scalar Sim3 blocks).
//
// The symmetric system is stored as its lower block envelope cut into 64 x 64 tiles: tile row I holds the tiles of
// columns [envT[I], I], contiguous from tileOff[I].  Skyline fill-in stays inside the envelope, so tiles left of a row's
// envelope are never touched.  The factorisation is tiled right-looking: the diagonal tile is factorised and inverted by
// one CTA, the panel (L_IK = A_IK Linv_KK^T) and the trailing update (A_IJ -= L_IK L_JK^T) run on many CTAs with
// mma.sync.m8n8k4.f64 (DMMA).  Panel and trailing launches cover only the tile rows whose envelope reaches the column
// (panel_rows): a pose graph is a narrow band plus a few long rows, so most of the dense triangle is empty.
// A non-positive or non-finite pivot sets *fail; every later kernel of the solve then returns at once.
// Everything here is static: each .cu that includes it gets its own copy of the kernels.
#pragma once
#include <algorithm>
#include <vector>

#include "common.cuh"

namespace b2s {
namespace chol {

constexpr int TS = 64;           // tile (scalar rows / columns)
constexpr int TT = TS * TS;      // doubles per stored tile (row-major, stride TS)
constexpr int LDT = 68;          // shared-memory row stride of a tile: the 8 rows of a DMMA fragment spread over the banks
constexpr int TILE_SMEM = TS * LDT * 8;
constexpr int RED_BLOCKS = 256;  // fixed grid of the deterministic sums

struct TileSys {
  int np;                    // scalar rows; rows of the last tile past np are padded with the identity
  const int* envT;           // per tile row: first tile column of its envelope
  const long long* tileOff;  // per tile row: index of tile (I, envT[I])
  double* tiles;
  double* linv;              // nT x TT: inverse of every diagonal factor
  double* rhs;               // npPad: right-hand side, consumed by the forward substitution
  double* ybuf;              // npPad
  double* x;                 // npPad: the solution
  int* fail;
};

// tile (I, K) of any struct with the TileSys envelope members
template <class S>
__device__ __forceinline__ double* tile_ptr(const S& a, int I, int K) {
  return a.tiles + (size_t)(a.tileOff[I] + (K - a.envT[I])) * TT;
}

// ================================================================================================ deterministic sums
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// part[blockIdx.x] = sum of v[chunk of this block] (fixed chunking, fixed tree); op 0 = sum, 1 = max |v|
template <int OP>
static __global__ void __launch_bounds__(256) k_reduce_part(const double* __restrict__ v, long long n, double* part) {
  __shared__ double sm[8];
  const long long chunk = (n + gridDim.x - 1) / gridDim.x;
  const long long beg = chunk * blockIdx.x, end = min(n, beg + chunk);
  double s = 0;
  for (long long i = beg + threadIdx.x; i < end; i += 256) s = OP == 0 ? s + v[i] : fmax(s, fabs(v[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double t = __shfl_xor_sync(0xffffffffu, s, o);
    s = OP == 0 ? s + t : fmax(s, t);
  }
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double r = sm[0];
    for (int i = 1; i < 8; i++) r = OP == 0 ? r + sm[i] : fmax(r, sm[i]);
    part[blockIdx.x] = r;
  }
}
template <int OP>
static __global__ void __launch_bounds__(256) k_reduce_final(const double* __restrict__ part, int n, double* out) {
  __shared__ double sm[8];
  double s = threadIdx.x < n ? part[threadIdx.x] : 0.0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double t = __shfl_xor_sync(0xffffffffu, s, o);
    s = OP == 0 ? s + t : fmax(s, t);
  }
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double r = sm[0];
    for (int i = 1; i < 8; i++) r = OP == 0 ? r + sm[i] : fmax(r, sm[i]);
    *out = r;
  }
}
// deterministic sum (OP 0) or max |.| (OP 1) of v[0, n) into *out (device); part holds RED_BLOCKS doubles
template <int OP>
static void reduce(const double* v, long long n, double* part, double* out, cudaStream_t s) {
  k_reduce_part<OP><<<RED_BLOCKS, 256, 0, s>>>(v, n, part);
  k_reduce_final<OP><<<1, 256, 0, s>>>(part, RED_BLOCKS, out);
}

// ================================================================================================ tiled Cholesky
__device__ __forceinline__ void load_tile(double* s, const double* g) {
  for (int k = threadIdx.x; k < TT; k += blockDim.x) s[(k / TS) * LDT + (k % TS)] = g[k];
}
// acc = X Y^T for the 8 output rows of this warp (rows 8 w + g, columns 8 n + 2 t + {0, 1}) on the DMMA pipe
__device__ __forceinline__ void gemm_nt(const double* __restrict__ X, const double* __restrict__ Y, double (&acc)[8][2]) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int n = 0; n < 8; n++) acc[n][0] = acc[n][1] = 0.0;
#pragma unroll 4
  for (int s = 0; s < TS / 4; s++) {
    const double av = X[(8 * w + g) * LDT + 4 * s + t];
#pragma unroll
    for (int n = 0; n < 8; n++) {
      const double bv = Y[(8 * n + g) * LDT + 4 * s + t];
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                   : "+d"(acc[n][0]), "+d"(acc[n][1])
                   : "d"(av), "d"(bv));
    }
  }
}

// diagonal tile K: Cholesky in shared memory (right-looking), then Linv = L^-1 (lower) to linv[K]
static __global__ void __launch_bounds__(256) k_potrf(TileSys a, int K) {
  extern __shared__ double sm[];
  double* sA = sm;
  double* sX = sm + TS * LDT;
  if (*(volatile int*)a.fail) return;
  const int tid = threadIdx.x;
  const double* g = tile_ptr(a, K, K);
  for (int k = tid; k < TT; k += 256) {
    const int r = k / TS, c = k % TS;
    const bool pad = K * TS + r >= a.np || K * TS + c >= a.np;  // padding rows / columns: identity
    sA[r * LDT + c] = pad ? (r == c ? 1.0 : 0.0) : g[k];
    sX[r * LDT + c] = 0.0;
  }
  for (int j = 0; j < TS; j++) {
    __syncthreads();
    const double d = sA[j * LDT + j];
    if (!(d > 0.0) || !isfinite(d)) {
      if (tid == 0) *a.fail = 1;
      return;
    }
    const double piv = sqrt(d);
    __syncthreads();
    if (tid == 0) sA[j * LDT + j] = piv;
    for (int i = j + 1 + tid; i < TS; i += 256) sA[i * LDT + j] /= piv;
    __syncthreads();
    for (int i = j + 1 + (tid >> 4); i < TS; i += 16) {
      const double lij = sA[i * LDT + j];
      for (int c = j + 1 + (tid & 15); c <= i; c += 16) sA[i * LDT + c] -= lij * sA[c * LDT + j];
    }
  }
  __syncthreads();
  // Linv column c by a group of 4 lanes: X[r][c] = (delta_rc - sum_{k=c}^{r-1} L[r][k] X[k][c]) / L[r][r]
  {
    const int c = tid >> 2, q = tid & 3;
    const unsigned mask = 0xFu << (threadIdx.x & 28);
    for (int r = c; r < TS; r++) {
      double s = 0;
      for (int k = c + q; k < r; k += 4) s += sA[r * LDT + k] * sX[k * LDT + c];
      s += __shfl_xor_sync(mask, s, 1);
      s += __shfl_xor_sync(mask, s, 2);
      if (q == 0) sX[r * LDT + c] = ((r == c ? 1.0 : 0.0) - s) / sA[r * LDT + r];
      __syncwarp(mask);
    }
  }
  __syncthreads();
  double* out = a.linv + (size_t)K * TT;
  for (int k = tid; k < TT; k += 256) out[k] = sX[(k / TS) * LDT + (k % TS)];
}

// panel: L_IK = A_IK Linv_KK^T for I = rows[blockIdx.x] (the tile rows below K whose envelope reaches column K)
static __global__ void __launch_bounds__(256) k_trsm(TileSys a, const int* __restrict__ rows, int K) {
  extern __shared__ double sm[];
  if (*(volatile int*)a.fail) return;
  const int I = rows[blockIdx.x];
  double* sA = sm;
  double* sL = sm + TS * LDT;
  double* g = tile_ptr(a, I, K);
  load_tile(sA, g);
  load_tile(sL, a.linv + (size_t)K * TT);
  __syncthreads();
  double acc[8][2];
  gemm_nt(sA, sL, acc);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, gi = lane >> 2, t = lane & 3;
#pragma unroll
  for (int n = 0; n < 8; n++) {
    const int r = 8 * w + gi, c = 8 * n + 2 * t;
    g[r * TS + c] = acc[n][0];
    g[r * TS + c + 1] = acc[n][1];
  }
}

// trailing update: A_IJ -= L_IK L_JK^T for every pair I >= J of the same row list (block = lower-triangle pair index)
static __global__ void __launch_bounds__(256) k_syrk(TileSys a, const int* __restrict__ rows, int K) {
  extern __shared__ double sm[];
  if (*(volatile int*)a.fail) return;
  const long long idx = blockIdx.x;
  long long ii = (long long)((sqrt(8.0 * (double)idx + 1.0) - 1.0) * 0.5);
  while (ii * (ii + 1) / 2 > idx) ii--;
  while ((ii + 1) * (ii + 2) / 2 <= idx) ii++;
  const int I = rows[ii], J = rows[idx - ii * (ii + 1) / 2];
  double* sI = sm;
  double* sJ = sm + TS * LDT;
  load_tile(sI, tile_ptr(a, I, K));
  load_tile(sJ, tile_ptr(a, J, K));
  __syncthreads();
  double acc[8][2];
  gemm_nt(sI, sJ, acc);
  double* g = tile_ptr(a, I, J);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, gi = lane >> 2, t = lane & 3;
#pragma unroll
  for (int n = 0; n < 8; n++) {
    const int r = 8 * w + gi, c = 8 * n + 2 * t;
    g[r * TS + c] -= acc[n][0];
    g[r * TS + c + 1] -= acc[n][1];
  }
}

// forward substitution step K: y_K = Linv_KK r_K (block 0 stores it), r_I -= L_IK y_K (block I - K)
static __global__ void __launch_bounds__(TS) k_fwd(TileSys a, int K) {
  __shared__ double y[TS];
  if (*(volatile int*)a.fail) return;
  const int t = threadIdx.x;
  const double* Li = a.linv + (size_t)K * TT + (size_t)t * TS;
  const double* r = a.rhs + (size_t)K * TS;
  double s = 0;
  for (int k = 0; k <= t; k++) s += Li[k] * r[k];
  y[t] = s;
  __syncthreads();
  if (blockIdx.x == 0) {
    a.ybuf[(size_t)K * TS + t] = s;
    return;
  }
  const int I = K + blockIdx.x;
  if (a.envT[I] > K) return;
  const double* L = tile_ptr(a, I, K) + (size_t)t * TS;
  double u = 0;
  for (int k = 0; k < TS; k++) u += L[k] * y[k];
  a.rhs[(size_t)I * TS + t] -= u;
}

// backward substitution step I: x_I = Linv_II^T z_I (block 0 stores it), z_K -= L_IK^T x_I for K in [envT[I], I)
static __global__ void __launch_bounds__(TS) k_bwd(TileSys a, int I) {
  __shared__ double x[TS];
  if (*(volatile int*)a.fail) return;
  const int t = threadIdx.x;
  const double* Li = a.linv + (size_t)I * TT;
  const double* z = a.ybuf + (size_t)I * TS;
  double s = 0;
  for (int k = t; k < TS; k++) s += Li[(size_t)k * TS + t] * z[k];
  x[t] = s;
  __syncthreads();
  if (blockIdx.x == 0) {
    a.x[(size_t)I * TS + t] = s;
    return;
  }
  const int K = a.envT[I] + blockIdx.x - 1;
  const double* L = tile_ptr(a, I, K);
  double u = 0;
  for (int r = 0; r < TS; r++) u += L[(size_t)r * TS + t] * x[r];
  a.ybuf[(size_t)K * TS + t] -= u;
}

// ================================================================================================ host side
// The host-driven LM loop's synchronisations.  busyMs adds up the stream segments between them (CUDA events): the device
// time of a solve, without the host's decisions in between.  start() opens the first segment.
struct HostSync {
  cudaStream_t s;
  cudaEvent_t* ev;        // ev[0]: start of the open segment, ev[1]: its end
  double* hScal;          // pinned host copy of the solver's scalars
  const double* scal;     // device scalars (chi2, scale / max |diag|)
  int* hFail;             // pinned host copy of the factorisation's fail flag
  const int* fail;
  float busyMs;

  int start() {
    B2S_CUDA(cudaEventRecord(ev[0], s));
    return B2S_OK;
  }
  // wait for the stream and close the segment
  int stream() {
    B2S_CUDA(cudaEventRecord(ev[1], s));
    B2S_CUDA(cudaStreamSynchronize(s));
    float ms = 0.f;
    B2S_CUDA(cudaEventElapsedTime(&ms, ev[0], ev[1]));
    busyMs += ms;
    B2S_CUDA(cudaEventRecord(ev[0], s));
    return B2S_OK;
  }
  // the first n scalars and the fail flag to the host, then stream()
  int scalars(int n) {
    B2S_CUDA(cudaMemcpyAsync(hScal, scal, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
    B2S_CUDA(cudaMemcpyAsync(hFail, fail, 4, cudaMemcpyDeviceToHost, s));
    return stream();
  }
};

// the kernels above need 2 tiles of dynamic shared memory
static cudaError_t set_smem_limits() {
  cudaError_t e = cudaFuncSetAttribute(k_potrf, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * TILE_SMEM);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_trsm, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * TILE_SMEM);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_syrk, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * TILE_SMEM);
  return e;
}

// The tile envelope of a system of nBlk blocks of B scalars whose block row i starts at block column envBlk[i]: the first
// tile column any scalar row of a tile row reaches, the tile offsets (nT + 1) and the panel row lists
// (rows[rowOff[K], rowOff[K + 1]): the tile rows I > K with envT[I] <= K, ascending).  Returns the number of tiles.
static long long tile_envelope(const std::vector<int>& envBlk, int nBlk, int B, std::vector<int>& envT,
                               std::vector<long long>& off, std::vector<int>& rowOff, std::vector<int>& rows) {
  const int nT = (nBlk * B + TS - 1) / TS;
  envT.assign((size_t)nT, 0);
  off.assign((size_t)nT + 1, 0);
  for (int T = 0; T < nT; T++) {
    int e0 = T;
    for (int i = T * TS / B; i < nBlk && i * B < (T + 1) * TS; i++) e0 = std::min(e0, envBlk[(size_t)i] * B / TS);
    envT[(size_t)T] = e0;
    off[(size_t)T + 1] = off[(size_t)T] + (T - e0 + 1);
  }
  std::vector<int> cnt((size_t)nT + 1, 0);
  for (int I = 0; I < nT; I++)
    for (int K = envT[(size_t)I]; K < I; K++) cnt[(size_t)K + 1]++;
  rowOff.assign((size_t)nT + 1, 0);
  for (int K = 0; K < nT; K++) rowOff[(size_t)K + 1] = rowOff[(size_t)K] + cnt[(size_t)K + 1];
  rows.assign((size_t)rowOff[(size_t)nT], 0);
  std::vector<int> fill(rowOff.begin(), rowOff.end() - 1);
  for (int I = 0; I < nT; I++)
    for (int K = envT[(size_t)I]; K < I; K++) rows[(size_t)fill[(size_t)K]++] = I;
  return off[(size_t)nT];
}

// Factorise the tiles in place and solve for a.x from a.rhs (a.rhs and a.ybuf are overwritten).  envT / rowOff are the
// host copies of tile_envelope's output; dRows is its row list on the device.
static void factor_solve(const TileSys& a, int nT, const std::vector<int>& envT, const std::vector<int>& rowOff,
                         const int* dRows, cudaStream_t s) {
  for (int K = 0; K < nT; K++) {
    k_potrf<<<1, 256, 2 * TILE_SMEM, s>>>(a, K);
    const int m = rowOff[(size_t)K + 1] - rowOff[(size_t)K];
    if (m > 0) {
      k_trsm<<<m, 256, 2 * TILE_SMEM, s>>>(a, dRows + rowOff[(size_t)K], K);
      k_syrk<<<(unsigned)((long long)m * (m + 1) / 2), 256, 2 * TILE_SMEM, s>>>(a, dRows + rowOff[(size_t)K], K);
    }
  }
  for (int K = 0; K < nT; K++) k_fwd<<<nT - K, TS, 0, s>>>(a, K);
  for (int I = nT - 1; I >= 0; I--) k_bwd<<<1 + I - envT[(size_t)I], TS, 0, s>>>(a, I);
}

}  // namespace chol
}  // namespace b2s
