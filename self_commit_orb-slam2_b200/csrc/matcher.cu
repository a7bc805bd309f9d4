// matcher.cu — H100 (sm_90a) ORBmatcher: 256-bit Hamming as warp POPC reductions over 32-byte descriptors.
//
//   SearchByBoW            /root/reference/src/ORBmatcher.cc:230-382 (KF,F) and :656-799 (KF,KF)
//   SearchByProjection     :1569-1728 (CurrentFrame, LastFrame) + Frame grid src/Frame.cc:461-491, 741-877
//   DescriptorDistance     :1913-1933
//
// The reference matchers are greedy and order dependent (a frame feature matched by an earlier keyframe feature is
// skipped by later ones, :288).  Distances are the parallel part: one warp per query row scans its candidates in the
// reference's iteration order and keeps the K best by (distance, order) — removing already-matched candidates from
// such a sorted list preserves both the first-minimum tie rule and the second-best value, so the order-dependent
// part becomes a cheap resolver walking K-entry lists (with an exact full rescan when a list runs dry).
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "distinctive.cuh"
#include "matcher.cuh"

namespace b2s {

constexpr int TOPK = 8;
constexpr int HISTO = 30;             // HISTO_LENGTH, src/ORBmatcher.cc:51
constexpr int GRID_COLS = 64, GRID_ROWS = 48;  // include/Frame.h:55,60
constexpr uint32_t EMPTY = 0xFFFFFFFFu;

struct MatchParams {
  int thLow;       // TH_LOW / TH_HIGH depending on the matcher
  float nnratio;
  int strictLt;
  int checkOri;
};

__device__ __forceinline__ u256 ld_desc(const uint8_t* base, int i) { return ld_u256(base + (size_t)i * 32); }
// 4-byte aligned descriptor (embedded in a query record)
__device__ __forceinline__ u256 ld_desc_w(const uint8_t* p) {
  u256 r;
  const uint32_t* w = reinterpret_cast<const uint32_t*>(p);
#pragma unroll
  for (int k = 0; k < 8; k++) r.w[k] = w[k];
  return r;
}

// keep the K smallest keys of a stream (ascending, registers)
__device__ __forceinline__ void topk_insert(uint32_t (&t)[TOPK], uint32_t key) {
  if (key >= t[TOPK - 1]) return;
  t[TOPK - 1] = key;
#pragma unroll
  for (int k = TOPK - 1; k > 0; k--) {
    if (t[k] < t[k - 1]) {
      const uint32_t tmp = t[k];
      t[k] = t[k - 1];
      t[k - 1] = tmp;
    }
  }
}

// merge the 32 per-lane sorted lists into the warp's global K smallest (result broadcast to all lanes)
__device__ __forceinline__ void topk_warp_merge(uint32_t (&t)[TOPK], uint32_t (&out)[TOPK]) {
  int head = 0;
#pragma unroll
  for (int k = 0; k < TOPK; k++) {
    uint32_t mine = EMPTY;
#pragma unroll
    for (int q = 0; q < TOPK; q++)
      if (q == head) mine = t[q];
    uint32_t m = mine;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
    out[k] = m;
    if (m != EMPTY && mine == m) head++;  // keys are unique (they embed the candidate order)
  }
}

__device__ __forceinline__ int rot_bin(float angA, float angB) {
  const float factor = HISTO / 360.0f;
  float rot = __fsub_rn(angA, angB);
  if (rot < 0.0f) rot = __fadd_rn(rot, 360.0f);
  int bin = (int)roundf(__fmul_rn(rot, factor));  // C round(): half away from zero
  if (bin == HISTO) bin = 0;
  return bin;
}

// ------------------------------------------------------------------------------------------------
// order[]: indices sorted by (key, index) — rank by counting (n <= a few thousand)
// ------------------------------------------------------------------------------------------------
__global__ void k_rank_by_key(const int32_t* __restrict__ keyBase, const int32_t* __restrict__ nArr, int cap,
                              int32_t* __restrict__ orderBase) {
  const int pair = blockIdx.y;
  const int n = min(nArr[pair], cap);  // counts come from device memory (another rank's record, a caller's array): never past the slice
  const int32_t* key = keyBase + (size_t)pair * cap;
  int32_t* order = orderBase + (size_t)pair * cap;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int ki = key[i];
  int r = 0;
  for (int k = 0; k < n; k++) {
    const int kk = key[k];
    r += (kk < ki) || (kk == ki && k < i);
  }
  order[r] = i;
}

// ------------------------------------------------------------------------------------------------
// SearchByBoW, stage 1: per keyframe-side row, K best frame-side candidates of the same vocabulary node
// key = dist<<16 | j   (j ascending == the reference's candidate iteration order inside a node)
// Only candidates closer than `cut` are listed and counted (bow_distance_cut below): no other candidate can change a
// decision of the resolver.
// The distances run on the integer tensor pipe.  popc(a ^ b) = popc(a) + popc(b) - 2 popc(a & b), and popc(a & b) of two
// 256-bit strings is the dot product of their bits written as 0 / 1 bytes: a 16 x 8 tile of distances is eight
// mma.sync.m16n8k32.u8 (IMMA.16832; bench.py reports the issue rate measured on the device, b2s_measure_peaks slot 5).
// A CTA owns 128 keyframe-side rows (4 warps x 32 rows, bit-expanded A fragments live in registers for the whole sweep) and
// walks the frame side in stages of 64 columns expanded into shared memory.  Because a dot product does not care about the
// order of its terms, the 256 byte positions are laid out in FRAGMENT order: lane (g, t) of k-step s owns the eight bits of
// descriptor byte 4 s + t, on both sides, so a B fragment is one conflict-free LDS.64 (column pitch 288 B).
// Selection: lane (g, t) sees rows {g, g+8, g+16, g+24} x columns {2t, 2t+1} of every 8-column block and keeps a K-list
// per row; keys are unique (column index in the low half), so the K smallest of the four lanes' lists are exactly the K
// smallest of the row.  The lists are merged once at the end: each row's K-list is written in ascending key order, i.e.
// by distance and then by frame-side index, with EMPTY filling the slots past the row's candidates.
// ------------------------------------------------------------------------------------------------
constexpr int BI_ROWS = 128, BI_COLS = 64, BI_PITCH = 288;
__device__ __forceinline__ void expand_byte(uint32_t x, uint32_t& lo, uint32_t& hi) {  // bit i of x -> byte i (0 / 1)
  lo = ((x & 0xFu) * 0x00204081u) & 0x01010101u;
  hi = (((x >> 4) & 0xFu) * 0x00204081u) & 0x01010101u;
}
__device__ __forceinline__ void imma_16832(int (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__global__ void __launch_bounds__(128, 3) k_bow_topk_imma(const uint8_t* __restrict__ descA, const int32_t* __restrict__ nodeA,
                                                       const uint8_t* __restrict__ validA, const int32_t* __restrict__ nAarr,
                                                       int capA, const uint8_t* __restrict__ descB,
                                                       const int32_t* __restrict__ nodeB, const uint8_t* __restrict__ validB,
                                                       const int32_t* __restrict__ nBarr, int capB, int cut,
                                                       uint32_t* __restrict__ topk, int32_t* __restrict__ candCnt) {
  __shared__ __align__(16) uint8_t sB[BI_COLS * BI_PITCH];
  __shared__ __align__(8) int32_t sNode[BI_COLS];
  // (popc(b) << 16 | column index); a column that is no candidate at all carries 0x7000 in the distance field, which no
  // popc(a) - 2 popc(a & b) in [-512, 256] can bring below the cut
  __shared__ __align__(8) uint32_t sBase[BI_COLS];
  const uint32_t cutKey = (uint32_t)cut << 16;
  const int pair = blockIdx.y;
  const int nA = min(nAarr[pair], capA), nB = min(nBarr[pair], capB);
  const int row0 = blockIdx.x * BI_ROWS;
  if (row0 >= nA) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
  const size_t oa = (size_t)pair * capA, ob = (size_t)pair * capB;
  // ---- A side: four rows per lane, expanded fragments for the 8 k-steps of both 16-row tiles
  uint32_t aF[2][8][4];
  int rowIdx[4], rowNode[4];
  uint32_t rowPa16[4];  // popc(a) << 16
  bool rowOk[4];
#pragma unroll
  for (int q = 0; q < 4; q++) {
    const int i = row0 + warp * 32 + g + 8 * q;
    rowIdx[q] = i;
    rowOk[q] = (i < nA) && (!validA || validA[oa + i]);
    u256 da;
    if (rowOk[q]) {
      da = ld_desc(descA + oa * 32, i);
      rowNode[q] = nodeA[oa + i];
    } else {
#pragma unroll
      for (int k = 0; k < 8; k++) da.w[k] = 0;
      rowNode[q] = -1;
    }
    int pa = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) pa += __popc(da.w[k]);
    rowPa16[q] = (uint32_t)pa << 16;
#pragma unroll
    for (int sx = 0; sx < 8; sx++) {
      uint32_t lo, hi;
      expand_byte((da.w[sx] >> (8 * t)) & 0xFFu, lo, hi);
      // rows g (q = 0, 2) fill a0 / a2, rows g + 8 (q = 1, 3) fill a1 / a3 of tile q >> 1
      aF[q >> 1][sx][q & 1] = lo;
      aF[q >> 1][sx][2 + (q & 1)] = hi;
    }
  }
  uint32_t kl[4][TOPK];
  int cnt[4] = {0, 0, 0, 0};
#pragma unroll
  for (int q = 0; q < 4; q++)
#pragma unroll
    for (int k = 0; k < TOPK; k++) kl[q][k] = EMPTY;
  for (int j0 = 0; j0 < nB; j0 += BI_COLS) {
    __syncthreads();
    for (int cbase = 0; cbase < BI_COLS; cbase += 64) {  // stage: thread (column, half) expands 16 bytes into 128
      const int col = cbase + (tid >> 1), half = tid & 1, j = j0 + col;
      uint4 w = make_uint4(0u, 0u, 0u, 0u);
      bool ok = j < nB;
      if (ok) {
        w = *reinterpret_cast<const uint4*>(descB + (ob + j) * 32 + half * 16);
        ok = !validB || validB[ob + j];
      }
      const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
      uint8_t* dst = sB + col * BI_PITCH + half * 128;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        uint32_t e[8];
#pragma unroll
        for (int bt = 0; bt < 4; bt++) expand_byte((ww[k] >> (8 * bt)) & 0xFFu, e[2 * bt], e[2 * bt + 1]);
        *reinterpret_cast<uint4*>(dst + k * 32) = make_uint4(e[0], e[1], e[2], e[3]);
        *reinterpret_cast<uint4*>(dst + k * 32 + 16) = make_uint4(e[4], e[5], e[6], e[7]);
      }
      int pb = __popc(w.x) + __popc(w.y) + __popc(w.z) + __popc(w.w);
      pb += __shfl_xor_sync(0xffffffffu, pb, 1);
      if (half == 0) {
        sBase[col] = ((uint32_t)(ok ? pb : 0x7000) << 16) | (uint32_t)(j & 0xffff);
        sNode[col] = (j < nB) ? nodeB[ob + j] : -2;
      }
    }
    __syncthreads();
#pragma unroll 2
    for (int nb = 0; nb < BI_COLS / 8; nb++) {
      int acc[2][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}};
      const uint8_t* bp = sB + (nb * 8 + g) * BI_PITCH + 8 * t;
#pragma unroll
      for (int sx = 0; sx < 8; sx++) {
        const uint2 bf = *reinterpret_cast<const uint2*>(bp + 32 * sx);
        imma_16832(acc[0], aF[0][sx], bf.x, bf.y);
        imma_16832(acc[1], aF[1][sx], bf.x, bf.y);
      }
      // this lane's two columns of the block: keys (dist << 16 | column) of its 8 elements; the common case is that none of
      // them is below the cut, which ONE comparison of their minimum decides
      const uint2 base = *reinterpret_cast<const uint2*>(&sBase[nb * 8 + 2 * t]);
      uint32_t key[4][2];
#pragma unroll
      for (int q = 0; q < 4; q++) {  // row g + 8 q: tile q >> 1, accumulators (q & 1) * 2 + {0, 1}
        key[q][0] = base.x + rowPa16[q] - ((uint32_t)acc[q >> 1][(q & 1) * 2] << 17);
        key[q][1] = base.y + rowPa16[q] - ((uint32_t)acc[q >> 1][(q & 1) * 2 + 1] << 17);
      }
      const uint32_t m01 = min(min(key[0][0], key[0][1]), min(key[1][0], key[1][1]));
      const uint32_t m23 = min(min(key[2][0], key[2][1]), min(key[3][0], key[3][1]));
      if (min(m01, m23) < cutKey) {  // rare: a candidate below the cut
        const int2 nd = *reinterpret_cast<const int2*>(&sNode[nb * 8 + 2 * t]);
#pragma unroll
        for (int q = 0; q < 4; q++) {
#pragma unroll
          for (int cc = 0; cc < 2; cc++) {
            const bool ok = (key[q][cc] < cutKey) && ((cc ? nd.y : nd.x) == rowNode[q]);
            if (ok) {
              cnt[q]++;
              topk_insert(kl[q], key[q][cc]);
            }
          }
        }
      }
    }
  }
  // ---- merge the four lanes of a row (t = 0..3): K rounds of "smallest head wins, its owner pops"
#pragma unroll
  for (int q = 0; q < 4; q++) {
    int c = cnt[q];
    c += __shfl_xor_sync(0xffffffffu, c, 1);
    c += __shfl_xor_sync(0xffffffffu, c, 2);
    uint32_t out[TOPK];
#pragma unroll
    for (int k = 0; k < TOPK; k++) {
      uint32_t m = kl[q][0];
      m = min(m, __shfl_xor_sync(0xffffffffu, m, 1));
      m = min(m, __shfl_xor_sync(0xffffffffu, m, 2));
      out[k] = m;
      if (m != EMPTY && kl[q][0] == m) {
#pragma unroll
        for (int z = 0; z < TOPK - 1; z++) kl[q][z] = kl[q][z + 1];
        kl[q][TOPK - 1] = EMPTY;
      }
    }
    if (t == 0 && rowIdx[q] < nA) {
      uint4* dst = reinterpret_cast<uint4*>(topk + (oa + rowIdx[q]) * TOPK);
      dst[0] = make_uint4(out[0], out[1], out[2], out[3]);
      dst[1] = make_uint4(out[4], out[5], out[6], out[7]);
      candCnt[oa + rowIdx[q]] = c;
    }
  }
}

// full rescan of row i against the still-unmatched candidates (exact fallback when the K-list runs dry)
__device__ void bow_rescan(const u256& da, int na, const uint8_t* descB, const int32_t* nodeB, const uint8_t* validB,
                           const int32_t* matchB, int nB, int lane, int& best1, int& idx1, int& best2) {
  int b1 = 256, i1 = -1, b2 = 256;
  for (int j = lane; j < nB; j += 32) {
    if (nodeB[j] != na) continue;
    if (validB && !validB[j]) continue;
    if (__ldcg(&matchB[j]) >= 0) continue;
    const int d = hamming256(da, ld_desc(descB, j));
    if (d < b1) {
      b2 = b1;
      b1 = d;
      i1 = j;
    } else if (d < b2) {
      b2 = d;
    }
  }
  uint32_t key = (i1 >= 0) ? (((uint32_t)b1 << 16) | (uint32_t)i1) : EMPTY;
  uint32_t m = key;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
  int second = (key == m && m != EMPTY) ? b2 : b1;  // the winner lane contributes its own second best
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) second = min(second, __shfl_xor_sync(0xffffffffu, second, o));
  if (m == EMPTY) {
    best1 = 256;
    idx1 = -1;
    best2 = 256;
  } else {
    best1 = (int)(m >> 16);
    idx1 = (int)(m & 0xffff);
    best2 = second;
  }
}

// stage 2: one warp per vocabulary node (the warp at the first sorted position of a node owns it).  The reference's
// greedy loop (:268) is sequential in the keyframe-side rows of a node; here 32 consecutive rows are resolved
// speculatively, one per lane, against the current `matched` state, and the longest prefix of lanes whose decision
// cannot have been changed by an earlier lane of the same block is committed — exactly the sequential result, in
// ~1 round per 32 rows when rows rarely compete for the same frame feature.
__global__ void __launch_bounds__(128) k_bow_resolve(const uint8_t* __restrict__ descA, const int32_t* __restrict__ nodeA,
                                                     const uint8_t* __restrict__ validA, const float* __restrict__ angA,
                                                     const int32_t* __restrict__ nAarr, int capA,
                                                     const uint8_t* __restrict__ descB, const int32_t* __restrict__ nodeB,
                                                     const uint8_t* __restrict__ validB, const float* __restrict__ angB,
                                                     const int32_t* __restrict__ nBarr, int capB,
                                                     const int32_t* __restrict__ orderA, const uint32_t* __restrict__ topk,
                                                     const int32_t* __restrict__ candCnt, MatchParams mp,
                                                     int32_t* matchB, int32_t* __restrict__ binB) {
  const int pair = blockIdx.y;
  const int nA = min(nAarr[pair], capA), nB = min(nBarr[pair], capB);  // (clamped: device-side counts are untrusted)
  const int lane = threadIdx.x & 31;
  const int r0 = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (r0 >= nA) return;
  const size_t oa = (size_t)pair * capA, ob = (size_t)pair * capB;
  const int32_t* order = orderA + oa;
  const int32_t* nodeAp = nodeA + oa;
  const int node = nodeAp[order[r0]];
  if (r0 > 0 && nodeAp[order[r0 - 1]] == node) return;  // not the head of a node segment
  int32_t* mB = matchB + ob;
  for (int base = r0; base < nA; base += 32) {
    // lane <-> row base+lane of the segment
    const int r = base + lane;
    int i = -1;
    bool inSeg = false;
    if (r < nA) {
      i = order[r];
      inSeg = nodeAp[i] == node;
    }
    const unsigned segMask = __ballot_sync(0xffffffffu, inSeg);
    if (segMask == 0) break;
    const int nrows = __popc(segMask);  // rows of this node are contiguous in sorted order -> a prefix of lanes
    const bool rowOk = inSeg && (!validA || validA[oa + i]);  // no MapPoint / bad (:272-277)
    uint32_t e[TOPK];
#pragma unroll
    for (int k = 0; k < TOPK; k++) e[k] = rowOk ? topk[(oa + i) * TOPK + k] : EMPTY;
    const bool complete = rowOk ? (candCnt[oa + i] <= TOPK) : true;
    int first = 0;  // lanes < first are committed
    while (first < nrows) {
      // speculative decision of every uncommitted lane against the current matched state
      int best1 = 256, idx1 = -1, best2 = 256, idx2 = -1, navail = 0;
      if (lane >= first && rowOk) {
#pragma unroll
        for (int k = 0; k < TOPK; k++) {
          const uint32_t ek = e[k];
          if (ek == EMPTY) continue;
          const int j = (int)(ek & 0xffff);
          if (__ldcg(&mB[j]) >= 0) continue;  // already matched (:288)
          if (navail == 0) {
            best1 = (int)(ek >> 16);
            idx1 = j;
          } else if (navail == 1) {
            best2 = (int)(ek >> 16);
            idx2 = j;
          }
          navail++;
        }
      }
      const bool hard = (lane >= first) && rowOk && !(navail >= 2 || complete);  // K-list ran dry: exact rescan
      bool pass = mp.strictLt ? (best1 < mp.thLow) : (best1 <= mp.thLow);
      bool accept = (lane >= first) && rowOk && !hard && pass && ((float)best1 < __fmul_rn(mp.nnratio, (float)best2));
      const int pick = accept ? idx1 : -1;
      bool dirty = hard;
      for (int src = first; src < nrows; src++) {
        const int pk = __shfl_sync(0xffffffffu, pick, src);
        if (src < lane && pk >= 0 && (pk == idx1 || pk == idx2)) dirty = true;
      }
      const unsigned dm = __ballot_sync(0xffffffffu, dirty && lane >= first && lane < nrows);
      const int d = dm ? (__ffs(dm) - 1) : nrows;  // first lane that must wait
      if (lane >= first && lane < d && accept) {
        mB[idx1] = i;
        binB[ob + idx1] = mp.checkOri ? rot_bin(angA[oa + i], angB[ob + idx1]) : 0;
      }
      __syncwarp();
      first = d;
      if (first < nrows) {
        const unsigned hm = __ballot_sync(0xffffffffu, hard);
        if (hm & (1u << first)) {
          // cooperative exact rescan of that row with all 32 lanes
          const int ih = __shfl_sync(0xffffffffu, i, first);
          const u256 da = ld_desc(descA + oa * 32, ih);
          int b1, i1, b2;
          bow_rescan(da, node, descB + ob * 32, nodeB + ob, validB ? validB + ob : nullptr, mB, nB, lane, b1, i1, b2);
          const bool ps = mp.strictLt ? (b1 < mp.thLow) : (b1 <= mp.thLow);
          if (ps && (float)b1 < __fmul_rn(mp.nnratio, (float)b2)) {
            if (lane == 0) {
              mB[i1] = ih;
              binB[ob + i1] = mp.checkOri ? rot_bin(angA[oa + ih], angB[ob + i1]) : 0;
            }
          }
          __syncwarp();
          first++;
        }
      }
    }
    if (nrows < 32) break;
  }
}

// ComputeThreeMaxima (:1866-1908), one thread: the bins of the three largest counts (strict >, so the earlier bin wins
// a tie); the second and third are dropped (-1) when they hold less than a tenth of the first.
__device__ __forceinline__ void three_maxima(const int* hist, int (&keep)[3]) {
  int max1 = 0, max2 = 0, max3 = 0, ind1 = -1, ind2 = -1, ind3 = -1;
  for (int i = 0; i < HISTO; i++) {
    const int s = hist[i];
    if (s > max1) {
      max3 = max2; max2 = max1; max1 = s;
      ind3 = ind2; ind2 = ind1; ind1 = i;
    } else if (s > max2) {
      max3 = max2; max2 = s;
      ind3 = ind2; ind2 = i;
    } else if (s > max3) {
      max3 = s;
      ind3 = i;
    }
  }
  if ((float)max2 < 0.1f * (float)max1) {
    ind2 = -1;
    ind3 = -1;
  } else if ((float)max3 < 0.1f * (float)max1) {
    ind3 = -1;
  }
  keep[0] = ind1;
  keep[1] = ind2;
  keep[2] = ind3;
}

// rotation-histogram consistency (:356-379); one CTA per pair
__global__ void __launch_bounds__(256) k_rot_cull(const int32_t* __restrict__ nBarr, int capB, int checkOri,
                                                  int32_t* __restrict__ matchB, const int32_t* __restrict__ binB,
                                                  const int32_t* __restrict__ extraCount,
                                                  int32_t* __restrict__ nmatches) {
  __shared__ int hist[HISTO];
  __shared__ int keep[3];
  __shared__ int total, culled;
  const int pair = blockIdx.x;
  const int nB = min(nBarr[pair], capB);
  int32_t* mB = matchB + (size_t)pair * capB;
  const int32_t* bB = binB + (size_t)pair * capB;
  if (threadIdx.x < HISTO) hist[threadIdx.x] = 0;
  if (threadIdx.x == 0) {
    total = 0;
    culled = 0;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < nB; j += blockDim.x)
    if (mB[j] >= 0) {
      atomicAdd(&total, 1);
      if (checkOri) atomicAdd(&hist[bB[j]], 1);
    }
  __syncthreads();
  if (threadIdx.x == 0) three_maxima(hist, keep);
  __syncthreads();
  if (checkOri) {
    for (int j = threadIdx.x; j < nB; j += blockDim.x)
      if (mB[j] >= 0) {
        const int bn = bB[j];
        if (bn != keep[0] && bn != keep[1] && bn != keep[2]) {
          mB[j] = -1;
          atomicAdd(&culled, 1);
        }
      }
  }
  __syncthreads();
  if (threadIdx.x == 0) nmatches[pair] = total - culled + (extraCount ? extraCount[pair] : 0);
}

__global__ void k_fill_i32(int32_t* p, int v, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

__global__ void k_desc_distance(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, int n,
                                int32_t* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = hamming256(ld_desc(a, i), ld_desc(b, i));
}

// ------------------------------------------------------------------------------------------------
// SearchByProjection(CurrentFrame, LastFrame): Frame grid + windowed candidates
// ------------------------------------------------------------------------------------------------
struct ProjGeom {
  float minX, minY, maxX, maxY, invW, invH, bf, th;
  int mode, thHigh, checkOri, nlevels;
  float scale[16];
  float invSigma2[16];  // mvInvLevelSigma2 (only the chi-square gate of the window search reads it)
  int winFlags;         // B2S_WIN_* of b2s_search_windows
  // batched launches (b2s_search_by_projection_last_device): blockIdx.y = pair; all zero / null for the one-pair entry points
  int strideF = 0, strideQ = 0;       // per-pair stride (entries) of the feature-side / query-side arrays
  const int32_t* nfArr = nullptr;     // per-pair feature / query counts (device)
  const int32_t* nqArr = nullptr;
};
constexpr int CELL_STRIDE = GRID_COLS * GRID_ROWS + 2;  // cellStart entries of one pair

// PosInGrid (src/Frame.cc:863-877): cell = round(), features outside the grid get key = big (sorted last, ignored)
__global__ void k_proj_cell_key(const float* __restrict__ kpx, const float* __restrict__ kpy, int nf, ProjGeom g,
                                int32_t* __restrict__ cellKey) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (g.nfArr) nf = min(g.nfArr[blockIdx.y], g.strideF);
  const size_t fo = (size_t)blockIdx.y * g.strideF;
  kpx += fo; kpy += fo; cellKey += fo;
  if (i >= nf) return;
  const int px = (int)roundf(__fmul_rn(__fsub_rn(kpx[i], g.minX), g.invW));
  const int py = (int)roundf(__fmul_rn(__fsub_rn(kpy[i], g.minY), g.invH));
  cellKey[i] = (px < 0 || px >= GRID_COLS || py < 0 || py >= GRID_ROWS) ? (GRID_COLS * GRID_ROWS) : (px * GRID_ROWS + py);
}

// cellStart[c] = first sorted position whose key >= c  (c in [0, 3072])
__global__ void k_proj_cell_start(const int32_t* __restrict__ cellKey, const int32_t* __restrict__ order, int nf,
                                  int32_t* __restrict__ cellStart, int strideF = 0, const int32_t* __restrict__ nfArr = nullptr) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (nfArr) nf = min(nfArr[blockIdx.y], strideF);
  cellKey += (size_t)blockIdx.y * strideF;
  order += (size_t)blockIdx.y * strideF;
  cellStart += (size_t)blockIdx.y * CELL_STRIDE;
  if (r > nf) return;
  const int kPrev = (r == 0) ? -1 : cellKey[order[r - 1]];
  const int kCur = (r == nf) ? (GRID_COLS * GRID_ROWS) : cellKey[order[r]];
  for (int c = kPrev + 1; c <= kCur; c++) cellStart[c] = r;
}

struct __align__(8) ProjQuery {  // == b2s_proj_query
  float u, v, invz, angle;
  int32_t octave, has_obs;
  uint8_t desc[32];
};
struct __align__(8) MapQuery {  // == b2s_map_query (SearchByProjection(Frame&, vector<MapPoint*>&, th), :70-175)
  float u, v, ur, view_cos;
  int32_t level;
  uint8_t in_view, has_obs, pad[2];
  uint8_t desc[32];
};

struct __align__(4) WinQuery {  // == b2s_win_query (Fuse / SearchByProjection(KeyFrame*, Scw, ...) search core)
  float u, v, ur, radius;
  int32_t min_level, max_level;
  uint8_t valid, pad[3];
  uint8_t desc[32];
};

// search window of one query: centre, radius, level range of GetFeaturesInArea and the right-image coordinate of the
// stereo gate
struct Win {
  bool ok;
  float u, v, r, ur;
  int minL, maxL;
  bool stereoGate = true;  // |ur - uRight| <= r on stereo features (:1662-1669 / :128-139)
  bool chi2Gate = false;   // Fuse reprojection gate (:1097-1124)
};
__device__ __forceinline__ Win make_win(const ProjQuery& Q, const ProjGeom& g) {  // :1607-1646
  Win w;
  w.u = Q.u; w.v = Q.v;
  w.ok = !(Q.invz < 0) && !(Q.u < g.minX || Q.u > g.maxX) && !(Q.v < g.minY || Q.v > g.maxY);  // :1616-1626
  const int oct = Q.octave;
  w.r = w.ok ? __fmul_rn(g.th, g.scale[oct]) : 0.f;
  if (g.mode == 1) { w.minL = oct; w.maxL = -1; }
  else if (g.mode == 2) { w.minL = 0; w.maxL = oct; }
  else { w.minL = oct - 1; w.maxL = oct + 1; }
  w.ur = __fsub_rn(Q.u, __fmul_rn(g.bf, Q.invz));
  return w;
}
__device__ __forceinline__ Win make_win(const MapQuery& Q, const ProjGeom& g) {  // :83-103
  Win w;
  w.u = Q.u; w.v = Q.v;
  w.ok = Q.in_view != 0;
  float r = ((double)Q.view_cos > 0.998) ? 2.5f : 4.0f;  // RadiusByViewingCos (:178-185)
  if (g.th != 1.0f) r = __fmul_rn(r, g.th);              // bFactor (:76,93-94)
  const int lv = min(max(Q.level, 0), 15);
  w.r = __fmul_rn(r, g.scale[lv]);
  w.minL = Q.level - 1;
  w.maxL = Q.level;
  w.ur = Q.ur;
  return w;
}
__device__ __forceinline__ Win make_win(const WinQuery& Q, const ProjGeom& g) {
  Win w;
  w.u = Q.u; w.v = Q.v; w.ur = Q.ur;
  w.ok = Q.valid != 0;
  w.r = Q.radius;
  w.minL = Q.min_level;  // max_level >= 0, so the GetFeaturesInArea-style test below is the plain range test
  w.maxL = max(Q.max_level, 0);
  w.stereoGate = false;
  w.chi2Gate = (g.winFlags & 1) != 0;
  return w;
}
// cell range of GetFeaturesInArea (src/Frame.cc:752-770); false = empty result
__device__ __forceinline__ bool win_cells(const Win& w, const ProjGeom& g, int& c0x, int& c1x, int& c0y, int& c1y) {
  c0x = max(0, (int)floorf(__fmul_rn(__fsub_rn(__fsub_rn(w.u, g.minX), w.r), g.invW)));
  c1x = min(GRID_COLS - 1, (int)ceilf(__fmul_rn(__fadd_rn(__fsub_rn(w.u, g.minX), w.r), g.invW)));
  c0y = max(0, (int)floorf(__fmul_rn(__fsub_rn(__fsub_rn(w.v, g.minY), w.r), g.invH)));
  c1y = min(GRID_ROWS - 1, (int)ceilf(__fmul_rn(__fadd_rn(__fsub_rn(w.v, g.minY), w.r), g.invH)));
  return !(c0x >= GRID_COLS || c1x < 0 || c0y >= GRID_ROWS || c1y < 0);
}
// one feature of the window's cells: level gate, |dx|,|dy| < r, stereo gate (:1648-1669 / :117-139)
__device__ __forceinline__ bool win_take(const Win& w, int id, const float* __restrict__ kpx, const float* __restrict__ kpy,
                                         const int32_t* __restrict__ octave, const float* __restrict__ uright) {
  if ((w.minL > 0) || (w.maxL >= 0)) {
    const int o = octave[id];
    if (o < w.minL) return false;
    if (w.maxL >= 0 && o > w.maxL) return false;
  }
  const float dx = __fsub_rn(kpx[id], w.u), dy = __fsub_rn(kpy[id], w.v);
  if (!(fabsf(dx) < w.r && fabsf(dy) < w.r)) return false;
  const float urr = uright[id];
  if (w.stereoGate && urr > 0 && fabsf(__fsub_rn(w.ur, urr)) > w.r) return false;
  return true;
}
// Fuse: reprojection error gate with the candidate's level sigma (src/ORBmatcher.cc:1097-1124)
__device__ __forceinline__ bool win_chi2_ok(const Win& w, int id, const float* __restrict__ kpx, const float* __restrict__ kpy,
                                            const int32_t* __restrict__ octave, const float* __restrict__ uright,
                                            const ProjGeom& g) {
  const float ex = __fsub_rn(w.u, kpx[id]), ey = __fsub_rn(w.v, kpy[id]);
  const float is2 = g.invSigma2[min(max(octave[id], 0), 15)];
  const float urr = uright[id];
  if (urr >= 0) {
    const float er = __fsub_rn(w.ur, urr);
    const float e2 = __fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(er, er));
    return !((double)__fmul_rn(e2, is2) > 7.8);
  }
  const float e2 = __fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey));
  return !((double)__fmul_rn(e2, is2) > 5.99);
}
// a candidate of the window: win_take, the Fuse gate when it is on, and never a feature occupied on entry (the test of
// k_proj_topk's loop, which keeps it written out)
__device__ __forceinline__ bool win_candidate(const Win& w, int id, const float* __restrict__ kpx,
                                              const float* __restrict__ kpy, const int32_t* __restrict__ octave,
                                              const float* __restrict__ uright, const uint8_t* __restrict__ occupied,
                                              const ProjGeom& g) {
  bool take = win_take(w, id, kpx, kpy, octave, uright);
  if (take && w.chi2Gate) take = win_chi2_ok(w, id, kpx, kpy, octave, uright, g);
  if (take && occupied && occupied[id]) take = false;
  return take;
}

// stage 1: one warp per query; candidates are enumerated in GetFeaturesInArea order (src/Frame.cc:741-850:
// ix outer, iy inner, insertion order inside a cell) and the K best by (distance, order) are kept.
// key = dist<<20 | ord  (ord < 2^20 = running index in enumeration order); cand index stored alongside.
template <class QT>
__global__ void __launch_bounds__(256) k_proj_topk(const QT* __restrict__ q, int nq, const float* __restrict__ kpx,
                                                   const float* __restrict__ kpy, const int32_t* __restrict__ octave,
                                                   const float* __restrict__ uright, const uint8_t* __restrict__ occupied,
                                                   const uint8_t* __restrict__ desc, const int32_t* __restrict__ order,
                                                   const int32_t* __restrict__ cellStart, ProjGeom g,
                                                   uint32_t* __restrict__ topk, int32_t* __restrict__ topkIdx,
                                                   int32_t* __restrict__ candCnt) {
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * 8 + (threadIdx.x >> 5);
  {
    const size_t fo = (size_t)blockIdx.y * g.strideF, qo = (size_t)blockIdx.y * g.strideQ;
    if (g.nqArr) nq = min(g.nqArr[blockIdx.y], g.strideQ);
    q += qo; kpx += fo; kpy += fo; octave += fo; uright += fo; desc += fo * 32; order += fo;
    if (occupied) occupied += fo;
    cellStart += (size_t)blockIdx.y * CELL_STRIDE;
    topk += qo * TOPK; topkIdx += qo * TOPK; candCnt += qo;
  }
  if (i >= nq) return;
  uint32_t t[TOPK];
#pragma unroll
  for (int k = 0; k < TOPK; k++) t[k] = EMPTY;
  int cnt = 0;
  const QT& Q = q[i];
  Win w = make_win(Q, g);
  int c0x = 0, c1x = -1, c0y = 0, c1y = -1;
  bool ok = w.ok;
  if (ok) ok = win_cells(w, g, c0x, c1x, c0y, c1y);
  if (ok) {
    const u256 dq = ld_desc_w(Q.desc);
    // columns of cells ix; inside a column the cells iy=c0y..c1y are contiguous in the sorted array
    int ord = 0;
    for (int ix = c0x; ix <= c1x; ix++) {
      const int beg = cellStart[ix * GRID_ROWS + c0y], end = cellStart[ix * GRID_ROWS + c1y + 1];
      for (int p = beg + lane; p < end; p += 32) {
        const int id = order[p];
        bool take = win_take(w, id, kpx, kpy, octave, uright);
        if (take && w.chi2Gate) take = win_chi2_ok(w, id, kpx, kpy, octave, uright, g);
        if (take && occupied && occupied[id]) take = false;  // initially occupied features are never candidates
        if (take) {
          const int d = hamming256(dq, ld_desc(desc, id));
          cnt++;
          // order inside the enumeration: position p-beg within column ix, columns ascending
          topk_insert(t, ((uint32_t)d << 20) | (uint32_t)(ord + (p - beg)));
        }
      }
      ord += end - beg;
    }
  }
  uint32_t out[TOPK];
  topk_warp_merge(t, out);
  cnt = warp_reduce_sum(cnt);
  if (lane < TOPK) {
    uint32_t e = EMPTY;
#pragma unroll
    for (int k = 0; k < TOPK; k++)
      if (k == lane) e = out[k];
    int id = -1;
    if (e != EMPTY) {
      // recover the feature index from the enumeration order
      int ordv = (int)(e & 0xFFFFF);
      for (int ix = c0x; ix <= c1x; ix++) {
        const int beg = cellStart[ix * GRID_ROWS + c0y], end = cellStart[ix * GRID_ROWS + c1y + 1];
        if (ordv < end - beg) {
          id = order[beg + ordv];
          break;
        }
        ordv -= end - beg;
      }
    }
    topk[(size_t)i * TOPK + lane] = e;
    topkIdx[(size_t)i * TOPK + lane] = id;
  }
  if (lane == 0) candCnt[i] = ok ? cnt : -1;
}

// Exact rescan of one query's window in enumeration order against the CURRENT state of the greedy loop: the NEED (1 or
// 2) smallest (distance, order) keys over the warp among the candidates whose distance is below bound(feature)
// (key2/id2 = EMPTY/-1 when there is no second candidate or NEED == 1).
template <int NEED, class QT, class Bound>
__device__ __forceinline__ void win_rescan_top2(const QT& Q, const ProjGeom& g, int lane, const float* __restrict__ kpx,
                                                const float* __restrict__ kpy, const int32_t* __restrict__ octave,
                                                const float* __restrict__ uright, const uint8_t* __restrict__ occupied,
                                                const uint8_t* __restrict__ desc, const int32_t* __restrict__ order,
                                                const int32_t* __restrict__ cellStart, Bound bound, uint32_t& key1,
                                                int& id1, uint32_t& key2, int& id2) {
  const Win w = make_win(Q, g);
  int c0x, c1x, c0y, c1y;
  win_cells(w, g, c0x, c1x, c0y, c1y);
  const u256 dq = ld_desc_w(Q.desc);
  uint32_t k1 = EMPTY, k2 = EMPTY;
  int i1 = -1, i2 = -1;
  int ord = 0;
  for (int ix = c0x; ix <= c1x; ix++) {
    const int beg = cellStart[ix * GRID_ROWS + c0y], end = cellStart[ix * GRID_ROWS + c1y + 1];
    for (int p = beg + lane; p < end; p += 32) {
      const int fid = order[p];
      if (!win_candidate(w, fid, kpx, kpy, octave, uright, occupied, g)) continue;
      const int lim = bound(fid);
      if (lim <= 0) continue;  // no distance is below it
      const int d = hamming256(dq, ld_desc(desc, fid));
      if (d >= lim) continue;
      const uint32_t key = ((uint32_t)d << 20) | (uint32_t)(ord + (p - beg));
      if (key < k1) {
        k2 = k1; i2 = i1;
        k1 = key; i1 = fid;
      } else if (key < k2) {
        k2 = key; i2 = fid;
      }
    }
    ord += end - beg;
  }
  // warp top-2 of the per-lane pairs (keys are unique: the order part differs)
  uint32_t m1 = k1;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m1 = min(m1, __shfl_xor_sync(0xffffffffu, m1, o));
  key1 = m1;
  id1 = -1;
  key2 = EMPTY;
  id2 = -1;
  if (m1 == EMPTY) return;
  const unsigned who = __ballot_sync(0xffffffffu, k1 == m1);
  const int wl = __ffs(who) - 1;
  id1 = __shfl_sync(0xffffffffu, i1, wl);
  if (NEED == 1) return;  // shuffles are not dead code to the compiler
  // second: the winner lane contributes its own runner-up, every other lane its best
  const uint32_t cand2 = (lane == wl) ? k2 : k1;
  const int cid2 = (lane == wl) ? i2 : i1;
  uint32_t m2 = cand2;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m2 = min(m2, __shfl_xor_sync(0xffffffffu, m2, o));
  if (m2 != EMPTY) {
    const unsigned who2 = __ballot_sync(0xffffffffu, cand2 == m2);
    key2 = m2;
    id2 = __shfl_sync(0xffffffffu, cid2, __ffs(who2) - 1);
  }
}

// The best and (NEED == 2) second-best candidates of query Q that are available NOW — a candidate counts while its
// distance is below bound(feature) — as keys ascending; key/id = EMPTY/-1 where there is none.  Removing unavailable
// entries from the query's K-list (topk / topkIdx, sorted by distance, then enumeration order) keeps the reference's
// first-minimum rule and its runner-up, so the list decides when it holds NEED available entries, or at least one and the
// window had no more than TOPK candidates (cc; the list is then the whole window).  Otherwise a window with more than TOPK candidates is rescanned exactly; otherwise there is none.
template <int NEED, class QT, class Bound>
__device__ __forceinline__ void best_two(const QT& Q, int cc, const uint32_t* __restrict__ topk,
                                         const int32_t* __restrict__ topkIdx, const ProjGeom& g, int lane,
                                         const float* __restrict__ kpx, const float* __restrict__ kpy,
                                         const int32_t* __restrict__ octave, const float* __restrict__ uright,
                                         const uint8_t* __restrict__ occupied, const uint8_t* __restrict__ desc,
                                         const int32_t* __restrict__ order, const int32_t* __restrict__ cellStart,
                                         Bound bound, uint32_t& key1, int& id1, uint32_t& key2, int& id2) {
  const uint32_t e = (lane < TOPK) ? topk[lane] : EMPTY;
  const int id = (lane < TOPK) ? topkIdx[lane] : -1;
  unsigned am = __ballot_sync(0xffffffffu, e != EMPTY && (int)(e >> 20) < bound(id));
  key1 = EMPTY; id1 = -1;
  key2 = EMPTY; id2 = -1;
  if (__popc(am) >= NEED || (am != 0u && cc <= TOPK)) {
    const int l1 = __ffs(am) - 1;
    key1 = __shfl_sync(0xffffffffu, e, l1);
    id1 = __shfl_sync(0xffffffffu, id, l1);
    am &= am - 1;
    if (NEED == 2 && am) {
      const int l2 = __ffs(am) - 1;
      key2 = __shfl_sync(0xffffffffu, e, l2);
      id2 = __shfl_sync(0xffffffffu, id, l2);
    }
  } else if (cc > TOPK) {
    win_rescan_top2<NEED>(Q, g, lane, kpx, kpy, octave, uright, occupied, desc, order, cellStart, bound, key1, id1, key2,
                          id2);
  }
}

// stage 2: the greedy loop of :1600-1706 — one warp walks the queries in order; `taken[j]` = feature j now holds a
// MapPoint with Observations()>0 (:1658-1660).  A query whose K-list ran dry is rescanned exactly.
__global__ void __launch_bounds__(32) k_proj_resolve(const ProjQuery* __restrict__ q, int nq,
                                                     const float* __restrict__ kpx, const float* __restrict__ kpy,
                                                     const int32_t* __restrict__ octave, const float* __restrict__ angle,
                                                     const float* __restrict__ uright,
                                                     const uint8_t* __restrict__ occupied, const uint8_t* __restrict__ desc,
                                                     const int32_t* __restrict__ order,
                                                     const int32_t* __restrict__ cellStart, ProjGeom g,
                                                     const uint32_t* __restrict__ topk, const int32_t* __restrict__ topkIdx,
                                                     const int32_t* __restrict__ candCnt, uint8_t* __restrict__ taken,
                                                     int32_t* __restrict__ matchCur, int32_t* __restrict__ pushList,
                                                     int32_t* __restrict__ accepted, int32_t* __restrict__ histOut) {
  const int lane = threadIdx.x;
  __shared__ int hist[HISTO];
  if (lane < HISTO) hist[lane] = 0;
  __syncwarp();
  {
    const size_t fo = (size_t)blockIdx.y * g.strideF, qo = (size_t)blockIdx.y * g.strideQ;
    if (g.nqArr) nq = min(g.nqArr[blockIdx.y], g.strideQ);
    q += qo; kpx += fo; kpy += fo; octave += fo; angle += fo; uright += fo; desc += fo * 32; order += fo;
    if (occupied) occupied += fo;
    cellStart += (size_t)blockIdx.y * CELL_STRIDE;
    topk += qo * TOPK; topkIdx += qo * TOPK; candCnt += qo;
    taken += fo; matchCur += fo; pushList += qo;
    accepted += (size_t)blockIdx.y * 4; histOut += (size_t)blockIdx.y * HISTO;
  }
  int nAccepted = 0;
  for (int i = 0; i < nq; i++) {
    const int cc = candCnt[i];
    if (cc <= 0) continue;
    uint32_t key1, key2;
    int id1, id2;
    best_two<1>(q[i], cc, topk + (size_t)i * TOPK, topkIdx + (size_t)i * TOPK, g, lane, kpx, kpy, octave, uright, occupied,
                desc, order, cellStart, [=](int f) { return taken[f] ? 0 : 257; }, key1, id1, key2, id2);
    if (id1 < 0 || (int)(key1 >> 20) > g.thHigh) continue;  // :1683
    if (lane == 0) {
      matchCur[id1] = i;
      taken[id1] = q[i].has_obs ? 1 : 0;
      if (g.checkOri) {
        const int bn = rot_bin(q[i].angle, angle[id1]);
        pushList[nAccepted] = (bn << 20) | id1;  // rotHist[bin].push_back(bestIdx2) (:1700)
        hist[bn]++;
      }
      nAccepted++;
    }
    __syncwarp();
  }
  __syncwarp();
  if (lane == 0) accepted[0] = nAccepted;
  if (lane < HISTO) histOut[lane] = hist[lane];
}

// ------------------------------------------------------------------------------------------------
// SearchForTriangulation (src/ORBmatcher.cc:810-1009): per vocabulary node, greedy in keyframe-1 feature order; the
// candidates of a row are the unmatched keyframe-2 features of the node without a MapPoint that pass the distance,
// epipole and epipolar-line gates; `dist > bestDist -> continue` (:893) makes the LAST minimum win.
// One warp per node: rows sequential, lanes over the node's keyframe-2 features (a node holds tens of features with a
// real vocabulary; nothing here is shared between nodes).
// ------------------------------------------------------------------------------------------------
struct TriParams {
  float F12[9];
  float ex, ey;
  float scale[16], sigma2[16];
  int thLow, checkOri;
};
__device__ __forceinline__ bool tri_epipolar_ok(float x1, float y1, float x2, float y2, int oct2, const TriParams& tp) {
  // CheckDistEpipolarLine (:186-215), float arithmetic in source order (this file is built with --fmad=false)
  const float a = __fadd_rn(__fadd_rn(__fmul_rn(x1, tp.F12[0]), __fmul_rn(y1, tp.F12[3])), tp.F12[6]);
  const float b = __fadd_rn(__fadd_rn(__fmul_rn(x1, tp.F12[1]), __fmul_rn(y1, tp.F12[4])), tp.F12[7]);
  const float c = __fadd_rn(__fadd_rn(__fmul_rn(x1, tp.F12[2]), __fmul_rn(y1, tp.F12[5])), tp.F12[8]);
  const float num = __fadd_rn(__fadd_rn(__fmul_rn(a, x2), __fmul_rn(b, y2)), c);
  const float den = __fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b));
  if (den == 0) return false;
  const float dsqr = __fdiv_rn(__fmul_rn(num, num), den);
  return (double)dsqr < 3.84 * (double)tp.sigma2[min(max(oct2, 0), 15)];
}
__global__ void __launch_bounds__(128) k_tri_match(const uint8_t* __restrict__ descA, const int32_t* __restrict__ nodeA,
                                                   const uint8_t* __restrict__ eligA, const uint8_t* __restrict__ stereoA,
                                                   const float* __restrict__ xA, const float* __restrict__ yA,
                                                   const float* __restrict__ angA, int nA,
                                                   const int32_t* __restrict__ orderA, const uint8_t* __restrict__ descB,
                                                   const int32_t* __restrict__ nodeB, const uint8_t* __restrict__ eligB,
                                                   const uint8_t* __restrict__ stereoB, const float* __restrict__ xB,
                                                   const float* __restrict__ yB, const int32_t* __restrict__ octB,
                                                   const float* __restrict__ angB, int nB,
                                                   const int32_t* __restrict__ orderB, TriParams tp, int32_t* matchB,
                                                   int32_t* __restrict__ binB) {
  const int lane = threadIdx.x & 31;
  const int r0 = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (r0 >= nA) return;
  const int node = nodeA[orderA[r0]];
  if (r0 > 0 && nodeA[orderA[r0 - 1]] == node) return;  // not the head of a node segment
  // keyframe-2 segment of the node: lower bound in the (node, index)-sorted order
  int lo = 0, hi = nB;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (nodeB[orderB[mid]] < node) lo = mid + 1;
    else hi = mid;
  }
  const int bBeg = lo;
  int bEnd = bBeg;
  while (bEnd < nB && nodeB[orderB[bEnd]] == node) bEnd++;
  if (bEnd == bBeg) return;
  for (int r = r0; r < nA; r++) {
    const int i = orderA[r];
    if (nodeA[i] != node) break;
    if (!eligA[i]) continue;  // has a MapPoint / not stereo when bOnlyStereo (:852-861)
    const u256 da = ld_desc(descA, i);
    const bool st1 = stereoA[i] != 0;
    const float x1 = xA[i], y1 = yA[i];
    uint32_t best = EMPTY;
    for (int p = bBeg + lane; p < bEnd; p += 32) {
      const int j = orderB[p];
      if (!eligB[j] || __ldcg(&matchB[j]) >= 0) continue;  // :877-885
      const int d = hamming256(da, ld_desc(descB, j));
      if (d > tp.thLow) continue;  // :893
      const float x2 = xB[j], y2 = yB[j];
      const int o2 = octB[j];
      if (!st1 && !stereoB[j]) {  // :899-906
        const float dx = __fsub_rn(tp.ex, x2), dy = __fsub_rn(tp.ey, y2);
        if (__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) < __fmul_rn(100.f, tp.scale[min(max(o2, 0), 15)])) continue;
      }
      if (!tri_epipolar_ok(x1, y1, x2, y2, o2, tp)) continue;
      best = min(best, ((uint32_t)d << 16) | (uint32_t)(0xFFFF - (p - bBeg)));  // smallest distance, LAST in node order
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
    if (best != EMPTY) {
      const int j = orderB[bBeg + (0xFFFF - (int)(best & 0xFFFFu))];
      if (lane == 0) {
        matchB[j] = i;  // vMatches12[idx1] = bestIdx2; vbMatched2[bestIdx2] = true (:913-916)
        binB[j] = tp.checkOri ? rot_bin(angA[i], angB[j]) : 0;
      }
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------
// DBoW2 TemplatedVocabulary<FORB>::transform (TemplatedVocabulary.h:1211-1256): descend the k-ary tree, at every level the
// child with the smallest Hamming distance (first minimum in file order); word id / weight of the leaf and the id of the
// node `levelsup` levels above the leaves.  One thread per feature; the children of a node are contiguous in cDesc.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_bow_transform(const uint8_t* __restrict__ feat, int n,
                                                       const int32_t* __restrict__ childStart,
                                                       const int32_t* __restrict__ childCount,
                                                       const int32_t* __restrict__ cNode, const uint8_t* __restrict__ cDesc,
                                                       const int32_t* __restrict__ wordOf, const double* __restrict__ wgt,
                                                       int nidLevel, int32_t* __restrict__ wordId,
                                                       double* __restrict__ weight, int32_t* __restrict__ nodeId) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u256 f = ld_desc(feat, i);
  int finalId = 0, level = 0, nid = 0;
  if (childCount[0] == 0) {
    wordId[i] = 0;
    if (weight) weight[i] = 0;
    nodeId[i] = 0;
    return;
  }
  do {
    ++level;
    const int beg = childStart[finalId], cnt = childCount[finalId];
    uint32_t best = 0xFFFFFFFFu;
    for (int c = 0; c < cnt; c++) {
      const uint32_t key = ((uint32_t)hamming256(f, ld_desc(cDesc, beg + c)) << 16) | (uint32_t)c;  // d < best_d: first minimum
      best = min(best, key);
    }
    finalId = cNode[beg + (int)(best & 0xFFFFu)];
    if (level == nidLevel) nid = finalId;
  } while (childCount[finalId] != 0);
  wordId[i] = wordOf[finalId];
  if (weight) weight[i] = wgt[finalId];
  nodeId[i] = nid;
}

// ------------------------------------------------------------------------------------------------
// MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:359-440): one warp per map point (distinctive.cuh).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_distinctive(const uint8_t* __restrict__ desc, const int32_t* __restrict__ offsets,
                                                     int nPoints, int32_t* __restrict__ bestIdx) {
  __shared__ int hist[8][264];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int p = blockIdx.x * 8 + wid;
  if (p >= nPoints) return;
  const int beg = offsets[p], N = offsets[p + 1] - beg;
  if (N <= 0) {
    if (lane == 0) bestIdx[p] = -1;
    return;
  }
  const int best = distinctive_best(N, [&](int i) { return ld_desc(desc, beg + i); }, hist[wid], lane);
  if (lane == 0) bestIdx[p] = best;
}

// Window search without occupancy (Fuse): the queries are independent, the answer is the head of each K-list.
__global__ void __launch_bounds__(256) k_win_pick(int nq, int thDist, const uint32_t* __restrict__ topk,
                                                  const int32_t* __restrict__ topkIdx, int32_t* __restrict__ bestIdx,
                                                  int32_t* __restrict__ bestDist, int32_t* __restrict__ nAccepted) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool acc = false;
  if (i < nq) {
    const uint32_t e = topk[(size_t)i * TOPK];
    const int d = (e == EMPTY) ? 256 : (int)(e >> 20);
    acc = d <= thDist;
    bestDist[i] = d;
    bestIdx[i] = acc ? topkIdx[(size_t)i * TOPK] : -1;
  }
  const int c = __syncthreads_count(acc);
  if (threadIdx.x == 0 && c) atomicAdd(nAccepted, c);
}

// Window search with greedy occupancy (SearchByProjection(KeyFrame*, Scw, vpPoints, vpMatched, th), :388-512): a
// feature chosen by an earlier query (or occupied on entry) is skipped; one warp walks the queries in order.
__global__ void __launch_bounds__(32) k_win_resolve(const WinQuery* __restrict__ q, int nq, int thDist,
                                                    const float* __restrict__ kpx, const float* __restrict__ kpy,
                                                    const int32_t* __restrict__ octave, const float* __restrict__ uright,
                                                    const uint8_t* __restrict__ occupied, const uint8_t* __restrict__ desc,
                                                    const int32_t* __restrict__ order, const int32_t* __restrict__ cellStart,
                                                    ProjGeom g, const uint32_t* __restrict__ topk,
                                                    const int32_t* __restrict__ topkIdx, const int32_t* __restrict__ candCnt,
                                                    uint8_t* __restrict__ taken, int32_t* __restrict__ bestIdx,
                                                    int32_t* __restrict__ bestDist, int32_t* __restrict__ nAccepted) {
  const int lane = threadIdx.x;
  int nAcc = 0;
  for (int i = 0; i < nq; i++) {
    const int cc = candCnt[i];
    int outIdx = -1, outDist = 256;
    if (cc > 0) {
      uint32_t key1, key2;
      int id1, id2;
      best_two<1>(q[i], cc, topk + (size_t)i * TOPK, topkIdx + (size_t)i * TOPK, g, lane, kpx, kpy, octave, uright,
                  occupied, desc, order, cellStart, [=](int f) { return taken[f] ? 0 : 257; }, key1, id1, key2, id2);
      if (id1 >= 0) {
        outDist = (int)(key1 >> 20);
        if (outDist <= thDist) {
          outIdx = id1;
          if (lane == 0) taken[id1] = 1;
          nAcc++;
        }
      }
    }
    if (lane == 0) {
      bestIdx[i] = outIdx;
      bestDist[i] = outDist;
    }
    __syncwarp();
  }
  if (lane == 0) nAccepted[0] = nAcc;
}

// SearchByProjection(Frame&, vector<MapPoint*>&, th) greedy loop (:78-172): one warp walks the map points in order.
// Best and second best among the features that are not occupied NOW (:123-125) are the first two available entries of
// the query's K-list (sorted by distance, then enumeration order — exactly the order in which the reference's
// best/second bookkeeping of :147-160 ranks them); if the list cannot supply two, the window is rescanned exactly.
// Ratio test only when both are on the same pyramid level (:164-166); no rotation check in this matcher.
__global__ void __launch_bounds__(32) k_map_resolve(const MapQuery* __restrict__ q, int nq, const float* __restrict__ kpx,
                                                    const float* __restrict__ kpy, const int32_t* __restrict__ octave,
                                                    const float* __restrict__ uright, const uint8_t* __restrict__ occupied,
                                                    const uint8_t* __restrict__ desc, const int32_t* __restrict__ order,
                                                    const int32_t* __restrict__ cellStart, ProjGeom g, float nnratio,
                                                    const uint32_t* __restrict__ topk, const int32_t* __restrict__ topkIdx,
                                                    const int32_t* __restrict__ candCnt, uint8_t* __restrict__ taken,
                                                    int32_t* __restrict__ matchCur, int32_t* __restrict__ nmatches) {
  const int lane = threadIdx.x;
  int nAccepted = 0;
  for (int i = 0; i < nq; i++) {
    const int cc = candCnt[i];
    if (cc <= 0) continue;
    uint32_t key1, key2;
    int id1, id2;
    best_two<2>(q[i], cc, topk + (size_t)i * TOPK, topkIdx + (size_t)i * TOPK, g, lane, kpx, kpy, octave, uright, occupied,
                desc, order, cellStart, [=](int f) { return taken[f] ? 0 : 257; }, key1, id1, key2, id2);
    if (id1 < 0) continue;
    const int bestDist = (int)(key1 >> 20);
    if (bestDist > g.thHigh) continue;  // :164
    if (id2 >= 0) {
      const int bestDist2 = (int)(key2 >> 20);
      if (octave[id1] == octave[id2] && (float)bestDist > __fmul_rn(nnratio, (float)bestDist2)) continue;  // :166
    }
    if (lane == 0) {
      matchCur[id1] = i;                       // :168 (last writer wins)
      taken[id1] = q[i].has_obs ? 1 : 0;       // the feature now holds a MapPoint; occupied iff Observations()>0
    }
    nAccepted++;
    __syncwarp();
  }
  if (lane == 0) nmatches[0] = nAccepted;
}

// rotation culling for SearchByProjection: the histogram holds every accepted push (a feature may have been pushed more
// than once when a MapPoint without observations was overwritten, :1686); entries of non-kept bins are nulled and
// nmatches decremented per entry (:1713-1724).
__global__ void __launch_bounds__(256) k_proj_cull(int checkOri, const int32_t* __restrict__ hist,
                                                   const int32_t* __restrict__ accepted, int32_t* __restrict__ matchCur,
                                                   const int32_t* __restrict__ pushBins, int32_t* __restrict__ nmatches,
                                                   int strideF = 0, int strideQ = 0) {
  __shared__ int keep[3];
  __shared__ int culled;
  hist += (size_t)blockIdx.y * HISTO; accepted += (size_t)blockIdx.y * 4; nmatches += blockIdx.y;
  matchCur += (size_t)blockIdx.y * strideF; pushBins += (size_t)blockIdx.y * strideQ;
  if (threadIdx.x == 0) {
    culled = 0;
    three_maxima(hist, keep);
  }
  __syncthreads();
  if (checkOri) {
    // every push in a culled bin: null the feature, nmatches--
    const int nPush = accepted[0];
    for (int k = threadIdx.x; k < nPush; k += blockDim.x) {
      const int packed = pushBins[k];
      const int bn = packed >> 20, j = packed & 0xFFFFF;
      if (bn != keep[0] && bn != keep[1] && bn != keep[2]) {
        matchCur[j] = -1;
        atomicAdd(&culled, 1);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) nmatches[0] = accepted[0] - culled;
}

// ---------------------------------------------------------------- SearchForInitialization (src/ORBmatcher.cc:515-643)
// The sequential loop of :527-610 — one warp walks F1's keypoints in order over their K-lists (sorted by distance, then
// enumeration order).  matchedDist / match21 are the reference's vMatchedDistance / vnMatches21; a query whose list cannot
// prove its best two remaining candidates is rescanned exactly.  Every accepted match is pushed to the rotation histogram
// with its F1 index; pushes of matches that are stolen later stay in the histogram, as in the reference.
__global__ void __launch_bounds__(32) k_init_resolve(const WinQuery* __restrict__ q, int nq, const float* __restrict__ angle1,
                                                     const float* __restrict__ kpx, const float* __restrict__ kpy,
                                                     const int32_t* __restrict__ octave, const float* __restrict__ angle2,
                                                     const float* __restrict__ uright, const uint8_t* __restrict__ desc,
                                                     const int32_t* __restrict__ order, const int32_t* __restrict__ cellStart,
                                                     ProjGeom g, int thLow, float nnratio,
                                                     const uint32_t* __restrict__ topk, const int32_t* __restrict__ topkIdx,
                                                     const int32_t* __restrict__ candCnt, int32_t* __restrict__ matchedDist,
                                                     int32_t* __restrict__ match21, int32_t* __restrict__ match12,
                                                     int32_t* __restrict__ pushList, int32_t* __restrict__ accepted,
                                                     int32_t* __restrict__ histOut) {
  const int lane = threadIdx.x;
  __shared__ int hist[HISTO];
  if (lane < HISTO) hist[lane] = 0;
  __syncwarp();
  int nPush = 0;
  for (int i = 0; i < nq; i++) {
    const int cc = candCnt[i];
    if (cc <= 0) continue;
    uint32_t key1, key2;
    int id1, id2;
    // a feature already matched at a distance <= the candidate's is no candidate (:563)
    best_two<2>(q[i], cc, topk + (size_t)i * TOPK, topkIdx + (size_t)i * TOPK, g, lane, kpx, kpy, octave, uright, nullptr,
                desc, order, cellStart, [=](int f) { return matchedDist[f]; }, key1, id1, key2, id2);
    if (id1 < 0) continue;
    const int bestDist = (int)(key1 >> 20);
    const int bestDist2 = key2 == EMPTY ? 2147483647 : (int)(key2 >> 20);
    if (bestDist > thLow) continue;                                         // :579
    if (!((float)bestDist < __fmul_rn((float)bestDist2, nnratio))) continue;  // :581
    if (lane == 0) {
      const int prev = match21[id1];
      if (prev >= 0) match12[prev] = -1;  // :583-587: the better match steals the feature
      match12[i] = id1;
      match21[id1] = i;
      matchedDist[id1] = bestDist;
      if (g.checkOri) {
        const int bn = rot_bin(angle1[i], angle2[id1]);
        hist[bn]++;
        pushList[nPush] = (bn << 20) | i;
      }
    }
    __syncwarp();
    nPush++;  // (the match count is taken from match12 by k_init_cull: it equals the reference's running nmatches)
  }
  __syncwarp();
  if (lane < HISTO) histOut[lane] = hist[lane];
  if (lane == 0) accepted[0] = nPush;
}

// Rotation cull (:612-633): pushes in bins outside the three maxima lose their match if they still hold one; nmatches =
// the surviving matches (the reference's running count equals the number of non-negative entries at every point).
__global__ void __launch_bounds__(256) k_init_cull(int checkOri, int n1, const int32_t* __restrict__ hist,
                                                   const int32_t* __restrict__ accepted, int32_t* __restrict__ match12,
                                                   const int32_t* __restrict__ pushBins, int32_t* __restrict__ nmatches) {
  __shared__ int keep[3];
  __shared__ int total;
  if (threadIdx.x == 0) {
    total = 0;
    three_maxima(hist, keep);
  }
  __syncthreads();
  if (checkOri) {
    const int nPush = accepted[0];
    for (int k = threadIdx.x; k < nPush; k += blockDim.x) {
      const int packed = pushBins[k];
      const int bn = packed >> 20, i1 = packed & 0xFFFFF;
      if (bn != keep[0] && bn != keep[1] && bn != keep[2]) match12[i1] = -1;  // (each F1 index is pushed at most once)
    }
  }
  __syncthreads();
  int c = 0;
  for (int i = threadIdx.x; i < n1; i += blockDim.x) c += match12[i] >= 0;
  atomicAdd(&total, c);
  __syncthreads();
  if (threadIdx.x == 0) nmatches[0] = total;
}

// ---------------------------------------------------------------- persistent Frame feature grid (SURVEY §8f rank 4)
// unpack device-resident extractor records (28-byte cv::KeyPoint layout) into the SoA the matchers read
__global__ void k_unpack_kps(const uint8_t* __restrict__ rec, int nf, float* __restrict__ kpx, float* __restrict__ kpy,
                             int32_t* __restrict__ oct, float* __restrict__ ang) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nf) return;
  const float* r = reinterpret_cast<const float*>(rec + (size_t)i * 28);
  kpx[i] = r[0];
  kpy[i] = r[1];
  ang[i] = r[3];
  oct[i] = reinterpret_cast<const int32_t*>(r)[5];
}

// Frame::GetFeaturesInArea (src/Frame.cc:741-852) on the resident grid: one warp, output in the reference's order
__global__ void __launch_bounds__(32) k_grid_query(float x, float y, float r, int minL, int maxL, const float* __restrict__ kpx,
                                                   const float* __restrict__ kpy, const int32_t* __restrict__ octave,
                                                   const float* __restrict__ uright, const int32_t* __restrict__ order,
                                                   const int32_t* __restrict__ cellStart, ProjGeom g, int32_t* __restrict__ out,
                                                   int cap, int32_t* __restrict__ nOut) {
  const int lane = threadIdx.x;
  Win w;
  w.ok = true; w.u = x; w.v = y; w.r = r; w.ur = 0.f; w.minL = minL; w.maxL = maxL; w.stereoGate = false; w.chi2Gate = false;
  int c0x, c1x, c0y, c1y;
  int n = 0;
  if (win_cells(w, g, c0x, c1x, c0y, c1y)) {
    for (int ix = c0x; ix <= c1x; ix++) {
      const int beg = cellStart[ix * GRID_ROWS + c0y], end = cellStart[ix * GRID_ROWS + c1y + 1];
      for (int p0 = beg; p0 < end; p0 += 32) {
        const int p = p0 + lane;
        int id = -1;
        bool take = false;
        if (p < end) {
          id = order[p];
          take = win_take(w, id, kpx, kpy, octave, uright);
        }
        const unsigned m = __ballot_sync(0xffffffffu, take);
        if (take) {
          const int pos = n + __popc(m & ((1u << lane) - 1u));
          if (pos < cap) out[pos] = id;
        }
        n += __popc(m);
      }
    }
  }
  if (lane == 0) nOut[0] = n;
}

}  // namespace b2s

using namespace b2s;

extern "C" int b2s_matcher_create(int max_features, int max_batch, int device, b2s_matcher** out) {
  if (!out || max_features < 1 || max_features > 65535 || max_batch < 1) {
    set_error("b2s_matcher_create: bad argument (max_features must be in [1,65535])");
    return B2S_ERR_BAD_ARG;
  }
  *out = nullptr;
  int rc = select_device(device);
  if (rc != B2S_OK) return rc;
  b2s_matcher* h = new b2s_matcher();
  h->maxF = max_features;
  h->maxBatch = max_batch;
  const size_t F = (size_t)max_features * max_batch;
  h->open(device);
  auto A = [h](auto* p, size_t bytes) { h->alloc(*p, bytes); };
  A(&h->dDescA, F * 32); A(&h->dDescB, F * 32);
  A(&h->dValidA, F); A(&h->dValidB, F); A(&h->dOcc, F); A(&h->dTaken, F);
  A(&h->dNodeA, F * 4); A(&h->dNodeB, F * 4);
  A(&h->dNA, max_batch * 4); A(&h->dNB, max_batch * 4);
  A(&h->dOrder, F * 4); A(&h->dCandCnt, F * 4);
  A(&h->dMatch, F * 4); A(&h->dBin, F * 4); A(&h->dNMatches, max_batch * 4);
  A(&h->dOct, F * 4); A(&h->dCellKey, F * 4);
  A(&h->dCellStart, (size_t)CELL_STRIDE * max_batch * 4);
  A(&h->dTopkIdx, F * TOPK * 4); A(&h->dExtra, (size_t)max_batch * 4 * 4);
  A(&h->dHist, (size_t)max_batch * HISTO * 4);
  A(&h->dPush, F * 4);
  A(&h->dAngA, F * 4); A(&h->dAngB, F * 4);
  A(&h->dKpx, F * 4); A(&h->dKpy, F * 4); A(&h->dURight, F * 4);
  A(&h->dTopk, F * TOPK * 4);
  A(&h->dQueries, F * 64);  // ProjQuery / MapQuery (56 B) or WinQuery (60 B)
  if (h->error != cudaSuccess) {
    set_error("b2s_matcher_create: %s", cudaGetErrorString(h->error));
    b2s_matcher_destroy(h);
    return B2S_ERR_CUDA;
  }
  *out = h;
  return B2S_OK;
}

extern "C" void b2s_matcher_destroy(b2s_matcher* h) {
  if (!h) return;
  h->close();
  delete h;
}

extern "C" long long b2s_matcher_launch_count(const b2s_matcher* h) { return h ? h->launches : 0; }

extern "C" int b2s_descriptor_distance(b2s_matcher* h, const uint8_t* a, const uint8_t* b, int n, int32_t* dist) {
  if (!h || !a || !b || !dist || n < 0 || n > h->maxF * h->maxBatch) return B2S_ERR_BAD_ARG;
  if (n == 0) return B2S_OK;
  B2S_CUDA(cudaSetDevice(h->device));
  B2S_CUDA(cudaMemcpyAsync(h->dDescA, a, (size_t)n * 32, cudaMemcpyHostToDevice, h->stream));
  B2S_CUDA(cudaMemcpyAsync(h->dDescB, b, (size_t)n * 32, cudaMemcpyHostToDevice, h->stream));
  k_desc_distance<<<div_up(n, 256), 256, 0, h->stream>>>(h->dDescA, h->dDescB, n, h->dMatch);
  h->launches++;
  B2S_CUDA(cudaMemcpyAsync(dist, h->dMatch, (size_t)n * 4, cudaMemcpyDeviceToHost, h->stream));
  B2S_CUDA(cudaStreamSynchronize(h->stream));
  return B2S_OK;
}

// Distance from which a frame-side candidate cannot influence SearchByBoW (src/ORBmatcher.cc:284-310): a best candidate is
// only accepted with bestDist1 <= TH_LOW, and a second best at distance b2 only enters through bestDist1 < ratio * b2, which
// holds for every acceptable bestDist1 as soon as ratio * b2 > TH_LOW.  With cut = floor(TH_LOW / ratio) + 2 every candidate
// at distance >= cut is (a) never an accepted best and (b) as second best indistinguishable from "no second candidate"
// (bestDist2 = 256).  The K-lists therefore hold, and candCnt counts, only the candidates below the cut; the resolver's
// "complete" test and its exact rescan keep their meaning on that set.  257 = no cut (distances are <= 256).
static int bow_distance_cut(int th_low, float nnratio) {
  if (!(nnratio > 0.f) || th_low < 0) return 257;
  double c = floor((double)th_low / (double)nnratio) + 2.0;
  if (c < th_low + 2.0) c = th_low + 2.0;  // (a ratio above 1: every distance up to TH_LOW can still be an accepted best)
  return c < 257.0 ? (int)c : 257;
}

extern "C" int b2s_debug_bow_distance_cut(int th_low, float nnratio) { return bow_distance_cut(th_low, nnratio); }

// device-resident, batched core (asynchronous)
extern "C" int b2s_search_by_bow_device(b2s_matcher* h, int batch, const uint8_t* d_descA, const int32_t* d_nodeA,
                                        const uint8_t* d_validA, const float* d_angA, const int32_t* d_nA, int capA,
                                        const uint8_t* d_descB, const int32_t* d_nodeB, const uint8_t* d_validB,
                                        const float* d_angB, const int32_t* d_nB, int capB, int th_low, float nnratio,
                                        int strict_lt, int check_ori, int32_t* d_matchB, int32_t* d_nmatches,
                                        void* stream) {
  if (!h || batch < 1 || batch > h->maxBatch || capA < 1 || capB < 1 || capA > h->maxF || capB > h->maxF || !d_descA ||
      !d_nodeA || !d_angA || !d_nA || !d_descB || !d_nodeB || !d_angB || !d_nB || !d_matchB || !d_nmatches) {
    set_error("b2s_search_by_bow_device: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
  MatchParams mp{th_low, nnratio, strict_lt, check_ori};
  k_fill_i32<<<div_up(batch * capB, 256), 256, 0, st>>>(d_matchB, -1, (size_t)batch * capB);
  k_rank_by_key<<<dim3(div_up(capA, 128), batch), 128, 0, st>>>(d_nodeA, d_nA, capA, h->dOrder);
  const int cut = bow_distance_cut(th_low, nnratio);
  k_bow_topk_imma<<<dim3(div_up(capA, BI_ROWS), batch), 128, 0, st>>>(d_descA, d_nodeA, d_validA, d_nA, capA, d_descB, d_nodeB,
                                                                     d_validB, d_nB, capB, cut, h->dTopk, h->dCandCnt);
  k_bow_resolve<<<dim3(div_up(capA, 4), batch), 128, 0, st>>>(d_descA, d_nodeA, d_validA, d_angA, d_nA, capA, d_descB,
                                                              d_nodeB, d_validB, d_angB, d_nB, capB, h->dOrder, h->dTopk,
                                                              h->dCandCnt, mp, d_matchB, h->dBin);
  k_rot_cull<<<batch, 256, 0, st>>>(d_nB, capB, check_ori, d_matchB, h->dBin, nullptr, d_nmatches);
  h->launches += 5;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

extern "C" int b2s_search_by_bow(b2s_matcher* h, const uint8_t* descA, const int32_t* nodeA, const uint8_t* validA,
                                 const float* angA, int nA, const uint8_t* descB, const int32_t* nodeB,
                                 const uint8_t* validB, const float* angB, int nB, int th_low, float nnratio,
                                 int strict_lt, int check_ori, int32_t* matchB, int* nmatches) {
  if (!h || nA < 0 || nB < 0 || nA > h->maxF || nB > h->maxF || !matchB || !nmatches) {
    set_error("b2s_search_by_bow: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  *nmatches = 0;
  for (int j = 0; j < nB; j++) matchB[j] = -1;
  if (nA == 0 || nB == 0) return B2S_OK;
  if (!descA || !nodeA || !angA || !descB || !nodeB || !angB) return B2S_ERR_BAD_ARG;
  return b2s_search_by_bow_batch(h, 1, descA, nodeA, validA, angA, &nA, nA, descB, nodeB, validB, angB, &nB, nB, th_low,
                                 nnratio, strict_lt, check_ori, matchB, nmatches);
}

extern "C" int b2s_search_by_bow_batch(b2s_matcher* h, int batch, const uint8_t* descA, const int32_t* nodeA,
                                       const uint8_t* validA, const float* angA, const int32_t* nA, int capA,
                                       const uint8_t* descB, const int32_t* nodeB, const uint8_t* validB,
                                       const float* angB, const int32_t* nB, int capB, int th_low, float nnratio,
                                       int strict_lt, int check_ori, int32_t* matchB, int32_t* nmatches) {
  if (!h || batch < 1 || batch > h->maxBatch || capA < 1 || capB < 1 || capA > h->maxF || capB > h->maxF || !descA ||
      !nodeA || !angA || !nA || !descB || !nodeB || !angB || !nB || !matchB || !nmatches) {
    set_error("b2s_search_by_bow_batch: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  for (int b = 0; b < batch; b++)
    if (nA[b] < 0 || nA[b] > capA || nB[b] < 0 || nB[b] > capB) return B2S_ERR_BAD_ARG;
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->stream;
  const size_t FA = (size_t)batch * capA, FB = (size_t)batch * capB;
  B2S_CUDA(cudaMemcpyAsync(h->dDescA, descA, FA * 32, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->dNodeA, nodeA, FA * 4, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->dAngA, angA, FA * 4, cudaMemcpyHostToDevice, st));
  if (validA) B2S_CUDA(cudaMemcpyAsync(h->dValidA, validA, FA, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->dDescB, descB, FB * 32, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->dNodeB, nodeB, FB * 4, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->dAngB, angB, FB * 4, cudaMemcpyHostToDevice, st));
  if (validB) B2S_CUDA(cudaMemcpyAsync(h->dValidB, validB, FB, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->dNA, nA, (size_t)batch * 4, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->dNB, nB, (size_t)batch * 4, cudaMemcpyHostToDevice, st));
  int rc = b2s_search_by_bow_device(h, batch, h->dDescA, h->dNodeA, validA ? h->dValidA : nullptr, h->dAngA, h->dNA, capA,
                                    h->dDescB, h->dNodeB, validB ? h->dValidB : nullptr, h->dAngB, h->dNB, capB, th_low,
                                    nnratio, strict_lt, check_ori, h->dMatch, h->dNMatches, st);
  if (rc != B2S_OK) return rc;
  B2S_CUDA(cudaMemcpyAsync(matchB, h->dMatch, FB * 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaMemcpyAsync(nmatches, h->dNMatches, (size_t)batch * 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaStreamSynchronize(st));
  return B2S_OK;
}

// ================================================================================================ projection searches
// Every projection search runs on a frame grid: a resident b2s_frame_grid, or the matcher's own work buffers seen as one
// (scratch_grid) for the host-buffer calls, which upload the frame's features and build the grid on every call.

// Grid bounds, cell scales (src/Frame.cc:213-214), bf and the level tables of one frame; a null table reads as zeros.
// th / mode / thHigh / checkOri / winFlags are left to each search.
static ProjGeom proj_geom(const b2s_frame_geom* g, const float* inv_level_sigma2) {
  ProjGeom pg;
  memset(&pg, 0, sizeof(pg));
  pg.minX = g->mnMinX; pg.minY = g->mnMinY; pg.maxX = g->mnMaxX; pg.maxY = g->mnMaxY;
  pg.invW = (float)GRID_COLS / (g->mnMaxX - g->mnMinX);
  pg.invH = (float)GRID_ROWS / (g->mnMaxY - g->mnMinY);
  pg.bf = g->bf; pg.nlevels = g->nlevels;
  for (int i = 0; i < 16 && i < g->nlevels; i++) {
    pg.scale[i] = g->scale_factors ? g->scale_factors[i] : 0.f;
    pg.invSigma2[i] = inv_level_sigma2 ? inv_level_sigma2[i] : 0.f;
  }
  return pg;
}

struct b2s_frame_grid {
  b2s_matcher* owner = nullptr;  // identity check only: never dereferenced after creation-time use by destroy
  int device = 0;
  int nf = 0;
  ProjGeom pg;  // geometry + scale tables (th / mode / thresholds are filled per search)
  float *kpx = nullptr, *kpy = nullptr, *ang = nullptr, *uright = nullptr;
  int32_t *oct = nullptr, *order = nullptr, *cellStart = nullptr, *cellKey = nullptr, *nB = nullptr, *qOut = nullptr;
  uint8_t* desc = nullptr;
};

// A grid of b2s_frame_grid_create*: the arrays above are its own buffers.
struct OwnedGrid : b2s_frame_grid {
  DevBuf own[11];
};

// The grid of a host-buffer search: it aliases the matcher's work buffers, owns nothing and is never passed to
// b2s_frame_grid_destroy.
static b2s_frame_grid scratch_grid(b2s_matcher* h, int nf, const ProjGeom& pg) {
  b2s_frame_grid gr;
  gr.owner = h; gr.device = h->device; gr.nf = nf; gr.pg = pg;
  gr.kpx = h->dKpx; gr.kpy = h->dKpy; gr.ang = h->dAngB; gr.uright = h->dURight; gr.oct = h->dOct; gr.desc = h->dDescB;
  gr.order = h->dOrder; gr.cellStart = h->dCellStart; gr.cellKey = h->dCellKey; gr.nB = h->dNB;
  return gr;
}

// Frame::AssignFeaturesToGrid (src/Frame.cc:461-491) on the arrays already in gr: cell key, stable rank, cell starts
static int grid_build(b2s_frame_grid& gr, cudaStream_t st) {
  const int nf = gr.nf;
  B2S_CUDA(cudaMemcpyAsync(gr.nB, &gr.nf, 4, cudaMemcpyHostToDevice, st));
  if (nf > 0) {
    k_proj_cell_key<<<div_up(nf, 256), 256, 0, st>>>(gr.kpx, gr.kpy, nf, gr.pg, gr.cellKey);
    k_rank_by_key<<<dim3(div_up(nf, 128), 1), 128, 0, st>>>(gr.cellKey, gr.nB, nf, gr.order);
  }
  k_proj_cell_start<<<div_up(nf + 1, 256), 256, 0, st>>>(gr.cellKey, gr.order, nf, gr.cellStart);
  gr.owner->launches += 3;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

// host feature arrays into gr, then grid_build.  A null angle or uright array is not uploaded: the searches that do not
// read it pass none.
static int grid_upload(b2s_frame_grid& gr, const float* kpx, const float* kpy, const int32_t* octave, const float* angle,
                       const float* uright, const uint8_t* desc, cudaStream_t st) {
  const size_t n = (size_t)gr.nf;
  if (n > 0) {
    B2S_CUDA(cudaMemcpyAsync(gr.kpx, kpx, n * 4, cudaMemcpyHostToDevice, st));
    B2S_CUDA(cudaMemcpyAsync(gr.kpy, kpy, n * 4, cudaMemcpyHostToDevice, st));
    B2S_CUDA(cudaMemcpyAsync(gr.oct, octave, n * 4, cudaMemcpyHostToDevice, st));
    if (angle) B2S_CUDA(cudaMemcpyAsync(gr.ang, angle, n * 4, cudaMemcpyHostToDevice, st));
    if (uright) B2S_CUDA(cudaMemcpyAsync(gr.uright, uright, n * 4, cudaMemcpyHostToDevice, st));
    B2S_CUDA(cudaMemcpyAsync(gr.desc, desc, n * 32, cudaMemcpyHostToDevice, st));
  }
  return grid_build(gr, st);
}

// The three searches on a built grid (nq > 0, gr.nf > 0): upload the queries and the occupancy flags, run, download.
// SearchByProjection(CurrentFrame, LastFrame) and relocalisation: 4 launches
static int proj_search_last(b2s_matcher* h, const b2s_frame_grid& gr, const b2s_proj_query* q, int nq, const uint8_t* occupied,
                            float th, int mode, int th_high, int check_ori, int32_t* match_cur, int* nmatches) {
  const int nf = gr.nf;
  cudaStream_t st = h->stream;
  ProjGeom pg = gr.pg;
  pg.th = th; pg.mode = mode; pg.thHigh = th_high; pg.checkOri = check_ori;
  const uint8_t* occ = occupied ? h->dOcc : nullptr;
  B2S_CUDA(cudaMemcpyAsync(h->dQueries, q, (size_t)nq * sizeof(ProjQuery), cudaMemcpyHostToDevice, st));
  if (occ) B2S_CUDA(cudaMemcpyAsync(h->dOcc, occupied, (size_t)nf, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemsetAsync(h->dTaken, 0, (size_t)nf, st));
  k_fill_i32<<<div_up(nf, 256), 256, 0, st>>>(h->dMatch, -1, (size_t)nf);
  k_proj_topk<ProjQuery><<<div_up(nq, 8), 256, 0, st>>>(h->dQueries, nq, gr.kpx, gr.kpy, gr.oct, gr.uright, occ, gr.desc,
                                                        gr.order, gr.cellStart, pg, h->dTopk, h->dTopkIdx, h->dCandCnt);
  k_proj_resolve<<<1, 32, 0, st>>>(h->dQueries, nq, gr.kpx, gr.kpy, gr.oct, gr.ang, gr.uright, occ, gr.desc, gr.order,
                                   gr.cellStart, pg, h->dTopk, h->dTopkIdx, h->dCandCnt, h->dTaken, h->dMatch, h->dPush,
                                   h->dExtra, h->dHist);
  k_proj_cull<<<1, 256, 0, st>>>(check_ori, h->dHist, h->dExtra, h->dMatch, h->dPush, h->dNMatches);
  h->launches += 4;
  B2S_CUDA(cudaGetLastError());
  B2S_CUDA(cudaMemcpyAsync(match_cur, h->dMatch, (size_t)nf * 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaMemcpyAsync(nmatches, h->dNMatches, 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaStreamSynchronize(st));
  return B2S_OK;
}

// SearchByProjection(Frame&, vector<MapPoint*>&, th): 3 launches
static int proj_search_map(b2s_matcher* h, const b2s_frame_grid& gr, const b2s_map_query* q, int nq, const uint8_t* occupied,
                           float th, int th_high, float nnratio, int32_t* match_cur, int* nmatches) {
  const int nf = gr.nf;
  cudaStream_t st = h->stream;
  ProjGeom pg = gr.pg;
  pg.th = th; pg.mode = 0; pg.thHigh = th_high; pg.checkOri = 0;
  const uint8_t* occ = occupied ? h->dOcc : nullptr;
  MapQuery* dQ = reinterpret_cast<MapQuery*>(h->dQueries);
  B2S_CUDA(cudaMemcpyAsync(dQ, q, (size_t)nq * sizeof(MapQuery), cudaMemcpyHostToDevice, st));
  if (occ) B2S_CUDA(cudaMemcpyAsync(h->dOcc, occupied, (size_t)nf, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemsetAsync(h->dTaken, 0, (size_t)nf, st));
  k_fill_i32<<<div_up(nf, 256), 256, 0, st>>>(h->dMatch, -1, (size_t)nf);
  k_proj_topk<MapQuery><<<div_up(nq, 8), 256, 0, st>>>(dQ, nq, gr.kpx, gr.kpy, gr.oct, gr.uright, occ, gr.desc, gr.order,
                                                       gr.cellStart, pg, h->dTopk, h->dTopkIdx, h->dCandCnt);
  k_map_resolve<<<1, 32, 0, st>>>(dQ, nq, gr.kpx, gr.kpy, gr.oct, gr.uright, occ, gr.desc, gr.order, gr.cellStart, pg, nnratio,
                                  h->dTopk, h->dTopkIdx, h->dCandCnt, h->dTaken, h->dMatch, h->dNMatches);
  h->launches += 3;
  B2S_CUDA(cudaGetLastError());
  B2S_CUDA(cudaMemcpyAsync(match_cur, h->dMatch, (size_t)nf * 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaMemcpyAsync(nmatches, h->dNMatches, 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaStreamSynchronize(st));
  return B2S_OK;
}

// window search core of Fuse / SearchByProjection(KeyFrame*, Scw, ...): 2 launches; only the greedy form reads occupancy
static int proj_search_windows(b2s_matcher* h, const b2s_frame_grid& gr, const b2s_win_query* q, int nq,
                               const uint8_t* occupied, int flags, int th_dist, int32_t* best_idx, int32_t* best_dist,
                               int* n_accepted) {
  const int nf = gr.nf;
  cudaStream_t st = h->stream;
  ProjGeom pg = gr.pg;
  pg.th = 1.f; pg.mode = 0; pg.thHigh = th_dist; pg.checkOri = 0; pg.winFlags = flags;
  const bool greedy = (flags & B2S_WIN_GREEDY) != 0;
  const uint8_t* occ = (greedy && occupied) ? h->dOcc : nullptr;
  WinQuery* dQ = reinterpret_cast<WinQuery*>(h->dQueries);
  B2S_CUDA(cudaMemcpyAsync(dQ, q, (size_t)nq * sizeof(WinQuery), cudaMemcpyHostToDevice, st));
  if (occ) B2S_CUDA(cudaMemcpyAsync(h->dOcc, occupied, (size_t)nf, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemsetAsync(h->dTaken, 0, (size_t)nf, st));
  B2S_CUDA(cudaMemsetAsync(h->dNMatches, 0, 4, st));
  k_proj_topk<WinQuery><<<div_up(nq, 8), 256, 0, st>>>(dQ, nq, gr.kpx, gr.kpy, gr.oct, gr.uright, occ, gr.desc, gr.order,
                                                       gr.cellStart, pg, h->dTopk, h->dTopkIdx, h->dCandCnt);
  // results: dMatch holds best_idx (nq <= maxF entries), dPush holds best_dist
  if (greedy)
    k_win_resolve<<<1, 32, 0, st>>>(dQ, nq, th_dist, gr.kpx, gr.kpy, gr.oct, gr.uright, occ, gr.desc, gr.order, gr.cellStart,
                                    pg, h->dTopk, h->dTopkIdx, h->dCandCnt, h->dTaken, h->dMatch, h->dPush, h->dNMatches);
  else
    k_win_pick<<<div_up(nq, 256), 256, 0, st>>>(nq, th_dist, h->dTopk, h->dTopkIdx, h->dMatch, h->dPush, h->dNMatches);
  h->launches += 2;
  B2S_CUDA(cudaGetLastError());
  B2S_CUDA(cudaMemcpyAsync(best_idx, h->dMatch, (size_t)nq * 4, cudaMemcpyDeviceToHost, st));
  if (best_dist) B2S_CUDA(cudaMemcpyAsync(best_dist, h->dPush, (size_t)nq * 4, cudaMemcpyDeviceToHost, st));
  int acc = 0;
  B2S_CUDA(cudaMemcpyAsync(&acc, h->dNMatches, 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaStreamSynchronize(st));
  if (n_accepted) *n_accepted = acc;
  return B2S_OK;
}

extern "C" int b2s_search_by_projection_last(b2s_matcher* h, const b2s_proj_query* q, int nq, const float* kpx,
                                             const float* kpy, const int32_t* octave, const float* angle,
                                             const float* uright, const uint8_t* occupied, const uint8_t* desc, int nf,
                                             const b2s_frame_geom* g, float th, int mode, int th_high, int check_ori,
                                             int32_t* match_cur, int* nmatches) {
  static_assert(sizeof(ProjQuery) == sizeof(b2s_proj_query), "query layout");
  if (!h || nq < 0 || nf < 0 || nq > h->maxF || nf > h->maxF || !match_cur || !nmatches || !g || !g->scale_factors ||
      g->nlevels < 1 || g->nlevels > 16) {
    set_error("b2s_search_by_projection_last: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  *nmatches = 0;
  for (int j = 0; j < nf; j++) match_cur[j] = -1;
  if (nq == 0 || nf == 0) return B2S_OK;
  if (!q || !kpx || !kpy || !octave || !angle || !uright || !desc) return B2S_ERR_BAD_ARG;
  B2S_CUDA(cudaSetDevice(h->device));
  b2s_frame_grid gr = scratch_grid(h, nf, proj_geom(g, nullptr));
  const int rc = grid_upload(gr, kpx, kpy, octave, angle, uright, desc, h->stream);
  if (rc != B2S_OK) return rc;
  return proj_search_last(h, gr, q, nq, occupied, th, mode, th_high, check_ori, match_cur, nmatches);
}

// ---------------------------------------------------------------- batched, device-resident SearchByProjection(Cur, Last)
// cv::KeyPoint-layout records -> the arrays the window search reads (one pair per blockIdx.y)
__global__ void k_proj_unpack(const b2s_keypoint* __restrict__ kps, const int32_t* __restrict__ nArr, int cap,
                              float* __restrict__ kpx, float* __restrict__ kpy, int32_t* __restrict__ oct,
                              float* __restrict__ ang) {
  const int pair = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= min(nArr[pair], cap)) return;
  const size_t o = (size_t)pair * cap + i;
  const b2s_keypoint k = kps[o];
  kpx[o] = k.x; kpy[o] = k.y; oct[o] = k.octave; ang[o] = k.angle;
}

// The projection half of SearchByProjection(CurrentFrame, LastFrame) (src/ORBmatcher.cc:1600-1626) for a stereo sequence:
// feature i of the last frame with a stereo depth z > 0 stands for the map point Frame::UnprojectStereo gives it
// (src/Frame.cc:679-696: x = (u-cx) z invfx, y = (v-cy) z invfy), moved into the current camera by the relative pose
// Tcl = [R | t] (3 x 4, row major) and projected (u = fx xc invzc + cx, :1614-1621).  Features without depth become skipped
// queries (invz < 0), like last-frame slots without a MapPoint (:1603-1606).  Single-precision, one rounding per operation.
__global__ void k_track_queries(const b2s_keypoint* __restrict__ kps, const uint8_t* __restrict__ desc,
                                const float* __restrict__ depth, const int32_t* __restrict__ nArr, int cap,
                                const float* __restrict__ Tcl, float fx, float fy, float cx, float cy, float invfx,
                                float invfy, int hasObs, ProjQuery* __restrict__ q, int32_t* __restrict__ nq) {
  const int pair = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = min(nArr[pair], cap);
  if (i == 0) nq[pair] = n;
  if (i >= n) return;
  const size_t o = (size_t)pair * cap + i;
  const b2s_keypoint k = kps[o];
  const float z = depth[o];
  ProjQuery Q;
  Q.u = 0.f; Q.v = 0.f; Q.invz = -1.f; Q.angle = k.angle; Q.octave = k.octave; Q.has_obs = hasObs;
  const uint4* d4 = reinterpret_cast<const uint4*>(desc + o * 32);
  if (z > 0.f) {
    const float* T = Tcl + (size_t)pair * 12;
    const float x = __fmul_rn(__fmul_rn(__fsub_rn(k.x, cx), z), invfx);
    const float y = __fmul_rn(__fmul_rn(__fsub_rn(k.y, cy), z), invfy);
    const float xc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[0], x), __fmul_rn(T[1], y)), __fmul_rn(T[2], z)), T[3]);
    const float yc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4], x), __fmul_rn(T[5], y)), __fmul_rn(T[6], z)), T[7]);
    const float zc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[8], x), __fmul_rn(T[9], y)), __fmul_rn(T[10], z)), T[11]);
    const float invzc = __fdiv_rn(1.0f, zc);
    if (!(invzc < 0.f)) {  // :1616-1617
      Q.u = __fadd_rn(__fmul_rn(__fmul_rn(fx, xc), invzc), cx);
      Q.v = __fadd_rn(__fmul_rn(__fmul_rn(fy, yc), invzc), cy);
      Q.invz = invzc;
    }
  }
  // (desc[] sits at byte 24 of the 56-byte record: 8-byte aligned only)
  const uint4 a = d4[0], b = d4[1];
  uint2* q2 = reinterpret_cast<uint2*>(Q.desc);
  q2[0] = make_uint2(a.x, a.y); q2[1] = make_uint2(a.z, a.w); q2[2] = make_uint2(b.x, b.y); q2[3] = make_uint2(b.z, b.w);
  q[o] = Q;
}

extern "C" int b2s_track_queries_device(b2s_matcher* h, int batch, const b2s_keypoint* d_kps_last, const uint8_t* d_desc_last,
                                        const float* d_depth_last, const int32_t* d_n_last, int cap, const float* d_Tcl,
                                        float fx, float fy, float cx, float cy, int has_obs, b2s_proj_query* d_q,
                                        int32_t* d_nq, void* stream) {
  if (!h || batch < 1 || batch > h->maxBatch || cap < 1 || cap > h->maxF || !d_kps_last || !d_desc_last || !d_depth_last ||
      !d_n_last || !d_Tcl || !d_q || !d_nq || !(fx != 0.f) || !(fy != 0.f)) {
    set_error("b2s_track_queries_device: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
  k_track_queries<<<dim3(div_up(cap, 128), batch), 128, 0, st>>>(d_kps_last, d_desc_last, d_depth_last, d_n_last, cap, d_Tcl,
                                                                 fx, fy, cx, cy, 1.0f / fx, 1.0f / fy, has_obs ? 1 : 0,
                                                                 reinterpret_cast<ProjQuery*>(d_q), d_nq);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

extern "C" int b2s_search_by_projection_last_device(b2s_matcher* h, int batch, const b2s_proj_query* d_q, const int32_t* d_nq,
                                                    int capQ, const b2s_keypoint* d_kps, const float* d_uright,
                                                    const uint8_t* d_desc, const int32_t* d_nf, int capF,
                                                    const b2s_frame_geom* g, float th, int mode, int th_high, int check_ori,
                                                    int32_t* d_match_cur, int32_t* d_nmatches, void* stream) {
  if (!h || batch < 1 || batch > h->maxBatch || capQ < 1 || capF < 1 || capQ > h->maxF || capF > h->maxF || !d_q || !d_nq ||
      !d_kps || !d_uright || !d_desc || !d_nf || !d_match_cur || !d_nmatches || !g || !g->scale_factors || g->nlevels < 1 ||
      g->nlevels > 16 || mode < 0 || mode > 2) {
    set_error("b2s_search_by_projection_last_device: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
  ProjGeom pg = proj_geom(g, nullptr);
  pg.th = th; pg.mode = mode; pg.thHigh = th_high; pg.checkOri = check_ori;
  pg.strideF = capF; pg.strideQ = capQ; pg.nfArr = d_nf; pg.nqArr = d_nq;
  const size_t FF = (size_t)batch * capF;
  const ProjQuery* dq = reinterpret_cast<const ProjQuery*>(d_q);
  B2S_CUDA(cudaMemsetAsync(h->dTaken, 0, FF, st));
  k_fill_i32<<<div_up((int)FF, 256), 256, 0, st>>>(d_match_cur, -1, FF);
  k_proj_unpack<<<dim3(div_up(capF, 256), batch), 256, 0, st>>>(d_kps, d_nf, capF, h->dKpx, h->dKpy, h->dOct, h->dAngB);
  k_proj_cell_key<<<dim3(div_up(capF, 256), batch), 256, 0, st>>>(h->dKpx, h->dKpy, capF, pg, h->dCellKey);
  k_rank_by_key<<<dim3(div_up(capF, 128), batch), 128, 0, st>>>(h->dCellKey, d_nf, capF, h->dOrder);
  k_proj_cell_start<<<dim3(div_up(capF + 1, 256), batch), 256, 0, st>>>(h->dCellKey, h->dOrder, capF, h->dCellStart, capF, d_nf);
  k_proj_topk<ProjQuery><<<dim3(div_up(capQ, 8), batch), 256, 0, st>>>(dq, capQ, h->dKpx, h->dKpy, h->dOct, d_uright, nullptr,
                                                                        d_desc, h->dOrder, h->dCellStart, pg, h->dTopk,
                                                                        h->dTopkIdx, h->dCandCnt);
  k_proj_resolve<<<dim3(1, batch), 32, 0, st>>>(dq, capQ, h->dKpx, h->dKpy, h->dOct, h->dAngB, d_uright, nullptr, d_desc,
                                                h->dOrder, h->dCellStart, pg, h->dTopk, h->dTopkIdx, h->dCandCnt, h->dTaken,
                                                d_match_cur, h->dPush, h->dExtra, h->dHist);
  k_proj_cull<<<dim3(1, batch), 256, 0, st>>>(check_ori, h->dHist, h->dExtra, d_match_cur, h->dPush, d_nmatches, capF, capQ);
  h->launches += 8;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

// host-buffer form of the batched search: one upload, the device path above, one download
extern "C" int b2s_search_by_projection_last_batch(b2s_matcher* h, int batch, const b2s_proj_query* q, const int32_t* nq, int capQ,
                                                   const b2s_keypoint* kps, const float* uright, const uint8_t* desc,
                                                   const int32_t* nf, int capF, const b2s_frame_geom* g, float th, int mode,
                                                   int th_high, int check_ori, int32_t* match_cur, int32_t* nmatches) {
  if (!h || batch < 1 || batch > h->maxBatch || capQ < 1 || capF < 1 || capQ > h->maxF || capF > h->maxF || !q || !nq ||
      !kps || !uright || !desc || !nf || !match_cur || !nmatches) {
    set_error("b2s_search_by_projection_last_batch: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  for (int b = 0; b < batch; b++)
    if (nq[b] < 0 || nq[b] > capQ || nf[b] < 0 || nf[b] > capF) return B2S_ERR_BAD_ARG;
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->stream;
  const size_t FQ = (size_t)batch * capQ, FF = (size_t)batch * capF;
  int rc = grow(h->dKpsStage, FF * sizeof(b2s_keypoint));
  if (rc != B2S_OK) return rc;
  const b2s_keypoint* dKps = (const b2s_keypoint*)h->dKpsStage.p;
  B2S_CUDA(cudaMemcpyAsync(h->dQueries, q, FQ * sizeof(ProjQuery), cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->dKpsStage.p, kps, FF * sizeof(b2s_keypoint), cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->dURight, uright, FF * 4, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->dDescB, desc, FF * 32, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->dNA, nq, (size_t)batch * 4, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->dNB, nf, (size_t)batch * 4, cudaMemcpyHostToDevice, st));
  rc = b2s_search_by_projection_last_device(h, batch, reinterpret_cast<const b2s_proj_query*>(h->dQueries), h->dNA, capQ,
                                            dKps, h->dURight, h->dDescB, h->dNB, capF, g, th, mode, th_high, check_ori,
                                            h->dMatch, h->dNMatches, st);
  if (rc != B2S_OK) return rc;
  B2S_CUDA(cudaMemcpyAsync(match_cur, h->dMatch, FF * 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaMemcpyAsync(nmatches, h->dNMatches, (size_t)batch * 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaStreamSynchronize(st));
  return B2S_OK;
}

// host-buffer form for a frame sequence: records of frames 0 .. batch (batch + 1 of them) are uploaded once, frame b + 1 is
// matched against frame b with the queries formed on the device (b2s_track_queries_device)
extern "C" int b2s_search_by_projection_sequence(b2s_matcher* h, int batch, const b2s_keypoint* kps, const uint8_t* desc,
                                                 const float* depth, const float* uright, const int32_t* n, int cap,
                                                 const float* Tcl, float fx, float fy, float cx, float cy, int has_obs,
                                                 const b2s_frame_geom* g, float th, int mode, int th_high, int check_ori,
                                                 int32_t* match_cur, int32_t* nmatches) {
  if (!h || batch < 1 || batch > h->maxBatch || cap < 1 || cap > h->maxF || !kps || !desc || !depth || !uright || !n || !Tcl ||
      !match_cur || !nmatches) {
    set_error("b2s_search_by_projection_sequence: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  for (int b = 0; b <= batch; b++)
    if (n[b] < 0 || n[b] > cap) return B2S_ERR_BAD_ARG;
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->stream;
  const size_t S = (size_t)(batch + 1) * cap, FF = (size_t)batch * cap;
  int rc = grow(h->dKpsStage, S * sizeof(b2s_keypoint));
  if (rc == B2S_OK) rc = grow(h->dSeqDesc, S * 32);
  if (rc == B2S_OK) rc = grow(h->dSeqDepth, S * 4);
  if (rc == B2S_OK) rc = grow(h->dSeqN, (size_t)(h->maxBatch + 1) * 4);
  if (rc == B2S_OK) rc = grow(h->dSeqT, (size_t)h->maxBatch * 12 * 4);
  if (rc != B2S_OK) return rc;
  const b2s_keypoint* dKps = (const b2s_keypoint*)h->dKpsStage.p;
  const uint8_t* dDesc = (const uint8_t*)h->dSeqDesc.p;
  const int32_t* dN = (const int32_t*)h->dSeqN.p;
  B2S_CUDA(cudaMemcpyAsync(h->dKpsStage.p, kps, S * sizeof(b2s_keypoint), cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->dSeqDesc.p, desc, S * 32, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->dSeqDepth.p, depth, S * 4, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->dURight, uright, FF * 4, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->dSeqN.p, n, (size_t)(batch + 1) * 4, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->dSeqT.p, Tcl, (size_t)batch * 12 * 4, cudaMemcpyHostToDevice, st));
  rc = b2s_track_queries_device(h, batch, dKps, dDesc, (const float*)h->dSeqDepth.p, dN, cap, (const float*)h->dSeqT.p, fx,
                                fy, cx, cy, has_obs, reinterpret_cast<b2s_proj_query*>(h->dQueries), h->dNA, st);
  if (rc != B2S_OK) return rc;
  rc = b2s_search_by_projection_last_device(h, batch, reinterpret_cast<const b2s_proj_query*>(h->dQueries), h->dNA, cap,
                                            dKps + cap, h->dURight, dDesc + (size_t)cap * 32, dN + 1, cap, g, th, mode, th_high,
                                            check_ori, h->dMatch, h->dNMatches, st);
  if (rc != B2S_OK) return rc;
  B2S_CUDA(cudaMemcpyAsync(match_cur, h->dMatch, FF * 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaMemcpyAsync(nmatches, h->dNMatches, (size_t)batch * 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaStreamSynchronize(st));
  return B2S_OK;
}

extern "C" int b2s_search_for_initialization(b2s_matcher* h, const float* prevx, const float* prevy, const int32_t* octave1,
                                             const float* angle1, const uint8_t* desc1, int n1, const float* kpx2,
                                             const float* kpy2, const int32_t* octave2, const float* angle2,
                                             const uint8_t* desc2, int n2, const b2s_frame_geom* g, int window, int th_low,
                                             float nnratio, int check_ori, int32_t* match12, int* nmatches) {
  static_assert(sizeof(WinQuery) == sizeof(b2s_win_query), "query layout");
  if (!h || n1 < 0 || n2 < 0 || n1 > h->maxF || n2 > h->maxF || !match12 || !nmatches || !g || window < 0) {
    set_error("b2s_search_for_initialization: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  *nmatches = 0;
  for (int i = 0; i < n1; i++) match12[i] = -1;
  if (n1 == 0 || n2 == 0) return B2S_OK;
  if (!prevx || !prevy || !octave1 || !angle1 || !desc1 || !kpx2 || !kpy2 || !octave2 || !angle2 || !desc2)
    return B2S_ERR_BAD_ARG;
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->stream;
  // one window query per F1 keypoint: level-0 keypoints only (:537), fixed radius, candidates of the same level (:541)
  std::vector<WinQuery> wq((size_t)n1);
  for (int i = 0; i < n1; i++) {
    WinQuery& Q = wq[i];
    memset(&Q, 0, sizeof(Q));
    Q.u = prevx[i];
    Q.v = prevy[i];
    Q.radius = (float)window;
    Q.min_level = octave1[i];
    Q.max_level = octave1[i];
    Q.valid = octave1[i] > 0 ? 0 : 1;
    memcpy(Q.desc, desc1 + (size_t)i * 32, 32);
  }
  ProjGeom pg = proj_geom(g, nullptr);
  pg.checkOri = check_ori;
  b2s_frame_grid gr = scratch_grid(h, n2, pg);
  WinQuery* dQ = reinterpret_cast<WinQuery*>(h->dQueries);
  int32_t* dMatchedDist = h->dNodeA;  // vMatchedDistance
  int32_t* dMatch21 = h->dBin;        // vnMatches21
  B2S_CUDA(cudaMemcpyAsync(dQ, wq.data(), (size_t)n1 * sizeof(WinQuery), cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemcpyAsync(h->dAngA, angle1, (size_t)n1 * 4, cudaMemcpyHostToDevice, st));
  B2S_CUDA(cudaMemsetAsync(h->dURight, 0, (size_t)n2 * 4, st));
  const int rc = grid_upload(gr, kpx2, kpy2, octave2, angle2, nullptr, desc2, st);
  if (rc != B2S_OK) return rc;
  B2S_CUDA(cudaStreamSynchronize(st));  // wq is a stack-owned staging vector
  k_fill_i32<<<div_up(n1, 256), 256, 0, st>>>(h->dMatch, -1, (size_t)n1);
  k_fill_i32<<<div_up(n2, 256), 256, 0, st>>>(dMatch21, -1, (size_t)n2);
  k_fill_i32<<<div_up(n2, 256), 256, 0, st>>>(dMatchedDist, 2147483647, (size_t)n2);
  k_proj_topk<WinQuery><<<div_up(n1, 8), 256, 0, st>>>(dQ, n1, h->dKpx, h->dKpy, h->dOct, h->dURight, nullptr, h->dDescB,
                                                       h->dOrder, h->dCellStart, pg, h->dTopk, h->dTopkIdx, h->dCandCnt);
  k_init_resolve<<<1, 32, 0, st>>>(dQ, n1, h->dAngA, h->dKpx, h->dKpy, h->dOct, h->dAngB, h->dURight, h->dDescB, h->dOrder,
                                   h->dCellStart, pg, th_low, nnratio, h->dTopk, h->dTopkIdx, h->dCandCnt, dMatchedDist,
                                   dMatch21, h->dMatch, h->dPush, h->dExtra, h->dHist);
  k_init_cull<<<1, 256, 0, st>>>(check_ori, n1, h->dHist, h->dExtra, h->dMatch, h->dPush, h->dNMatches);
  h->launches += 6;
  B2S_CUDA(cudaGetLastError());
  B2S_CUDA(cudaMemcpyAsync(match12, h->dMatch, (size_t)n1 * 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaMemcpyAsync(nmatches, h->dNMatches, 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaStreamSynchronize(st));
  return B2S_OK;
}

extern "C" int b2s_search_by_projection_map(b2s_matcher* h, const b2s_map_query* q, int nq, const float* kpx,
                                            const float* kpy, const int32_t* octave, const float* uright,
                                            const uint8_t* occupied, const uint8_t* desc, int nf, const b2s_frame_geom* g,
                                            float th, int th_high, float nnratio, int32_t* match_cur, int* nmatches) {
  static_assert(sizeof(MapQuery) == sizeof(b2s_map_query), "query layout");
  static_assert(sizeof(MapQuery) == sizeof(ProjQuery), "the query staging buffer is shared");
  if (!h || nq < 0 || nf < 0 || nq > h->maxF || nf > h->maxF || !match_cur || !nmatches || !g || !g->scale_factors ||
      g->nlevels < 1 || g->nlevels > 16) {
    set_error("b2s_search_by_projection_map: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  *nmatches = 0;
  for (int j = 0; j < nf; j++) match_cur[j] = -1;
  if (nq == 0 || nf == 0) return B2S_OK;
  if (!q || !kpx || !kpy || !octave || !uright || !desc) return B2S_ERR_BAD_ARG;
  for (int i = 0; i < nq; i++)
    if (q[i].in_view && (q[i].level < 0 || q[i].level >= g->nlevels)) {
      set_error("b2s_search_by_projection_map: query %d has a predicted level outside the scale table", i);
      return B2S_ERR_BAD_ARG;
    }
  B2S_CUDA(cudaSetDevice(h->device));
  b2s_frame_grid gr = scratch_grid(h, nf, proj_geom(g, nullptr));
  const int rc = grid_upload(gr, kpx, kpy, octave, nullptr, uright, desc, h->stream);
  if (rc != B2S_OK) return rc;
  return proj_search_map(h, gr, q, nq, occupied, th, th_high, nnratio, match_cur, nmatches);
}

extern "C" int b2s_search_windows(b2s_matcher* h, const b2s_win_query* q, int nq, const float* kpx, const float* kpy,
                                  const int32_t* octave, const float* uright, const float* inv_level_sigma2,
                                  const uint8_t* occupied, const uint8_t* desc, int nf, const b2s_frame_geom* g, int flags,
                                  int th_dist, int32_t* best_idx, int32_t* best_dist, int* n_accepted) {
  static_assert(sizeof(WinQuery) == sizeof(b2s_win_query), "query layout");
  if (!h || nq < 0 || nf < 0 || nq > h->maxF || nf > h->maxF || !best_idx || !g || g->nlevels < 1 || g->nlevels > 16 ||
      ((flags & B2S_WIN_CHI2) && !inv_level_sigma2)) {
    set_error("b2s_search_windows: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  if (n_accepted) *n_accepted = 0;
  for (int i = 0; i < nq; i++) {
    best_idx[i] = -1;
    if (best_dist) best_dist[i] = 256;
  }
  if (nq == 0 || nf == 0) return B2S_OK;
  if (!q || !kpx || !kpy || !octave || !uright || !desc) return B2S_ERR_BAD_ARG;
  B2S_CUDA(cudaSetDevice(h->device));
  b2s_frame_grid gr = scratch_grid(h, nf, proj_geom(g, inv_level_sigma2));
  const int rc = grid_upload(gr, kpx, kpy, octave, nullptr, uright, desc, h->stream);
  if (rc != B2S_OK) return rc;
  return proj_search_windows(h, gr, q, nq, occupied, flags, th_dist, best_idx, best_dist, n_accepted);
}

// ================================================================================================ persistent feature grid
extern "C" void b2s_frame_grid_destroy(b2s_frame_grid* gr) {
  if (!gr) return;
  cudaSetDevice(gr->device);
  delete static_cast<OwnedGrid*>(gr);
}

static int grid_alloc(b2s_matcher* h, int nf, const b2s_frame_geom* g, const float* inv_level_sigma2, b2s_frame_grid** out) {
  if (!h || !out || nf < 0 || nf > h->maxF || !g || !g->scale_factors || g->nlevels < 1 || g->nlevels > 16) {
    set_error("b2s_frame_grid_create: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  *out = nullptr;
  B2S_CUDA(cudaSetDevice(h->device));
  OwnedGrid* gr = new OwnedGrid();
  gr->owner = h;
  gr->device = h->device;
  gr->nf = nf;
  gr->pg = proj_geom(g, inv_level_sigma2);
  const size_t n = (size_t)std::max(nf, 1);
  int k = 0, rc = B2S_OK;
  auto A = [&](auto** p, size_t bytes) {  // array *p in the next of the grid's own buffers
    DevBuf& b = gr->own[k++];
    if (rc == B2S_OK) rc = grow(b, bytes);
    *(void**)p = b.p;
  };
  A(&gr->kpx, n * 4); A(&gr->kpy, n * 4); A(&gr->ang, n * 4); A(&gr->uright, n * 4);
  A(&gr->oct, n * 4); A(&gr->order, n * 4); A(&gr->cellKey, n * 4);
  A(&gr->cellStart, (GRID_COLS * GRID_ROWS + 2) * 4); A(&gr->nB, 4); A(&gr->qOut, (n + 1) * 4);
  A(&gr->desc, n * 32);
  if (rc != B2S_OK) {
    set_error("b2s_frame_grid_create: %s", g_last_error.c_str());
    b2s_frame_grid_destroy(gr);
    return B2S_ERR_CUDA;
  }
  *out = gr;
  return B2S_OK;
}

static int stream_sync(cudaStream_t st) {
  B2S_CUDA(cudaStreamSynchronize(st));
  return B2S_OK;
}

extern "C" int b2s_frame_grid_create(b2s_matcher* h, const float* kpx, const float* kpy, const int32_t* octave, const float* angle,
                                     const float* uright, const uint8_t* desc, int nf, const b2s_frame_geom* g,
                                     const float* inv_level_sigma2, b2s_frame_grid** out) {
  if (nf > 0 && (!kpx || !kpy || !octave || !angle || !uright || !desc)) return B2S_ERR_BAD_ARG;
  int rc = grid_alloc(h, nf, g, inv_level_sigma2, out);
  if (rc != B2S_OK) return rc;
  b2s_frame_grid* gr = *out;
  rc = grid_upload(*gr, kpx, kpy, octave, angle, uright, desc, h->stream);
  if (rc == B2S_OK) rc = stream_sync(h->stream);
  if (rc != B2S_OK) {
    b2s_frame_grid_destroy(gr);
    *out = nullptr;
  }
  return rc;
}

extern "C" int b2s_frame_grid_create_device(b2s_matcher* h, const b2s_keypoint* d_kps, const uint8_t* d_desc, int nf,
                                            const float* d_uright, const b2s_frame_geom* g, const float* inv_level_sigma2,
                                            void* stream, b2s_frame_grid** out) {
  if (nf > 0 && (!d_kps || !d_desc)) return B2S_ERR_BAD_ARG;
  int rc = grid_alloc(h, nf, g, inv_level_sigma2, out);
  if (rc != B2S_OK) return rc;
  b2s_frame_grid* gr = *out;
  cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
  if (nf > 0) {
    k_unpack_kps<<<div_up(nf, 256), 256, 0, st>>>(reinterpret_cast<const uint8_t*>(d_kps), nf, gr->kpx, gr->kpy, gr->oct, gr->ang);
    h->launches += 1;
    if (d_uright) B2S_CUDA(cudaMemcpyAsync(gr->uright, d_uright, (size_t)nf * 4, cudaMemcpyDeviceToDevice, st));
    else k_fill_i32<<<div_up(nf, 256), 256, 0, st>>>(reinterpret_cast<int32_t*>(gr->uright), (int)0xBF800000, (size_t)nf);  // -1.0f
    B2S_CUDA(cudaMemcpyAsync(gr->desc, d_desc, (size_t)nf * 32, cudaMemcpyDeviceToDevice, st));
  }
  rc = grid_build(*gr, st);
  if (rc == B2S_OK) rc = stream_sync(st);
  if (rc != B2S_OK) {
    b2s_frame_grid_destroy(gr);
    *out = nullptr;
  }
  return rc;
}

extern "C" int b2s_frame_grid_size(const b2s_frame_grid* gr) { return gr ? gr->nf : 0; }

extern "C" int b2s_frame_grid_features_in_area(b2s_frame_grid* gr, float x, float y, float r, int min_level, int max_level,
                                               int32_t* out, int cap, int* n) {
  if (!gr || !n || cap < 0 || (cap > 0 && !out)) return B2S_ERR_BAD_ARG;
  *n = 0;
  if (gr->nf == 0) return B2S_OK;
  b2s_matcher* h = gr->owner;
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->stream;
  const int c = std::min(cap, gr->nf);
  k_grid_query<<<1, 32, 0, st>>>(x, y, r, min_level, max_level, gr->kpx, gr->kpy, gr->oct, gr->uright, gr->order, gr->cellStart,
                                 gr->pg, gr->qOut + 1, c, gr->qOut);
  h->launches += 1;
  B2S_CUDA(cudaGetLastError());
  int cnt = 0;
  B2S_CUDA(cudaMemcpyAsync(&cnt, gr->qOut, 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaStreamSynchronize(st));
  *n = cnt;
  if (cnt > cap) {
    set_error("b2s_frame_grid_features_in_area: %d features, capacity %d", cnt, cap);
    return B2S_ERR_CAPACITY;
  }
  if (cnt > 0) B2S_CUDA(cudaMemcpy(out, gr->qOut + 1, (size_t)cnt * 4, cudaMemcpyDeviceToHost));
  return B2S_OK;
}

// the three projection searches on a resident grid: only the queries (and the occupancy flags) travel
extern "C" int b2s_search_by_projection_last_grid(b2s_matcher* h, b2s_frame_grid* gr, const b2s_proj_query* q, int nq,
                                                  const uint8_t* occupied, float th, int mode, int th_high, int check_ori,
                                                  int32_t* match_cur, int* nmatches) {
  if (!h || !gr || gr->owner != h || nq < 0 || nq > h->maxF || !match_cur || !nmatches) {
    set_error("b2s_search_by_projection_last_grid: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  const int nf = gr->nf;
  *nmatches = 0;
  for (int j = 0; j < nf; j++) match_cur[j] = -1;
  if (nq == 0 || nf == 0) return B2S_OK;
  if (!q) return B2S_ERR_BAD_ARG;
  B2S_CUDA(cudaSetDevice(h->device));
  return proj_search_last(h, *gr, q, nq, occupied, th, mode, th_high, check_ori, match_cur, nmatches);
}

extern "C" int b2s_search_by_projection_map_grid(b2s_matcher* h, b2s_frame_grid* gr, const b2s_map_query* q, int nq,
                                                 const uint8_t* occupied, float th, int th_high, float nnratio,
                                                 int32_t* match_cur, int* nmatches) {
  if (!h || !gr || gr->owner != h || nq < 0 || nq > h->maxF || !match_cur || !nmatches) {
    set_error("b2s_search_by_projection_map_grid: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  const int nf = gr->nf;
  *nmatches = 0;
  for (int j = 0; j < nf; j++) match_cur[j] = -1;
  if (nq == 0 || nf == 0) return B2S_OK;
  if (!q) return B2S_ERR_BAD_ARG;
  for (int i = 0; i < nq; i++)
    if (q[i].in_view && (q[i].level < 0 || q[i].level >= gr->pg.nlevels)) {
      set_error("b2s_search_by_projection_map_grid: query %d has a predicted level outside the scale table", i);
      return B2S_ERR_BAD_ARG;
    }
  B2S_CUDA(cudaSetDevice(h->device));
  return proj_search_map(h, *gr, q, nq, occupied, th, th_high, nnratio, match_cur, nmatches);
}

extern "C" int b2s_search_windows_grid(b2s_matcher* h, b2s_frame_grid* gr, const b2s_win_query* q, int nq,
                                       const uint8_t* occupied, int flags, int th_dist, int32_t* best_idx, int32_t* best_dist,
                                       int* n_accepted) {
  if (!h || !gr || gr->owner != h || nq < 0 || nq > h->maxF || !best_idx) {
    set_error("b2s_search_windows_grid: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  const int nf = gr->nf;
  if (n_accepted) *n_accepted = 0;
  for (int i = 0; i < nq; i++) {
    best_idx[i] = -1;
    if (best_dist) best_dist[i] = 256;
  }
  if (nq == 0 || nf == 0) return B2S_OK;
  if (!q) return B2S_ERR_BAD_ARG;
  B2S_CUDA(cudaSetDevice(h->device));
  return proj_search_windows(h, *gr, q, nq, occupied, flags, th_dist, best_idx, best_dist, n_accepted);
}

extern "C" int b2s_search_for_triangulation(b2s_matcher* h, const b2s_kf_features* kf1, const b2s_kf_features* kf2,
                                            const float* F12, float ex, float ey, const float* scale_factors,
                                            const float* level_sigma2, int nlevels, int only_stereo, int check_ori,
                                            int32_t* match12, int* nmatches) {
  if (!h || !kf1 || !kf2 || !F12 || !scale_factors || !level_sigma2 || nlevels < 1 || nlevels > 16 || !match12 ||
      !nmatches || kf1->n < 0 || kf2->n < 0 || kf1->n > h->maxF || kf2->n > h->maxF) {
    set_error("b2s_search_for_triangulation: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  const int nA = kf1->n, nB = kf2->n;
  *nmatches = 0;
  for (int i = 0; i < nA; i++) match12[i] = -1;
  if (nA == 0 || nB == 0) return B2S_OK;
  for (const b2s_kf_features* k : {kf1, kf2})
    if (!k->desc || !k->node || !k->has_mp || !k->stereo || !k->x || !k->y || !k->octave || !k->angle) return B2S_ERR_BAD_ARG;
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->stream;
  // eligibility on the host: no MapPoint, and a stereo observation when bOnlyStereo (:852-861, :877-885)
  std::vector<uint8_t> eA(nA), eB(nB);
  for (int i = 0; i < nA; i++) eA[i] = !kf1->has_mp[i] && (!only_stereo || kf1->stereo[i]);
  for (int j = 0; j < nB; j++) eB[j] = !kf2->has_mp[j] && (!only_stereo || kf2->stereo[j]);
  TriParams tp;
  memset(&tp, 0, sizeof(tp));
  for (int k = 0; k < 9; k++) tp.F12[k] = F12[k];
  tp.ex = ex; tp.ey = ey; tp.thLow = 50; tp.checkOri = check_ori;
  for (int l = 0; l < nlevels; l++) {
    tp.scale[l] = scale_factors[l];
    tp.sigma2[l] = level_sigma2[l];
  }
  const size_t F = (size_t)h->maxF * h->maxBatch;
  float* scratch = reinterpret_cast<float*>(h->dQueries);  // 16 floats per feature slot
  float *dxA = scratch, *dyA = scratch + F, *dxB = scratch + 2 * F, *dyB = scratch + 3 * F;
  uint8_t* dStA = reinterpret_cast<uint8_t*>(scratch + 4 * F);
  uint8_t* dStB = dStA + F;
  int32_t* dOrderB = h->dCandCnt;
  auto up = [&](void* d, const void* s, size_t bytes) { return cudaMemcpyAsync(d, s, bytes, cudaMemcpyHostToDevice, st); };
  B2S_CUDA(up(h->dDescA, kf1->desc, (size_t)nA * 32)); B2S_CUDA(up(h->dDescB, kf2->desc, (size_t)nB * 32));
  B2S_CUDA(up(h->dNodeA, kf1->node, (size_t)nA * 4)); B2S_CUDA(up(h->dNodeB, kf2->node, (size_t)nB * 4));
  B2S_CUDA(up(h->dValidA, eA.data(), nA)); B2S_CUDA(up(h->dValidB, eB.data(), nB));
  B2S_CUDA(up(dStA, kf1->stereo, nA)); B2S_CUDA(up(dStB, kf2->stereo, nB));
  B2S_CUDA(up(dxA, kf1->x, (size_t)nA * 4)); B2S_CUDA(up(dyA, kf1->y, (size_t)nA * 4));
  B2S_CUDA(up(dxB, kf2->x, (size_t)nB * 4)); B2S_CUDA(up(dyB, kf2->y, (size_t)nB * 4));
  B2S_CUDA(up(h->dOct, kf2->octave, (size_t)nB * 4));
  B2S_CUDA(up(h->dAngA, kf1->angle, (size_t)nA * 4)); B2S_CUDA(up(h->dAngB, kf2->angle, (size_t)nB * 4));
  B2S_CUDA(up(h->dNA, &nA, 4)); B2S_CUDA(up(h->dNB, &nB, 4));
  k_fill_i32<<<div_up(nB, 256), 256, 0, st>>>(h->dMatch, -1, (size_t)nB);
  k_rank_by_key<<<dim3(div_up(nA, 128), 1), 128, 0, st>>>(h->dNodeA, h->dNA, nA, h->dOrder);
  k_rank_by_key<<<dim3(div_up(nB, 128), 1), 128, 0, st>>>(h->dNodeB, h->dNB, nB, dOrderB);
  k_tri_match<<<div_up(nA, 4), 128, 0, st>>>(h->dDescA, h->dNodeA, h->dValidA, dStA, dxA, dyA, h->dAngA, nA, h->dOrder,
                                            h->dDescB, h->dNodeB, h->dValidB, dStB, dxB, dyB, h->dOct, h->dAngB, nB,
                                            dOrderB, tp, h->dMatch, h->dBin);
  k_rot_cull<<<1, 256, 0, st>>>(h->dNB, nB, check_ori, h->dMatch, h->dBin, nullptr, h->dNMatches);
  h->launches += 5;
  B2S_CUDA(cudaGetLastError());
  std::vector<int32_t> mB(nB);
  B2S_CUDA(cudaMemcpyAsync(mB.data(), h->dMatch, (size_t)nB * 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaMemcpyAsync(nmatches, h->dNMatches, 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaStreamSynchronize(st));
  for (int j = 0; j < nB; j++)
    if (mB[j] >= 0) match12[mB[j]] = j;  // every keyframe-2 feature is matched at most once (vbMatched2)
  return B2S_OK;
}

// ---------------------------------------------------------------- DBoW2 vocabulary
struct b2s_vocabulary : b2s::Stage {
  int k = 0, L = 0, nNodes = 0, nWords = 0;
  int32_t *dChildStart = nullptr, *dChildCount = nullptr, *dCNode = nullptr, *dWordOf = nullptr;
  uint8_t* dCDesc = nullptr;
  double* dWeight = nullptr;
  // scratch of the host-buffer entry point
  DevBuf dFeat, dWord, dNode, dW;
};

extern "C" void b2s_vocabulary_destroy(b2s_vocabulary* v) {
  if (!v) return;
  v->close();
  delete v;
}

extern "C" int b2s_vocabulary_create(const b2s_vocabulary_desc* d, int device, b2s_vocabulary** out) {
  if (!out || !d || d->n_nodes < 1 || !d->parent || !d->leaf_flag || !d->desc || !d->weight || d->k < 1 || d->L < 1) {
    set_error("b2s_vocabulary_create: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  *out = nullptr;
  int rc = select_device(device);
  if (rc != B2S_OK) return rc;
  const int N = d->n_nodes;
  // children in file order (loadFromTextFile :1378-1418), word ids to the flagged leaves in file order
  std::vector<int32_t> cnt(N, 0), start(N + 1, 0), wordOf(N, 0);
  int nWords = 0;
  for (int nid = 1; nid < N; nid++) {
    const int p = d->parent[nid];
    if (p < 0 || p >= nid) {
      set_error("b2s_vocabulary_create: node %d has parent %d (parents must precede their children)", nid, p);
      return B2S_ERR_BAD_ARG;
    }
    cnt[p]++;
    if (d->leaf_flag[nid]) wordOf[nid] = nWords++;
  }
  for (int i = 0; i < N; i++) start[i + 1] = start[i] + cnt[i];
  std::vector<int32_t> fill(start.begin(), start.end() - 1), cNode(std::max(N - 1, 1));
  std::vector<uint8_t> cDesc((size_t)std::max(N - 1, 1) * 32);
  for (int nid = 1; nid < N; nid++) {
    const int pos = fill[d->parent[nid]]++;
    cNode[pos] = nid;
    memcpy(&cDesc[(size_t)pos * 32], d->desc + (size_t)nid * 32, 32);
  }
  b2s_vocabulary* v = new b2s_vocabulary();
  v->k = d->k; v->L = d->L; v->nNodes = N; v->nWords = nWords;
  v->open(device);
  auto A = [v](auto** p, size_t bytes, const void* src) {
    v->alloc(*p, bytes);
    if (v->error == cudaSuccess) v->error = cudaMemcpy(*p, src, bytes, cudaMemcpyHostToDevice);
  };
  A(&v->dChildStart, (size_t)N * 4, start.data());
  A(&v->dChildCount, (size_t)N * 4, cnt.data());
  A(&v->dCNode, cNode.size() * 4, cNode.data());
  A(&v->dCDesc, cDesc.size(), cDesc.data());
  A(&v->dWordOf, (size_t)N * 4, wordOf.data());
  A(&v->dWeight, (size_t)N * 8, d->weight);
  if (v->error != cudaSuccess) {
    set_error("b2s_vocabulary_create: %s", cudaGetErrorString(v->error));
    b2s_vocabulary_destroy(v);
    return B2S_ERR_CUDA;
  }
  *out = v;
  return B2S_OK;
}

extern "C" int b2s_vocabulary_words(const b2s_vocabulary* v) { return v ? v->nWords : 0; }

extern "C" int b2s_bow_transform_device(b2s_vocabulary* v, const uint8_t* d_features, int n, int levelsup, int32_t* d_word_id,
                                        double* d_weight, int32_t* d_node_id, void* stream) {
  if (!v || n < 0 || !d_word_id || !d_node_id || (n && !d_features)) {
    set_error("b2s_bow_transform_device: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  if (n == 0) return B2S_OK;
  B2S_CUDA(cudaSetDevice(v->device));
  cudaStream_t st = stream ? (cudaStream_t)stream : v->stream;
  k_bow_transform<<<div_up(n, 128), 128, 0, st>>>(d_features, n, v->dChildStart, v->dChildCount, v->dCNode, v->dCDesc,
                                                v->dWordOf, v->dWeight, v->L - levelsup, d_word_id, d_weight, d_node_id);
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

extern "C" int b2s_bow_transform(b2s_vocabulary* v, const uint8_t* features, int n, int levelsup, int32_t* word_id,
                                 double* weight, int32_t* node_id) {
  if (!v || n < 0 || !word_id || !node_id || (n && !features)) {
    set_error("b2s_bow_transform: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  if (n == 0) return B2S_OK;
  B2S_CUDA(cudaSetDevice(v->device));
  const size_t c = std::max<size_t>(n, 4096);
  int rc = grow(v->dFeat, c * 32);
  if (rc == B2S_OK) rc = grow(v->dWord, c * 4);
  if (rc == B2S_OK) rc = grow(v->dNode, c * 4);
  if (rc == B2S_OK) rc = grow(v->dW, c * 8);
  if (rc != B2S_OK) return rc;
  cudaStream_t st = v->stream;
  B2S_CUDA(cudaMemcpyAsync(v->dFeat.p, features, (size_t)n * 32, cudaMemcpyHostToDevice, st));
  rc = b2s_bow_transform_device(v, (const uint8_t*)v->dFeat.p, n, levelsup, (int32_t*)v->dWord.p, (double*)v->dW.p,
                                (int32_t*)v->dNode.p, st);
  if (rc != B2S_OK) return rc;
  B2S_CUDA(cudaMemcpyAsync(word_id, v->dWord.p, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
  if (weight) B2S_CUDA(cudaMemcpyAsync(weight, v->dW.p, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaMemcpyAsync(node_id, v->dNode.p, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaStreamSynchronize(st));
  return B2S_OK;
}

extern "C" int b2s_distinctive_descriptors(b2s_matcher* h, const uint8_t* desc, const int32_t* offsets, int n_points,
                                           int32_t* best_idx) {
  if (!h || n_points < 0 || !best_idx || (n_points && !offsets)) {
    set_error("b2s_distinctive_descriptors: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  if (n_points == 0) return B2S_OK;
  const int total = offsets[n_points];
  if (total < 0 || (total && !desc)) return B2S_ERR_BAD_ARG;
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->stream;
  int rc = grow(h->dDistDesc, (size_t)std::max(total, 1) * 32);
  if (rc == B2S_OK) rc = grow(h->dDistOff, (size_t)(n_points + 1) * 4);
  if (rc == B2S_OK) rc = grow(h->dDistBest, (size_t)n_points * 4);
  if (rc != B2S_OK) return rc;
  uint8_t* dDesc = (uint8_t*)h->dDistDesc.p;
  int32_t *dOff = (int32_t*)h->dDistOff.p, *dBest = (int32_t*)h->dDistBest.p;
  cudaError_t e = cudaSuccess;
  if (total) e = cudaMemcpyAsync(dDesc, desc, (size_t)total * 32, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dOff, offsets, (size_t)(n_points + 1) * 4, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) {
    k_distinctive<<<div_up(n_points, 8), 256, 0, st>>>(dDesc, dOff, n_points, dBest);
    h->launches++;
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(best_idx, dBest, (size_t)n_points * 4, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    set_error("b2s_distinctive_descriptors: %s", cudaGetErrorString(e));
    return B2S_ERR_CUDA;
  }
  return B2S_OK;
}
