// extractor.cu — H100 (sm_90a) ORB extractor: per-cell minThFAST fallback, parallel order-preserving quadtree,
// intensity-centroid orientation, steered rBRIEF and the host side (pyramid, FAST strength and Q8 Gaussian blur are the
// fused front end of extractor_tile.cu).
//
// Replaces the body of ORBextractor::operator() (/root/reference/src/ORBextractor.cc:1544-1668) and the OpenCV
// primitives it calls.  Every stage is integer- or explicitly-rounded-float arithmetic so results are bit-identical
// to the reference CPU path (tests/test_extractor_gpu.py checks against oracle/).
#include <math.h>

#include <algorithm>
#include <mutex>

#include "extractor.cuh"

namespace b2s {

// rBRIEF pattern: 256 x (x0,y0,x1,y1) int8 (data/orb_pattern_31.inc; reference table src/ORBextractor.cc:231-489)
static const int8_t h_pattern[1024] = {
#include "../../data/orb_pattern_31.inc"
};
__constant__ int8_t c_pattern[1024];
__constant__ int c_umax[16];

// ------------------------------------------------------------------------------------------------
// K2: the minThFAST pass of the cells that the fused front end (extractor_tile.cu) found without a maximum above
//     iniThFAST: per listed 30-px cell of src/ORBextractor.cc:1089-1157 (cv::FAST on the cell ROI, :1126,1135) one CTA
//     computes the FAST-9/16 score, the 3x3 NMS and the ini->min threshold rule.
//     M = max over the 16 arcs of min|v-p| (same sign); corner at th <=> M > th; response = M-1.
// ------------------------------------------------------------------------------------------------
constexpr int FP = 80;   // byte pitch of the raw ROI / score map (ROI width <= 66, + alignment slack)
constexpr int FR = 68;   // max ROI rows
constexpr int PW = 40;   // word pitch of the packed pixel-pair planes (<= 38 pair words per row, even => 8-byte stores)
// a cell's detectable area is at most 60 x 62 (plan_geometry) and its strict 3x3 maxima take one pixel of each 2x2
// block at most, so the survivor list of fast_cell never overflows
static_assert(((60 + 1) / 2) * ((FR - 6 + 1) / 2) <= kFastCellCap, "fast_cell survivor list");

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void sts_v2(uint32_t a, uint32_t x, uint32_t y) {
  asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void sts_zero16(uint32_t a) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(a), "r"(0u) : "memory");
}

// FAST-9/16 arc strength of a horizontal PIXEL PAIR in packed 16-bit lanes (DPX VIMNMX3.U16x2).
// d'_k = 256 + v - p_k per lane (in [1,511], so one 32-bit subtract never borrows across lanes).
// dark  strength = max_s min_{j<9} d'_{s+j} - 256 ; bright strength = 256 - min_s max_{j<9} d'_{s+j}.
// Returns M(lo) | M(hi)<<16, each clamped at 0.  quick: exact reject through the 8 opposite pairs (k,k+8).
__device__ __forceinline__ void fast_pair_load(const uint32_t* __restrict__ E, const uint32_t* __restrict__ O, int wrd,
                                               uint32_t (&d)[16]) {
  // center pair starts at odd ROI x = 2*wrd+1 -> O plane word `wrd`.  Neighbour (dx,dy): dx even -> O[wrd + dx/2],
  // dx odd -> E[wrd + (dx+1)/2]; row offset dy*PW.
  const uint32_t vb = O[wrd] + 0x01000100u;
  d[0] = vb - O[3 * PW + wrd];        // ( 0, 3)
  d[1] = vb - E[3 * PW + wrd + 1];    // ( 1, 3)
  d[2] = vb - O[2 * PW + wrd + 1];    // ( 2, 2)
  d[3] = vb - E[1 * PW + wrd + 2];    // ( 3, 1)
  d[4] = vb - E[wrd + 2];             // ( 3, 0)
  d[5] = vb - E[-1 * PW + wrd + 2];   // ( 3,-1)
  d[6] = vb - O[-2 * PW + wrd + 1];   // ( 2,-2)
  d[7] = vb - E[-3 * PW + wrd + 1];   // ( 1,-3)
  d[8] = vb - O[-3 * PW + wrd];       // ( 0,-3)
  d[9] = vb - E[-3 * PW + wrd];       // (-1,-3)
  d[10] = vb - O[-2 * PW + wrd - 1];  // (-2,-2)
  d[11] = vb - E[-1 * PW + wrd - 1];  // (-3,-1)
  d[12] = vb - E[wrd - 1];            // (-3, 0)
  d[13] = vb - E[1 * PW + wrd - 1];   // (-3, 1)
  d[14] = vb - O[2 * PW + wrd - 1];   // (-2, 2)
  d[15] = vb - E[3 * PW + wrd];       // (-1, 3)
}

// exact reject through the 8 opposite pairs (k,k+8): true if either lane can still be a corner at minTh
__device__ __forceinline__ bool fast_pair_quick(const uint32_t (&d)[16], int minTh) {
  uint32_t dk = __vimin3_u16x2(__vmaxu2(d[0], d[8]), __vmaxu2(d[1], d[9]), __vmaxu2(d[2], d[10]));
  dk = __vimin3_u16x2(dk, __vmaxu2(d[3], d[11]), __vmaxu2(d[4], d[12]));
  dk = __vimin3_u16x2(dk, __vmaxu2(d[5], d[13]), __vmaxu2(d[6], d[14]));
  dk = __vminu2(dk, __vmaxu2(d[7], d[15]));
  uint32_t br = __vimax3_u16x2(__vminu2(d[0], d[8]), __vminu2(d[1], d[9]), __vminu2(d[2], d[10]));
  br = __vimax3_u16x2(br, __vminu2(d[3], d[11]), __vminu2(d[4], d[12]));
  br = __vimax3_u16x2(br, __vminu2(d[5], d[13]), __vminu2(d[6], d[14]));
  br = __vmaxu2(br, __vminu2(d[7], d[15]));
  // lane passes if dk-256 > minTh or 256-br > minTh
  const uint32_t thHi = (uint32_t)(256 + minTh) * 0x00010001u, thLo = (uint32_t)(256 - minTh) * 0x00010001u;
  return (__vcmpgtu2(dk, thHi) | __vcmpgtu2(thLo, br)) != 0u;
}

// M(lo) | M(hi)<<16 : max over the 16 arcs of min|v-p| (same sign), clamped at 0
__device__ __forceinline__ uint32_t fast_pair_full(const uint32_t (&d)[16]) {
  uint32_t t3n[16], t3x[16];
#pragma unroll
  for (int k = 0; k < 16; k++) {
    t3n[k] = __vimin3_u16x2(d[k], d[(k + 1) & 15], d[(k + 2) & 15]);
    t3x[k] = __vimax3_u16x2(d[k], d[(k + 1) & 15], d[(k + 2) & 15]);
  }
  uint32_t dark = 0u, bright = 0xFFFFFFFFu;
#pragma unroll
  for (int sft = 0; sft < 16; sft += 2) {
    const uint32_t a0 = __vimin3_u16x2(t3n[sft], t3n[(sft + 3) & 15], t3n[(sft + 6) & 15]);
    const uint32_t a1 = __vimin3_u16x2(t3n[sft + 1], t3n[(sft + 4) & 15], t3n[(sft + 7) & 15]);
    dark = __vimax3_u16x2(dark, a0, a1);
    const uint32_t b0 = __vimax3_u16x2(t3x[sft], t3x[(sft + 3) & 15], t3x[(sft + 6) & 15]);
    const uint32_t b1 = __vimax3_u16x2(t3x[sft + 1], t3x[(sft + 4) & 15], t3x[(sft + 7) & 15]);
    bright = __vimin3_u16x2(bright, b0, b1);
  }
  const int dl = (int)(dark & 0xffffu) - 256, dh = (int)(dark >> 16) - 256;
  const int bl = 256 - (int)(bright & 0xffffu), bh = 256 - (int)(bright >> 16);
  const int Ml = __vimax3_s32(dl, bl, 0), Mh = __vimax3_s32(dh, bh, 0);
  return (uint32_t)Ml | ((uint32_t)Mh << 16);
}

// one cell, one CTA of 128 threads (every early return is CTA-uniform: it depends on the cell geometry only)
__device__ __forceinline__ void fast_cell(const ExtractGeom& g, const uint8_t* __restrict__ pyr,
                                          const uint32_t* __restrict__ cellInfo, uint32_t* __restrict__ candXY,
                                          uint32_t* __restrict__ candKey, uint8_t* __restrict__ candResp,
                                          int32_t* __restrict__ candCount, int32_t* __restrict__ status, const int b,
                                          const int cid) {
  __shared__ __align__(16) uint8_t score[FR * FP];   // arc strength M per pixel, indexed by the ALIGNED column X
  __shared__ __align__(16) uint32_t planeE[FR * PW];  // (P[2i], P[2i+1])   P = pixels of the 4-byte aligned row
  __shared__ __align__(16) uint32_t planeO[FR * PW];  // (P[2i+1], P[2i+2])
  __shared__ uint32_t list[1024];
  __shared__ int sN, sHi, sBase, sEmit, sPass;
  const uint32_t info = cellInfo[cid];  // level | cell row | cell column (built with the geometry)
  const int l = info >> 28, ci = (info >> 14) & 0x3fff, cj = info & 0x3fff;
  const LevelGeom& L = g.lv[l];
  const int c = ci * L.nCols + cj;
  const int iniY = kMinBorder + ci * L.hCell;
  int maxY = iniY + L.hCell + 6;
  if (iniY >= L.maxBY - 3) return;  // :1099
  if (maxY > L.maxBY) maxY = L.maxBY;
  const int iniX = kMinBorder + cj * L.wCell;
  int maxX = iniX + L.wCell + 6;
  if (iniX >= L.maxBX - 6) return;  // :1116
  if (maxX > L.maxBX) maxX = L.maxBX;
  const int rw = maxX - iniX, rh = maxY - iniY;
  if (rw < 7 || rh < 7) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // ---- pixel-pair planes straight from aligned 32-bit global loads (one word per lane, PRMT unpack, 8-byte stores).
  // Column coordinates below are ALIGNED columns X = x_roi + a0, with a0 = iniX & 3.
  const int a0 = iniX & 3;
  const int nWords = (a0 + rw + 4 + 3) >> 2;  // <= 19
  const int pitch = L.pitch;
  {
    // each warp owns rows warp, warp+4, ...; the (up to) nine global loads of a chunk are issued before any is
    // consumed, shared addresses are plain 32-bit offsets (one memory latency per chunk instead of one per row)
    const bool colOK = lane < nWords && (iniX - a0) + lane * 4 + 3 < pitch;
    const uint8_t* p0 = pyr + (size_t)b * g.pyrBytes + L.off + (size_t)(iniY + warp) * pitch + (iniX - a0) + lane * 4;
    const uint32_t eA = smem_u32(planeE) + (uint32_t)(warp * PW + 2 * lane) * 4u;
    const uint32_t oA = smem_u32(planeO) + (uint32_t)(warp * PW + 2 * lane) * 4u;
    for (int r0 = warp; r0 < rh; r0 += 36) {
      uint32_t wv[9];
#pragma unroll
      for (int i = 0; i < 9; i++) {
        const int r = r0 + 4 * i;
        wv[i] = 0u;
        if (colOK && r < rh) wv[i] = __ldg(reinterpret_cast<const uint32_t*>(p0 + (size_t)(r - warp) * pitch));
      }
#pragma unroll
      for (int i = 0; i < 9; i++) {
        const int r = r0 + 4 * i;
        if (r >= rh) break;  // (warp-uniform)
        const uint32_t w0 = wv[i];
        const uint32_t wn = __shfl_down_sync(0xffffffffu, w0, 1);
        if (lane < nWords) {
          const uint32_t rowOff = (uint32_t)(r - warp) * (PW * 4u);
          sts_v2(eA + rowOff, __byte_perm(w0, 0u, 0x4140), __byte_perm(w0, 0u, 0x4342));             // (b0,b1) (b2,b3)
          sts_v2(oA + rowOff, __byte_perm(w0, 0u, 0x4241), (w0 >> 24) | ((wn & 0xffu) << 16));        // (b1,b2) (b3,b4)
        }
      }
    }
    const uint32_t sA = smem_u32(score);
    for (int k = tid; k < (rh * FP) / 16; k += 128) sts_zero16(sA + (uint32_t)k * 16u);
  }
  if (tid == 0) {
    sN = 0;
    sHi = 0;
    sPass = 0;
  }
  __syncthreads();
  // ---- arc strength, two pixels per thread.  Pass 1: load the 16 circle pairs and run the exact quick reject on every
  // pair; survivors go to a compact list.  Pass 2: the full 16-arc evaluation runs densely on the list.
  const int xLo = a0 + 3, xHi = a0 + rw - 3;        // interior columns [xLo, xHi)
  const int xFirst = (xLo & 1) ? xLo : xLo - 1;     // pairs start at odd aligned columns
  const int ih = rh - 6;
  const int npair = (xHi - xFirst + 1) >> 1;
  const int ppr = (npair <= 16) ? 16 : 32;          // lanes per row slot
  const int rowsPerPass = 4 * (32 / ppr);
  const int myRow = warp * (32 / ppr) + (ppr == 16 ? (lane >> 4) : 0);
  const int myPair = (ppr == 16) ? (lane & 15) : lane;
  for (int y0 = 0; y0 < ih; y0 += rowsPerPass) {
    const int y = y0 + myRow + 3;
    bool pass = false;
    uint32_t d[16];
    if (y < rh - 3 && myPair < npair) {
      fast_pair_load(&planeE[y * PW], &planeO[y * PW], (xFirst - 1) / 2 + myPair, d);  // X = xFirst + 2*myPair
      pass = fast_pair_quick(d, g.minTh);
    }
    const unsigned pm = __ballot_sync(0xffffffffu, pass);
    if (pm) {  // warp-aggregated append
      int base = 0;
      if (lane == 0) base = atomicAdd(&sPass, __popc(pm));
      base = __shfl_sync(0xffffffffu, base, 0);
      if (pass) {
        const int slot = base + __popc(pm & ((1u << lane) - 1u));
        if (slot < 1024) {
          list[slot] = (uint32_t)myPair | ((uint32_t)y << 8);
        } else {  // list full (only possible for very large cells): evaluate in place
          const uint32_t M2 = fast_pair_full(d);
          const int X = xFirst + 2 * myPair;
          if (X >= xLo) score[y * FP + X] = (uint8_t)min((int)(M2 & 0xffffu), 255);
          if (X + 1 < xHi) score[y * FP + X + 1] = (uint8_t)min((int)(M2 >> 16), 255);
        }
      }
    }
  }
  __syncthreads();
  {
    const int nPass = min(sPass, 1024);
    for (int k = tid; k < nPass; k += 128) {
      const uint32_t e = list[k];
      const int pr = e & 0xff, y = e >> 8;
      uint32_t d[16];
      fast_pair_load(&planeE[y * PW], &planeO[y * PW], (xFirst - 1) / 2 + pr, d);
      const uint32_t M2 = fast_pair_full(d);
      const int X = xFirst + 2 * pr;
      if (X >= xLo) score[y * FP + X] = (uint8_t)min((int)(M2 & 0xffffu), 255);
      if (X + 1 < xHi) score[y * FP + X + 1] = (uint8_t)min((int)(M2 >> 16), 255);
    }
  }
  __syncthreads();
  // ---- 3x3 NMS inside the cell's detectable area (rim scores are 0 == "not a corner" in OpenCV's buffers).
  // Only pixels of pairs that passed the quick test can have a non-zero score, so the NMS walks the pass list; the
  // survivors (X | y<<8 | M<<16) go to `surv`, which reuses the pixel-pair plane E (dead after pass 2).
  uint32_t* surv = planeE;
  const int minTh = g.minTh, iniTh = g.iniTh;
  auto nms_pair = [&](int pr, int y) -> uint32_t {  // two adjacent pixels can never both survive a strict 3x3 NMS
    uint32_t ent = 0;
#pragma unroll
    for (int h2 = 0; h2 < 2; h2++) {
      const int X = xFirst + 2 * pr + h2;
      if (X < xLo || X >= xHi) continue;
      const uint8_t* sc = &score[y * FP + X];
      const int M = sc[0];
      if (M <= minTh) continue;
      const int nb =
          max(max(max(sc[-FP - 1], sc[-FP]), max(sc[-FP + 1], sc[-1])), max(max(sc[1], sc[FP - 1]), max(sc[FP], sc[FP + 1])));
      if (M > nb) ent = (uint32_t)X | ((uint32_t)y << 8) | ((uint32_t)M << 16);
    }
    return ent;
  };
  auto append = [&](uint32_t ent) {  // warp-aggregated append of the survivors (all lanes call)
    const unsigned sm = __ballot_sync(0xffffffffu, ent != 0u);
    if (sm) {
      const unsigned hm = __ballot_sync(0xffffffffu, ent != 0u && (int)(ent >> 16) > iniTh);
      int base = 0;
      if (lane == 0) {
        base = atomicAdd(&sN, __popc(sm));
        if (hm) atomicAdd(&sHi, __popc(hm));
      }
      base = __shfl_sync(0xffffffffu, base, 0);
      if (ent) {
        const int slot = base + __popc(sm & ((1u << lane) - 1u));
        if (slot < 1024) surv[slot] = ent;
      }
    }
  };
  if (sPass <= 1024) {
    const int nPass = sPass;
    for (int k0 = 0; k0 < nPass; k0 += 128) {
      const int k = k0 + tid;
      uint32_t ent = 0;
      if (k < nPass) {
        const uint32_t e = list[k];
        ent = nms_pair((int)(e & 0xff), (int)(e >> 8));
      }
      append(ent);
    }
  } else {  // pass list overflowed (very large cells only): dense NMS over every pixel pair
    for (int y0 = 0; y0 < ih; y0 += rowsPerPass) {
      const int y = y0 + myRow + 3;
      uint32_t ent = 0;
      if (y < rh - 3 && myPair < npair) ent = nms_pair(myPair, y);
      append(ent);
    }
  }
  __syncthreads();
  const int nList = min(sN, 1024);
  const bool useHi = sHi > 0;  // cell produced corners at iniThFAST -> keep only those (:1132-1139)
  if (tid == 0) {
    sEmit = 0;
    const int nEmit = useHi ? sHi : sN;
    sBase = nEmit ? atomicAdd(&candCount[b * kMaxLevels + l], nEmit) : 0;
    if (sN > 1024 || (nEmit && sBase + nEmit > L.candCap)) atomicOr(status, 1);
  }
  __syncthreads();
  const size_t cbase = (size_t)b * g.totalCandCap + L.candOff;
  for (int k = tid; k < nList; k += 128) {
    const uint32_t e = surv[k];
    const int x = (int)(e & 0xff) - a0, y = (e >> 8) & 0xff, M = e >> 16;  // back to ROI columns
    if (useHi && M <= iniTh) continue;
    const int slot = sBase + atomicAdd(&sEmit, 1);
    if (slot >= L.candCap) continue;
    candXY[cbase + slot] = (uint32_t)(x + cj * L.wCell) | ((uint32_t)(y + ci * L.hCell) << 16);  // :1150-1151
    candKey[cbase + slot] = ((uint32_t)c << 12) | ((uint32_t)(y - 3) << 6) | (uint32_t)(x - 3);
    candResp[cbase + slot] = (uint8_t)(M - 1);
  }
}

// the fused front end's minThFAST fallback: only the cells listed by k_cells (those without a maximum above iniThFAST,
// src/ORBextractor.cc:1132-1139), persistent CTAs striding over the list
__global__ void __launch_bounds__(128) k_fast_cells_list(ExtractGeom g, const uint8_t* __restrict__ pyr,
                                                         const uint32_t* __restrict__ cellInfo,
                                                         uint32_t* __restrict__ candXY, uint32_t* __restrict__ candKey,
                                                         uint8_t* __restrict__ candResp, int32_t* __restrict__ candCount,
                                                         int32_t* __restrict__ status, const uint2* __restrict__ fbList,
                                                         const int32_t* __restrict__ fbCount) {
  const int n = *fbCount;
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    const uint2 e = fbList[i];  // (image, cell)
    fast_cell(g, pyr, cellInfo, candXY, candKey, candResp, candCount, status, (int)e.x, (int)e.y);
    __syncthreads();  // the cell's shared state is reused by the next one
  }
}

int launch_fast_fallback(const ExtractGeom& g, const DeviceBuffers& d, const uint2* fbList, const int32_t* fbCount, int gridCtas,
                         cudaStream_t st) {
  k_fast_cells_list<<<gridCtas, 128, 0, st>>>(g, d.pyr, d.cellInfo, d.candXY, d.candKey, d.candResp, d.candCount, d.status,
                                              fbList, fbCount);
  return B2S_OK;
}

// ------------------------------------------------------------------------------------------------
// K3: DistributeOctTree (src/ORBextractor.cc:706-1049) as a data-parallel, order-preserving emulation.
//     One CTA per (image, level).  The std::list is an array in list order; a pass over the list becomes:
//     histogram the keypoints of every splittable node into 4 quadrants, scan to get the new list positions
//     (children are push_front'ed -> the new front section is in reverse creation order, untouched nodes keep
//     their relative order behind it), relabel the keypoints.  The "expand largest first" phase (:929-1010)
//     sorts candidates by (count desc, creation order desc), prefix-sums the growth and cuts where size>=N.
//     The first-max-response-in-insertion-order rule (:1022-1045) is an atomicMax over (response, ~orderkey).
// ------------------------------------------------------------------------------------------------
struct QtNodes {
  int16_t *x0, *x1, *y0, *y1;
  int* cnt;
  uint8_t* created;
};

__device__ void warp0_excl_scan(int* a, int n, int* total) {  // call from all threads; caller syncs afterwards
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    const int chunk = (n + 31) / 32;
    const int beg = min(lane * chunk, n), end = min(beg + chunk, n);
    int s = 0;
    for (int i = beg; i < end; i++) s += a[i];
    const int incl = warp_incl_scan(s, lane);
    int run = incl - s;
    for (int i = beg; i < end; i++) {
      const int v = a[i];
      a[i] = run;
      run += v;
    }
    if (lane == 31) *total = incl;
  }
}

__device__ __forceinline__ int qt_quadrant(int x, int y, int x0, int x1, int y0, int y1) {
  const int mx = x0 + ((x1 - x0 + 1) >> 1);  // ceil(w/2), :641-642
  const int my = y0 + ((y1 - y0 + 1) >> 1);
  return (x < mx ? 0 : 1) + (y < my ? 0 : 2);  // n1=UL n2=UR n3=BL n4=BR
}

__global__ void __launch_bounds__(256) k_quadtree(ExtractGeom g, int capMax, const uint32_t* __restrict__ candXY,
                                                  const uint32_t* __restrict__ candKey,
                                                  const uint8_t* __restrict__ candResp, uint16_t* __restrict__ candNode,
                                                  uint8_t* __restrict__ candQ, const int32_t* __restrict__ candCount,
                                                  uint32_t* __restrict__ selXYR, int32_t* __restrict__ selCount,
                                                  int32_t* __restrict__ status) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int l = blockIdx.x, b = blockIdx.y;
  const LevelGeom& L = g.lv[l];
  const int tid = threadIdx.x, T = blockDim.x;
  const int n = min(candCount[b * kMaxLevels + l], L.candCap);
  int32_t* selCnt = selCount + b * kMaxLevels + l;
  if (n == 0) {
    if (tid == 0) *selCnt = 0;
    return;
  }
  const size_t cbase = (size_t)b * g.totalCandCap + L.candOff;
  const uint32_t* xy = candXY + cbase;
  const uint32_t* key = candKey + cbase;
  const uint8_t* resp = candResp + cbase;
  uint16_t* node = candNode + cbase;
  uint8_t* Q = candQ + cbase;
  const int CAP = capMax;
  // carve shared memory
  uint8_t* p = smem;
  unsigned long long* best = (unsigned long long*)p; p += sizeof(unsigned long long) * CAP;
  int* cc = (int*)p; p += sizeof(int) * CAP * 4;
  int* childPos = (int*)p; p += sizeof(int) * CAP * 4;
  int* newPos = (int*)p; p += sizeof(int) * CAP;
  int* aux1 = (int*)p; p += sizeof(int) * CAP;
  int* aux2 = (int*)p; p += sizeof(int) * CAP;
  int* aux3 = (int*)p; p += sizeof(int) * CAP;
  int* aux4 = (int*)p; p += sizeof(int) * CAP;
  QtNodes nb[2];
  for (int k = 0; k < 2; k++) {
    nb[k].cnt = (int*)p; p += sizeof(int) * CAP;
  }
  for (int k = 0; k < 2; k++) {
    nb[k].x0 = (int16_t*)p; p += 2 * CAP;
    nb[k].x1 = (int16_t*)p; p += 2 * CAP;
    nb[k].y0 = (int16_t*)p; p += 2 * CAP;
    nb[k].y1 = (int16_t*)p; p += 2 * CAP;
  }
  for (int k = 0; k < 2; k++) {
    nb[k].created = p; p += CAP;
  }
  __shared__ int sTot1, sTot2, sSize, sNToExpand, sFlag, sCut;
  int cur = 0;

  const int N = L.N;
  const int Hq = L.maxBY - kMinBorder;
  // ---- roots (:719-767) ----
  const int nIni = L.nIni;
  if (tid < nIni) {
    nb[0].x0[tid] = (int16_t)(int)__fmul_rn(L.hX, (float)tid);
    nb[0].x1[tid] = (int16_t)(int)__fmul_rn(L.hX, (float)(tid + 1));
    nb[0].y0[tid] = 0;
    nb[0].y1[tid] = (int16_t)Hq;
    nb[0].cnt[tid] = 0;
    nb[0].created[tid] = 0;
  }
  __syncthreads();
  for (int i = tid; i < n; i += T) {
    const int x = xy[i] & 0xffff;
    int r = (int)__fdiv_rn((float)x, L.hX);  // vpIniNodes[kp.pt.x/hX] :766
    r = min(r, nIni - 1);
    node[i] = (uint16_t)r;
    atomicAdd(&nb[0].cnt[r], 1);
  }
  __syncthreads();
  if (tid == 0) {  // erase empty roots, keep order (:771-786); nIni is tiny
    int m = 0;
    for (int r = 0; r < nIni; r++) {
      if (nb[0].cnt[r] > 0) {
        newPos[r] = m;
        nb[1].x0[m] = nb[0].x0[r]; nb[1].x1[m] = nb[0].x1[r];
        nb[1].y0[m] = nb[0].y0[r]; nb[1].y1[m] = nb[0].y1[r];
        nb[1].cnt[m] = nb[0].cnt[r];
        nb[1].created[m] = 0;
        m++;
      } else
        newPos[r] = 0;
    }
    sSize = m;
  }
  __syncthreads();
  for (int i = tid; i < n; i += T) node[i] = (uint16_t)newPos[node[i]];
  cur = 1;
  int size = sSize;
  __syncthreads();

  bool finish = false;
  bool overflow = false;
  while (!finish) {
    const int prevSize = size;
    QtNodes A = nb[cur], B = nb[cur ^ 1];
    // ---- full pass over the list (:801-905) ----
    for (int k = tid; k < size * 4; k += T) cc[k] = 0;
    if (tid == 0) sNToExpand = 0;
    __syncthreads();
    for (int i = tid; i < n; i += T) {
      const int nd = node[i];
      if (A.cnt[nd] > 1) {
        const uint32_t v = xy[i];
        const int q = qt_quadrant(v & 0xffff, v >> 16, A.x0[nd], A.x1[nd], A.y0[nd], A.y1[nd]);
        Q[i] = (uint8_t)q;
        atomicAdd(&cc[nd * 4 + q], 1);
      }
    }
    __syncthreads();
    for (int nd = tid; nd < size; nd += T) {
      const bool e = A.cnt[nd] > 1;
      const int nch = e ? ((cc[nd * 4] > 0) + (cc[nd * 4 + 1] > 0) + (cc[nd * 4 + 2] > 0) + (cc[nd * 4 + 3] > 0)) : 0;
      aux1[nd] = nch;
      aux3[nd] = nch;
      aux2[nd] = e ? 0 : 1;
    }
    __syncthreads();
    warp0_excl_scan(aux1, size, &sTot1);
    __syncthreads();
    warp0_excl_scan(aux2, size, &sTot2);
    __syncthreads();
    const int totalCh = sTot1, totalStay = sTot2;
    const int newSize = totalCh + totalStay;
    if (newSize > CAP) {
      overflow = true;
      break;
    }
    for (int nd = tid; nd < size; nd += T) {
      if (A.cnt[nd] > 1) {
        const int x0 = A.x0[nd], x1 = A.x1[nd], y0 = A.y0[nd], y1 = A.y1[nd];
        const int mx = x0 + ((x1 - x0 + 1) >> 1), my = y0 + ((y1 - y0 + 1) >> 1);
        int pos = totalCh - aux1[nd] - aux3[nd];
        for (int q = 3; q >= 0; q--) {  // n4 was pushed last -> frontmost
          const int cq = cc[nd * 4 + q];
          if (cq == 0) continue;
          B.x0[pos] = (int16_t)((q & 1) ? mx : x0);
          B.x1[pos] = (int16_t)((q & 1) ? x1 : mx);
          B.y0[pos] = (int16_t)((q & 2) ? my : y0);
          B.y1[pos] = (int16_t)((q & 2) ? y1 : my);
          B.cnt[pos] = cq;
          B.created[pos] = 1;
          childPos[nd * 4 + q] = pos;
          if (cq > 1) atomicAdd(&sNToExpand, 1);
          pos++;
        }
      } else {
        const int pos = totalCh + aux2[nd];
        B.x0[pos] = A.x0[nd]; B.x1[pos] = A.x1[nd];
        B.y0[pos] = A.y0[nd]; B.y1[pos] = A.y1[nd];
        B.cnt[pos] = A.cnt[nd];
        B.created[pos] = 0;
        newPos[nd] = pos;
      }
    }
    __syncthreads();
    for (int i = tid; i < n; i += T) {
      const int nd = node[i];
      node[i] = (uint16_t)((A.cnt[nd] > 1) ? childPos[nd * 4 + Q[i]] : newPos[nd]);
    }
    const int nToExpand = sNToExpand;
    __syncthreads();
    cur ^= 1;
    size = newSize;
    if (size >= N || size == prevSize) {
      finish = true;
    } else if (size + nToExpand * 3 > N) {
      // ---- expand-largest-first phase (:929-1010) ----
      while (!finish) {
        const int prevSize2 = size;
        QtNodes C = nb[cur], D = nb[cur ^ 1];
        for (int k = tid; k < size * 4; k += T) cc[k] = 0;
        __syncthreads();
        for (int i = tid; i < n; i += T) {
          const int nd = node[i];
          if (C.created[nd] && C.cnt[nd] > 1) {
            const uint32_t v = xy[i];
            const int q = qt_quadrant(v & 0xffff, v >> 16, C.x0[nd], C.x1[nd], C.y0[nd], C.y1[nd]);
            Q[i] = (uint8_t)q;
            atomicAdd(&cc[nd * 4 + q], 1);
          }
        }
        __syncthreads();
        // rank candidates by (count desc, list position asc == creation order desc)
        for (int a = tid; a < size; a += T) {
          const bool isC = C.created[a] && C.cnt[a] > 1;
          int r = -1;
          if (isC) {
            r = 0;
            const int ca = C.cnt[a];
            for (int o = 0; o < size; o++) {
              if (!(C.created[o] && C.cnt[o] > 1)) continue;
              const int co = C.cnt[o];
              r += (co > ca) || (co == ca && o < a);
            }
          }
          aux4[a] = r;  // rank of node a, -1 if not a candidate
        }
        for (int k = tid; k < size; k += T) aux1[k] = 0;
        if (tid == 0) sFlag = 0;
        __syncthreads();
        for (int a = tid; a < size; a += T) {
          const int r = aux4[a];
          if (r >= 0) {
            const int nch = (cc[a * 4] > 0) + (cc[a * 4 + 1] > 0) + (cc[a * 4 + 2] > 0) + (cc[a * 4 + 3] > 0);
            aux1[r] = nch;  // children in rank order
            aux3[r] = a;    // rank -> node
            atomicAdd(&sFlag, 1);
          }
        }
        __syncthreads();
        const int m = sFlag;  // number of candidates
        if (m == 0) {
          finish = true;  // nothing to split: size == prevSize
          break;
        }
        // inclusive prefix of children count in rank order (aux2), find the cut where size reaches N
        for (int k = tid; k < m; k += T) aux2[k] = aux1[k];
        __syncthreads();
        warp0_excl_scan(aux2, m, &sTot1);
        __syncthreads();
        if (tid == 0) sCut = m - 1;
        __syncthreads();
        for (int r = tid; r < m; r += T) {
          // size after processing ranks 0..r : size + sum(nch) - (r+1)
          const int after = size + aux2[r] + aux1[r] - (r + 1);
          if (after >= N) atomicMin(&sCut, r);
        }
        __syncthreads();
        const int cut = sCut;
        const int totalChP = aux2[cut] + aux1[cut];
        const int np = cut + 1;
        const int newSize2 = totalChP + (size - np);
        if (newSize2 > CAP) {
          overflow = true;
          break;
        }
        // unprocessed nodes keep their relative order behind the new children
        for (int a = tid; a < size; a += T) {
          const int r = aux4[a];
          newPos[a] = (r >= 0 && r <= cut) ? 0 : 1;
        }
        __syncthreads();
        warp0_excl_scan(newPos, size, &sTot2);
        __syncthreads();
        for (int a = tid; a < size; a += T) {
          const int r = aux4[a];
          if (r >= 0 && r <= cut) {
            const int x0 = C.x0[a], x1 = C.x1[a], y0 = C.y0[a], y1 = C.y1[a];
            const int mx = x0 + ((x1 - x0 + 1) >> 1), my = y0 + ((y1 - y0 + 1) >> 1);
            int pos = totalChP - (aux2[r] + aux1[r]);  // later-processed parents' children sit in front
            for (int q = 3; q >= 0; q--) {
              const int cq = cc[a * 4 + q];
              if (cq == 0) continue;
              D.x0[pos] = (int16_t)((q & 1) ? mx : x0);
              D.x1[pos] = (int16_t)((q & 1) ? x1 : mx);
              D.y0[pos] = (int16_t)((q & 2) ? my : y0);
              D.y1[pos] = (int16_t)((q & 2) ? y1 : my);
              D.cnt[pos] = cq;
              D.created[pos] = 1;
              childPos[a * 4 + q] = pos;
              pos++;
            }
          } else {
            const int pos = totalChP + newPos[a];
            D.x0[pos] = C.x0[a]; D.x1[pos] = C.x1[a];
            D.y0[pos] = C.y0[a]; D.y1[pos] = C.y1[a];
            D.cnt[pos] = C.cnt[a];
            D.created[pos] = 0;
            newPos[a] = pos;
          }
        }
        __syncthreads();
        for (int i = tid; i < n; i += T) {
          const int nd = node[i];
          const int r = aux4[nd];
          node[i] = (uint16_t)((r >= 0 && r <= cut) ? childPos[nd * 4 + Q[i]] : newPos[nd]);
        }
        __syncthreads();
        cur ^= 1;
        size = newSize2;
        if (size >= N || size == prevSize2) finish = true;
      }
      if (overflow) break;
    }
  }
  if (overflow) {
    if (tid == 0) {
      atomicOr(status, 4);
      *selCnt = 0;
    }
    return;
  }
  // ---- keep the best keypoint of every node (:1022-1045) ----
  for (int k = tid; k < size; k += T) best[k] = 0ull;
  __syncthreads();
  for (int i = tid; i < n; i += T) {
    const unsigned long long v = ((unsigned long long)(resp[i] + 1u) << 32) | (unsigned long long)(0xFFFFFFFFu - key[i]);
    atomicMax(&best[node[i]], v);
  }
  __syncthreads();
  uint32_t* sel = selXYR + ((size_t)b * g.totalSelCap + L.selOff) * 2;
  for (int k = tid; k < size; k += T) {
    const unsigned long long v = best[k];
    const uint32_t ky = 0xFFFFFFFFu - (uint32_t)(v & 0xFFFFFFFFull);
    const uint32_t r = (uint32_t)(v >> 32) - 1u;
    const int cell = ky >> 12, yl = (ky >> 6) & 63, xl = ky & 63;
    const int ci = cell / L.nCols, cj = cell - ci * L.nCols;
    const int x = cj * L.wCell + xl + 3 + kMinBorder;  // :1184-1185
    const int y = ci * L.hCell + yl + 3 + kMinBorder;
    sel[k * 2] = (uint32_t)x | ((uint32_t)y << 16);
    sel[k * 2 + 1] = r;
  }
  if (tid == 0) *selCnt = size;
}

// ------------------------------------------------------------------------------------------------
// K4+K5b: IC_Angle (:108-161) + cv::fastAtan2 (:160) + computeOrbDescriptor (:173-227), one warp per keypoint.
//      cosf/sinf restate glibc 2.39's FMA sincosf kernels operation by operation (DESIGN.md "float trig");
//      tap coordinates use unfused float mul/add and round-half-even, like the oracle's -ffp-contract=off build.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float dev_fast_atan2(float y, float x) {
  const float scale = (float)(180.0 / 3.14159265358979323846);
  const float p1 = 0.9997878412794807f * scale, p3 = -0.3258083974640975f * scale, p5 = 0.1555786518463281f * scale,
              p7 = -0.04432655554792128f * scale;
  const float eps = (float)2.2204460492503131e-16;
  const float ax = fabsf(x), ay = fabsf(y);
  float a, c, c2;
  if (ax >= ay) {
    c = __fdiv_rn(ay, __fadd_rn(ax, eps));
    c2 = __fmul_rn(c, c);
    a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
  } else {
    c = __fdiv_rn(ax, __fadd_rn(ay, eps));
    c2 = __fmul_rn(c, c);
    a = __fsub_rn(90.f,
                  __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c));
  }
  if (x < 0) a = __fsub_rn(180.f, a);
  if (y < 0) a = __fsub_rn(360.f, a);
  return a;
}

// glibc 2.39 x86_64 __sinf_fma/__cosf_fma for |y| < 120 (sysdeps/ieee754/flt-32/s_sincosf.h), verified
// exhaustively against libm over every float in [0, 2*pi] (tests/test_sincosf_mirror.py).
__device__ __forceinline__ double sc_sinpoly(double xs, double x2) {
  const double S1 = -0x1.555545995a603p-3, S2 = 0x1.1107605230bc4p-7, S3 = -0x1.994eb3774cf24p-13;
  const double s1 = __fma_rn(S3, x2, S2);
  const double x3 = __dmul_rn(x2, xs);
  const double x5 = __dmul_rn(x2, x3);
  const double s = __fma_rn(x3, S1, xs);
  return __fma_rn(s1, x5, s);
}
__device__ __forceinline__ double sc_cospoly(double x2, double sg) {
  const double C0 = 1.0, C1 = -0x1.ffffffd0c621cp-2, C2 = 0x1.55553e1068f19p-5, C3 = -0x1.6c087e89a359dp-10,
               C4 = 0x1.99343027bf8c3p-16;
  const double x4 = __dmul_rn(x2, x2);
  const double c1 = __fma_rn(sg * C1, x2, sg * C0);
  const double c2 = __fma_rn(sg * C4, x2, sg * C3);
  const double x6 = __dmul_rn(x2, x4);
  const double c = __fma_rn(x4, sg * C2, c1);
  return __fma_rn(c2, x6, c);
}
__device__ __forceinline__ void dev_sincosf(float y, float* sn, float* cs) {
  const double HPI_INV = 0x1.45f306dc9c883p+23, HPI = 0x1.921fb54442d18p+0;
  const double x = (double)y;
  const uint32_t t = (__float_as_uint(y) >> 20) & 0x7ff;
  if (t < 0x3f4) {
    const double x2 = __dmul_rn(x, x);
    if (t < 0x398) {
      *sn = y;
      *cs = 1.0f;
      return;
    }
    *sn = (float)sc_sinpoly(x, x2);
    *cs = (float)sc_cospoly(x2, 1.0);
    return;
  }
  const double r = __dmul_rn(x, HPI_INV);
  const int n = (__double2int_rz(r) + 0x800000) >> 24;
  const double xr = __fma_rn(-(double)n, HPI, x);
  const double x2 = __dmul_rn(xr, xr);
  const double sg = (n & 2) ? -1.0 : 1.0;
  const double sgn = ((n & 3) == 1 || (n & 3) == 2) ? -1.0 : 1.0;
  const double sp = sc_sinpoly(__dmul_rn(xr, sgn), x2);
  const double cp = sc_cospoly(x2, sg);
  if ((n & 1) == 0) {
    *sn = (float)sp;
    *cs = (float)cp;
  } else {
    *sn = (float)cp;
    *cs = (float)sp;
  }
}

__global__ void k_sincos_test(const float* __restrict__ in, int n, float* __restrict__ s, float* __restrict__ c) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dev_sincosf(in[i], &s[i], &c[i]);
}

__global__ void __launch_bounds__(256) k_orient_describe(ExtractGeom g, const uint8_t* __restrict__ pyr,
                                                         const uint8_t* __restrict__ blur,
                                                         const uint32_t* __restrict__ selXYR,
                                                         const int32_t* __restrict__ selCount,
                                                         b2s_keypoint* __restrict__ outKps, uint8_t* __restrict__ outDesc,
                                                         int32_t* __restrict__ outCounts, int cap,
                                                         int32_t* __restrict__ status) {
  __shared__ uint32_t pat[256];
  const int b = blockIdx.y;
  const int tid = threadIdx.x;
  {
    const int8_t* cp = c_pattern + tid * 4;
    pat[(tid & 7) * 32 + (tid >> 3)] = (uint32_t)(uint8_t)cp[0] | ((uint32_t)(uint8_t)cp[1] << 8) | ((uint32_t)(uint8_t)cp[2] << 16) |
               ((uint32_t)(uint8_t)cp[3] << 24);
  }
  __syncthreads();
  const int lane = tid & 31;
  const int wi = blockIdx.x * 8 + (tid >> 5);
  const int32_t* sc = selCount + b * kMaxLevels;
  if (wi == 0 && lane == 0) {
    int tot = 0;
    for (int k = 0; k < g.nlevels; k++) tot += sc[k];
    if (tot > cap) {
      atomicOr(status, 2);
      tot = cap;
    }
    outCounts[b] = tot;
  }
  if (wi >= g.totalSelCap) return;
  int l = 0;
  while (l + 1 < g.nlevels && wi >= g.lv[l + 1].selOff) l++;
  const LevelGeom& L = g.lv[l];
  const int idx = wi - L.selOff;
  if (idx >= sc[l]) return;
  int outIdx = idx;
  for (int k = 0; k < l; k++) outIdx += sc[k];
  if (outIdx >= cap) return;
  const uint32_t* sel = selXYR + ((size_t)b * g.totalSelCap + wi) * 2;
  const int cx = sel[0] & 0xffff, cy = sel[0] >> 16;
  const uint32_t resp = sel[1];
  // IC_Angle: m10 = sum u*I, m01 = sum v*I over the 31-row circular patch (lane = column)
  const uint8_t* img = pyr + (size_t)b * g.pyrBytes + L.off;
  int m01 = 0, m10 = 0;
  // all 31 row loads are independent: fully unrolled so that they are in flight together (integer sums: any order)
  const int pitch = L.pitch;
  const uint8_t* ctr = img + (size_t)cy * pitch + cx;
#pragma unroll
  for (int v = -kHalfPatch; v <= kHalfPatch; v++) {
    const int d = c_umax[v < 0 ? -v : v];
    const int u = lane - d;
    const int val = (u <= d) ? (int)ctr[v * pitch + u] : 0;
    m10 += u * val;
    m01 += v * val;
  }
  m01 = warp_reduce_sum(m01);
  m10 = warp_reduce_sum(m10);
  const float angle = dev_fast_atan2((float)m01, (float)m10);
  // steered BRIEF: lane i builds descriptor byte i from pattern pairs 8i..8i+7
  const float factorPI = (float)(3.14159265358979323846 / 180.f);
  float a, bsn;
  dev_sincosf(__fmul_rn(angle, factorPI), &bsn, &a);  // a = cos, b = sin (:181)
  const uint8_t* bl = blur + (size_t)b * g.pyrBytes + L.off + (size_t)cy * pitch + cx;
  uint32_t val = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const uint32_t pp = pat[k * 32 + lane];  // pair 8*lane+k, stored transposed (bank-conflict free)
    const float x0 = (float)(int8_t)(pp & 0xff), y0 = (float)(int8_t)((pp >> 8) & 0xff);
    const float x1 = (float)(int8_t)((pp >> 16) & 0xff), y1 = (float)(int8_t)(pp >> 24);
    const int r0 = __float2int_rn(__fadd_rn(__fmul_rn(x0, bsn), __fmul_rn(y0, a)));
    const int c0 = __float2int_rn(__fsub_rn(__fmul_rn(x0, a), __fmul_rn(y0, bsn)));
    const int r1 = __float2int_rn(__fadd_rn(__fmul_rn(x1, bsn), __fmul_rn(y1, a)));
    const int c1 = __float2int_rn(__fsub_rn(__fmul_rn(x1, a), __fmul_rn(y1, bsn)));
    const int t0 = bl[r0 * pitch + c0];
    const int t1 = bl[r1 * pitch + c1];
    val |= (uint32_t)(t0 < t1) << k;
  }
  // gather the 32 bytes into 8 words on lanes 0..7, then one 32-byte store from lane 0
  uint32_t w = val | (__shfl_down_sync(0xffffffffu, val, 1) << 8) | (__shfl_down_sync(0xffffffffu, val, 2) << 16) |
               (__shfl_down_sync(0xffffffffu, val, 3) << 24);
  u256 dsc;
#pragma unroll
  for (int k = 0; k < 8; k++) dsc.w[k] = __shfl_sync(0xffffffffu, w, k * 4);
  if (lane == 0) {
    st_u256(outDesc + ((size_t)b * cap + outIdx) * 32, dsc);
    b2s_keypoint kp;
    kp.x = (l != 0) ? __fmul_rn((float)cx, L.scale) : (float)cx;  // keypoint->pt *= scale (:1651-1660)
    kp.y = (l != 0) ? __fmul_rn((float)cy, L.scale) : (float)cy;
    kp.size = L.kpsize;
    kp.angle = angle;
    kp.response = (float)resp;
    kp.octave = l;
    kp.class_id = -1;
    outKps[(size_t)b * cap + outIdx] = kp;
  }
}

// ================================================================================================
// host side
// ================================================================================================
static inline int cv_roundf(float v) { return (int)lrintf(v); }
static inline int cv_floor(double v) {
  int i = (int)v;
  return i - (i > v);
}

static std::once_flag g_const_once[64];
static int upload_constants(int device) {
  int rc = B2S_OK;
  std::call_once(g_const_once[device & 63], [&]() {
    // umax (src/ORBextractor.cc:579-608)
    int umax[16];
    int v, v0, vmax = cv_floor(kHalfPatch * sqrt(2.f) / 2 + 1);
    int vminc = (int)ceil(kHalfPatch * sqrt(2.f) / 2);
    const double hp2 = kHalfPatch * kHalfPatch;
    for (v = 0; v < 16; v++) umax[v] = 0;
    for (v = 0; v <= vmax; ++v) umax[v] = (int)lrint(sqrt(hp2 - v * v));
    for (v = kHalfPatch, v0 = 0; v >= vminc; --v) {
      while (umax[v0] == umax[v0 + 1]) ++v0;
      umax[v] = v0;
      ++v0;
    }
    if (cudaMemcpyToSymbol(c_umax, umax, sizeof(umax)) != cudaSuccess) rc = B2S_ERR_CUDA;
    if (cudaMemcpyToSymbol(c_pattern, h_pattern, sizeof(h_pattern)) != cudaSuccess) rc = B2S_ERR_CUDA;
  });
  return rc;
}

static size_t quadtree_smem_bytes(int cap) {
  return (size_t)cap * (8 + 16 + 16 + 4 * 5 + 2 * 4 + 2 * 8 + 2) + 64;
}

// Level size (:1680-1682) and 30-px FAST cell grid (:1064-1086) of a WxH image at inverse scale s.  A level too small
// for the grid gets nCols or nRows <= 0.
static void level_grid(int W, int H, float s, LevelGeom& L) {
  L.w = cv_roundf((float)W * s);
  L.h = cv_roundf((float)H * s);
  L.maxBX = L.w - kEdge + 3;
  L.maxBY = L.h - kEdge + 3;
  const float width = (float)(L.maxBX - kMinBorder), height = (float)(L.maxBY - kMinBorder);
  L.nCols = (int)(width / 30.f);
  L.nRows = (int)(height / 30.f);
  L.wCell = L.nCols > 0 ? (int)ceilf(width / L.nCols) : 0;
  L.hCell = L.nRows > 0 ? (int)ceilf(height / L.nRows) : 0;
}

// Sum over the n cells of one grid row (or column) of ceil(d / 2), d = the extent of the cell's detectable area; cells
// the reference skips (:1099 with margin 3, :1116 with margin 6) count 0.  A strict 3x3 maximum of the cell NMS takes at
// most one pixel of each 2x2 block inside a cell, and the NMS never looks across a seam, so (column sum) x (row sum)
// bounds a level's candidates whatever the texture.  (ceil(band / 2) over the whole band is NOT a bound: two cells can
// both keep a maximum on their common seam.)
static int half_span_sum(int n, int cell, int maxB, int skipMargin) {
  int s = 0;
  for (int j = 0; j < n; j++) {
    const int ini = kMinBorder + j * cell;
    if (ini >= maxB - skipMargin) break;
    const int mx = std::min(ini + cell + 6, maxB);
    if (mx - ini >= 7) s += (mx - ini - 6 + 1) / 2;
  }
  return s;
}
static int cand_bound(const LevelGeom& L) {
  return half_span_sum(L.nCols, L.wCell, L.maxBX, 6) * half_span_sum(L.nRows, L.hCell, L.maxBY, 3);
}

// Builds per-level geometry for a WxH image (host arithmetic only) and checks it against the handle's allocations; the
// resize tables and the cell list go to the vectors for build_geometry to upload.
static int plan_geometry(b2s_extractor* h, int W, int H, std::vector<int16_t>& rxOfs, std::vector<uint32_t>& rxAlpha,
                         std::vector<int16_t>& ryOfs, std::vector<uint32_t>& ryBeta, std::vector<uint32_t>& info) {
  ExtractGeom& g = h->geom;
  memset(&g, 0, sizeof(g));
  g.nlevels = h->nlevels;
  g.iniTh = h->iniTh;
  g.minTh = h->minTh;
  uint32_t off = 0;
  int cellStart = 0, candOff = 0, selOff = 0;
  uint32_t rxOff = 0, ryOff = 0;
  for (int l = 0; l < g.nlevels; l++) {
    LevelGeom& L = g.lv[l];
    level_grid(W, H, h->invScale[l], L);
    L.pitch = (int)align_up((size_t)L.w, 16);
    L.off = off;
    off += (uint32_t)align_up((size_t)L.pitch * L.h, 256);
    if (L.nCols <= 0 || L.nRows <= 0) {
      set_error("pyramid level %d (%dx%d) is too small for the 30-px FAST cell grid", l, L.w, L.h);
      return B2S_ERR_BAD_ARG;
    }
    const float width = (float)(L.maxBX - kMinBorder), height = (float)(L.maxBY - kMinBorder);
    // (nCols = floor(width / 30) gives wCell <= 60; hCell <= 60 likewise: never refused, kept as the kernels' limits)
    if (L.wCell + 6 > 66 || L.hCell + 6 > FR || L.wCell > 63 || L.hCell > 63) {
      set_error("cell %dx%d at level %d exceeds the kernel tile", L.wCell, L.hCell, l);
      return B2S_ERR_BAD_ARG;
    }
    L.cellStart = cellStart;
    cellStart += L.nCols * L.nRows;
    L.N = h->nFeat[l];
    L.nIni = (int)roundf(width / height);  // :719 (C round)
    if (L.nIni < 1) {
      set_error("portrait level %dx%d: quadtree needs width >= height/2", L.w, L.h);
      return B2S_ERR_BAD_ARG;
    }
    L.hX = width / L.nIni;
    L.candCap = cand_bound(L);
    L.candOff = candOff;
    candOff += (int)align_up((size_t)L.candCap, 64);
    // k_cells: whole cells per CTA such that their maxima fit its shared list (>= 8: a cell is at most 60 x 60), the
    // row split into equal column ranges
    const int maxPerCta = std::min(kCellsMaxCols, kCellsListCap / (((L.wCell + 1) / 2) * ((L.hCell + 1) / 2)));
    L.nChunks = div_up(L.nCols, maxPerCta);
    L.cellsPerCta = div_up(L.nCols, L.nChunks);
    L.nodeCap = (int)align_up((size_t)std::max(L.N + 4, 4 * L.nIni), 8);
    L.selOff = selOff;
    selOff += L.nodeCap;
    L.scale = h->scale[l];
    L.kpsize = (float)(int)(kPatch * h->scale[l]);
    L.rxOff = rxOff;
    L.ryOff = ryOff;
    if (l > 0) {
      const LevelGeom& S = g.lv[l - 1];
      const double scale_x = 1. / ((double)L.w / S.w), scale_y = 1. / ((double)L.h / S.h);
      for (int dx = 0; dx < L.w; dx++) {
        float fx = (float)((dx + 0.5) * scale_x - 0.5);
        int sx = cv_floor(fx);
        fx -= sx;
        if (sx < 0) { fx = 0; sx = 0; }
        if (sx >= S.w - 1) { fx = 0; sx = S.w - 1; }
        rxOfs.push_back((int16_t)sx);
        const int16_t a0 = (int16_t)cv_roundf((1.f - fx) * 2048.f), a1 = (int16_t)cv_roundf(fx * 2048.f);
        rxAlpha.push_back((uint32_t)(uint16_t)a0 | ((uint32_t)(uint16_t)a1 << 16));
      }
      for (int dy = 0; dy < L.h; dy++) {
        float fy = (float)((dy + 0.5) * scale_y - 0.5);
        int sy = cv_floor(fy);
        fy -= sy;
        ryOfs.push_back((int16_t)sy);
        const int16_t b0 = (int16_t)cv_roundf((1.f - fy) * 2048.f), b1 = (int16_t)cv_roundf(fy * 2048.f);
        ryBeta.push_back((uint32_t)(uint16_t)b0 | ((uint32_t)(uint16_t)b1 << 16));
      }
      rxOff += L.w;
      ryOff += L.h;
    }
  }
  g.pyrBytes = off;
  g.totalCells = cellStart;
  info.assign(cellStart, 0u);
  for (int l = 0; l < g.nlevels; l++)
    for (int ci = 0; ci < g.lv[l].nRows; ci++)
      for (int cj = 0; cj < g.lv[l].nCols; cj++)
        info[g.lv[l].cellStart + ci * g.lv[l].nCols + cj] = ((uint32_t)l << 28) | ((uint32_t)ci << 14) | (uint32_t)cj;
  if ((size_t)cellStart > h->cellAlloc) {
    set_error("image %dx%d needs %d FAST cells, more than allocated", W, H, cellStart);
    return B2S_ERR_BAD_ARG;
  }
  g.totalCandCap = candOff;
  g.totalSelCap = selOff;
  if (g.pyrBytes > h->pyrBytesAlloc || (size_t)g.totalCandCap > h->candCapAlloc || (size_t)g.totalSelCap > h->selCapAlloc ||
      rxOfs.size() > h->rxAlloc || ryOfs.size() > h->ryAlloc) {
    set_error("image %dx%d exceeds the extractor's max_width/max_height (%dx%d)", W, H, h->maxW, h->maxH);
    return B2S_ERR_BAD_ARG;
  }
  int capMax = 0;
  for (int l = 0; l < g.nlevels; l++) capMax = std::max(capMax, g.lv[l].nodeCap);
  if (quadtree_smem_bytes(capMax) > 220 * 1024) {
    set_error("quadtree node capacity %d needs %zu B of shared memory", capMax, quadtree_smem_bytes(capMax));
    return B2S_ERR_BAD_ARG;
  }
  return B2S_OK;
}

// Builds the geometry of a WxH image and uploads its tables.  Until it succeeds the handle has no current size, so a
// refused image never leaves a half-built geometry behind for the next call.
static int build_geometry(b2s_extractor* h, int W, int H) {
  h->curW = h->curH = 0;
  std::vector<int16_t> rxOfs, ryOfs;
  std::vector<uint32_t> rxAlpha, ryBeta, info;
  const int rc0 = plan_geometry(h, W, H, rxOfs, rxAlpha, ryOfs, ryBeta, info);
  if (rc0 != B2S_OK) return rc0;
  const ExtractGeom& g = h->geom;
  B2S_CUDA(cudaMemcpy(h->d.cellInfo, info.data(), info.size() * 4, cudaMemcpyHostToDevice));
  if (!rxOfs.empty()) {
    B2S_CUDA(cudaMemcpyAsync(h->d.rxOfs, rxOfs.data(), rxOfs.size() * 2, cudaMemcpyHostToDevice, h->stream));
    B2S_CUDA(cudaMemcpyAsync(h->d.rxAlpha, rxAlpha.data(), rxAlpha.size() * 4, cudaMemcpyHostToDevice, h->stream));
    B2S_CUDA(cudaMemcpyAsync(h->d.ryOfs, ryOfs.data(), ryOfs.size() * 2, cudaMemcpyHostToDevice, h->stream));
    B2S_CUDA(cudaMemcpyAsync(h->d.ryBeta, ryBeta.data(), ryBeta.size() * 4, cudaMemcpyHostToDevice, h->stream));
    B2S_CUDA(cudaStreamSynchronize(h->stream));  // the host vectors die here
  }
  {
    int capMax = 0;
    for (int l = 0; l < g.nlevels; l++) capMax = std::max(capMax, g.lv[l].nodeCap);
    const size_t qsm = quadtree_smem_bytes(capMax);
    B2S_CUDA(cudaFuncSetAttribute(k_quadtree, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max(qsm, (size_t)49152)));
  }
  {
    const int rc = tile_build(h);
    if (rc != B2S_OK) return rc;
  }
  h->curW = W;
  h->curH = H;
  return B2S_OK;
}

static void b2s_extractor_timing_collect(b2s_extractor* h);

// per-image arrays advanced by `off` images (a chunk of a batch uses a disjoint slice of every buffer)
static DeviceBuffers shifted(const DeviceBuffers& d, const ExtractGeom& g, int off) {
  DeviceBuffers r = d;
  r.pyr += (size_t)off * g.pyrBytes;
  r.blur += (size_t)off * g.pyrBytes;
  r.candXY += (size_t)off * g.totalCandCap;
  r.candKey += (size_t)off * g.totalCandCap;
  r.candResp += (size_t)off * g.totalCandCap;
  r.candNode += (size_t)off * g.totalCandCap;
  r.candQ += (size_t)off * g.totalCandCap;
  r.candCount += (size_t)off * kMaxLevels;
  r.selXYR += (size_t)off * g.totalSelCap * 2;
  r.selCount += (size_t)off * kMaxLevels;
  return r;
}

// Dense host layout [image][row][width bytes] (one 1-D H2D copy per contiguous run of images; 2-D copies of 1241-byte
// rows run far below PCIe speed) -> level 0 of the pyramid (rows padded to 16 bytes, padding written as 0).
__global__ void __launch_bounds__(128) k_repitch(const uint8_t* __restrict__ raw, uint8_t* __restrict__ pyr, size_t pyrBytes,
                                                 uint32_t off0, int w, int h, int pitch, int bBase) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;  // destination word of the row
  const int y = blockIdx.y, b = blockIdx.z;
  if (4 * k >= pitch) return;
  const int rem = w - 4 * k;
  uint32_t v = 0;
  if (rem > 0) {
    const size_t o = ((size_t)(bBase + b) * h + y) * (size_t)w + 4 * (size_t)k;  // `raw` itself is 256-byte aligned
    const uint32_t* W = reinterpret_cast<const uint32_t*>(raw);
    const size_t a = o >> 2;
    v = __funnelshift_r(W[a], W[a + 1], (unsigned)(o & 3) * 8);
    if (rem < 4) v &= (1u << (8 * rem)) - 1u;
  }
  *reinterpret_cast<uint32_t*>(pyr + (size_t)b * pyrBytes + off0 + (size_t)y * pitch + 4 * k) = v;
}

// Upload `n` host images (each `height` rows of `width` bytes, row stride `stride`) into level 0 of images [b0, b0+n).
static int upload_level0(b2s_extractor* h, const uint8_t* const* imgs, int b0, int n, int width, int height, int stride,
                         cudaStream_t st) {
  const ExtractGeom& g = h->geom;
  if (stride != width || !h->d.raw) {
    for (int b = b0; b < b0 + n; b++)
      B2S_CUDA(cudaMemcpy2DAsync(h->d.pyr + (size_t)b * g.pyrBytes + g.lv[0].off, g.lv[0].pitch, imgs[b], stride, width,
                                 height, cudaMemcpyHostToDevice, st));
    return B2S_OK;
  }
  const size_t img = (size_t)width * height;
  for (int b = b0; b < b0 + n;) {
    int e = b + 1;
    while (e < b0 + n && imgs[e] == imgs[e - 1] + img) e++;  // contiguous run on the host
    B2S_CUDA(cudaMemcpyAsync(h->d.raw + (size_t)b * img, imgs[b], (size_t)(e - b) * img, cudaMemcpyHostToDevice, st));
    b = e;
  }
  k_repitch<<<dim3(div_up(g.lv[0].pitch / 4, 128), height, n), 128, 0, st>>>(
      h->d.raw, h->d.pyr + (size_t)b0 * g.pyrBytes, g.pyrBytes, g.lv[0].off, width, height, g.lv[0].pitch, b0);
  h->launches++;
  return B2S_OK;
}

// Enqueue the whole pipeline for `batch` images whose level-0 pixels are already in d.pyr.
static int run_pipeline(b2s_extractor* h, const DeviceBuffers& d, int batch, b2s_keypoint* dKps, uint8_t* dDesc,
                        int32_t* dCounts, int cap, cudaStream_t st, bool allowTiming = true) {
  const ExtractGeom& g = h->geom;
  B2S_CUDA(cudaMemsetAsync(d.candCount, 0, sizeof(int32_t) * kMaxLevels * batch, st));
  const bool tm = allowTiming && h->timing != 0;
  if (tm) {
    if (h->evPending) b2s_extractor_timing_collect(h);
    cudaEventRecord(h->ev[0], st);
  }
  // fused front end: per level one tile kernel (TMA-staged tile -> FAST strength map, blur, level l+1), then the per-cell
  // NMS / threshold rules.  `d` may be a slice of the handle's buffers: pass its image offset.
  const int bBase = (int)((size_t)(d.pyr - h->d.pyr) / g.pyrBytes);
  const int rc = tile_run(h, bBase, batch, st);
  if (rc != B2S_OK) return rc;
  if (tm) cudaEventRecord(h->ev[1], st);
  int capMax = 0;
  for (int l = 0; l < g.nlevels; l++) capMax = std::max(capMax, g.lv[l].nodeCap);
  const size_t qsm = quadtree_smem_bytes(capMax);
  k_quadtree<<<dim3(g.nlevels, batch), 256, qsm, st>>>(g, capMax, d.candXY, d.candKey, d.candResp, d.candNode, d.candQ,
                                                       d.candCount, d.selXYR, d.selCount, d.status);
  h->launches++;
  if (tm) cudaEventRecord(h->ev[2], st);
  k_orient_describe<<<dim3(div_up(g.totalSelCap, 8), batch), 256, 0, st>>>(g, d.pyr, d.blur, d.selXYR, d.selCount, dKps,
                                                                           dDesc, dCounts, cap, d.status);
  h->launches++;
  if (tm) {
    cudaEventRecord(h->ev[3], st);
    h->evPending = 1;
  }
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

static void b2s_extractor_timing_collect(b2s_extractor* h) {
  if (!h->evPending) return;
  static const int kSlot[3] = {1, 2, 4};  // stage slot of the span ev[k] -> ev[k + 1]: tiles + cells, quadtree, describe
  if (cudaEventSynchronize(h->ev[3]) != cudaSuccess) return;
  for (int k = 0; k < 3; k++) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, h->ev[k], h->ev[k + 1]) == cudaSuccess) h->stageMs[kSlot[k]] += ms;
  }
  h->timedCalls++;
  h->evPending = 0;
}

// ------------------------------------------------------------------------------------------------
// Frame::ComputeStereoMatches (src/Frame.cc:1026-1421) on the device-resident pyramids of a batch.
// ------------------------------------------------------------------------------------------------
struct StereoParams {
  float invScale[kMaxLevels];  // mvInvScaleFactors
  float bf, mb;
  int firstLeft, firstRight;   // image indices of pair 0 inside the batch (pair p = firstLeft+p, firstRight+p)
  int cap;
};
constexpr int ST_WARPS = 16;      // left keypoints per CTA
constexpr int ST_MAXR = 4096;     // right keypoints staged per CTA (cap is checked on the host)

// One warp per left keypoint.  Stage 1 (:1169-1219): the right keypoints whose row band [floor(y-r), ceil(y+r)],
// r = 2*scale[octave] (:1060-1097) contains the left keypoint's row, within one pyramid level and with uR in
// [uL-maxD, uL], minimum Hamming distance, first minimum in right-keypoint order.  Stage 2 (:1222-1391): 11x11 L1 block
// matching over +-5 px on the keypoint's own pyramid level, parabola fit, disparity gate.  sad = best SAD or -1.
__global__ void __launch_bounds__(ST_WARPS * 32) k_stereo_match(ExtractGeom g, StereoParams sp, const uint8_t* __restrict__ pyr,
                                                                const b2s_keypoint* __restrict__ kps,
                                                                const uint8_t* __restrict__ desc,
                                                                const int32_t* __restrict__ counts,
                                                                float* __restrict__ uRight, float* __restrict__ depth,
                                                                int32_t* __restrict__ sad) {
  __shared__ int16_t sMinr[ST_MAXR], sMaxr[ST_MAXR];
  __shared__ int8_t sOct[ST_MAXR];
  __shared__ float sU[ST_MAXR];
  const int pairI = blockIdx.y;
  const int imgL = sp.firstLeft + pairI, imgR = sp.firstRight + pairI;
  const int nL = min(counts[imgL], sp.cap), nR = min(counts[imgR], min(sp.cap, ST_MAXR));
  if ((int)(blockIdx.x * ST_WARPS) >= nL) {  // beyond the left image's features: "no match"
    const int i = blockIdx.x * ST_WARPS + (threadIdx.x >> 5);
    if ((threadIdx.x & 31) == 0 && i < sp.cap) {
      uRight[(size_t)pairI * sp.cap + i] = -1.0f;
      depth[(size_t)pairI * sp.cap + i] = -1.0f;
      sad[(size_t)pairI * sp.cap + i] = -1;
    }
    return;
  }
  const b2s_keypoint* kR = kps + (size_t)imgR * sp.cap;
  for (int j = threadIdx.x; j < nR; j += blockDim.x) {
    const b2s_keypoint k = kR[j];
    const float r = __fmul_rn(2.0f, g.lv[k.octave].scale);
    sMaxr[j] = (int16_t)(int)ceilf(__fadd_rn(k.y, r));
    sMinr[j] = (int16_t)(int)floorf(__fsub_rn(k.y, r));
    sOct[j] = (int8_t)k.octave;
    sU[j] = k.x;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * ST_WARPS + (threadIdx.x >> 5);
  if (i >= nL) {
    if (lane == 0 && i < sp.cap) {
      uRight[(size_t)pairI * sp.cap + i] = -1.0f;
      depth[(size_t)pairI * sp.cap + i] = -1.0f;
      sad[(size_t)pairI * sp.cap + i] = -1;
    }
    return;
  }
  const size_t oi = (size_t)pairI * sp.cap + i;
  const b2s_keypoint kL = kps[(size_t)imgL * sp.cap + i];
  const int levelL = kL.octave;
  const float uL = kL.x, vL = kL.y;
  const int row = (int)vL;  // vRowIndices[vL]
  const float minD = 0.f, maxD = __fdiv_rn(sp.bf, sp.mb);  // :1108-1112 (mb == 0 -> +inf)
  const float minU = __fsub_rn(uL, maxD), maxU = __fsub_rn(uL, minD);
  float outU = -1.0f, outD = -1.0f;
  int outSad = -1;
  // ---- stage 1
  uint32_t best = 0xFFFFFFFFu;
  if (!(maxU < 0) && row >= 0 && row < g.lv[0].h) {
    const u256 dL = ld_u256(desc + ((size_t)imgL * sp.cap + i) * 32);
    const uint8_t* dR = desc + (size_t)imgR * sp.cap * 32;
    for (int j = lane; j < nR; j += 32) {
      const int o = sOct[j];
      if (row < sMinr[j] || row > sMaxr[j] || o < levelL - 1 || o > levelL + 1) continue;
      const float uR = sU[j];
      if (!(uR >= minU && uR <= maxU)) continue;
      const uint32_t key = ((uint32_t)hamming256(dL, ld_u256(dR + (size_t)j * 32)) << 16) | (uint32_t)j;
      best = min(best, key);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
  const int bestDist = (best == 0xFFFFFFFFu) ? 256 : (int)(best >> 16);
  // dist < bestDist with bestDist initialised to TH_HIGH (:1166,1205); then bestDist < thOrbDist = (TH_HIGH+TH_LOW)/2
  if (bestDist < 100 && bestDist < (100 + 50) / 2) {
    // ---- stage 2
    const int bestIdxR = (int)(best & 0xFFFFu);
    const float uR0 = sU[bestIdxR];
    const float scaleFactor = sp.invScale[levelL];
    const float scaleduL = roundf(__fmul_rn(uL, scaleFactor));
    const float scaledvL = roundf(__fmul_rn(vL, scaleFactor));
    const float scaleduR0 = roundf(__fmul_rn(uR0, scaleFactor));
    const LevelGeom& LV = g.lv[levelL];
    const int w = 5, L = 5;
    const float iniu = scaleduR0 + L - w, endu = scaleduR0 + L + w + 1;
    const int cy = (int)scaledvL, cxL = (int)scaleduL, cxR0 = (int)scaleduR0;
    bool ok = !(iniu < 0 || endu >= (float)LV.w);  // :1290
    ok = ok && !(cy - w < 0 || cy + w >= LV.h || cxL - w < 0 || cxL + w >= LV.w || cxR0 - L - w < 0);  // cv::Mat range asserts
    if (ok) {
      const uint8_t* IL = pyr + (size_t)imgL * g.pyrBytes + LV.off;
      const uint8_t* IR = pyr + (size_t)imgR * g.pyrBytes + LV.off;
      const int pitch = LV.pitch;
      const int cL = IL[(size_t)cy * pitch + cxL];
      int aL[4], off[4];
#pragma unroll
      for (int t = 0; t < 4; t++) {
        const int p = lane + 32 * t;  // pixel of the 11x11 window
        const int dy = p / 11 - w, dx = p - (p / 11) * 11 - w;
        off[t] = (p < 121) ? (cy + dy) * pitch + dx : -1;
        aL[t] = (p < 121) ? (int)IL[off[t] + cxL] - cL : 0;
      }
      int bestSad = 0x7fffffff, bestinc = 0;
      int d0 = 0, d1 = 0, d2 = 0;  // SAD at bestinc-1, bestinc, bestinc+1
      int prev = 0;
      bool needNext = false;
#pragma unroll 1
      for (int incR = -L; incR <= L; incR++) {
        const int cxR = cxR0 + incR;
        const int cR = IR[(size_t)cy * pitch + cxR];
        int sum = 0;
#pragma unroll
        for (int t = 0; t < 4; t++)
          if (off[t] >= 0) sum += abs(aL[t] - ((int)IR[off[t] + cxR] - cR));
        sum = warp_reduce_sum(sum);
        sum = __shfl_sync(0xffffffffu, sum, 0);
        if (needNext) {
          d2 = sum;
          needNext = false;
        }
        if (sum < bestSad) {  // (float)dist < bestDist, strict: first minimum wins (:1308)
          bestSad = sum;
          bestinc = incR;
          d0 = prev;
          d1 = sum;
          needNext = true;
        }
        prev = sum;
      }
      if (!(bestinc == -L || bestinc == L)) {
        const float dist1 = (float)d0, dist2 = (float)d1, dist3 = (float)d2;
        const float deltaR =
            __fdiv_rn(__fsub_rn(dist1, dist3), __fmul_rn(2.0f, __fsub_rn(__fadd_rn(dist1, dist3), __fmul_rn(2.0f, dist2))));
        if (!(deltaR < -1 || deltaR > 1)) {
          float bestuR = __fmul_rn(LV.scale, __fadd_rn(__fadd_rn(scaleduR0, (float)bestinc), deltaR));
          float disparity = __fsub_rn(uL, bestuR);
          if (disparity >= minD && disparity < maxD) {
            if (disparity <= 0) {
              disparity = 0.01f;
              bestuR = (float)((double)uL - 0.01);
            }
            outD = __fdiv_rn(sp.bf, disparity);
            outU = bestuR;
            outSad = bestSad;
          }
        }
      }
    }
  }
  if (lane == 0) {
    uRight[oi] = outU;
    depth[oi] = outD;
    sad[oi] = outSad;
  }
}

// Median-based cull (:1395-1415): thDist = 1.5f*1.4f*median(SAD) over the accepted matches (element size/2 of the
// list sorted by (SAD, index)); matches with SAD >= thDist are removed.  One CTA per stereo pair.
__global__ void __launch_bounds__(1024) k_stereo_cull(StereoParams sp, const int32_t* __restrict__ counts,
                                                      float* __restrict__ uRight, float* __restrict__ depth,
                                                      const int32_t* __restrict__ sad, int32_t* __restrict__ nMatched) {
  __shared__ int32_t sSad[ST_MAXR];
  __shared__ int sM, sMedian, sKept;
  const int pairI = blockIdx.x;
  const int nL = min(counts[sp.firstLeft + pairI], min(sp.cap, ST_MAXR));
  const size_t base = (size_t)pairI * sp.cap;
  if (threadIdx.x == 0) {
    sM = 0;
    sMedian = 0;
    sKept = 0;
  }
  __syncthreads();
  int mine = 0;
  for (int i = threadIdx.x; i < nL; i += blockDim.x) {
    const int v = sad[base + i];
    sSad[i] = v;
    mine += v >= 0;
  }
  if (mine) atomicAdd(&sM, mine);
  __syncthreads();
  const int M = sM;
  if (M == 0) {
    if (threadIdx.x == 0) nMatched[pairI] = 0;
    return;
  }
  const int target = M / 2;
  for (int i = threadIdx.x; i < nL; i += blockDim.x) {
    const int v = sSad[i];
    if (v < 0) continue;
    int rank = 0;
    for (int j = 0; j < nL; j++) {
      const int u = sSad[j];
      rank += (u >= 0) && (u < v || (u == v && j < i));
    }
    if (rank == target) sMedian = v;
  }
  __syncthreads();
  const float thDist = __fmul_rn(__fmul_rn(1.5f, 1.4f), (float)sMedian);
  int kept = 0;
  for (int i = threadIdx.x; i < nL; i += blockDim.x) {
    const int v = sSad[i];
    if (v < 0) continue;
    if ((float)v < thDist) {
      kept++;
    } else {
      uRight[base + i] = -1.0f;
      depth[base + i] = -1.0f;
    }
  }
  if (kept) atomicAdd(&sKept, kept);
  __syncthreads();
  if (threadIdx.x == 0) nMatched[pairI] = sKept;
}

}  // namespace b2s

using namespace b2s;

extern "C" int b2s_extractor_set_timing(b2s_extractor* h, int enable) {
  if (!h) return B2S_ERR_BAD_ARG;
  B2S_CUDA(cudaSetDevice(h->device));
  if (enable && !h->ev[0])
    for (int k = 0; k < 4; k++) B2S_CUDA(cudaEventCreate(&h->ev[k]));
  b2s_extractor_timing_collect(h);
  h->timing = enable;
  for (int k = 0; k < 5; k++) h->stageMs[k] = 0;
  h->timedCalls = 0;
  return B2S_OK;
}

/* accumulated device milliseconds per stage since set_timing(1): resize chain, FAST, quadtree, blur, orient+describe;
 * the resize chain and the blur run inside the tile kernels, whose time is slot 1, so slots 0 and 3 stay 0 */
extern "C" int b2s_extractor_get_timing(b2s_extractor* h, double* stage_ms5, long long* calls) {
  if (!h || !stage_ms5) return B2S_ERR_BAD_ARG;
  B2S_CUDA(cudaSetDevice(h->device));
  b2s_extractor_timing_collect(h);
  for (int k = 0; k < 5; k++) stage_ms5[k] = h->stageMs[k];
  if (calls) *calls = h->timedCalls;
  return B2S_OK;
}

// scale tables and per-level quotas — src/ORBextractor.cc:500-554 (from h->nfeatures, nlevels, scaleFactor)
static void init_tables(b2s_extractor* h) {
  const int nlevels = h->nlevels;
  h->scale.resize(nlevels);
  h->sigma2.resize(nlevels);
  h->scale[0] = 1.0f;
  h->sigma2[0] = 1.0f;
  for (int i = 1; i < nlevels; i++) {
    h->scale[i] = (float)(h->scale[i - 1] * h->scaleFactor);
    h->sigma2[i] = h->scale[i] * h->scale[i];
  }
  h->invScale.resize(nlevels);
  h->invSigma2.resize(nlevels);
  for (int i = 0; i < nlevels; i++) {
    h->invScale[i] = 1.0f / h->scale[i];
    h->invSigma2[i] = 1.0f / h->sigma2[i];
  }
  h->nFeat.resize(nlevels);
  float factor = (float)(1.0f / h->scaleFactor);
  float nDesired = h->nfeatures * (1 - factor) / (1 - (float)pow((double)factor, (double)nlevels));
  int sum = 0;
  for (int l = 0; l < nlevels - 1; l++) {
    h->nFeat[l] = cv_roundf(nDesired);
    sum += h->nFeat[l];
    nDesired *= factor;
  }
  h->nFeat[nlevels - 1] = std::max(h->nfeatures - sum, 0);
}

// Per-image buffer sizes for images up to maxW x maxH, from the geometry arithmetic itself (no device access).  Level
// sizes grow monotonically with the image size, and so do the cell grid (nCols = floor((w - 32) / 30)) and the tile
// grid, so the largest image bounds every smaller one.  Candidates: plan_geometry gives each level its exact bound
// cand_bound, which is not monotonic in the size; the allocation uses a monotonic bound of it.
static void size_buffers(b2s_extractor* h) {
  size_t pyrBytes = 0, candCap = 0, selCap = 0, rx = 0, ry = 0, cells = 0, bmWords = 0, tiles = 0;
  for (int l = 0; l < h->nlevels; l++) {
    LevelGeom L;
    level_grid(h->maxW, h->maxH, h->invScale[l], L);
    pyrBytes += align_up(align_up((size_t)L.w, 16) * L.h, 256);
    // cand_bound's column sum adds ceil(d / 2) over at most nCols cells whose extents d sum to at most w - 38, so it is
    // <= (w - 38 + nCols) / 2, which grows with w (rows alike)
    const size_t colHalf = (size_t)std::max(L.w - 2 * kEdge + std::max(L.nCols, 0), 0) / 2;
    const size_t rowHalf = (size_t)std::max(L.h - 2 * kEdge + std::max(L.nRows, 0), 0) / 2;
    candCap += align_up(colHalf * rowHalf, 64);
    // quadtree nodes: plan_geometry's nodeCap = max(N + 4, 4 * nIni), nIni = round(width / height) with height >= 30
    const int nIniMax = std::max(1, (int)roundf((float)std::max(L.w - 2 * kMinBorder, 0) / 30.f));
    selCap += align_up((size_t)std::max({h->nFeat[l] + 4, 4 * nIniMax, 64}), 8);
    if (l > 0) {
      rx += L.w;
      ry += L.h;
    }
    cells += (size_t)std::max(L.nCols, 0) * (size_t)std::max(L.nRows, 0);
    bmWords += (size_t)(div_up(L.w, 128) * 4) * (size_t)(div_up(L.h, 32) * 32);  // tile_build: per 128 x 32 tile 4 x 32 words
    tiles = std::max(tiles, (size_t)(div_up(L.w, 128) + div_up(L.h, 32) + 2));
  }
  h->pyrBytesAlloc = pyrBytes + 4096;  // (slack for the 256-byte level alignment of smaller images)
  h->candCapAlloc = candCap;
  h->selCapAlloc = selCap + 64 * h->nlevels;
  h->rxAlloc = rx + 16;
  h->ryAlloc = ry + 16;
  h->cellAlloc = cells;
  h->bmWordsAlloc = bmWords;
  h->tileTabAlloc = tiles * h->nlevels;
  h->outCap = h->nfeatures + 4 * h->nlevels + 16;
}

/* test hook, host only (no device): the buffer sizes b2s_extractor_create gives a handle for max_width x max_height and
 * the geometry of a width x height image in it.  out[0..7]: candidate entries allocated / needed per image, FAST cells
 * allocated / needed, NMS bitmap words allocated, k_cells list capacity, k_cells cell columns per CTA at most,
 * k_fast_cells_list maxima per cell; then per level 8 entries: w, h, nCols, nRows, wCell, hCell, candCap, cellsPerCta.
 * Returns plan_geometry's status (B2S_ERR_BAD_ARG with b2s_last_error() for a refused image). */
extern "C" int b2s_debug_extractor_plan(int nfeatures, float scaleFactor, int nlevels, int max_width, int max_height, int width,
                                        int height, int64_t* out) {
  if (!out || nfeatures <= 0 || nlevels < 1 || nlevels > kMaxLevels || !(scaleFactor > 1.0f)) return B2S_ERR_BAD_ARG;
  b2s_extractor h;
  h.nfeatures = nfeatures;
  h.nlevels = nlevels;
  h.iniTh = 20;
  h.minTh = 7;
  h.scaleFactor = scaleFactor;
  h.maxW = max_width;
  h.maxH = max_height;
  h.maxBatch = 1;
  h.device = 0;
  init_tables(&h);
  size_buffers(&h);
  std::vector<int16_t> rxOfs, ryOfs;
  std::vector<uint32_t> rxAlpha, ryBeta, info;
  const int rc = plan_geometry(&h, width, height, rxOfs, rxAlpha, ryOfs, ryBeta, info);
  const ExtractGeom& g = h.geom;
  const int64_t head[8] = {(int64_t)h.candCapAlloc, g.totalCandCap, (int64_t)h.cellAlloc, g.totalCells, (int64_t)h.bmWordsAlloc,
                           kCellsListCap, kCellsMaxCols, kFastCellCap};
  for (int k = 0; k < 8; k++) out[k] = head[k];
  for (int l = 0; l < nlevels; l++) {
    const LevelGeom& L = g.lv[l];
    const int64_t v[8] = {L.w, L.h, L.nCols, L.nRows, L.wCell, L.hCell, L.candCap, L.cellsPerCta};
    for (int k = 0; k < 8; k++) out[8 + 8 * l + k] = v[k];
  }
  return rc;
}

extern "C" int b2s_extractor_create(int nfeatures, float scaleFactor, int nlevels, int iniThFAST, int minThFAST,
                                    int max_width, int max_height, int max_batch, int device, b2s_extractor** out) {
  if (!out) return B2S_ERR_BAD_ARG;
  *out = nullptr;
  if (nfeatures <= 0 || nlevels < 1 || nlevels > kMaxLevels || !(scaleFactor > 1.0f) || minThFAST < 1 ||
      iniThFAST < minThFAST || iniThFAST > 254 || max_width < 64 || max_height < 64 || max_width > 8192 ||
      max_height > 8192 || max_batch < 1) {
    set_error("b2s_extractor_create: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  int rc = select_device(device);
  if (rc != B2S_OK) return rc;
  rc = upload_constants(device);
  if (rc != B2S_OK) {
    set_error("constant upload failed");
    return rc;
  }
  int sms = 0;
  B2S_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  b2s_extractor* h = new b2s_extractor();
  h->numSMs = sms;
  h->nfeatures = nfeatures;
  h->nlevels = nlevels;
  h->iniTh = iniThFAST;
  h->minTh = minThFAST;
  h->scaleFactor = scaleFactor;  // `double scaleFactor` member initialised from the float ctor argument
  h->maxW = max_width;
  h->maxH = max_height;
  h->maxBatch = max_batch;
  h->device = device;
  init_tables(h);
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&h->stream2, cudaStreamNonBlocking) != cudaSuccess) {
    set_error("cudaStreamCreate failed");
    delete h;
    return B2S_ERR_CUDA;
  }
  size_buffers(h);
  const size_t candCap = h->candCapAlloc, selCap = h->selCapAlloc, pyrBytes = h->pyrBytesAlloc;
  DeviceBuffers& d = h->d;
  const size_t B = (size_t)max_batch;
  cudaError_t e = cudaSuccess;
  auto A = [&](void** p, size_t bytes) {
    if (e == cudaSuccess) e = cudaMalloc(p, bytes);
  };
  A((void**)&d.pyr, B * pyrBytes);
  A((void**)&d.blur, B * pyrBytes);
  A((void**)&d.score, B * pyrBytes);
  A((void**)&d.bitmap, B * h->bmWordsAlloc * 4);
  A((void**)&d.tileDx, h->tileTabAlloc * 2);
  A((void**)&d.tileDy, h->tileTabAlloc * 2);
  if (max_batch > 1) A((void**)&d.raw, B * (size_t)max_width * max_height + 64);  // dense upload staging (batch path)
  A((void**)&d.candXY, B * candCap * 4);
  A((void**)&d.candKey, B * candCap * 4);
  A((void**)&d.candResp, B * candCap);
  A((void**)&d.candNode, B * candCap * 2);
  A((void**)&d.candQ, B * candCap);
  A((void**)&d.candCount, B * kMaxLevels * 4);
  A((void**)&d.selXYR, B * selCap * 8);
  A((void**)&d.selCount, B * kMaxLevels * 4);
  A((void**)&d.status, 4);
  A((void**)&d.cellInfo, h->cellAlloc * 4);
  A((void**)&d.fbList, B * h->cellAlloc * sizeof(uint2));
  A((void**)&d.fbCount, B * 4);  // one counter per possible first image of a chunk (chunks of a batch run on two streams)
  A((void**)&d.rxOfs, h->rxAlloc * 2);
  A((void**)&d.rxAlpha, h->rxAlloc * 4);
  A((void**)&d.ryOfs, h->ryAlloc * 2);
  A((void**)&d.ryBeta, h->ryAlloc * 4);
  A((void**)&d.outKps, B * h->outCap * sizeof(b2s_keypoint));
  A((void**)&d.outDesc, B * h->outCap * 32);
  A((void**)&d.outCounts, B * 4);
  if (e == cudaSuccess) e = cudaMemset(d.status, 0, 4);
  if (e == cudaSuccess) e = cudaMallocHost((void**)&h->hKps, B * h->outCap * sizeof(b2s_keypoint));
  if (e == cudaSuccess) e = cudaMallocHost((void**)&h->hDesc, B * h->outCap * 32);
  if (e == cudaSuccess) e = cudaMallocHost((void**)&h->hCounts, B * 4);
  if (e == cudaSuccess) e = cudaMallocHost((void**)&h->hStatus, 4);
  if (e == cudaSuccess) {
    int capMax = 0;
    for (int l = 0; l < nlevels; l++) capMax = std::max(capMax, (int)align_up((size_t)std::max(h->nFeat[l] + 4, 64), 8));
    const size_t qsm = quadtree_smem_bytes(capMax);
    if (qsm > 220 * 1024) {
      set_error("nfeatures per level (%d) too large for the quadtree kernel's shared memory", capMax);
      b2s_extractor_destroy(h);
      return B2S_ERR_BAD_ARG;
    }
    e = cudaFuncSetAttribute(k_quadtree, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max(qsm, (size_t)49152));
  }
  if (e != cudaSuccess) {
    set_error("b2s_extractor_create: %s", cudaGetErrorString(e));
    b2s_extractor_destroy(h);
    return B2S_ERR_CUDA;
  }
  *out = h;
  return B2S_OK;
}

extern "C" void b2s_extractor_destroy(b2s_extractor* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  DeviceBuffers& d = h->d;
  void* ptrs[] = {d.pyr, d.blur, d.candXY, d.candKey, d.candResp, d.candNode, d.candQ, d.candCount, d.selXYR,
                  d.selCount, d.status, d.rxOfs, d.rxAlpha, d.ryOfs, d.ryBeta, d.outKps, d.outDesc, d.outCounts, d.cellInfo,
                  d.raw, d.score, d.tileDx, d.tileDy, d.bitmap, d.fbList, d.fbCount};
  for (void* p : ptrs)
    if (p) cudaFree(p);
  if (h->hKps) cudaFreeHost(h->hKps);
  if (h->hDesc) cudaFreeHost(h->hDesc);
  if (h->hCounts) cudaFreeHost(h->hCounts);
  if (h->hStatus) cudaFreeHost(h->hStatus);
  if (h->dStereoSad) cudaFree(h->dStereoSad);
  if (h->dStereoU) cudaFree(h->dStereoU);
  if (h->dStereoD) cudaFree(h->dStereoD);
  if (h->dStereoN) cudaFree(h->dStereoN);
  if (h->stream) cudaStreamDestroy(h->stream);
  if (h->stream2) cudaStreamDestroy(h->stream2);
  delete h;
}

extern "C" int b2s_extractor_tables(const b2s_extractor* h, float* scale, float* inv_scale, float* sigma2,
                                    float* inv_sigma2, int32_t* nfeatures_per_level) {
  if (!h) return B2S_ERR_BAD_ARG;
  for (int i = 0; i < h->nlevels; i++) {
    if (scale) scale[i] = h->scale[i];
    if (inv_scale) inv_scale[i] = h->invScale[i];
    if (sigma2) sigma2[i] = h->sigma2[i];
    if (inv_sigma2) inv_sigma2[i] = h->invSigma2[i];
    if (nfeatures_per_level) nfeatures_per_level[i] = h->nFeat[i];
  }
  return B2S_OK;
}

extern "C" int b2s_extractor_max_keypoints(const b2s_extractor* h) { return h ? h->outCap : 0; }
extern "C" long long b2s_extractor_launch_count(const b2s_extractor* h) { return h ? h->launches : 0; }

static int ensure_geometry(b2s_extractor* h, int W, int H) {
  if (h->curW == W && h->curH == H) return B2S_OK;
  if (W > h->maxW || H > h->maxH) {
    set_error("image %dx%d exceeds max %dx%d", W, H, h->maxW, h->maxH);
    return B2S_ERR_BAD_ARG;
  }
  return build_geometry(h, W, H);
}

static int check_status(b2s_extractor* h) {
  // d.status was copied to hStatus by the caller and the stream synchronised
  const int s = *h->hStatus;
  if (s) {
    cudaMemsetAsync(h->d.status, 0, 4, h->stream);
    set_error("extractor capacity exceeded (status bits %d: 1=candidates 2=output cap 4=quadtree nodes)", s);
    return B2S_ERR_CAPACITY;
  }
  return B2S_OK;
}

extern "C" int b2s_extract_batch(b2s_extractor* h, const uint8_t* const* imgs, int batch, int width, int height, int stride,
                                 b2s_keypoint* kps, uint8_t* desc, int cap, int* n_out) {
  if (!h || !n_out || batch < 1 || batch > h->maxBatch) {
    set_error("b2s_extract_batch: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  if (!imgs || width <= 0 || height <= 0) {  // empty image -> silent return (src/ORBextractor.cc:1553)
    for (int b = 0; b < batch; b++) n_out[b] = 0;
    return B2S_OK;
  }
  if (!kps || !desc || stride < width) return B2S_ERR_BAD_ARG;
  B2S_CUDA(cudaSetDevice(h->device));
  int rc = ensure_geometry(h, width, height);
  if (rc != B2S_OK) return rc;
  const ExtractGeom& g = h->geom;
  for (int b = 0; b < batch; b++)
    if (!imgs[b]) return B2S_ERR_BAD_ARG;
  const int icap = h->outCap;
  if (cap <= icap) {
    // Records are produced with the caller's stride and copied straight into the caller's arrays (full PCIe speed when
    // those are pinned).  Large batches are cut into chunks on two streams so that the H2D copy of chunk k+1, the kernels
    // of chunk k and the D2H copy of chunk k-1 overlap.
    const int nChunks = (batch >= 16 && h->stream2) ? 4 : 1;
    for (int c = 0; c < nChunks; c++) {
      const int b0 = (int)((long long)batch * c / nChunks), b1 = (int)((long long)batch * (c + 1) / nChunks);
      if (b1 <= b0) continue;
      cudaStream_t st = (nChunks > 1 && (c & 1)) ? h->stream2 : h->stream;
      rc = upload_level0(h, imgs, b0, b1 - b0, width, height, stride, st);
      if (rc != B2S_OK) return rc;
      const DeviceBuffers dc = shifted(h->d, g, b0);
      rc = run_pipeline(h, dc, b1 - b0, h->d.outKps + (size_t)b0 * cap, h->d.outDesc + (size_t)b0 * cap * 32,
                        h->d.outCounts + b0, cap, st, nChunks == 1);
      if (rc != B2S_OK) return rc;
      B2S_CUDA(cudaMemcpyAsync(kps + (size_t)b0 * cap, h->d.outKps + (size_t)b0 * cap,
                               (size_t)(b1 - b0) * cap * sizeof(b2s_keypoint), cudaMemcpyDeviceToHost, st));
      B2S_CUDA(cudaMemcpyAsync(desc + (size_t)b0 * cap * 32, h->d.outDesc + (size_t)b0 * cap * 32,
                               (size_t)(b1 - b0) * cap * 32, cudaMemcpyDeviceToHost, st));
      B2S_CUDA(cudaMemcpyAsync(h->hCounts + b0, h->d.outCounts + b0, (size_t)(b1 - b0) * 4, cudaMemcpyDeviceToHost, st));
    }
    if (nChunks > 1) B2S_CUDA(cudaStreamSynchronize(h->stream2));
    B2S_CUDA(cudaMemcpyAsync(h->hStatus, h->d.status, 4, cudaMemcpyDeviceToHost, h->stream));
    B2S_CUDA(cudaStreamSynchronize(h->stream));
    rc = check_status(h);
    if (rc != B2S_OK) return rc;
    for (int b = 0; b < batch; b++) n_out[b] = h->hCounts[b];
    h->lastCap = cap;  // the records of this call stay on the device (b2s_stereo_match)
    h->lastBatch = batch;
    return B2S_OK;
  }
  rc = upload_level0(h, imgs, 0, batch, width, height, stride, h->stream);
  if (rc != B2S_OK) return rc;
  rc = run_pipeline(h, h->d, batch, h->d.outKps, h->d.outDesc, h->d.outCounts, icap, h->stream);
  if (rc != B2S_OK) return rc;
  B2S_CUDA(cudaMemcpyAsync(h->hKps, h->d.outKps, (size_t)batch * icap * sizeof(b2s_keypoint), cudaMemcpyDeviceToHost,
                           h->stream));
  B2S_CUDA(cudaMemcpyAsync(h->hDesc, h->d.outDesc, (size_t)batch * icap * 32, cudaMemcpyDeviceToHost, h->stream));
  B2S_CUDA(cudaMemcpyAsync(h->hCounts, h->d.outCounts, (size_t)batch * 4, cudaMemcpyDeviceToHost, h->stream));
  B2S_CUDA(cudaMemcpyAsync(h->hStatus, h->d.status, 4, cudaMemcpyDeviceToHost, h->stream));
  B2S_CUDA(cudaStreamSynchronize(h->stream));
  rc = check_status(h);
  if (rc != B2S_OK) return rc;
  for (int b = 0; b < batch; b++) {
    const int n = h->hCounts[b];
    n_out[b] = n;
    memcpy(kps + (size_t)b * cap, h->hKps + (size_t)b * icap, (size_t)n * sizeof(b2s_keypoint));
    memcpy(desc + (size_t)b * cap * 32, h->hDesc + (size_t)b * icap * 32, (size_t)n * 32);
  }
  h->lastCap = icap;
  h->lastBatch = batch;
  return B2S_OK;
}

extern "C" int b2s_extract(b2s_extractor* h, const uint8_t* img, int width, int height, int stride, b2s_keypoint* kps,
                           uint8_t* desc, int cap, int* n_out, uint8_t* const* pyr_out) {
  if (!h || !n_out) return B2S_ERR_BAD_ARG;
  if (!img || width <= 0 || height <= 0) {
    *n_out = 0;
    return B2S_OK;
  }
  const uint8_t* imgs[1] = {img};
  int rc = b2s_extract_batch(h, imgs, 1, width, height, stride, kps, desc, cap, n_out);
  if (rc != B2S_OK) return rc;
  if (pyr_out) {  // mvImagePyramid for Frame::ComputeStereoMatches (src/Frame.cc:1044)
    const ExtractGeom& g = h->geom;
    for (int l = 0; l < g.nlevels; l++) {
      if (!pyr_out[l]) continue;
      B2S_CUDA(cudaMemcpy2DAsync(pyr_out[l], g.lv[l].w, h->d.pyr + g.lv[l].off, g.lv[l].pitch, g.lv[l].w, g.lv[l].h,
                                 cudaMemcpyDeviceToHost, h->stream));
    }
    B2S_CUDA(cudaStreamSynchronize(h->stream));
  }
  return B2S_OK;
}

extern "C" int b2s_extract_batch_device(b2s_extractor* h, const uint8_t* d_imgs, size_t img_pitch_bytes, int batch,
                                        int width, int height, int stride, b2s_keypoint* d_kps, uint8_t* d_desc,
                                        int32_t* d_counts, int cap, void* stream) {
  if (!h || !d_imgs || !d_kps || !d_desc || !d_counts || batch < 1 || batch > h->maxBatch || width <= 0 || height <= 0 ||
      stride < width || cap < 1) {
    set_error("b2s_extract_batch_device: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  B2S_CUDA(cudaSetDevice(h->device));
  int rc = ensure_geometry(h, width, height);
  if (rc != B2S_OK) return rc;
  cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
  const ExtractGeom& g = h->geom;
  // level 0 = copy of the input (src/ORBextractor.cc:1728); one strided 2D copy per image
  for (int b = 0; b < batch; b++)
    B2S_CUDA(cudaMemcpy2DAsync(h->d.pyr + (size_t)b * g.pyrBytes + g.lv[0].off, g.lv[0].pitch,
                               d_imgs + (size_t)b * img_pitch_bytes, stride, width, height, cudaMemcpyDeviceToDevice, st));
  return run_pipeline(h, h->d, batch, d_kps, d_desc, d_counts, cap, st);
}

extern "C" int b2s_extractor_check(b2s_extractor* h) {
  if (!h) return B2S_ERR_BAD_ARG;
  B2S_CUDA(cudaSetDevice(h->device));
  B2S_CUDA(cudaDeviceSynchronize());
  B2S_CUDA(cudaMemcpy(h->hStatus, h->d.status, 4, cudaMemcpyDeviceToHost));
  return check_status(h);
}

extern "C" int b2s_extractor_debug_level(b2s_extractor* h, int b, int level, int blurred, uint8_t* out, int* w, int* hgt) {
  if (!h || level < 0 || level >= h->nlevels || b < 0 || b >= h->maxBatch || !h->curW) return B2S_ERR_BAD_ARG;
  const LevelGeom& L = h->geom.lv[level];
  if (w) *w = L.w;
  if (hgt) *hgt = L.h;
  if (out) {
    B2S_CUDA(cudaSetDevice(h->device));
    B2S_CUDA(cudaDeviceSynchronize());
    const uint8_t* src = (blurred ? h->d.blur : h->d.pyr) + (size_t)b * h->geom.pyrBytes + L.off;
    B2S_CUDA(cudaMemcpy2D(out, L.w, src, L.pitch, L.w, L.h, cudaMemcpyDeviceToHost));
  }
  return B2S_OK;
}

extern "C" int b2s_extractor_debug_candidates(b2s_extractor* h, int b, int level, int32_t* xy, int32_t* resp, int cap,
                                              int* n) {
  if (!h || level < 0 || level >= h->nlevels || b < 0 || b >= h->maxBatch || !h->curW || !n) return B2S_ERR_BAD_ARG;
  B2S_CUDA(cudaSetDevice(h->device));
  B2S_CUDA(cudaDeviceSynchronize());
  const LevelGeom& L = h->geom.lv[level];
  int cnt = 0;
  B2S_CUDA(cudaMemcpy(&cnt, h->d.candCount + b * kMaxLevels + level, 4, cudaMemcpyDeviceToHost));
  cnt = std::min(cnt, L.candCap);
  *n = cnt;
  if (xy && resp && cnt > 0) {
    std::vector<uint32_t> vxy(cnt), vkey(cnt);
    std::vector<uint8_t> vr(cnt);
    const size_t base = (size_t)b * h->geom.totalCandCap + L.candOff;
    B2S_CUDA(cudaMemcpy(vxy.data(), h->d.candXY + base, (size_t)cnt * 4, cudaMemcpyDeviceToHost));
    B2S_CUDA(cudaMemcpy(vkey.data(), h->d.candKey + base, (size_t)cnt * 4, cudaMemcpyDeviceToHost));
    B2S_CUDA(cudaMemcpy(vr.data(), h->d.candResp + base, (size_t)cnt, cudaMemcpyDeviceToHost));
    // return in reference insertion order (sort by order key)
    std::vector<int> idx(cnt);
    for (int i = 0; i < cnt; i++) idx[i] = i;
    std::sort(idx.begin(), idx.end(), [&](int a, int c) { return vkey[a] < vkey[c]; });
    for (int i = 0; i < cnt && i < cap; i++) {
      xy[2 * i] = vxy[idx[i]] & 0xffff;
      xy[2 * i + 1] = vxy[idx[i]] >> 16;
      resp[i] = vr[idx[i]];
    }
  }
  return B2S_OK;
}

// test hook: device sincosf mirror over n floats (host buffers)
extern "C" int b2s_debug_sincosf(const float* in, int n, float* s, float* c) {
  int rc = select_device(0);
  if (rc != B2S_OK) return rc;
  float *din, *ds, *dc;
  B2S_CUDA(cudaMalloc(&din, (size_t)n * 4));
  B2S_CUDA(cudaMalloc(&ds, (size_t)n * 4));
  B2S_CUDA(cudaMalloc(&dc, (size_t)n * 4));
  B2S_CUDA(cudaMemcpy(din, in, (size_t)n * 4, cudaMemcpyHostToDevice));
  k_sincos_test<<<div_up(n, 256), 256>>>(din, n, ds, dc);
  B2S_CUDA(cudaMemcpy(s, ds, (size_t)n * 4, cudaMemcpyDeviceToHost));
  B2S_CUDA(cudaMemcpy(c, dc, (size_t)n * 4, cudaMemcpyDeviceToHost));
  cudaFree(din);
  cudaFree(ds);
  cudaFree(dc);
  return B2S_OK;
}


// ---------------------------------------------------------------- stereo matching on the resident pyramids
static int stereo_launch(b2s_extractor* h, int first_left, int first_right, int n_pairs, const b2s_keypoint* d_kps,
                         const uint8_t* d_desc, const int32_t* d_counts, int cap, float bf, float mb, float* d_uright,
                         float* d_depth, int32_t* d_nmatched, cudaStream_t st) {
  const ExtractGeom& g = h->geom;
  StereoParams sp;
  for (int l = 0; l < kMaxLevels; l++) sp.invScale[l] = l < h->nlevels ? h->invScale[l] : 0.f;
  sp.bf = bf; sp.mb = mb; sp.firstLeft = first_left; sp.firstRight = first_right; sp.cap = cap;
  if ((size_t)n_pairs * cap > h->stereoCap) {
    if (h->dStereoSad) cudaFree(h->dStereoSad);
    h->dStereoSad = nullptr;
    h->stereoCap = 0;
    B2S_CUDA(cudaMalloc((void**)&h->dStereoSad, (size_t)n_pairs * cap * 4));
    h->stereoCap = (size_t)n_pairs * cap;
  }
  k_stereo_match<<<dim3(div_up(cap, ST_WARPS), n_pairs), ST_WARPS * 32, 0, st>>>(g, sp, h->d.pyr, d_kps, d_desc, d_counts,
                                                                               d_uright, d_depth, h->dStereoSad);
  k_stereo_cull<<<n_pairs, 1024, 0, st>>>(sp, d_counts, d_uright, d_depth, h->dStereoSad, d_nmatched);
  h->launches += 2;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

extern "C" int b2s_stereo_match_device(b2s_extractor* h, int first_left, int first_right, int n_pairs,
                                       const b2s_keypoint* d_kps, const uint8_t* d_desc, const int32_t* d_counts, int cap,
                                       float bf, float mb, float* d_uright, float* d_depth, int32_t* d_nmatched,
                                       void* stream) {
  if (!h || !h->curW || n_pairs < 1 || first_left < 0 || first_right < 0 || first_left + n_pairs > h->maxBatch ||
      first_right + n_pairs > h->maxBatch || !d_kps || !d_desc || !d_counts || cap < 1 || cap > ST_MAXR || !d_uright ||
      !d_depth || !d_nmatched) {
    set_error("b2s_stereo_match_device: bad argument (extract a batch with this handle first; cap <= %d)", ST_MAXR);
    return B2S_ERR_BAD_ARG;
  }
  B2S_CUDA(cudaSetDevice(h->device));
  return stereo_launch(h, first_left, first_right, n_pairs, d_kps, d_desc, d_counts, cap, bf, mb, d_uright, d_depth,
                       d_nmatched, stream ? (cudaStream_t)stream : h->stream);
}

extern "C" int b2s_stereo_match(b2s_extractor* h, int first_left, int first_right, int n_pairs, float bf, float mb,
                                float* uright, float* depth, int cap_out, int32_t* n_matched) {
  if (!h || !h->curW || h->lastCap < 1 || n_pairs < 1 || first_left < 0 || first_right < 0 ||
      first_left + n_pairs > h->lastBatch || first_right + n_pairs > h->lastBatch || !uright || !depth ||
      cap_out < h->lastCap || h->lastCap > ST_MAXR) {
    set_error("b2s_stereo_match: call b2s_extract_batch first; cap_out must be >= the cap of that call");
    return B2S_ERR_BAD_ARG;
  }
  B2S_CUDA(cudaSetDevice(h->device));
  const int cap = h->lastCap;
  const size_t need = (size_t)n_pairs * cap;
  if (need > h->stereoOutCap) {
    if (h->dStereoU) cudaFree(h->dStereoU);
    if (h->dStereoD) cudaFree(h->dStereoD);
    if (h->dStereoN) cudaFree(h->dStereoN);
    h->dStereoU = h->dStereoD = nullptr;
    h->dStereoN = nullptr;
    h->stereoOutCap = 0;
    B2S_CUDA(cudaMalloc((void**)&h->dStereoU, need * 4));
    B2S_CUDA(cudaMalloc((void**)&h->dStereoD, need * 4));
    B2S_CUDA(cudaMalloc((void**)&h->dStereoN, (size_t)h->maxBatch * 4));
    h->stereoOutCap = need;
  }
  cudaStream_t st = h->stream;
  int rc = stereo_launch(h, first_left, first_right, n_pairs, h->d.outKps, h->d.outDesc, h->d.outCounts, cap, bf, mb,
                         h->dStereoU, h->dStereoD, h->dStereoN, st);
  if (rc != B2S_OK) return rc;
  B2S_CUDA(cudaMemcpy2DAsync(uright, (size_t)cap_out * 4, h->dStereoU, (size_t)cap * 4, (size_t)cap * 4, n_pairs,
                             cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaMemcpy2DAsync(depth, (size_t)cap_out * 4, h->dStereoD, (size_t)cap * 4, (size_t)cap * 4, n_pairs,
                             cudaMemcpyDeviceToHost, st));
  if (n_matched) B2S_CUDA(cudaMemcpyAsync(n_matched, h->dStereoN, (size_t)n_pairs * 4, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaStreamSynchronize(st));
  return B2S_OK;
}
