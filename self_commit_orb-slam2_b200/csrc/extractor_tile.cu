// extractor_tile.cu — the fused front end of the H100 ORB extractor: ONE tile kernel per pyramid level that
//   * stages a 128 x 32 pixel tile (+ halo) of level l in shared memory with TMA (cp.async.bulk.tensor, mbarrier),
//   * computes the FAST-9/16 arc strength of EVERY pixel of the tile once (packed u16x2 DPX min/max; one strength map
//     serves both thresholds, SURVEY.md §8c),
//   * computes the Q8 7x7 Gaussian blur of the tile (REFLECT_101 at the image border),
//   * produces the part of pyramid level l+1 whose bilinear source samples start inside the tile,
// and writes the strength map / blurred tile back with TMA stores.  A light per-cell kernel then applies the reference's
// cell rules (3x3 NMS that never crosses a cell seam, iniThFAST -> minThFAST fallback per cell) and emits the candidate
// lists the quadtree kernel consumes.
//
// Replaces ComputePyramid (/root/reference/src/ORBextractor.cc:1674-1734), the cell loop + cv::FAST of
// ComputeKeyPointsOctTree (:1060-1157) and the GaussianBlur of operator() (:1626-1634).  Bit-exact: the arithmetic is
// the integer recipe of cv::resize INTER_LINEAR, FAST and the Q8 GaussianBlur (SURVEY.md §8c), checked level by level
// against the oracle (tests/test_extractor_gpu.py).
#include <cuda.h>  // CUtensorMap (types only: the encoder is fetched through cudaGetDriverEntryPoint, libcuda is not linked)

#include <algorithm>
#include <vector>

#include "extractor.cuh"

namespace b2s {

constexpr int TW = 128, TH = 32;          // tile interior
// halo left / top (right / bottom are HX / HY as well).  Only 3 pixels are needed, but the innermost TMA coordinate must
// be a multiple of 16 BYTES (an 8-byte-aligned start, x = tx*128 - 8, is an illegal instruction)
// 4 halo rows: the strength is also computed on a 1-pixel ring around the interior (the in-tile NMS needs it).
constexpr int HX = 16, HY = 4;
constexpr int BW = TW + 2 * HX;           // 160: TMA box width in bytes (multiple of 16)
constexpr int BH = TH + 2 * HY;           // 40
constexpr int SPW = 136;                  // byte pitch of the padded strength tile: column c of the interior at c + 4
constexpr int SPH = TH + 2;               // rows -1 .. 32 of the interior
constexpr int PASS_SUB = 288;             // >= ceil(34 * 66 / 256) * 32 items a warp can see
constexpr int CAND_CAP = 2048;            // candidate pixels per tile handled by the sparse NMS (more: dense fallback)
constexpr int PWD = TW / 2 + 8;           // 72 pair words per plane row: box columns [HX - 8, HX + TW + 8), word 0 = column HX - 8
constexpr int PJ0 = HX / 2 - 4;           // box pair-word index of plane word 0
constexpr int TILE_THREADS = 256;

// Shared memory of one CTA (43.3 KB: five CTAs per SM).  Phases reuse space: the pixel-pair planes die when the strength
// pass is over and the blur's horizontal sums take their place; the quick-reject pass list shares the blurred tile.
struct TileSmem {
  alignas(128) uint8_t raw[BH * BW];        // TMA destination: rows ty*32-4 .., columns tx*128-16 ..
  alignas(128) uint8_t scoreT[TH * TW];     // TMA store source: FAST arc strength M (0..255) per interior pixel
  union {
    alignas(128) uint8_t blurT[TH * TW];    // TMA store source: blurred interior
    uint16_t passList[(TILE_THREADS / 32) * PASS_SUB];  // pixel pairs that survive the quick reject, one sub-list per warp
  };
  union {
    struct {
      alignas(16) uint32_t planeE[BH * PWD];  // (raw[2j], raw[2j+1]) as u16x2
      alignas(16) uint32_t planeO[BH * PWD];  // (raw[2j+1], raw[2j+2])
    };
    alignas(16) uint16_t blurH[BH * TW];    // horizontal pass of the blur, rows of the box x interior columns
  };
  alignas(16) uint8_t scoreP[SPH * SPW];    // strength of the interior + 1-pixel ring (+ one more column each side)
  alignas(16) uint32_t bm[TH * 4];          // NMS bitmap of the tile: per row even / odd pixel words of two 64-pixel groups
  uint16_t candList[CAND_CAP];              // interior pixels with M > iniThFAST (offset into scoreP)
  alignas(8) unsigned long long bar;        // mbarrier of the tile load
  int nPass, nCand;
  uint32_t rzB[TH + 2];                     // per destination row of the tile: vertical weights b0 | b1 << 16
  int16_t rzO0[TH + 2], rzO1[TH + 2];       // ... and the box rows of its two source rows
  uint8_t colFlag[TW], rowFlag[TH];         // per interior column / row: bit0 = in the FAST band, bit1 = the left / upper
                                            // neighbour is in the same cell, bit2 = the right / lower neighbour is
};
static_assert(sizeof(TileSmem) <= 56 * 1024, "four CTAs per SM");

__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* tm, uint32_t bar, int x, int y, int z) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(dst),
      "l"(tm), "r"(x), "r"(y), "r"(z), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* tm, uint32_t src, int x, int y, int z) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(tm), "r"(src), "r"(x),
               "r"(y), "r"(z)
               : "memory");
}

struct TileArgs {
  int level, bBase;
  uint8_t* pyr;  // base of the batch's pyramids (image 0 of the handle), for the level l+1 stores
  const int16_t* rxOfs;
  const uint32_t* rxAlpha;
  const int16_t* ryOfs;
  const uint32_t* ryBeta;
  const int16_t* tileDx;  // per (level, tile column) first destination column owned; one sentinel per level
  const int16_t* tileDy;
  uint32_t* bitmap;  // per image g.bmWords words: NMS bitmap, per level rows of tilesX * 4 words (even / odd pixel words)
};

// FAST-9/16 arc strength of the pixel pair whose left pixel sits at EVEN box column 2*j (row pointers at the pair's row).
// With I_k the 16 circle pixels, A = max_s min_{9 window} I, B = min_s max_{9 window} I and c the centre:
// bright strength = A - c, dark strength = c - B, M = max(bright, dark, 0) — identical to max over the 16 arcs of
// min |v - p| with one sign (extractor.cu fast_pair_full); corner at th <=> M > th, response = M - 1.
__device__ __forceinline__ void fast_pair_load(const uint32_t* __restrict__ E, const uint32_t* __restrict__ O, int j,
                                               uint32_t (&d)[16], uint32_t& c) {
  d[0] = E[3 * PWD + j];        // ( 0, 3)
  d[1] = O[3 * PWD + j];        // ( 1, 3)
  d[2] = E[2 * PWD + j + 1];    // ( 2, 2)
  d[3] = O[1 * PWD + j + 1];    // ( 3, 1)
  d[4] = O[j + 1];              // ( 3, 0)
  d[5] = O[-1 * PWD + j + 1];   // ( 3,-1)
  d[6] = E[-2 * PWD + j + 1];   // ( 2,-2)
  d[7] = O[-3 * PWD + j];       // ( 1,-3)
  d[8] = E[-3 * PWD + j];       // ( 0,-3)
  d[9] = O[-3 * PWD + j - 1];   // (-1,-3)
  d[10] = E[-2 * PWD + j - 1];  // (-2,-2)
  d[11] = O[-1 * PWD + j - 2];  // (-3,-1)
  d[12] = O[j - 2];             // (-3, 0)
  d[13] = O[1 * PWD + j - 2];   // (-3, 1)
  d[14] = E[2 * PWD + j - 1];   // (-2, 2)
  d[15] = O[3 * PWD + j - 1];   // (-1, 3)
  c = E[j];
}

// Exact reject: any 9 contiguous circle pixels contain one of every opposite pair (k, k+8), so
// bright strength <= min_k max(I_k, I_k+8) - c and dark strength <= c - max_k min(I_k, I_k+8).
// Returns 0x8000 in every 16-bit lane whose bound exceeds th (only those lanes can have M > th).
__device__ __forceinline__ uint32_t fast_pair_quick(const uint32_t (&d)[16], uint32_t c, int th) {
  uint32_t X = __vimin3_u16x2(__vmaxu2(d[0], d[8]), __vmaxu2(d[1], d[9]), __vmaxu2(d[2], d[10]));
  X = __vimin3_u16x2(X, __vmaxu2(d[3], d[11]), __vmaxu2(d[4], d[12]));
  X = __vimin3_u16x2(X, __vmaxu2(d[5], d[13]), __vmaxu2(d[6], d[14]));
  X = __vminu2(X, __vmaxu2(d[7], d[15]));
  uint32_t Y = __vimax3_u16x2(__vminu2(d[0], d[8]), __vminu2(d[1], d[9]), __vminu2(d[2], d[10]));
  Y = __vimax3_u16x2(Y, __vminu2(d[3], d[11]), __vminu2(d[4], d[12]));
  Y = __vimax3_u16x2(Y, __vminu2(d[5], d[13]), __vminu2(d[6], d[14]));
  Y = __vmaxu2(Y, __vminu2(d[7], d[15]));
  const uint32_t ub = __vmaxu2((X + 0x01000100u) - c, (c + 0x01000100u) - Y);  // 256 + bound, per lane
  return (ub + 0x7fff7fffu - (uint32_t)(256 + th) * 0x00010001u) & 0x80008000u;
}

// With I_k the 16 circle pixels, A = max_s min_{9 window} I, B = min_s max_{9 window} I and c the centre:
// bright strength = A - c, dark strength = c - B, M = max(bright, dark, 0) — identical to max over the 16 arcs of
// min |v - p| with one sign (extractor.cu fast_pair_full); corner at th <=> M > th, response = M - 1.
__device__ __forceinline__ uint32_t fast_pair_full(const uint32_t (&d)[16], uint32_t c) {
  uint32_t t3n[16], t3x[16];
#pragma unroll
  for (int k = 0; k < 16; k++) {
    t3n[k] = __vimin3_u16x2(d[k], d[(k + 1) & 15], d[(k + 2) & 15]);
    t3x[k] = __vimax3_u16x2(d[k], d[(k + 1) & 15], d[(k + 2) & 15]);
  }
  uint32_t A = 0u, B = 0xFFFFFFFFu;
#pragma unroll
  for (int s = 0; s < 16; s += 2) {
    const uint32_t a0 = __vimin3_u16x2(t3n[s], t3n[(s + 3) & 15], t3n[(s + 6) & 15]);
    const uint32_t a1 = __vimin3_u16x2(t3n[s + 1], t3n[(s + 4) & 15], t3n[(s + 7) & 15]);
    A = __vimax3_u16x2(A, a0, a1);
    const uint32_t b0 = __vimax3_u16x2(t3x[s], t3x[(s + 3) & 15], t3x[(s + 6) & 15]);
    const uint32_t b1 = __vimax3_u16x2(t3x[s + 1], t3x[(s + 4) & 15], t3x[(s + 7) & 15]);
    B = __vimin3_u16x2(B, b0, b1);
  }
  // biased per-lane differences stay in [1, 511]: a plain 32-bit add / subtract never carries across the lanes
  const uint32_t bright = (A + 0x01000100u) - c;
  const uint32_t dark = (c + 0x01000100u) - B;
  return __vimax3_u16x2(bright, dark, 0x01000100u) - 0x01000100u;  // M(lo) | M(hi) << 16, each in [0, 255]
}

__global__ void __launch_bounds__(TILE_THREADS) k_tile(const __grid_constant__ CUtensorMap tmPyr,
                                                       const __grid_constant__ CUtensorMap tmScore,
                                                       const __grid_constant__ CUtensorMap tmBlur,
                                                       const __grid_constant__ ExtractGeom g, const TileArgs a) {
  // (no static shared memory in this kernel: the dynamic window starts at the CTA's shared base, which satisfies the
  // 128-byte alignment TMA needs; indexing the array directly keeps every access an LDS / STS instead of a generic LD / ST)
  extern __shared__ __align__(1024) TileSmem smemTile[];
  TileSmem& S = smemTile[0];
  const LevelGeom& L = g.lv[a.level];
  const int tx = blockIdx.x, ty = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x;
  const int X0 = tx * TW - HX, Y0 = ty * TH - HY;  // image coordinates of box (0, 0)
  const uint32_t bar = s32(&S.bar);
  // strengths default to 0 (pairs the quick reject drops are never written)
  for (int k = tid; k < (SPH * SPW) / 16; k += TILE_THREADS) reinterpret_cast<uint4*>(S.scoreP)[k] = make_uint4(0u, 0u, 0u, 0u);
  for (int k = tid; k < (TH * TW) / 16; k += TILE_THREADS) reinterpret_cast<uint4*>(S.scoreT)[k] = make_uint4(0u, 0u, 0u, 0u);
  if (tid < TH * 4) S.bm[tid] = 0u;
  if (tid == 0) {
    S.nPass = 0;
    S.nCand = 0;
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    mbar_expect_tx(bar, BH * BW);
    tma_load_3d(s32(S.raw), &tmPyr, bar, X0, Y0, a.bBase + b);  // out-of-image bytes arrive as 0
  }
  __syncthreads();  // the barrier is initialised for everyone
  while (!mbar_try_wait(bar, 0)) {
  }

  // ---- REFLECT_101 border of cv::GaussianBlur for tiles that touch the image edge: columns first, then whole rows
  const int Wd = L.w, Hd = L.h;
  const bool edgeX = (X0 + HX - 3 < 0) || (X0 + HX + TW + 3 > Wd);
  const bool edgeY = (Y0 + HY - 3 < 0) || (Y0 + HY + TH + 3 > Hd);
  if (edgeX || edgeY) {
    if (edgeX) {
      for (int k = tid; k < BH * 6; k += TILE_THREADS) {
        const int ly = k / 6, c6 = k - ly * 6;
        const int gy = Y0 + ly;
        if (gy < 0 || gy >= Hd) continue;
        const int gx = (c6 < 3) ? (c6 - 3) : (Wd + c6 - 3);
        const int lx = gx - X0;
        if (lx < 0 || lx >= BW) continue;
        const int rx = (gx < 0) ? -gx : 2 * (Wd - 1) - gx;
        const int lsx = rx - X0;
        if (lsx >= 0 && lsx < BW) S.raw[ly * BW + lx] = S.raw[ly * BW + lsx];
      }
      __syncthreads();
    }
    if (edgeY) {
      for (int k = tid; k < 6 * (BW / 4); k += TILE_THREADS) {
        const int r6 = k / (BW / 4), wq = k - r6 * (BW / 4);
        const int gy = (r6 < 3) ? (r6 - 3) : (Hd + r6 - 3);
        const int ly = gy - Y0;
        if (ly < 0 || ly >= BH) continue;
        const int ry = (gy < 0) ? -gy : 2 * (Hd - 1) - gy;
        const int lsy = ry - Y0;
        if (lsy >= 0 && lsy < BH)
          reinterpret_cast<uint32_t*>(S.raw)[ly * (BW / 4) + wq] = reinterpret_cast<const uint32_t*>(S.raw)[lsy * (BW / 4) + wq];
      }
      __syncthreads();
    }
  }

  // ---- FAST: pixel-pair planes, then the dense arc strength of the interior and of a 1-pixel ring around it
  {
    const uint32_t* rw = reinterpret_cast<const uint32_t*>(S.raw);
    // (only the words the 16-point circles can reach: box columns [HX - 8, HX + TW + 8))
    constexpr int Q0 = HX / 4 - 2, QN = TW / 4 + 4;
    for (int k = tid; k < BH * QN; k += TILE_THREADS) {
      const int r = k / QN, q = Q0 + (k - r * QN);
      const uint32_t w0 = rw[r * (BW / 4) + q];
      const uint32_t w1 = rw[r * (BW / 4) + q + 1];
      uint2 e, o;
      e.x = __byte_perm(w0, 0u, 0x4140);                 // (b0, b1)
      e.y = __byte_perm(w0, 0u, 0x4342);                 // (b2, b3)
      o.x = __byte_perm(w0, 0u, 0x4241);                 // (b1, b2)
      o.y = (w0 >> 24) | ((w1 & 0xffu) << 16);           // (b3, b4)
      *reinterpret_cast<uint2*>(&S.planeE[r * PWD + 2 * q - PJ0]) = e;
      *reinterpret_cast<uint2*>(&S.planeO[r * PWD + 2 * q - PJ0]) = o;
    }
    // cell seams of ComputeKeyPointsOctTree (:1089-1120): the detectable areas of the cells tile the band
    // [19, maxBorder - 3) in steps of wCell / hCell; a neighbour across a seam (or outside the band) is not compared
    const int xLo = kMinBorder + 3, xHi = L.maxBX - 3, yLo = kMinBorder + 3, yHi = L.maxBY - 3;
    if (tid < TW) {
      const int gx = tx * TW + tid;
      uint8_t f = 0;
      if (gx >= xLo && gx < xHi) {
        const int m = (gx - xLo) % L.wCell;
        f = 1 | (m > 0 ? 2 : 0) | ((m < L.wCell - 1 && gx + 1 < xHi) ? 4 : 0);
      }
      S.colFlag[tid] = f;
    } else if (tid < TW + TH) {
      const int r = tid - TW, gy = ty * TH + r;
      uint8_t f = 0;
      if (gy >= yLo && gy < yHi) {
        const int m = (gy - yLo) % L.hCell;
        f = 1 | (m > 0 ? 2 : 0) | ((m < L.hCell - 1 && gy + 1 < yHi) ? 4 : 0);
      }
      S.rowFlag[r] = f;
    }
    __syncthreads();
    // Pass 1 — every pixel pair of the interior + ring, in the FAST band: the exact quick reject at iniThFAST.  Only pairs
    // that can still hold a corner at iniThFAST go to the compact list; everything else keeps strength 0 (a pixel with
    // M <= iniThFAST neither is a keypoint at iniThFAST nor can it suppress one).  Cells that end up without a maximum
    // above iniThFAST are re-done at minThFAST by the per-cell kernel (k_fast_cells_list), as :1132-1139 asks.
    constexpr int PCN = TW / 2 + 2;  // pair columns -1 .. 64
    const int iniTh = g.iniTh;
    int rrI = tid / PCN, pcI = tid - rrI * PCN;  // (row, pair column) of item q = q0 + tid, advanced by 256 = 3 * 66 + 58
    int warpCnt = 0;
#pragma unroll 1
    for (int q0 = 0; q0 < SPH * PCN; q0 += TILE_THREADS) {
      const int q = q0 + tid;
      bool pass = false;
      if (q < SPH * PCN) {
        const int rr = rrI, pc = pcI - 1;  // rr = interior row + 1
        const int gy = ty * TH + rr - 1;
        if (gy >= yLo && gy < yHi) {
          const int ly = rr - 1 + HY;
          uint32_t d[16], c;
          fast_pair_load(&S.planeE[ly * PWD], &S.planeO[ly * PWD], HX / 2 + pc - PJ0, d, c);
          pass = fast_pair_quick(d, c, iniTh) != 0u;
        }
      }
      pcI += TILE_THREADS - 3 * PCN;
      rrI += 3;
      if (pcI >= PCN) {
        pcI -= PCN;
        rrI++;
      }
      // survivors go to the WARP's own sub-list (the running count is warp-uniform: no atomics, no shuffles)
      const unsigned pm = __ballot_sync(0xffffffffu, pass);
      if (pass) S.passList[(tid >> 5) * PASS_SUB + warpCnt + __popc(pm & ((1u << (tid & 31)) - 1u))] = (uint16_t)q;
      warpCnt += __popc(pm);
    }
    __syncthreads();
    // Pass 2 — the full 16-arc strength, densely over the survivors
    {  // every warp works through its own sub-list (rows are interleaved over the warps, so the lists are balanced)
#pragma unroll 1
      for (int k = tid & 31; k < warpCnt; k += 32) {
        const int q = S.passList[(tid >> 5) * PASS_SUB + k];
        const int rr = q / PCN, pc = q - rr * PCN - 1;
        const int ly = rr - 1 + HY;
        uint32_t d[16], c;
        fast_pair_load(&S.planeE[ly * PWD], &S.planeO[ly * PWD], HX / 2 + pc - PJ0, d, c);
        const uint32_t M2 = fast_pair_full(d, c);
        const uint16_t m16 = (uint16_t)((M2 & 0xffu) | ((M2 >> 8) & 0xff00u));
        *reinterpret_cast<uint16_t*>(&S.scoreP[rr * SPW + 2 * pc + 4]) = m16;
        if (rr >= 1 && rr <= TH && pc >= 0 && pc < TW / 2) {
          reinterpret_cast<uint16_t*>(S.scoreT)[(rr - 1) * (TW / 2) + pc] = m16;
          // keypoint candidates at iniThFAST: interior pixels of the FAST band above the threshold (a few per cent)
          if ((int)(M2 & 0xffffu) > iniTh) {
            const int slot = atomicAdd(&S.nCand, 1);
            if (slot < CAND_CAP) S.candList[slot] = (uint16_t)(rr * SPW + 2 * pc + 4);
          }
          if ((int)(M2 >> 16) > iniTh) {
            const int slot = atomicAdd(&S.nCand, 1);
            if (slot < CAND_CAP) S.candList[slot] = (uint16_t)(rr * SPW + 2 * pc + 5);
          }
        }
      }
    }
    __syncthreads();
    // 3x3 non-maximum suppression inside the cells -> one bit per pixel ("local maximum of its cell above iniThFAST");
    // per 64 pixels of a row an even-pixel word and an odd-pixel word.  Sparse: one thread per candidate; if a tile has more
    // candidates than the list holds, every pixel is tested instead (warp ballots assemble the words).
    uint32_t* bmRow = a.bitmap + (size_t)(a.bBase + b) * g.bmWords + L.bmOff + (size_t)(ty * TH) * (L.tilesX * 4) + tx * 4;
    auto is_max = [&](const uint8_t* p, int M, int cf, int rf) -> bool {
      const bool lOK = cf & 2, rOK = cf & 4;
      int nb = 0;
      if (lOK) nb = max(nb, (int)p[-1]);
      if (rOK) nb = max(nb, (int)p[1]);
      if (rf & 2) {
        nb = max(nb, (int)p[-SPW]);
        if (lOK) nb = max(nb, (int)p[-SPW - 1]);
        if (rOK) nb = max(nb, (int)p[-SPW + 1]);
      }
      if (rf & 4) {
        nb = max(nb, (int)p[SPW]);
        if (lOK) nb = max(nb, (int)p[SPW - 1]);
        if (rOK) nb = max(nb, (int)p[SPW + 1]);
      }
      return M > nb;
    };
    const int nCand = S.nCand;
    if (nCand <= CAND_CAP) {
      for (int k = tid; k < nCand; k += TILE_THREADS) {
        const int off = S.candList[k];
        const int rr = off / SPW, col = off - rr * SPW - 4;  // interior row + 1, interior column
        const int cf = S.colFlag[col], rf = S.rowFlag[rr - 1];
        if (!(cf & 1) || !(rf & 1)) continue;
        const uint8_t* p = &S.scoreP[off];
        if (is_max(p, p[0], cf, rf)) atomicOr(&S.bm[(rr - 1) * 4 + ((col >> 6) << 1) + (col & 1)], 1u << ((col & 63) >> 1));
      }
    } else {
#pragma unroll 1
      for (int it = 0; it < (TW / 2) * TH / TILE_THREADS; it++) {
        const int q = it * TILE_THREADS + tid;
        const int row = q >> 6, pc = q & 63;
        const uint8_t* sp = &S.scoreP[(row + 1) * SPW + 2 * pc + 4];
        const int rf = S.rowFlag[row];
        bool keep[2] = {false, false};
#pragma unroll
        for (int h2 = 0; h2 < 2; h2++) {
          const int M = sp[h2];
          const int cf = S.colFlag[2 * pc + h2];
          if (M > iniTh && (rf & 1) && (cf & 1)) keep[h2] = is_max(sp + h2, M, cf, rf);
        }
        const uint32_t we = __ballot_sync(0xffffffffu, keep[0]);
        const uint32_t wo = __ballot_sync(0xffffffffu, keep[1]);
        if ((tid & 31) == 0) {
          S.bm[row * 4 + ((pc >> 5) << 1)] = we;
          S.bm[row * 4 + ((pc >> 5) << 1) + 1] = wo;
        }
      }
    }
    __syncthreads();
    if (tid < TH * 4) bmRow[(size_t)(tid >> 2) * (L.tilesX * 4) + (tid & 3)] = S.bm[tid];
  }

  // ---- Gaussian blur 7x7, sigma 2, Q8 taps [18,34,48,56,48,34,18] (OpenCV >= 4 fixed point; SURVEY.md §8c)
  // (its horizontal sums overwrite the pixel-pair planes: every warp is past the strength passes after the barrier that
  // precedes the NMS loop)
  {
    const uint32_t* rw = reinterpret_cast<const uint32_t*>(S.raw);
    const uint32_t KA = 0x38302212u, KB = 0x00122230u;  // taps (18,34,48,56) and (48,34,18,0)
    for (int k = tid; k < (TH + 6) * (TW / 4); k += TILE_THREADS) {
      const int r = (k >> 5) + (HY - 3), q = k & 31;  // box row, group of 4 interior columns
      const int wq = r * (BW / 4) + HX / 4 + q;
      const uint32_t w0 = rw[wq - 1], w1 = rw[wq], w2 = rw[wq + 1];
      const uint32_t h0 = __dp4a(__byte_perm(w1, w2, 0x4321), KB, __dp4a(__byte_perm(w0, w1, 0x4321), KA, 0u));
      const uint32_t h1 = __dp4a(__byte_perm(w1, w2, 0x5432), KB, __dp4a(__byte_perm(w0, w1, 0x5432), KA, 0u));
      const uint32_t h2 = __dp4a(__byte_perm(w1, w2, 0x6543), KB, __dp4a(__byte_perm(w0, w1, 0x6543), KA, 0u));
      const uint32_t h3 = __dp4a(w2, KB, __dp4a(w1, KA, 0u));
      uint2 hv;
      hv.x = h0 | (h1 << 16);
      hv.y = h2 | (h3 << 16);
      *reinterpret_cast<uint2*>(&S.blurH[r * TW + 4 * q]) = hv;
    }
    __syncthreads();
    {
      // 32 column groups (4 pixels) x 8 strips of 4 output rows: a register window of 7 horizontal sums slides down
      const int q = tid & 31, strip = tid >> 5;
      const uint2* hp = reinterpret_cast<const uint2*>(&S.blurH[(strip * 4 + HY - 3) * TW + 4 * q]);
      uint32_t win[7][4];
#pragma unroll
      for (int i = 0; i < 10; i++) {
        const uint2 hv = hp[i * (TW / 4)];
        const int u = i % 7;
        win[u][0] = hv.x & 0xffffu;
        win[u][1] = hv.x >> 16;
        win[u][2] = hv.y & 0xffffu;
        win[u][3] = hv.y >> 16;
        if (i >= 6) {
          uint32_t outw = 0;
#pragma unroll
          for (int j = 0; j < 4; j++) {
            const uint32_t q0 = win[(u + 1) % 7][j], q1 = win[(u + 2) % 7][j], q2 = win[(u + 3) % 7][j],
                           q3 = win[(u + 4) % 7][j], q4 = win[(u + 5) % 7][j], q5 = win[(u + 6) % 7][j], q6 = win[u][j];
            const uint32_t acc = 18u * (q0 + q6) + 34u * (q1 + q5) + 48u * (q2 + q4) + 56u * q3;
            outw |= ((acc + 32768u) >> 16) << (8 * j);
          }
          reinterpret_cast<uint32_t*>(S.blurT)[(strip * 4 + i - 6) * (TW / 4) + q] = outw;
        }
      }
    }
  }

  // ---- level l+1: cv::resize INTER_LINEAR fixed point, every destination pixel whose top-left source sample lies in
  // this tile's interior (the +1 neighbours are inside the halo)
  if (a.level + 1 < g.nlevels) {
    const LevelGeom& D = g.lv[a.level + 1];
    const int16_t* tdx = a.tileDx + L.tdxOff;
    const int16_t* tdy = a.tileDy + L.tdyOff;
    const int dx0 = tdx[tx], nw = tdx[tx + 1] - dx0, dy0 = tdy[ty], nh = tdy[ty + 1] - dy0;
    // (nw <= TW and nh <= TH + 1: tile_build refuses scale factors so close to 1 that a tile would own more; at 1.1 a
    // tile owns up to 117 columns)
    if (tid < nh) {  // row parameters once per tile
      const int dy = dy0 + tid;
      const int sy = a.ryOfs[D.ryOff + dy];
      S.rzB[tid] = a.ryBeta[D.ryOff + dy];
      S.rzO0[tid] = (int16_t)(min(max(sy, 0), Hd - 1) - Y0);      // box row of the upper source row
      S.rzO1[tid] = (int16_t)(min(max(sy + 1, 0), Hd - 1) - Y0);  // ... and of the lower one
    }
    __syncthreads();
    // horizontal pass: for every source row of the tile that a destination row reads (<= TH + 1) and every destination
    // column, h = S[sx] * a0 + S[sx + 1] * a1 (>> 4 as the vertical stage wants it); the buffer reuses the blur's
    // horizontal sums (the blur is finished: barrier above)
    uint16_t* hb = S.blurH;  // [row of the box][destination column], pitch RZP
    constexpr int RZP = TW + 2;  // >= nw; box rows <= HY + TH, so the rows fit the blur's horizontal-sum buffer
    static_assert((HY + TH) * RZP + TW + 1 < BH * TW, "resize rows fit blurH");
    {
      const int rowLo = nh > 0 ? S.rzO0[0] : 0, rowHi = nh > 0 ? S.rzO1[nh - 1] : -1;  // box rows
      const int c = tid & 127;
      if (c < nw) {  // thread = (destination column, every second source row): column parameters stay in registers
        const int dx = dx0 + c;
        const int sx = a.rxOfs[D.rxOff + dx];
        const uint32_t aa = a.rxAlpha[D.rxOff + dx];
        const int a0 = (int16_t)(aa & 0xffffu), a1 = (int16_t)(aa >> 16);
        const uint8_t* cl = S.raw + (sx - X0);
        const uint8_t* cr = S.raw + (min(sx + 1, Wd - 1) - X0);
#pragma unroll 2
        for (int r = rowLo + (tid >> 7); r <= rowHi; r += 2) hb[r * RZP + c] = (uint16_t)((cl[r * BW] * a0 + cr[r * BW] * a1) >> 4);
      }
    }
    __syncthreads();
    // vertical pass: thread = (destination column, half of the rows)
    const int c = tid & 127, strip = tid >> 7;
    const int half = (nh + 1) >> 1;
    const int rBeg = strip * half, rEnd = min(nh, rBeg + half);
    if (c < nw && rBeg < rEnd) {
      uint8_t* dst = a.pyr + (size_t)(a.bBase + b) * g.pyrBytes + D.off + (size_t)(dy0 + rBeg) * D.pitch + dx0 + c;
#pragma unroll 2
      for (int r = rBeg; r < rEnd; r++) {
        const uint32_t bb = S.rzB[r];
        const int b0 = (int16_t)(bb & 0xffffu), b1 = (int16_t)(bb >> 16);
        const int h0 = hb[S.rzO0[r] * RZP + c], h1 = hb[S.rzO1[r] * RZP + c];
        *dst = (uint8_t)((((b0 * h0) >> 16) + ((b1 * h1) >> 16) + 2) >> 2);
        dst += D.pitch;
      }
    }
  }

  // ---- results out: the generic-proxy writes to shared memory become visible to the async proxy, then one thread issues
  // the bulk tensor stores (clipped at the image edge by the hardware)
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  if (tid == 0) {
    tma_store_3d(&tmScore, s32(S.scoreT), tx * TW, ty * TH, a.bBase + b);
    tma_store_3d(&tmBlur, s32(S.blurT), tx * TW, ty * TH, a.bBase + b);
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
  }
}

// ------------------------------------------------------------------------------------------------
// Per-cell rules of ComputeKeyPointsOctTree (src/ORBextractor.cc:1089-1157) on the strength map: one CTA per
// (image, level, row of cells).  A pixel is a keypoint at threshold th iff M > th and M is strictly greater than its 8
// neighbours INSIDE the cell's detectable area (cv::FAST runs on the cell ROI: the 3-pixel rim scores 0, so maxima never
// see across a seam).  Because M is the threshold-independent arc strength, the same maxima serve iniThFAST and
// minThFAST; a cell falls back to minThFAST only if it has no maximum above iniThFAST.
// The detectable areas of a level's cells tile [19, maxBorderX-3) x [19, maxBorderY-3) without gaps (cell j owns
// x in [19 + j*wCell, 19 + (j+1)*wCell)); cells the reference skips (:1099, :1116) own no pixel of that band.
// A row of cells is split by column range over L.nChunks CTAs of L.cellsPerCta cells: a strict 3x3 maximum of a cell
// occupies at most one pixel of each 2x2 block, so one CTA collects at most cellsPerCta * ceil(wCell/2) * ceil(hCell/2)
// <= CL_CAP maxima whatever the texture (build_geometry picks cellsPerCta).  The emission order does not matter: the
// quadtree orders candidates by candKey.
// ------------------------------------------------------------------------------------------------
constexpr int CL_CAP = kCellsListCap;
constexpr int CL_MAXCOLS = kCellsMaxCols;

__global__ void __launch_bounds__(256) k_cells(const __grid_constant__ ExtractGeom g, const uint8_t* __restrict__ score,
                                               const uint32_t* __restrict__ bitmap, uint32_t* __restrict__ candXY,
                                               uint32_t* __restrict__ candKey, uint8_t* __restrict__ candResp,
                                               int32_t* __restrict__ candCount, int32_t* __restrict__ status,
                                               uint2* __restrict__ fbList, int32_t* __restrict__ fbCount, int bAbs) {
  __shared__ uint32_t list[CL_CAP];
  __shared__ int cellAll[CL_MAXCOLS], cellHi[CL_MAXCOLS];
  __shared__ int sN, sBase, sEmit, sTotal;
  const int tid = threadIdx.x;
  const int b = blockIdx.y;
  int l = 0, k0 = blockIdx.x;  // CTA index -> (level, row of cells, column chunk)
  while (l < g.nlevels && k0 >= g.lv[l].nRows * g.lv[l].nChunks) {
    k0 -= g.lv[l].nRows * g.lv[l].nChunks;
    l++;
  }
  if (l >= g.nlevels) return;
  const LevelGeom& L = g.lv[l];
  const int ci = k0 / L.nChunks, chunk = k0 - ci * L.nChunks;
  const int cj0 = chunk * L.cellsPerCta, nc = min(L.nCols - cj0, L.cellsPerCta);  // cell columns [cj0, cj0 + nc)
  const int iniY = kMinBorder + ci * L.hCell;
  if (iniY >= L.maxBY - 3) return;  // :1099
  const int maxY = min(iniY + L.hCell + 6, L.maxBY);
  if (maxY - iniY < 7) return;
  const int ay0 = iniY + 3, ay1 = maxY - 3;          // detectable rows of this row of cells
  const int ax0 = kMinBorder + 3, ax1 = L.maxBX - 3;  // detectable columns of the level
  if (ax1 <= ax0) return;
  const int x0 = ax0 + cj0 * L.wCell, x1 = min(ax1, ax0 + (cj0 + nc) * L.wCell);  // this CTA's detectable columns
  for (int k = tid; k < nc; k += 256) {
    cellAll[k] = 0;
    cellHi[k] = 0;
  }
  if (tid == 0) {
    sN = 0;
    sEmit = 0;
  }
  __syncthreads();
  const int pitch = L.pitch, wCell = L.wCell;
  const uint8_t* img = score + (size_t)b * g.pyrBytes + L.off;
  const int iniTh = g.iniTh;
  // the tile kernel left one bit per pixel: "maximum of its cell above minThFAST" (row = tilesX*4 words; per 64 pixels an
  // even-pixel word and an odd-pixel word)
  // (this CTA reads the words of the 64-pixel groups that overlap [x0, x1) and keeps the bits inside it)
  const int bmPitch = L.tilesX * 4, ah = ay1 - ay0;
  const int wLo = (x0 >> 6) * 2, nw = x1 > x0 ? ((x1 - 1) >> 6) * 2 + 2 - wLo : 0;
  const uint32_t* bm = bitmap + (size_t)b * g.bmWords + L.bmOff + (size_t)ay0 * bmPitch + wLo;
  for (int k = tid; k < nw * ah; k += 256) {
    const int r = k / nw, wi = k - r * nw;
    uint32_t bits = bm[(size_t)r * bmPitch + wi];
    if (!bits) continue;
    const int xBase = ((wLo + wi) >> 1) * 64 + (wi & 1);
    while (bits) {
      const int bi = __ffs(bits) - 1;
      bits &= bits - 1;
      const int x = xBase + 2 * bi;
      if (x < x0 || x >= x1) continue;
      const int M = img[(size_t)(ay0 + r) * pitch + x];
      const int cj = (x - ax0) / wCell - cj0;
      const int slot = atomicAdd(&sN, 1);
      if (slot < CL_CAP) list[slot] = (uint32_t)x | ((uint32_t)r << 13) | ((uint32_t)M << 19);
      atomicAdd(&cellAll[cj], 1);
      if (M > iniTh) atomicAdd(&cellHi[cj], 1);
    }
  }
  __syncthreads();
  if (tid < 32) {  // candidates these cells emit: per cell the maxima above iniThFAST if it has any, else all
    int t = 0;
    for (int k = tid; k < nc; k += 32) t += cellHi[k] > 0 ? cellHi[k] : cellAll[k];
    t = warp_reduce_sum(t);
    if (tid == 0) {
      sTotal = t;
      sBase = t ? atomicAdd(&candCount[b * kMaxLevels + l], t) : 0;
      // (neither can happen: CL_CAP and candCap hold the geometric maximum; kept so that a sizing bug is an error)
      if (sN > CL_CAP || (t && sBase + t > L.candCap)) atomicOr(status, 1);
    }
  }
  __syncthreads();
  // cells without a maximum above iniThFAST: the minThFAST pass re-does them (k_fast_cells_list)
  for (int c = tid; c < nc; c += 256) {
    const int cj = cj0 + c;
    if (cellHi[c] > 0 || kMinBorder + cj * wCell >= L.maxBX - 6) continue;
    const int slot = atomicAdd(fbCount, 1);
    fbList[slot] = make_uint2((uint32_t)(bAbs + b), (uint32_t)(L.cellStart + ci * L.nCols + cj));
  }
  if (sTotal == 0) return;
  const int nList = min(sN, CL_CAP);
  const size_t cbase = (size_t)b * g.totalCandCap + L.candOff;
  for (int k = tid; k < nList; k += 256) {
    const uint32_t e = list[k];
    const int x = e & 0x1fff, r = (e >> 13) & 0x3f, M = e >> 19;
    const int cj = (x - ax0) / wCell;
    if (cellHi[cj - cj0] > 0 && M <= iniTh) continue;  // :1132-1139
    const int slot = sBase + atomicAdd(&sEmit, 1);
    if (slot >= L.candCap) continue;
    // kp.pt += (j*wCell, i*hCell) (:1150-1151) -> coordinates relative to the 16-pixel border
    candXY[cbase + slot] = (uint32_t)(x - kMinBorder) | ((uint32_t)(ay0 + r - kMinBorder) << 16);
    candKey[cbase + slot] = ((uint32_t)(ci * L.nCols + cj) << 12) | ((uint32_t)r << 6) | (uint32_t)(x - ax0 - cj * wCell);
    candResp[cbase + slot] = (uint8_t)(M - 1);
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qr;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) != cudaSuccess || !p) return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

static int encode_level_map(CUtensorMap* tm, uint8_t* base, const LevelGeom& L, uint32_t pyrBytes, int maxBatch, int boxW,
                            int boxH) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled is not available from the driver");
    return B2S_ERR_CUDA;
  }
  const cuuint64_t dims[3] = {(cuuint64_t)L.w, (cuuint64_t)L.h, (cuuint64_t)maxBatch};
  const cuuint64_t strides[2] = {(cuuint64_t)L.pitch, (cuuint64_t)pyrBytes};
  const cuuint32_t box[3] = {(cuuint32_t)boxW, (cuuint32_t)boxH, 1u};
  const cuuint32_t estr[3] = {1u, 1u, 1u};
  const CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, base + L.off, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) for a %dx%d level, pitch %d", (int)r, L.w, L.h, L.pitch);
    return B2S_ERR_CUDA;
  }
  return B2S_OK;
}

// Called at the end of build_geometry: tensor maps of every level (pyramid load, strength store, blur store) and the
// destination ranges each source tile owns in the bilinear resize.
int tile_build(b2s_extractor* h) {
  ExtractGeom& g = h->geom;
  std::vector<int16_t> tdx, tdy;
  uint32_t bmWords = 0;
  for (int l = 0; l < g.nlevels; l++) {
    LevelGeom& L = g.lv[l];
    L.tilesX = div_up(L.w, TW);
    L.tilesY = div_up(L.h, TH);
    L.bmOff = bmWords;
    bmWords += (uint32_t)(L.tilesX * 4) * (uint32_t)(L.tilesY * TH);
    L.tdxOff = (uint32_t)tdx.size();
    L.tdyOff = (uint32_t)tdy.size();
    if (l + 1 < g.nlevels) {
      // same float arithmetic as the resize tables (build_geometry): sx(dx), sy(dy) are non-decreasing
      const int dw = g.lv[l + 1].w, dh = g.lv[l + 1].h;
      const double scale_x = 1. / ((double)dw / L.w), scale_y = 1. / ((double)dh / L.h);
      int dx = 0;
      for (int t = 0; t <= L.tilesX; t++) {
        while (dx < dw) {
          float fx = (float)((dx + 0.5) * scale_x - 0.5);
          int sx = (int)floor((double)fx);
          if (sx < 0) sx = 0;
          if (sx >= L.w - 1) sx = L.w - 1;
          if (sx >= t * TW) break;
          dx++;
        }
        tdx.push_back((int16_t)dx);
      }
      int dy = 0;
      for (int t = 0; t <= L.tilesY; t++) {
        while (dy < dh) {
          float fy = (float)((dy + 0.5) * scale_y - 0.5);
          int sy = (int)floor((double)fy);
          sy = std::min(std::max(sy, 0), L.h - 1);
          if (sy >= t * TH) break;
          dy++;
        }
        tdy.push_back((int16_t)dy);
      }
    } else {
      for (int t = 0; t <= L.tilesX; t++) tdx.push_back(0);
      for (int t = 0; t <= L.tilesY; t++) tdy.push_back(0);
    }
  }
  g.bmWords = bmWords;
  // k_tile resizes with one thread per destination column a tile owns (at most TW) and keeps TH + 2 rows of parameters
  for (int l = 0; l + 1 < g.nlevels; l++) {
    const LevelGeom& L = g.lv[l];
    for (int t = 0; t < L.tilesX; t++)
      if (tdx[L.tdxOff + t + 1] - tdx[L.tdxOff + t] > TW) {
        set_error("scale factor %.6f is too close to 1: a 128-column tile of level %d owns more than 128 columns of level %d",
                  h->scaleFactor, l, l + 1);
        return B2S_ERR_BAD_ARG;
      }
    for (int t = 0; t < L.tilesY; t++)
      if (tdy[L.tdyOff + t + 1] - tdy[L.tdyOff + t] > TH + 2) {
        set_error("scale factor %.6f is too close to 1: a 32-row tile of level %d owns more than 34 rows of level %d",
                  h->scaleFactor, l, l + 1);
        return B2S_ERR_BAD_ARG;
      }
  }
  if ((size_t)bmWords > h->bmWordsAlloc) {
    set_error("NMS bitmap (%u words per image) exceeds its allocation", bmWords);
    return B2S_ERR_BAD_ARG;
  }
  if (tdx.size() > h->tileTabAlloc || tdy.size() > h->tileTabAlloc) {
    set_error("tile tables exceed their allocation");
    return B2S_ERR_BAD_ARG;
  }
  B2S_CUDA(cudaMemcpy(h->d.tileDx, tdx.data(), tdx.size() * 2, cudaMemcpyHostToDevice));
  B2S_CUDA(cudaMemcpy(h->d.tileDy, tdy.data(), tdy.size() * 2, cudaMemcpyHostToDevice));
  static_assert(sizeof(CUtensorMap) == 128, "CUtensorMap is 128 bytes");
  for (int l = 0; l < g.nlevels; l++) {
    int rc = encode_level_map(reinterpret_cast<CUtensorMap*>(h->tmPyr[l]), h->d.pyr, g.lv[l], g.pyrBytes, h->maxBatch, BW, BH);
    if (rc == B2S_OK)
      rc = encode_level_map(reinterpret_cast<CUtensorMap*>(h->tmScore[l]), h->d.score, g.lv[l], g.pyrBytes, h->maxBatch, TW, TH);
    if (rc == B2S_OK)
      rc = encode_level_map(reinterpret_cast<CUtensorMap*>(h->tmBlur[l]), h->d.blur, g.lv[l], g.pyrBytes, h->maxBatch, TW, TH);
    if (rc != B2S_OK) return rc;
  }
  B2S_CUDA(cudaFuncSetAttribute(k_tile, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TileSmem)));
  return B2S_OK;
}

// Enqueue the fused front end for `batch` images starting at image `bBase` of the handle's buffers.
int tile_run(b2s_extractor* h, int bBase, int batch, cudaStream_t st) {
  const ExtractGeom& g = h->geom;
  const DeviceBuffers& d = h->d;
  for (int l = 0; l < g.nlevels; l++) {
    TileArgs a;
    a.level = l;
    a.bBase = bBase;
    a.pyr = d.pyr;
    a.rxOfs = d.rxOfs;
    a.rxAlpha = d.rxAlpha;
    a.ryOfs = d.ryOfs;
    a.ryBeta = d.ryBeta;
    a.tileDx = d.tileDx;
    a.tileDy = d.tileDy;
    a.bitmap = d.bitmap;
    k_tile<<<dim3(g.lv[l].tilesX, g.lv[l].tilesY, batch), TILE_THREADS, sizeof(TileSmem), st>>>(
        *reinterpret_cast<const CUtensorMap*>(h->tmPyr[l]), *reinterpret_cast<const CUtensorMap*>(h->tmScore[l]),
        *reinterpret_cast<const CUtensorMap*>(h->tmBlur[l]), g, a);
    h->launches++;
  }
  // chunks of one batch run concurrently on two streams: each owns a slice of the fallback list and its own counter
  uint2* fbList = d.fbList + (size_t)bBase * g.totalCells;
  int32_t* fbCount = d.fbCount + bBase;
  B2S_CUDA(cudaMemsetAsync(fbCount, 0, 4, st));
  int cellCtas = 0;
  for (int l = 0; l < g.nlevels; l++) cellCtas += g.lv[l].nRows * g.lv[l].nChunks;
  k_cells<<<dim3(cellCtas, batch), 256, 0, st>>>(
      g, d.score + (size_t)bBase * g.pyrBytes, d.bitmap + (size_t)bBase * g.bmWords, d.candXY + (size_t)bBase * g.totalCandCap,
      d.candKey + (size_t)bBase * g.totalCandCap, d.candResp + (size_t)bBase * g.totalCandCap,
      d.candCount + (size_t)bBase * kMaxLevels, d.status, fbList, fbCount, bBase);
  h->launches++;
  // minThFAST pass for the listed cells (persistent CTAs, 16 per SM; the list length stays on the device)
  launch_fast_fallback(g, d, fbList, fbCount, std::min(g.totalCells * batch, h->numSMs * 16), st);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

}  // namespace b2s
