// extractor.cuh — geometry + handle of the H100 ORB extractor (see extractor.cu for the kernels).
#pragma once
#include <vector>

#include "common.cuh"

namespace b2s {

constexpr int kMaxLevels = 12;
constexpr int kEdge = 19;       // EDGE_THRESHOLD, src/ORBextractor.cc:86
constexpr int kMinBorder = 16;  // EDGE_THRESHOLD-3, :1064
constexpr int kPatch = 31;      // PATCH_SIZE, :82
constexpr int kHalfPatch = 15;  // HALF_PATCH_SIZE, :84

// Per-level constants, passed to kernels by value inside ExtractGeom.
struct LevelGeom {
  int w, h, pitch;        // level image (no border), row pitch in bytes (multiple of 16)
  uint32_t off;           // byte offset of the level inside one image's pyramid
  int maxBX, maxBY;       // maxBorderX/Y = dim-16 (:1066-1070)
  int nCols, nRows, wCell, hCell;  // cell grid (:1082-1086)
  int cellStart;          // first FAST CTA index of this level
  int N;                  // mnFeaturesPerLevel[level]
  int nIni;               // quadtree roots (:719)
  float hX;               // root width (:722)
  int candCap, candOff;   // candidate capacity (the level's exact maximum, cand_bound) / offset (entries) inside one
                          // image's candidate arrays
  int cellsPerCta, nChunks;  // k_cells: cell columns per CTA (their NMS maxima always fit its list) and CTAs per row
  int nodeCap, selOff;    // quadtree node capacity / offset of the level's selected keypoints
  float scale;            // mvScaleFactor[level]
  float kpsize;           // (float)(int)(PATCH_SIZE*scale) (:1175,1189)
  uint32_t rxOff, ryOff;  // resize tables (entries) for producing this level from level-1
  int tilesX, tilesY;     // 128 x 32 tiles of the fused front end (extractor_tile.cu)
  uint32_t tdxOff, tdyOff;  // per tile column / row: first level l+1 column / row whose source sample starts in it
  uint32_t bmOff;           // word offset of the level inside one image's NMS bitmap
};

struct ExtractGeom {
  int nlevels;
  int iniTh, minTh;
  int totalCells, totalCandCap, totalSelCap;
  uint32_t pyrBytes;  // bytes of one image's pyramid
  uint32_t bmWords;   // words of one image's NMS bitmap (fused front end)
  LevelGeom lv[kMaxLevels];
};

struct DeviceBuffers {
  uint8_t* pyr = nullptr;      // B x pyrBytes
  uint8_t* blur = nullptr;     // B x pyrBytes
  uint8_t* raw = nullptr;      // B x width*height dense upload staging (host-buffer batch path)
  uint8_t* score = nullptr;    // B x pyrBytes: FAST arc strength of every pixel (fused front end)
  uint32_t* bitmap = nullptr;  // B x bmWords: 1 bit per pixel, maxima of their cell above minThFAST (fused front end)
  uint2* fbList = nullptr;     // (image, cell) pairs that need the minThFAST pass (no maximum above iniThFAST); the chunk that
                               // starts at image b owns the entries from b * totalCells on and the counter fbCount[b]
  int32_t* fbCount = nullptr;
  int16_t* tileDx = nullptr;   // resize ownership tables of the fused front end
  int16_t* tileDy = nullptr;
  uint32_t* candXY = nullptr;  // B x totalCandCap   (x | y<<16, border-relative)
  uint32_t* candKey = nullptr; // B x totalCandCap   (order key: cell<<12 | ylocal<<6 | xlocal)
  uint8_t* candResp = nullptr; // B x totalCandCap
  uint16_t* candNode = nullptr;
  uint8_t* candQ = nullptr;
  int32_t* candCount = nullptr;  // B x kMaxLevels
  uint32_t* selXYR = nullptr;    // B x totalSelCap x 2 (x|y<<16 level coords, response)
  int32_t* selCount = nullptr;   // B x kMaxLevels
  uint32_t* cellInfo = nullptr;  // per FAST cell: level<<28 | cell row<<14 | cell column
  int32_t* status = nullptr;     // 1 int: bit0 cand overflow, bit1 output overflow, bit2 node overflow
  int16_t* rxOfs = nullptr;      // resize tables
  uint32_t* rxAlpha = nullptr;
  int16_t* ryOfs = nullptr;
  uint32_t* ryBeta = nullptr;
  b2s_keypoint* outKps = nullptr;  // B x outCap (internal result records for the host-buffer entry points)
  uint8_t* outDesc = nullptr;
  int32_t* outCounts = nullptr;
};

}  // namespace b2s

struct b2s_extractor;
namespace b2s {
int tile_build(b2s_extractor* h);  // tensor maps + resize ownership tables for the current geometry
int tile_run(b2s_extractor* h, int bBase, int batch, cudaStream_t st);
int launch_fast_fallback(const ExtractGeom& g, const DeviceBuffers& d, const uint2* fbList, const int32_t* fbCount, int gridCtas,
                         cudaStream_t st);  // extractor.cu
constexpr int kCellsListCap = 8192;  // k_cells: NMS maxima one CTA collects in shared memory (extractor_tile.cu)
constexpr int kCellsMaxCols = 64;    // k_cells: cell columns one CTA owns at most
constexpr int kFastCellCap = 1024;   // k_fast_cells_list: maxima of one cell it keeps in shared memory (extractor.cu)
}  // namespace b2s

struct b2s_extractor {
  int nfeatures, nlevels, iniTh, minTh;
  double scaleFactor;
  int maxW, maxH, maxBatch, device;
  int numSMs = 0;  // multiprocessors of `device` (grid of the persistent kernels)
  std::vector<float> scale, invScale, sigma2, invSigma2;
  std::vector<int> nFeat;
  int outCap;  // per-image record capacity of the internal output buffers
  // geometry cache for the current image size
  int curW = 0, curH = 0;
  b2s::ExtractGeom geom;
  b2s::DeviceBuffers d;
  size_t pyrBytesAlloc = 0, candCapAlloc = 0, selCapAlloc = 0, rxAlloc = 0, ryAlloc = 0, cellAlloc = 0;
  cudaStream_t stream = nullptr, stream2 = nullptr;
  // stereo matching scratch + bookkeeping of the last host-buffer batch extraction (b2s_stereo_match)
  int32_t* dStereoSad = nullptr;
  size_t stereoCap = 0, stereoOutCap = 0;
  float *dStereoU = nullptr, *dStereoD = nullptr;
  int32_t* dStereoN = nullptr;
  int lastCap = 0, lastBatch = 0;
  // pinned staging for the host-buffer entry points
  b2s_keypoint* hKps = nullptr;
  uint8_t* hDesc = nullptr;
  int32_t* hCounts = nullptr;
  int32_t* hStatus = nullptr;
  long long launches = 0;
  // fused front end (extractor_tile.cu)
  size_t tileTabAlloc = 0, bmWordsAlloc = 0;
  alignas(64) unsigned char tmPyr[b2s::kMaxLevels][128];    // CUtensorMap: level images (TMA load, 144 x 38 box)
  alignas(64) unsigned char tmScore[b2s::kMaxLevels][128];  // strength map (TMA store, 128 x 32 box)
  alignas(64) unsigned char tmBlur[b2s::kMaxLevels][128];   // blurred level (TMA store)
  // optional per-stage CUDA-event timing (bench.py roofline): resize chain, FAST, quadtree, blur, describe; events
  // around the tile front end, the quadtree and the description (resize chain and blur are part of the tile front end)
  int timing = 0;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  double stageMs[5] = {0, 0, 0, 0, 0};
  long long timedCalls = 0;
  int evPending = 0;
};
