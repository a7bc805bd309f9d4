// matcher.cuh — the b2s_matcher handle, shared by matcher.cu and the per-point map routines of mappoint.cu.
#pragma once
#include "common.cuh"

namespace b2s {
struct ProjQuery;
}

struct b2s_matcher : b2s::Stage {
  int maxF, maxBatch;
  long long launches = 0;
  // device work buffers
  uint8_t *dDescA = nullptr, *dDescB = nullptr, *dValidA = nullptr, *dValidB = nullptr, *dOcc = nullptr, *dTaken = nullptr;
  int32_t *dNodeA = nullptr, *dNodeB = nullptr, *dNA = nullptr, *dNB = nullptr, *dOrder = nullptr, *dCandCnt = nullptr;
  int32_t *dMatch = nullptr, *dBin = nullptr, *dNMatches = nullptr, *dOct = nullptr, *dCellKey = nullptr;
  int32_t *dCellStart = nullptr, *dTopkIdx = nullptr, *dExtra = nullptr, *dHist = nullptr, *dPush = nullptr;
  float *dAngA = nullptr, *dAngB = nullptr, *dKpx = nullptr, *dKpy = nullptr, *dURight = nullptr;
  uint32_t* dTopk = nullptr;
  b2s::ProjQuery* dQueries = nullptr;
  // record staging of b2s_search_by_projection_last_batch and b2s_search_by_projection_sequence (grown on first use)
  b2s::DevBuf dKpsStage;
  // the rest of the staging of b2s_search_by_projection_sequence: records of batch + 1 frames
  b2s::DevBuf dSeqDesc, dSeqDepth, dSeqT, dSeqN;
  // b2s_distinctive_descriptors: descriptors, point offsets and results
  b2s::DevBuf dDistDesc, dDistOff, dDistBest;
  // b2s_update_normal_and_depth and b2s_process_new_keyframe: packed inputs (descriptors included); outputs, then scratch
  b2s::Packed mpIn, mpOut;
};
