// distinctive.cuh — the per-point body of MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:359-440), shared by
// k_distinctive (matcher.cu) and the keyframe insertion (mappoint.cu).
#pragma once
#include "common.cuh"

namespace b2s {

// One warp, N >= 1 descriptors, desc(i) loads descriptor i; h: 257+ ints of shared memory owned by the warp.  For every
// descriptor i the median (sorted row element floor(0.5*(N-1))) of its distances to all N is read off a 257-bin
// histogram; returns the first i with the smallest median (on every lane).
template <class Desc>
__device__ __forceinline__ int distinctive_best(int N, Desc desc, int* h, int lane) {
  const int kth = (int)(0.5 * (double)(N - 1));
  int bestMedian = 0x7fffffff, best = 0;
  for (int i = 0; i < N; i++) {
    for (int b = lane; b < 257; b += 32) h[b] = 0;
    __syncwarp();
    const u256 di = desc(i);
    for (int j = lane; j < N; j += 32) atomicAdd(&h[(j == i) ? 0 : hamming256(di, desc(j))], 1);
    __syncwarp();
    // smallest value v with #(distances <= v) > kth: warp scan over 257 bins (9 per lane)
    int local[9], sum = 0;
#pragma unroll
    for (int t = 0; t < 9; t++) {
      const int b = lane * 9 + t;
      local[t] = (b < 257) ? h[b] : 0;
      sum += local[t];
    }
    int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    int run = incl - sum, med = 0x7fffffff;
#pragma unroll
    for (int t = 0; t < 9; t++) {
      run += local[t];
      if (med == 0x7fffffff && run > kth && lane * 9 + t < 257) med = lane * 9 + t;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) med = min(med, __shfl_xor_sync(0xffffffffu, med, o));
    if (med < bestMedian) {  // strict: the first minimum wins (:424-428)
      bestMedian = med;
      best = i;
    }
    __syncwarp();
  }
  return best;
}

}  // namespace b2s
