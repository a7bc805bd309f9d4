// common.cuh — shared helpers for libb200slam.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <string>

#include "../../include/b200slam.h"

namespace b2s {

extern thread_local std::string g_last_error;
void set_error(const char* fmt, ...);

#define B2S_CUDA(call)                                                                                  \
  do {                                                                                                  \
    cudaError_t e__ = (call);                                                                           \
    if (e__ != cudaSuccess) {                                                                           \
      b2s::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__));            \
      return (e__ == cudaErrorNoDevice || e__ == cudaErrorInsufficientDriver) ? B2S_ERR_NO_DEVICE       \
                                                                               : B2S_ERR_CUDA;          \
    }                                                                                                   \
  } while (0)

int select_device(int device);  // returns B2S_OK / B2S_ERR_NO_DEVICE

// Device buffer grown on demand.  grow() reallocates when `bytes` exceeds the capacity, without keeping the contents
// (cudaFree synchronises the device); returns B2S_OK or a B2S_CUDA error.
struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
};
int grow(DevBuf& b, size_t bytes);

static inline int div_up(int a, int b) { return (a + b - 1) / b; }
static inline size_t align_up(size_t a, size_t b) { return (a + b - 1) / b * b; }

// ---- device helpers ----
__device__ __forceinline__ int warp_reduce_sum(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_incl_scan(int v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  return v;
}

// 256-bit descriptor load/store as two 128-bit global transactions per thread (LDG.E.128 / STG.E.128: sm_90 has no
// 256-bit load/store); descriptors are 32-byte aligned, so both halves stay in one 32-byte sector.
struct __align__(32) u256 {
  uint32_t w[8];
};
__device__ __forceinline__ u256 ld_u256(const void* p) {
  u256 r;
  asm volatile("ld.global.v4.b32 {%0,%1,%2,%3}, [%8];\n\tld.global.v4.b32 {%4,%5,%6,%7}, [%8+16];"
               : "=r"(r.w[0]), "=r"(r.w[1]), "=r"(r.w[2]), "=r"(r.w[3]), "=r"(r.w[4]), "=r"(r.w[5]), "=r"(r.w[6]),
                 "=r"(r.w[7])
               : "l"(p));
  return r;
}
__device__ __forceinline__ void st_u256(void* p, const u256& r) {
  asm volatile("st.global.v4.b32 [%0], {%1,%2,%3,%4};\n\tst.global.v4.b32 [%0+16], {%5,%6,%7,%8};" ::"l"(p), "r"(r.w[0]),
               "r"(r.w[1]), "r"(r.w[2]), "r"(r.w[3]), "r"(r.w[4]), "r"(r.w[5]), "r"(r.w[6]), "r"(r.w[7])
               : "memory");
}
// 256-bit Hamming distance with 4 instead of 8 POPC: the eight XOR words are compressed by a carry-save adder tree
// (sum = a^b^c, carry = maj(a,b,c): one LOP3 each) into bit planes of weight 1, 1, 2, 4.  POPC issues at a quarter of
// the LOP3 rate, and the brute-force matchers are bound by it.
__device__ __forceinline__ uint32_t csa_sum(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t r;
  asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
  return r;
}
__device__ __forceinline__ uint32_t csa_carry(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t r;
  asm("lop3.b32 %0, %1, %2, %3, 0xE8;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
  return r;
}
__device__ __forceinline__ int hamming256_words(uint32_t x0, uint32_t x1, uint32_t x2, uint32_t x3, uint32_t x4, uint32_t x5,
                                                uint32_t x6, uint32_t x7) {
  const uint32_t s1 = csa_sum(x0, x1, x2), c1 = csa_carry(x0, x1, x2);
  const uint32_t s2 = csa_sum(x3, x4, x5), c2 = csa_carry(x3, x4, x5);
  const uint32_t s3 = csa_sum(s1, s2, x6), c3 = csa_carry(s1, s2, x6);
  const uint32_t s4 = csa_sum(c1, c2, c3), c4 = csa_carry(c1, c2, c3);
  return __popc(s3) + __popc(x7) + 2 * __popc(s4) + 4 * __popc(c4);
}
__device__ __forceinline__ int hamming256(const u256& a, const u256& b) {
  return hamming256_words(a.w[0] ^ b.w[0], a.w[1] ^ b.w[1], a.w[2] ^ b.w[2], a.w[3] ^ b.w[3], a.w[4] ^ b.w[4],
                          a.w[5] ^ b.w[5], a.w[6] ^ b.w[6], a.w[7] ^ b.w[7]);
}

}  // namespace b2s
