// common.cuh — shared helpers for libb200slam.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

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

static inline size_t align_up(size_t a, size_t b) { return (a + b - 1) / b * b; }

// Device buffer grown on demand, freed by its destructor.  grow() reallocates when `bytes` exceeds the capacity, without
// keeping the contents (cudaFree synchronises the device); returns B2S_OK or a B2S_CUDA error.
struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() {
    if (p) cudaFree(p);
  }
};
int grow(DevBuf& b, size_t bytes);
// Exchanges two buffers: a buffer whose contents must survive a reallocation is filled in a new one, then swapped in.
void swap(DevBuf& a, DevBuf& b);
// Its pinned host counterpart (cudaMallocHost), with the same grow().
struct HostBuf {
  void* p = nullptr;
  size_t bytes = 0;
  HostBuf() = default;
  HostBuf(const HostBuf&) = delete;
  HostBuf& operator=(const HostBuf&) = delete;
  ~HostBuf() {
    if (p) cudaFreeHost(p);
  }
};
int grow(HostBuf& b, size_t bytes);

// n values of T at byte offset `off` of a Packed area.
template <class T>
struct Seg {
  size_t off = 0, n = 0;
  size_t end() const { return off + n * sizeof(T); }
};

// The arrays of a batched call, packed into one pinned host area and one device area at the same offsets: the host side
// is filled or read, the device side goes into the kernels' arguments, and each direction is one copy.  Every array
// starts at a 256-byte boundary, the start alignment of a cudaMalloc of its own.
//   layout:  clear(), then add<T>(n) for each array in order; `used` is the bytes they span.
//   sizing:  reserve() once at create, after a layout at the handle's capacities; a later layout that outgrows it is
//            refused by fit() with B2S_ERR_CAPACITY.  Without reserve(), fit() grows both areas to max(used, 2 x their
//            size), without keeping their contents: call sizes vary and cudaFree synchronises the device.
//   moving:  upload() copies [0, used) to the device; download() copies a byte range of it back (by default all of it).
struct Packed {
  HostBuf h;
  DevBuf d;
  size_t used = 0;
  bool reserved = false;

  void clear() { used = 0; }
  template <class T>
  Seg<T> add(size_t n) {
    const Seg<T> s{align_up(used, 256), n};
    used = s.end();
    return s;
  }
  template <class T>
  T* host(Seg<T> s) const {
    return reinterpret_cast<T*>(static_cast<char*>(h.p) + s.off);
  }
  template <class T>
  T* dev(Seg<T> s) const {
    return reinterpret_cast<T*>(static_cast<char*>(d.p) + s.off);
  }
  // Copies the segment's n values from src into the host area; returns the segment's device address.
  template <class T>
  T* stage(Seg<T> s, const T* src) {
    if (s.n) memcpy(host(s), src, s.n * sizeof(T));
    return dev(s);
  }
  // Allocates `used` bytes on the device and, when `pinned`, on the host (a device-only area holds scratch no copy
  // touches).  Like Stage::alloc, it does nothing once `error` is set and records its own failure there.
  void reserve(cudaError_t& error, bool pinned = true);
  int fit(const char* fn);  // B2S_OK when both areas hold `used` bytes; `fn` names the entry point in the error
  int upload(cudaStream_t s) const;
  int download(cudaStream_t s, size_t from = 0, size_t to = SIZE_MAX) const;
};

// The host side every device stage's handle shares (the handle struct derives from it): its device, a non-blocking
// stream, the two events around the timed segment of a call and that segment's device time, and the buffers allocated
// for the handle's lifetime.
//   create:  open(device), then alloc / alloc_pinned for each buffer; `error` holds the first failure, after which
//            every later open / alloc does nothing, so a create function checks it once at the end.
//   a call:  begin() before the timed segment, finish() after it (waits for the stream, reads lastMs).
//   destroy: close(), then delete the handle; buffers the handle holds itself (DevBuf, HostBuf) are freed by their
//            destructors after close() has synchronised the stream.
struct Stage {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  float lastMs = 0.f;
  cudaError_t error = cudaSuccess;
  std::vector<void*> devAllocs, pinnedAllocs;

  void open(int dev);
  template <class T>
  void alloc(T*& p, size_t bytes) {
    alloc_bytes(reinterpret_cast<void**>(&p), bytes, false);
  }
  template <class T>
  void alloc_pinned(T*& p, size_t bytes) {
    alloc_bytes(reinterpret_cast<void**>(&p), bytes, true);
  }
  int begin();   // records ev[0] on the stream
  int finish();  // records ev[1], waits for the stream, checks for a launch error and sets lastMs
  void close();  // sets the device, waits for the stream, frees the recorded buffers, destroys the events and stream

 private:
  void alloc_bytes(void** p, size_t bytes, bool pinned);
};

// Host-side checks of caller CSRs: off[0] == 0, non-decreasing, off[rows] <= cap.
bool csr_ok(const int32_t* off, int rows, int64_t cap);
// Every entry of the rows of a valid CSR in [lo, hi); each row strictly ascending when `ascending`.
bool entries_ok(const int32_t* off, const int32_t* v, int rows, int lo, int hi, bool ascending);
// k minimal sets of `width` indices each (row-major): true when every entry is in [0, n) and differs from the earlier
// entries of its row, else false with the first bad (set, entry) written to *set / *entry.
bool sets_ok(const int32_t* sets, int k, int width, int n, int* set, int* entry);

static inline int div_up(int a, int b) { return (a + b - 1) / b; }

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
