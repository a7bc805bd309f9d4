// common.cu — error text, device selection, version for libb200slam.so
#include <stdarg.h>

#include "common.cuh"

namespace b2s {
thread_local std::string g_last_error;

void set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
}

int select_device(int device) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0) {
    set_error("no CUDA device available (%s): libb200slam has no CPU fallback",
              e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
    cudaGetLastError();
    return B2S_ERR_NO_DEVICE;
  }
  if (device < 0 || device >= n) {
    set_error("device %d out of range (have %d)", device, n);
    return B2S_ERR_BAD_ARG;
  }
  e = cudaSetDevice(device);
  if (e != cudaSuccess) {
    set_error("cudaSetDevice(%d): %s", device, cudaGetErrorString(e));
    return B2S_ERR_CUDA;
  }
  return B2S_OK;
}

int grow(DevBuf& b, size_t bytes) {
  if (bytes == 0) bytes = 16;
  if (b.bytes >= bytes) return B2S_OK;
  if (b.p) cudaFree(b.p);
  b.p = nullptr;
  b.bytes = 0;
  B2S_CUDA(cudaMalloc(&b.p, bytes));
  b.bytes = bytes;
  return B2S_OK;
}
}  // namespace b2s

extern "C" const char* b2s_last_error(void) { return b2s::g_last_error.c_str(); }
extern "C" int b2s_version(void) { return 100; }
extern "C" int b2s_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

// ------------------------------------------------------------------------------------------------
// b2s_measure_peaks: issue-rate micro-benchmarks of the pipes the hot kernels are bound by (bench.py reports them next to
// the kernel figures: MEASURED_PEAKS.json only has HBM copy bandwidth and bf16 GEMM throughput).
//   [0] packed u16x2 3-input min/max (VIMNMX3, ALU pipe: the FAST strength of the front end)  G warp-instr/s
//   [1] IMAD (FMA pipe)                                                                         G warp-instr/s
//   [2] FP64 DFMA (the LocalBA / PoseOptimization solvers)                                      TFLOP/s
//   [3] POPC (the Hamming matchers)                                                             G warp-instr/s
//   [4] VIMNMX3 + IMAD interleaved 1:1 (ALU and FMA pipes issue side by side)                   G warp-instr/s
// ------------------------------------------------------------------------------------------------
namespace b2s {
template <int MODE>
__global__ void __launch_bounds__(256) k_peak(uint32_t* out, int iters, uint32_t seed) {
  uint32_t a[8], b[8];
  double da[8], db[8];
#pragma unroll
  for (int i = 0; i < 8; i++) {
    a[i] = (seed * (threadIdx.x + i + 1)) & 0x00ff00ffu;
    b[i] = (seed + i * 77 + threadIdx.x) & 0x00ff00ffu;
    da[i] = 1.0 + 1e-9 * (double)(threadIdx.x + i);
    db[i] = 1e-12 * (double)(seed & 255u);
  }
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < 8; i++) {
      if (MODE == 0) {
        a[i] = __vimin3_u16x2(a[i], b[i], b[(i + 1) & 7]);
        b[i] = __vimax3_u16x2(b[i], a[i], a[(i + 3) & 7]);
      } else if (MODE == 1) {
        a[i] = a[i] * 3u + b[i];
        b[i] = b[i] * 5u + a[(i + 3) & 7];
      } else if (MODE == 2) {
        da[i] = fma(da[i], 1.0000001, db[i]);
        db[i] = fma(db[i], 0.9999999, da[(i + 3) & 7]);
      } else if (MODE == 3) {
        a[i] = __popc(a[i] ^ b[i]) + b[(i + 1) & 7];
        b[i] = __popc(b[i] + a[(i + 3) & 7]) ^ a[i];
      } else if (MODE == 5) {
        // four independent IMMA.16832.U8.U8 accumulator tiles (a[0..3], a[4..7], b[0..3], b[4..7]); one per statement pair
        if (i < 4) {
          uint32_t* t = (i & 1) ? b : a;
          const int o = (i & 2) ? 4 : 0;
          asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                       : "+r"(t[o]), "+r"(t[o + 1]), "+r"(t[o + 2]), "+r"(t[o + 3])
                       : "r"(seed), "r"(seed + 1u), "r"(seed + 2u), "r"(seed + 3u), "r"(seed + 4u), "r"(seed + 5u));
        }
      } else {
        a[i] = __vimin3_u16x2(a[i], b[i], b[(i + 1) & 7]);
        b[i] = b[i] * 5u + a[(i + 3) & 7];
      }
    }
  }
  uint32_t s = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) s ^= a[i] ^ b[i] ^ (uint32_t)__double2int_rn(da[i] + db[i]);
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
}  // namespace b2s

extern "C" int b2s_measure_peaks(int device, double* out8) {
  using namespace b2s;
  if (!out8) return B2S_ERR_BAD_ARG;
  int rc = select_device(device);
  if (rc != B2S_OK) return rc;
  for (int i = 0; i < 8; i++) out8[i] = 0;
  cudaDeviceProp prop;
  B2S_CUDA(cudaGetDeviceProperties(&prop, device));
  const int ctas = prop.multiProcessorCount * 8, iters = 2000;
  uint32_t* d = nullptr;
  B2S_CUDA(cudaMalloc(&d, (size_t)ctas * 256 * 4));
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  for (int m = 0; m < 6; m++) {
    float best = 1e30f;
    for (int rep = 0; rep < 4; rep++) {
      cudaEventRecord(e0);
      switch (m) {
        case 0: k_peak<0><<<ctas, 256>>>(d, iters, 12345u); break;
        case 1: k_peak<1><<<ctas, 256>>>(d, iters, 12345u); break;
        case 2: k_peak<2><<<ctas, 256>>>(d, iters, 12345u); break;
        case 3: k_peak<3><<<ctas, 256>>>(d, iters, 12345u); break;
        case 4: k_peak<4><<<ctas, 256>>>(d, iters, 12345u); break;
        default: k_peak<5><<<ctas, 256>>>(d, iters, 12345u); break;
      }
      cudaEventRecord(e1);
      cudaEventSynchronize(e1);
      float ms = 0;
      cudaEventElapsedTime(&ms, e0, e1);
      if (rep > 0 && ms < best) best = ms;
    }
    const double winstr = (double)ctas * 8 /*warps*/ * 16 /*per iteration*/ * iters;
    if (m == 2)
      out8[2] = winstr * 32 * 2 / (best * 1e-3) / 1e12;  // DFMA = 2 flop per lane
    else if (m == 3)
      out8[3] = winstr / (best * 1e-3) / 1e9;  // (POPC + one integer op per statement: POPC issue is what bounds it)
    else if (m == 5)
      out8[5] = winstr / 4.0 / (best * 1e-3) / 1e9;  // 4 IMMA per iteration (the other statements compile to nothing)
    else
      out8[m] = winstr / (best * 1e-3) / 1e9;
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaFree(d);
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}
