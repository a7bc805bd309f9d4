// ingest.cu — what happens to a camera frame before the grey image exists: Tracking::GrabImage*'s colour-to-grey step
// (src/Tracking.cc:252-278, :313-326, :371-384), optionally preceded by the stereo examples' rectification
// cv::remap(src, dst, mapx, mapy, INTER_LINEAR) with CV_32FC1 maps and BORDER_CONSTANT 0
// (Examples/Stereo/stereo_euroc.cc:124-189).  Both are integer arithmetic pinned to OpenCV 4 (include/b200slam.h):
//   grey:  Y = (9798 R + 19235 G + 3735 B + 16384) >> 15 (alpha ignored; mbRGB, not the data, says which byte is R);
//   remap: X = cvRound(mapx * 32), Y likewise; taps (X >> 5, Y >> 5) .. +1 with weights (32 - ax)(32 - ay), ax (32 - ay),
//          (32 - ax) ay, ax ay (ax = X & 31, ay = Y & 31); a tap outside the source adds 0; dst = (sum + 512) >> 10.
// A colour image is remapped channel by channel and converted afterwards (the two do not commute).  One thread per 4
// consecutive output pixels of a row, one 32-bit store where the output address allows it.
#include <cmath>

#include "extractor.cuh"

namespace b2s {
namespace {

constexpr int kMaxDim = 8192;

struct IngestArgs {
  const uint8_t* src;
  size_t srcRow, srcImg;
  int srcW, srcH;
  const float* mapx;
  const float* mapy;
  size_t mapRow;  // bytes
  int w, h;
  uint8_t* out;
  size_t outRow, outImg;
  int r, b;  // byte offsets of R and B inside a pixel (rgb: 0, 2; bgr: 2, 0)
};

__device__ __forceinline__ uint32_t grey(uint32_t r, uint32_t g, uint32_t b) {
  return (9798u * r + 19235u * g + 3735u * b + 16384u) >> 15;
}

// cvRound(m * 32) as x86 computes it keeps NaN outside the image (INT_MIN); cvt.rni turns NaN into 0, which is inside,
// so NaN is sent outside explicitly.  m * 32 is exact; +-inf and huge values saturate to INT_MIN / INT_MAX, outside too.
__device__ __forceinline__ int fixed5(float m) { return isnan(m) ? INT_MIN : __float2int_rn(m * 32.f); }

// one output pixel: the remapped channels (C = 1: the grey value) -> grey
template <int C>
__device__ __forceinline__ uint32_t remap_pixel(const IngestArgs& a, const uint8_t* __restrict__ img, float mx, float my) {
  const int X = fixed5(mx), Y = fixed5(my);
  const int sx = X >> 5, sy = Y >> 5;
  const int ax = X & 31, ay = Y & 31;
  const bool x0 = sx >= 0 && sx < a.srcW, x1 = sx >= -1 && sx < a.srcW - 1;
  const bool y0 = sy >= 0 && sy < a.srcH, y1 = sy >= -1 && sy < a.srcH - 1;
  const int w00 = (32 - ax) * (32 - ay), w01 = ax * (32 - ay), w10 = (32 - ax) * ay, w11 = ax * ay;
  const uint8_t* r0 = img + (ptrdiff_t)sy * (ptrdiff_t)a.srcRow + (ptrdiff_t)sx * C;
  const uint8_t* r1 = r0 + a.srcRow;
  constexpr int NC = C == 1 ? 1 : 3;  // alpha cannot reach the output
  uint32_t v[NC];
#pragma unroll
  for (int c = 0; c < NC; c++) {
    int s = 0;
    if (y0 && x0) s += (int)__ldg(r0 + c) * w00;
    if (y0 && x1) s += (int)__ldg(r0 + C + c) * w01;
    if (y1 && x0) s += (int)__ldg(r1 + c) * w10;
    if (y1 && x1) s += (int)__ldg(r1 + C + c) * w11;
    v[c] = (uint32_t)((s + 512) >> 10);
  }
  if constexpr (C == 1)
    return v[0];
  else
    return a.r == 0 ? grey(v[0], v[1], v[2]) : grey(v[2], v[1], v[0]);  // no dynamic index into registers
}

template <int C>
__device__ __forceinline__ uint32_t copy_pixel(const IngestArgs& a, const uint8_t* __restrict__ row, int x) {
  const uint8_t* p = row + (size_t)x * C;
  if constexpr (C == 1)
    return __ldg(p);
  else
    return grey(__ldg(p + a.r), __ldg(p + 1), __ldg(p + a.b));
}

// grid: (ceil(ceil(w / 4) * h / 128), batch); thread t of image b owns row t / ceil(w / 4), pixels 4 (t % ceil(w / 4)) ..
template <int C, bool MAPS>
__global__ void __launch_bounds__(128) k_prepare(IngestArgs a) {
  const int qw = (a.w + 3) >> 2;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= qw * a.h) return;
  const int y = t / qw, x0 = (t - y * qw) * 4;
  const int n = min(4, a.w - x0);
  const uint8_t* img = a.src + (size_t)blockIdx.y * a.srcImg;
  uint32_t px[4] = {0, 0, 0, 0};
  if constexpr (MAPS) {
    const float* mxr = reinterpret_cast<const float*>(reinterpret_cast<const uint8_t*>(a.mapx) + (size_t)y * a.mapRow) + x0;
    const float* myr = reinterpret_cast<const float*>(reinterpret_cast<const uint8_t*>(a.mapy) + (size_t)y * a.mapRow) + x0;
    float mx[4], my[4];
    if (n == 4 && !((reinterpret_cast<uintptr_t>(mxr) | reinterpret_cast<uintptr_t>(myr)) & 15)) {
      const float4 fx = __ldg(reinterpret_cast<const float4*>(mxr)), fy = __ldg(reinterpret_cast<const float4*>(myr));
      mx[0] = fx.x; mx[1] = fx.y; mx[2] = fx.z; mx[3] = fx.w;
      my[0] = fy.x; my[1] = fy.y; my[2] = fy.z; my[3] = fy.w;
    } else {
#pragma unroll
      for (int k = 0; k < 4; k++) {
        mx[k] = k < n ? __ldg(mxr + k) : 0.f;
        my[k] = k < n ? __ldg(myr + k) : 0.f;
      }
    }
#pragma unroll
    for (int k = 0; k < 4; k++)
      if (k < n) px[k] = remap_pixel<C>(a, img, mx[k], my[k]);
  } else {
    const uint8_t* row = img + (size_t)y * a.srcRow;
#pragma unroll
    for (int k = 0; k < 4; k++)
      if (k < n) px[k] = copy_pixel<C>(a, row, x0 + k);
  }
  uint8_t* o = a.out + (size_t)blockIdx.y * a.outImg + (size_t)y * a.outRow + x0;
  if (n == 4 && !(reinterpret_cast<uintptr_t>(o) & 3)) {
    *reinterpret_cast<uint32_t*>(o) = px[0] | px[1] << 8 | px[2] << 16 | px[3] << 24;
  } else {
#pragma unroll
    for (int k = 0; k < 4; k++)
      if (k < n) o[k] = (uint8_t)px[k];
  }
}

template <int C>
void launch_prepare(const IngestArgs& a, int batch, bool maps, cudaStream_t st) {
  const dim3 grid(div_up(((a.w + 3) >> 2) * a.h, 128), batch);
  if (maps)
    k_prepare<C, true><<<grid, 128, 0, st>>>(a);
  else
    k_prepare<C, false><<<grid, 128, 0, st>>>(a);
}

}  // namespace
}  // namespace b2s

using namespace b2s;

extern "C" int b2s_prepare_images_device(b2s_extractor* h, const uint8_t* d_src, size_t src_row_bytes,
                                         size_t src_image_bytes, int batch, int src_width, int src_height, int channels,
                                         int rgb, const float* d_mapx, const float* d_mapy, size_t map_row_bytes, int width,
                                         int height, uint8_t* d_out, size_t out_row_bytes, size_t out_image_bytes,
                                         void* stream) {
  const bool maps = d_mapx && d_mapy;
  auto dim_ok = [](int v) { return v >= 1 && v <= kMaxDim; };
  if (!h || !d_src || !d_out || (!d_mapx != !d_mapy) || batch < 1 || batch > 65535 ||
      (channels != 1 && channels != 3 && channels != 4) || !dim_ok(src_width) || !dim_ok(src_height) || !dim_ok(width) ||
      !dim_ok(height) || src_row_bytes < (size_t)src_width * channels || src_image_bytes < src_row_bytes * src_height ||
      out_row_bytes < (size_t)width || out_image_bytes < out_row_bytes * height ||
      (maps && (map_row_bytes % 4 || map_row_bytes < (size_t)width * 4)) ||
      (!maps && (width != src_width || height != src_height)))
    return refuse(h, "b2s_prepare_images_device");
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
  IngestArgs a{d_src, src_row_bytes, src_image_bytes, src_width, src_height, d_mapx, d_mapy, map_row_bytes, width, height,
               d_out, out_row_bytes, out_image_bytes, rgb ? 0 : 2, rgb ? 2 : 0};
  if (channels == 1)
    launch_prepare<1>(a, batch, maps, st);
  else if (channels == 3)
    launch_prepare<3>(a, batch, maps, st);
  else
    launch_prepare<4>(a, batch, maps, st);
  h->launches += 1;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}
