// undistort.cu — Frame::UndistortKeyPoints and Frame::ComputeStereoFromRGBD (src/Frame.cc:899-964, :1423-1461) on the
// extractor's device-resident keypoint records, and cv::undistortPoints on host points (the corners of
// Frame::ComputeImageBounds, :967-1014).
//
// The undistortion restates OpenCV 4's cvUndistortPointsInternal for P = K, R = I, no tilt and its default criteria
// (COUNT, 5 iterations): everything in double, the float K and coefficients widened, each operation rounded on its own.
// Built with --fmad=false (build.py): a contracted a*b+c would round once where the x86 code rounds twice, and the
// result is meant to be bit-identical to cv2.undistortPoints.  One thread per keypoint.
#include <cmath>

#include "extractor.cuh"

namespace b2s {
namespace {

struct Undistort {
  double fx, fy, cx, cy, ifx, ify;
  double k[5];  // k1 k2 p1 p2 k3 (k3 = 0 for a 4-coefficient model)
};

// cvUndistortPointsInternal, one point.  The identity tilt and rectification multiply by exact ones and zeros and are
// left out; the projection through P = K keeps its `0*y` term (it only matters for a non-finite coordinate).
__host__ __device__ inline void undistort_point(const Undistort& p, float u, float v, float* xo, float* yo) {
  const double* k = p.k;
  const double k5 = 0, k6 = 0, k7 = 0, k8 = 0, k9 = 0, k10 = 0, k11 = 0;  // the 8- and 12-coefficient terms
  double x = ((double)u - p.cx) * p.ifx;
  double y = ((double)v - p.cy) * p.ify;
  const double x0 = x, y0 = y;
  for (int j = 0; j < 5; j++) {
    const double r2 = x * x + y * y;
    const double icdist = (1 + ((k7 * r2 + k6) * r2 + k5) * r2) / (1 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2);
    if (icdist < 0) {  // OpenCV 4 only (regression 14583): back to the first normalised point
      x = ((double)u - p.cx) * p.ifx;
      y = ((double)v - p.cy) * p.ify;
      break;
    }
    const double deltaX = 2 * k[2] * x * y + k[3] * (r2 + 2 * x * x) + k8 * r2 + k9 * r2 * r2;
    const double deltaY = k[2] * (r2 + 2 * y * y) + 2 * k[3] * x * y + k10 * r2 + k11 * r2 * r2;
    x = (x0 - deltaX) * icdist;
    y = (y0 - deltaY) * icdist;
  }
  *xo = (float)(p.fx * x + 0 * y + p.cx);
  *yo = (float)(p.fy * y + 0 * x + p.cy);
}

// records [b][cap]: the first min(counts[b], cap) of image b are rewritten with the undistorted x, y (apply = 1) or
// copied (apply = 0: k1 == 0, src/Frame.cc:905-909); in == out is allowed.
__global__ void k_undistort_kps(const b2s_keypoint* __restrict__ in, const int32_t* __restrict__ counts, int cap,
                                Undistort p, int apply, b2s_keypoint* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (i >= min(counts[b], cap)) return;
  const size_t r = (size_t)b * cap + i;
  b2s_keypoint kp = in[r];
  if (apply) undistort_point(p, kp.x, kp.y, &kp.x, &kp.y);
  out[r] = kp;
}

// n host points (x, y pairs) undistorted in place on the device
__global__ void k_undistort_xy(float2* __restrict__ xy, int n, Undistort p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float2 q = xy[i];
  undistort_point(p, q.x, q.y, &q.x, &q.y);
  xy[i] = q;
}

// ComputeStereoFromRGBD: the depth at the distorted keypoint (coordinates truncated to int), mvuRight from the
// undistorted x.  `d > 0` is false for 0, negatives and NaN.  A keypoint whose truncated position is outside the depth
// image has no depth.  T = float: metres; T = uint16_t: the sensor's raw depth, converted at the keypoint as
// GrabImageRGBD's convertTo(CV_32F, factor) converts every pixel (src/Tracking.cc:334-338): the product of a u16 and a
// float is exact in double, so the one float rounding of (float)raw * factor is OpenCV's result whatever its precision.
template <typename T>
__global__ void k_stereo_from_depth(const b2s_keypoint* __restrict__ kps, const b2s_keypoint* __restrict__ kpsUn,
                                    const int32_t* __restrict__ counts, int cap, const uint8_t* __restrict__ depth,
                                    size_t pitch, size_t imgBytes, int width, int height, float factor, float bf,
                                    float* __restrict__ uright, float* __restrict__ depthOut) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (i >= min(counts[b], cap)) return;
  const size_t r = (size_t)b * cap + i;
  const float x = kps[r].x, y = kps[r].y;
  float ur = -1.f, dd = -1.f;
  if (x > -1.f && x < (float)width && y > -1.f && y < (float)height) {
    const int u = (int)x, v = (int)y;
    const T raw = *reinterpret_cast<const T*>(depth + (size_t)b * imgBytes + (size_t)v * pitch + (size_t)u * sizeof(T));
    float d;
    if constexpr (sizeof(T) == 2)
      d = __fmul_rn((float)raw, factor);
    else
      d = raw;
    if (d > 0) {
      dd = d;
      ur = __fsub_rn(kpsUn[r].x, __fdiv_rn(bf, d));
    }
  }
  uright[r] = ur;
  depthOut[r] = dd;
}

// K4 = fx, fy, cx, cy; dist = k1 k2 p1 p2 [k3]
bool make_params(const float* K4, const float* dist, int n_dist, Undistort* p) {
  if (!K4 || !dist || (n_dist != 4 && n_dist != 5)) return false;
  for (int i = 0; i < 4; i++)
    if (!std::isfinite(K4[i])) return false;
  for (int i = 0; i < n_dist; i++)
    if (!std::isfinite(dist[i])) return false;
  if (K4[0] == 0.f || K4[1] == 0.f) return false;
  p->fx = K4[0]; p->fy = K4[1]; p->cx = K4[2]; p->cy = K4[3];
  p->ifx = 1. / p->fx;
  p->ify = 1. / p->fy;
  for (int i = 0; i < 5; i++) p->k[i] = i < n_dist ? (double)dist[i] : 0.;
  return true;
}

}  // namespace
}  // namespace b2s

using namespace b2s;

extern "C" int b2s_undistort_keypoints_device(b2s_extractor* h, const b2s_keypoint* d_kps, const int32_t* d_counts, int batch,
                                              int cap, const float* K4, const float* dist, int n_dist, b2s_keypoint* d_kps_un,
                                              void* stream) {
  Undistort p;
  if (!h || !d_kps || !d_counts || !d_kps_un || batch < 1 || cap < 1 || batch > 65535 || !make_params(K4, dist, n_dist, &p))
    return refuse(h, "b2s_undistort_keypoints_device");
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
  k_undistort_kps<<<dim3(div_up(cap, 128), batch), 128, 0, st>>>(d_kps, d_counts, cap, p, dist[0] != 0.f, d_kps_un);
  h->launches += 1;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

extern "C" int b2s_undistort_points(b2s_extractor* h, const float* xy, int n, const float* K4, const float* dist, int n_dist,
                                    float* xy_out) {
  Undistort p;
  if (!h || n < 0 || (n > 0 && (!xy || !xy_out)) || !make_params(K4, dist, n_dist, &p)) return refuse(h, "b2s_undistort_points");
  B2S_CUDA(cudaSetDevice(h->device));
  if (n == 0) return B2S_OK;
  const size_t bytes = (size_t)n * 8;
  int rc = grow(h->dUndistortXY, bytes);
  if (rc != B2S_OK) return rc;
  cudaStream_t st = h->stream;
  float2* d = (float2*)h->dUndistortXY.p;
  B2S_CUDA(cudaMemcpyAsync(d, xy, bytes, cudaMemcpyHostToDevice, st));
  k_undistort_xy<<<div_up(n, 128), 128, 0, st>>>(d, n, p);
  h->launches += 1;
  B2S_CUDA(cudaGetLastError());
  B2S_CUDA(cudaMemcpyAsync(xy_out, d, bytes, cudaMemcpyDeviceToHost, st));
  B2S_CUDA(cudaStreamSynchronize(st));
  return B2S_OK;
}

extern "C" int b2s_stereo_from_depth_device(b2s_extractor* h, const b2s_keypoint* d_kps, const b2s_keypoint* d_kps_un,
                                            const int32_t* d_counts, int batch, int cap, const float* d_depth,
                                            size_t depth_pitch_bytes, int width, int height, float bf, float* d_uright,
                                            float* d_depth_out, void* stream) {
  if (!h || !d_kps || !d_kps_un || !d_counts || !d_depth || !d_uright || !d_depth_out || batch < 1 || batch > 65535 ||
      cap < 1 || width < 1 || height < 1 || depth_pitch_bytes < (size_t)width * 4 || depth_pitch_bytes % 4)
    return refuse(h, "b2s_stereo_from_depth_device");
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
  k_stereo_from_depth<float><<<dim3(div_up(cap, 128), batch), 128, 0, st>>>(
      d_kps, d_kps_un, d_counts, cap, reinterpret_cast<const uint8_t*>(d_depth), depth_pitch_bytes,
      depth_pitch_bytes * height, width, height, 1.f, bf, d_uright, d_depth_out);
  h->launches += 1;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

extern "C" int b2s_stereo_from_depth_u16_device(b2s_extractor* h, const b2s_keypoint* d_kps, const b2s_keypoint* d_kps_un,
                                                const int32_t* d_counts, int batch, int cap, const uint16_t* d_depth,
                                                size_t depth_row_bytes, int width, int height, float depth_map_factor,
                                                float bf, float* d_uright, float* d_depth_out, void* stream) {
  if (!h || !d_kps || !d_kps_un || !d_counts || !d_depth || !d_uright || !d_depth_out || batch < 1 || batch > 65535 ||
      cap < 1 || width < 1 || height < 1 || depth_row_bytes < (size_t)width * 2 || depth_row_bytes % 2 ||
      !std::isfinite(depth_map_factor))
    return refuse(h, "b2s_stereo_from_depth_u16_device");
  // the Tracking constructor (src/Tracking.cc:212-216): float mDepthMapFactor; fabs(float) < 1e-5 compares in double
  const float factor = (double)std::fabs(depth_map_factor) < 1e-5 ? 1.f : 1.0f / depth_map_factor;
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
  k_stereo_from_depth<uint16_t><<<dim3(div_up(cap, 128), batch), 128, 0, st>>>(
      d_kps, d_kps_un, d_counts, cap, reinterpret_cast<const uint8_t*>(d_depth), depth_row_bytes, depth_row_bytes * height,
      width, height, factor, bf, d_uright, d_depth_out);
  h->launches += 1;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}
