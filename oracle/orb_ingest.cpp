// CPU restatement of the frame ingest (test infrastructure): OpenCV 4's cvtColor(*2GRAY) on 8-bit images, remap with
// CV_32FC1 maps, INTER_LINEAR and BORDER_CONSTANT 0 on 8-bit images, and Tracking's 16-bit depth conversion.  Written
// statement by statement from OpenCV 4.x (modules/imgproc/src/color_rgb.simd.hpp, imgwarp.cpp) and the reference's
// src/Tracking.cc; checked byte for byte against cv2 4.13 by tests/test_ingest_oracle.py.
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <climits>

#include "ingest_oracle.h"

namespace {

// color_rgb.simd.hpp, RGB2Gray<uchar>: yuv_shift = 15 fixed-point BT.601 coefficients, R2Y + G2Y + B2Y = 1 << 15
constexpr int kShift = 15, R2Y = 9798, G2Y = 19235, B2Y = 3735;

inline int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }  // CV_DESCALE

// saturate_cast<int>(float) = cvRound on x86: cvtss2si, round half to even; NaN and out-of-range give INT_MIN
// ("integer indefinite")
inline int cv_round(float v) {
  if (std::isnan(v) || !(v >= -2147483648.f && v < 2147483648.f)) return INT_MIN;
  return (int)std::nearbyint(v);
}

inline short saturate_short(int v) { return (short)(v < SHRT_MIN ? SHRT_MIN : v > SHRT_MAX ? SHRT_MAX : v); }

// imgwarp.cpp: INTER_BITS = 5, INTER_TAB_SIZE = 32, INTER_REMAP_COEF_BITS = 15
constexpr int kBits = 5, kTab = 1 << kBits, kCoefBits = 15;

// initInterTab2D(INTER_LINEAR, fixpt): interpolateLinear gives (1 - t, t) for t = k / 32; the 2-D table is the outer
// product, scaled by 1 << 15 and rounded (saturate_cast<short>); every entry is exact, so the sum correction (the loop
// that moves the rounding error of a row of weights onto its largest entry) never changes anything.
void linear_tab(int ax, int ay, int w[4]) {
  const float tx[2] = {1.f - (float)ax / kTab, (float)ax / kTab};
  const float ty[2] = {1.f - (float)ay / kTab, (float)ay / kTab};
  for (int i = 0; i < 2; i++)
    for (int j = 0; j < 2; j++) w[i * 2 + j] = (int)std::lrint(ty[i] * tx[j] * (1 << kCoefBits));
}

}  // namespace

extern "C" {

// src/Tracking.cc:252-278 (stereo), :313-326 (RGB-D), :371-384 (monocular): 3 channels -> RGB2GRAY if mbRGB else
// BGR2GRAY; 4 channels -> RGBA2GRAY / BGRA2GRAY (alpha ignored, same coefficients); 1 channel is left as it is
void orc_gray_from_color(const uint8_t* src, size_t src_row_bytes, int width, int height, int channels, int rgb,
                         uint8_t* out, size_t out_row_bytes) {
  const int bidx = rgb ? 0 : 2;  // byte of R (RGB2Gray's blueIdx is the other end)
  for (int y = 0; y < height; y++) {
    const uint8_t* s = src + (size_t)y * src_row_bytes;
    uint8_t* d = out + (size_t)y * out_row_bytes;
    for (int x = 0; x < width; x++, s += channels) {
      if (channels == 1) {
        d[x] = s[0];
        continue;
      }
      d[x] = (uint8_t)descale(s[bidx] * R2Y + s[1] * G2Y + s[bidx ^ 2] * B2Y, kShift);
    }
  }
}

// cv::remap(src, dst, mapx, mapy, INTER_LINEAR, BORDER_CONSTANT, 0) with CV_32FC1 maps (RemapInvoker + remapBilinear):
// the float maps are first turned into short (sx, sy) pairs and a table index, then every channel is interpolated.
// dst: width x height x channels, dense.
void orc_remap_linear(const uint8_t* src, size_t src_row_bytes, int src_width, int src_height, int channels,
                      const float* mapx, const float* mapy, size_t map_row_bytes, int width, int height, uint8_t* dst) {
  for (int y = 0; y < height; y++) {
    const float* mx = (const float*)((const uint8_t*)mapx + (size_t)y * map_row_bytes);
    const float* my = (const float*)((const uint8_t*)mapy + (size_t)y * map_row_bytes);
    for (int x = 0; x < width; x++) {
      // RemapInvoker, m1 CV_32FC1 / m2 CV_32FC1, INTER_LINEAR
      const int X = cv_round(mx[x] * kTab), Y = cv_round(my[x] * kTab);
      const int sx = saturate_short(X >> kBits), sy = saturate_short(Y >> kBits);
      const int a = (Y & (kTab - 1)) * kTab + (X & (kTab - 1));
      int w[4];
      linear_tab(a % kTab, a / kTab, w);
      uint8_t* D = dst + ((size_t)y * width + x) * channels;
      // remapBilinear, BORDER_CONSTANT: a pixel whose 2 x 2 block misses the image entirely is the border value; else
      // each tap outside the image reads the border value (0)
      if (sx >= src_width || sx + 1 < 0 || sy >= src_height || sy + 1 < 0) {
        for (int k = 0; k < channels; k++) D[k] = 0;
        continue;
      }
      for (int k = 0; k < channels; k++) {
        int v[4];
        for (int i = 0; i < 2; i++)
          for (int j = 0; j < 2; j++) {
            const int xs = sx + j, ys = sy + i;
            v[i * 2 + j] = (xs >= 0 && xs < src_width && ys >= 0 && ys < src_height)
                               ? src[(size_t)ys * src_row_bytes + (size_t)xs * channels + k]
                               : 0;
          }
        // FixedPtCast<int, uchar, INTER_REMAP_COEF_BITS>: (sum + (1 << 14)) >> 15, saturated to uchar
        const int sum = v[0] * w[0] + v[1] * w[1] + v[2] * w[2] + v[3] * w[3];
        const int r = (sum + (1 << (kCoefBits - 1))) >> kCoefBits;
        D[k] = (uint8_t)(r < 0 ? 0 : r > 255 ? 255 : r);
      }
    }
  }
}

// src/Tracking.cc:212-216: mDepthMapFactor = 1 when fabs(DepthMapFactor) < 1e-5, else 1.0f / DepthMapFactor (float);
// :334-338: a 16-bit image is always converted, imDepth.convertTo(imDepth, CV_32F, mDepthMapFactor).  Returns the
// multiplier.
float orc_depth_u16(const uint16_t* raw, size_t n, float depth_map_factor, float* out) {
  float f = depth_map_factor;
  if (std::fabs(f) < 1e-5)
    f = 1;
  else
    f = 1.0f / f;
  for (size_t i = 0; i < n; i++) out[i] = (float)raw[i] * f;
  return f;
}

}  // extern "C"
