// cv_compat.h — the few OpenCV types the hot-path signatures mention.
// With -DB2S_HAVE_OPENCV the real OpenCV headers are used (drop-in build inside ORB-SLAM2), or whichever
// <opencv2/core/core.hpp> the include path finds first: the parity builds of oracle/frame.mk put oracle/refshim's cv
// stand-in there, so the drop-in ORBextractor and Frame compile behind the reference's glue without OpenCV; otherwise
// layout-compatible stand-ins are declared so the shim and its tests build where OpenCV C++ is absent.
#pragma once
#ifdef B2S_HAVE_OPENCV
#include <opencv2/core/core.hpp>
namespace b2s_cv = cv;
#else
#include <cstdint>
#include <cstring>
#include <vector>
namespace b2s_cv {
struct Point2f {
  float x = 0, y = 0;
};
// same 28-byte layout as cv::KeyPoint: pt, size, angle, response, octave, class_id
struct KeyPoint {
  Point2f pt;
  float size = 0, angle = -1, response = 0;
  int octave = 0, class_id = -1;
};
static_assert(sizeof(KeyPoint) == 28, "cv::KeyPoint layout");
// minimal CV_8UC1 / CV_32F matrix: owns its pixels, row-major, contiguous
struct Mat {
  int rows = 0, cols = 0;
  size_t step = 0;
  std::vector<uint8_t> buf;
  uint8_t* data = nullptr;
  Mat() {}
  Mat(int r, int c) { create(r, c); }
  void create(int r, int c) {
    rows = r;
    cols = c;
    step = (size_t)c;
    buf.assign((size_t)r * c, 0);
    data = buf.data();
  }
  void release() {
    rows = cols = 0;
    step = 0;
    buf.clear();
    data = nullptr;
  }
  bool empty() const { return rows == 0 || cols == 0 || !data; }
  uint8_t* ptr(int r) { return data + (size_t)r * step; }
  const uint8_t* ptr(int r) const { return data + (size_t)r * step; }
};
typedef const Mat& InputArray;
typedef Mat& OutputArray;
}  // namespace b2s_cv
#endif
