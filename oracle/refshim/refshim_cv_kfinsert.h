// oracle/refshim/refshim_cv_kfinsert.h — TEST INFRASTRUCTURE ONLY.
// The OpenCV C++ API as src/LocalMapping.cc, src/KeyFrame.cc, src/MapPoint.cc and the headers they include use it, for
// the keyframe-insertion checkers (oracle/kfinsert.mk -> _ref/libref_kfinsert.so; the include directory refshim/kfinsert
// puts it behind the OpenCV headers).  It is refshim_cv_localmapping.h (a float Mat with shared storage and row / column
// views, evaluated eagerly) with the arithmetic MapPoint::UpdateNormalAndDepth runs pinned to OpenCV's.  A descriptor row is 8 floats holding the 32 bytes.  What only CreateNewMapPoints uses is there to compile,
// not to run.
#pragma once
#include <algorithm>  // the real OpenCV headers bring these in
#include <climits>
#include <cmath>
#include <cstring>
#include <memory>
#include <vector>

#define CV_32F 5
#define CV_8U 0

namespace cv {

struct Scalar {
  double v;
  Scalar(double x = 0) : v(x) {}
};

template <typename T>
struct Point_ {
  T x = 0, y = 0;
  Point_() {}
  Point_(T a, T b) : x(a), y(b) {}
};
typedef Point_<float> Point2f;
typedef Point_<int> Point2i;
typedef Point2i Point;

struct KeyPoint {
  Point2f pt;
  float size = 0, angle = -1, response = 0;
  int octave = 0, class_id = -1;
};

class Mat {
 public:
  int rows = 0, cols = 0, step = 0;  // step: elements between rows
  float* data = nullptr;
  std::shared_ptr<std::vector<float> > buf;

  Mat() {}
  Mat(int r, int c, int = CV_32F) { create(r, c); }
  Mat(int r, int c, int t, Scalar s) : Mat(r, c, t) {
    for (int i = 0; i < r * c; i++) data[i] = (float)s.v;
  }
  void create(int r, int c, int = CV_32F) {
    if (data && rows == r && cols == c) return;
    buf = std::make_shared<std::vector<float> >((size_t)r * c, 0.f);
    rows = r;
    cols = c;
    step = c;
    data = buf->data();
  }
  bool empty() const { return !data || rows * cols == 0; }
  int type() const { return CV_32F; }
  template <typename T>
  T& at(int r, int c) {
    return reinterpret_cast<T&>(data[r * step + c]);
  }
  template <typename T>
  const T& at(int r, int c) const {
    return reinterpret_cast<const T&>(data[r * step + c]);
  }
  template <typename T>
  T& at(int i) {
    return cols == 1 ? at<T>(i, 0) : at<T>(i / cols, i % cols);
  }
  template <typename T>
  const T& at(int i) const {
    return cols == 1 ? at<T>(i, 0) : at<T>(i / cols, i % cols);
  }
  template <typename T>
  T* ptr(int r = 0) {
    return reinterpret_cast<T*>(data + r * step);
  }
  float f(int r, int c) const { return data[r * step + c]; }
  Mat view(int r0, int r1, int c0, int c1) const {
    Mat m = *this;
    m.data = data + r0 * step + c0;
    m.rows = r1 - r0;
    m.cols = c1 - c0;
    return m;
  }
  Mat rowRange(int a, int b) const { return view(a, b, 0, cols); }
  Mat colRange(int a, int b) const { return view(0, rows, a, b); }
  Mat row(int r) const { return view(r, r + 1, 0, cols); }
  Mat col(int c) const { return view(0, rows, c, c + 1); }
  Mat clone() const {
    Mat m(rows, cols);
    for (int r = 0; r < rows; r++)
      for (int c = 0; c < cols; c++) m.data[r * cols + c] = f(r, c);
    return m;
  }
  // into a view of the same size: its elements; otherwise the destination is reallocated
  void copyTo(Mat& dst) const {
    const Mat s = clone();
    if (!dst.data || dst.rows != rows || dst.cols != cols) dst.create(rows, cols);
    for (int r = 0; r < rows; r++)
      for (int c = 0; c < cols; c++) dst.data[r * dst.step + c] = s.data[r * cols + c];
  }
  void copyTo(Mat&& dst) const { copyTo(static_cast<Mat&>(dst)); }
  Mat t() const {
    Mat m(cols, rows);
    for (int r = 0; r < rows; r++)
      for (int c = 0; c < cols; c++) m.data[c * rows + r] = f(r, c);
    return m;
  }
  Mat inv() const {  // Gauss-Jordan with partial pivoting, in double
    const int n = rows;
    std::vector<double> a((size_t)n * 2 * n, 0.0);
    for (int r = 0; r < n; r++) {
      for (int c = 0; c < n; c++) a[(size_t)r * 2 * n + c] = f(r, c);
      a[(size_t)r * 2 * n + n + r] = 1.0;
    }
    for (int c = 0; c < n; c++) {
      int p = c;
      for (int r = c + 1; r < n; r++)
        if (std::fabs(a[(size_t)r * 2 * n + c]) > std::fabs(a[(size_t)p * 2 * n + c])) p = r;
      for (int k = 0; k < 2 * n; k++) std::swap(a[(size_t)c * 2 * n + k], a[(size_t)p * 2 * n + k]);
      const double d = a[(size_t)c * 2 * n + c];
      if (d == 0) return Mat(n, n, CV_32F, Scalar(0));
      for (int k = 0; k < 2 * n; k++) a[(size_t)c * 2 * n + k] /= d;
      for (int r = 0; r < n; r++)
        if (r != c) {
          const double g = a[(size_t)r * 2 * n + c];
          for (int k = 0; k < 2 * n; k++) a[(size_t)r * 2 * n + k] -= g * a[(size_t)c * 2 * n + k];
        }
    }
    Mat m(n, n);
    for (int r = 0; r < n; r++)
      for (int c = 0; c < n; c++) m.data[r * n + c] = (float)a[(size_t)r * 2 * n + n + c];
    return m;
  }
  double dot(const Mat& b) const {
    double s = 0;
    for (int i = 0; i < rows * cols; i++) s += (double)at<float>(i) * b.at<float>(i);
    return s;
  }
  static Mat zeros(int r, int c, int t) { return Mat(r, c, t, Scalar(0)); }
  static Mat eye(int r, int c, int t) {
    Mat m = zeros(r, c, t);
    for (int i = 0; i < r && i < c; i++) m.data[i * c + i] = 1.f;
    return m;
  }
};

typedef const Mat& InputArray;
typedef Mat& OutputArray;

template <typename T>
class Mat_ : public Mat {
 public:
  Mat_(int r, int c) : Mat(r, c, CV_32F) {}
};
// Mat_<float>(r, c) << a, b, ...
template <typename T>
struct MatCommaInitializer_ {
  Mat m;
  int i;
  template <typename V>
  MatCommaInitializer_& operator,(V v) {
    m.at<float>(i++) = (float)v;
    return *this;
  }
  operator Mat() const { return m; }
};
template <typename T, typename V>
MatCommaInitializer_<T> operator<<(const Mat_<T>& m, V v) {
  MatCommaInitializer_<T> w{m, 0};
  w.m.template at<float>(w.i++) = (float)v;
  return w;
}

inline Mat scaled(const Mat& a, double s) {
  Mat m(a.rows, a.cols);
  for (int r = 0; r < a.rows; r++)
    for (int c = 0; c < a.cols; c++) m.data[r * a.cols + c] = (float)(a.f(r, c) * s);
  return m;
}
inline Mat added(const Mat& a, double x, const Mat& b, double y) {
  Mat m(a.rows, a.cols);
  for (int r = 0; r < a.rows; r++)
    for (int c = 0; c < a.cols; c++) m.data[r * a.cols + c] = (float)(a.f(r, c) * x + b.f(r, c) * y);
  return m;
}
inline Mat operator*(const Mat& a, const Mat& b) {
  Mat m(a.rows, b.cols);
  for (int r = 0; r < a.rows; r++)
    for (int c = 0; c < b.cols; c++) {
      double s = 0;
      for (int k = 0; k < a.cols; k++) s += (double)a.f(r, k) * b.f(k, c);
      m.data[r * b.cols + c] = (float)s;
    }
  return m;
}
inline Mat operator*(double s, const Mat& a) { return scaled(a, s); }
inline Mat operator*(const Mat& a, double s) { return scaled(a, s); }
inline Mat operator-(const Mat& a) { return scaled(a, -1); }
inline Mat operator+(const Mat& a, const Mat& b) { return added(a, 1, b, 1); }

// The forms MapPoint::UpdateNormalAndDepth takes, as OpenCV evaluates them (DESIGN.md §7).  Mat / s stays a scaled
// expression (MatOp_AddEx, alpha = 1./s) until it is used: assigned, it is convertTo with alpha rounded to float; added to a Mat, it is scaleAdd with alpha rounded to
// float, fused and rounded once (pinned against cv2.scaleAdd).  Mat - Mat subtracts in float; norm sums the squares in
// double in order, as cv2.norm does for the 3 x 1 columns it is given here.  Build with -ffp-contract=off.
struct MatScaled {
  Mat a;
  double alpha;
  operator Mat() const {
    Mat m(a.rows, a.cols);
    const float al = (float)alpha;
    for (int r = 0; r < a.rows; r++)
      for (int c = 0; c < a.cols; c++) m.data[r * a.cols + c] = a.f(r, c) * al + 0.f;
    return m;
  }
};
inline MatScaled operator/(const Mat& a, double s) { return MatScaled{a, 1. / s}; }
inline Mat operator+(const Mat& b, const MatScaled& e) {
  Mat m(b.rows, b.cols);
  const float al = (float)e.alpha;
  for (int r = 0; r < b.rows; r++)
    for (int c = 0; c < b.cols; c++) m.data[r * b.cols + c] = std::fmaf(e.a.f(r, c), al, b.f(r, c));
  return m;
}
inline Mat operator-(const Mat& a, const Mat& b) {
  Mat m(a.rows, a.cols);
  for (int r = 0; r < a.rows; r++)
    for (int c = 0; c < a.cols; c++) m.data[r * a.cols + c] = a.f(r, c) - b.f(r, c);
  return m;
}
inline double norm(const Mat& a) {
  double s = 0;
  for (int i = 0; i < a.rows * a.cols; i++) {
    const double v = a.at<float>(i);
    s += v * v;
  }
  return std::sqrt(s);
}

struct SVD {
  enum { MODIFY_A = 1, NO_UV = 2, FULL_UV = 4 };
  static void compute(const Mat&, Mat&, Mat&, Mat&, int = 0) {}
};

}  // namespace cv
