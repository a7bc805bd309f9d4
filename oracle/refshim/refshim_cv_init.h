// oracle/refshim/refshim_cv_init.h — TEST INFRASTRUCTURE ONLY.
// The OpenCV C++ API as src/Initializer.cc uses it, so that the reference's own file compiles in place
// (oracle/init.mk -> _ref/libref_init.so; the include directory refshim/init puts it behind <opencv2/opencv.hpp>).  It
// is a separate stand-in from refshim_cv.h, which every other oracle library uses unchanged, because Initializer.cc
// needs OpenCV's expression semantics that refshim_cv.h does not model:
//   - assigning an expression writes into the existing data when the size matches (A.row(0) = x*P.row(2) - P.row(0)
//     fills A; copyTo into a rowRange/colRange view fills the view), while assigning a Mat rebinds the header;
//   - expressions stay lazy the way cv::MatExpr keeps them: s*U*Rp is one gemm with alpha = s, R*x + t one gemm with C,
//     K.t()*F a gemm with the first operand transposed, x*a - b an addWeighted, m*s / m/s / -m a convertTo.
// The arithmetic is delegated to the oracle primitives that tests/test_oracle_init.py pins bit for bit against cv2:
// orc_svd (SVD::compute / SVDecomp), orc_inv3 (Mat::inv), orc_det3 (cv::determinant), orc_gemm (gemm).  CV_32F only.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <memory>
#include <vector>

#include "../init_oracle.h"

#define CV_PI 3.1415926535897932384626433832795
#define CV_32F 5

namespace cv {

struct Scalar {
  double v;
  Scalar(double x = 0) : v(x) {}
};
template <typename T>
struct Point_ {
  T x, y;
  Point_() : x(0), y(0) {}
  Point_(T _x, T _y) : x(_x), y(_y) {}
};
typedef Point_<float> Point2f;
template <typename T>
struct Point3_ {
  T x, y, z;
  Point3_() : x(0), y(0), z(0) {}
  Point3_(T _x, T _y, T _z) : x(_x), y(_y), z(_z) {}
};
typedef Point3_<float> Point3f;
struct KeyPoint {
  Point2f pt;
  float size = 0, angle = -1, response = 0;
  int octave = 0, class_id = -1;
};

class MatExpr;

class Mat {
 public:
  int rows = 0, cols = 0, step = 0;  // step in floats
  float* data = nullptr;

  Mat() {}
  Mat(int r, int c, int) { create(r, c); }
  Mat(int r, int c, int, Scalar s) {
    create(r, c);
    for (int i = 0; i < r * c; i++) data[i] = (float)s.v;
  }
  Mat(int r, int c, int, void* d) : rows(r), cols(c), step(c), data((float*)d) {}  // user data, not copied
  Mat(const MatExpr& e);
  Mat& operator=(const MatExpr& e);

  void create(int r, int c) {
    if (data && rows == r && cols == c) return;
    buf_ = std::make_shared<std::vector<float> >((size_t)r * c);
    rows = r;
    cols = c;
    step = c;
    data = buf_->data();
  }
  bool empty() const { return !data || rows == 0 || cols == 0; }
  int type() const { return CV_32F; }
  template <typename T>
  T& at(int r, int c) {
    return data[r * step + c];
  }
  template <typename T>
  const T& at(int r, int c) const {
    return data[r * step + c];
  }
  template <typename T>
  T& at(int i) {
    return rows == 1 ? data[i] : data[i * step];
  }
  template <typename T>
  const T& at(int i) const {
    return rows == 1 ? data[i] : data[i * step];
  }
  float f(int r, int c) const { return data[r * step + c]; }
  Mat view(int r0, int c0, int nr, int nc) const {
    Mat m = *this;
    m.data = data + r0 * step + c0;
    m.rows = nr;
    m.cols = nc;
    return m;
  }
  Mat row(int r) const { return view(r, 0, 1, cols); }
  Mat col(int c) const { return view(0, c, rows, 1); }
  Mat rowRange(int a, int b) const { return view(a, 0, b - a, cols); }
  Mat colRange(int a, int b) const { return view(0, a, rows, b - a); }
  Mat reshape(int, int r) const {  // a continuous matrix (here: a row) seen as r rows
    Mat m = *this;
    const int n = rows * cols;
    m.rows = r;
    m.cols = n / r;
    m.step = m.cols;
    return m;
  }
  Mat clone() const {
    Mat m(rows, cols, CV_32F);
    for (int r = 0; r < rows; r++)
      for (int c = 0; c < cols; c++) m.data[r * cols + c] = f(r, c);
    return m;
  }
  // copyTo(OutputArray): create() keeps a destination of the same size, so a view is filled in place
  void copyTo(Mat& dst) const {
    const Mat src = clone();
    dst.create(rows, cols);
    for (int r = 0; r < rows; r++)
      for (int c = 0; c < cols; c++) dst.data[r * dst.step + c] = src.data[r * cols + c];
  }
  void copyTo(Mat&& dst) const { copyTo(static_cast<Mat&>(dst)); }
  double dot(const Mat& b) const {
    double s = 0;
    for (int r = 0; r < rows; r++)
      for (int c = 0; c < cols; c++) s += (double)f(r, c) * (double)b.f(r, c);
    return s;
  }
  MatExpr t() const;
  MatExpr inv() const;
  static MatExpr eye(int r, int c, int type);
  static MatExpr zeros(int r, int c, int type);
  static MatExpr diag(const Mat& d);

 private:
  std::shared_ptr<std::vector<float> > buf_;
};

// cv::MatExpr, reduced to the forms Initializer.cc builds:
//   MAT    a
//   SCALE  alpha*a                          (convertTo: each element times (float)alpha)
//   ADD    alpha*a + beta*b                 (add / subtract / addWeighted: double, rounded once)
//   GEMM   alpha*op(a)*op(b) [+ c]          (gemm; flags GEMM_1_T / GEMM_2_T)
//   T      alpha*a^T
//   INV    a^-1
class MatExpr {
 public:
  enum Op { MAT, SCALE, ADD, GEMM, T, INV };
  enum { T1 = 1, T2 = 2 };
  Op op = MAT;
  Mat a, b, c;
  double alpha = 1, beta = 0;
  int flags = 0;
  MatExpr() {}
  MatExpr(const Mat& m) : op(MAT), a(m) {}
  static MatExpr make(Op op, const Mat& a, double alpha = 1, const Mat& b = Mat(), double beta = 0, int flags = 0,
                      const Mat& c = Mat()) {
    MatExpr e;
    e.op = op;
    e.a = a;
    e.b = b;
    e.c = c;
    e.alpha = alpha;
    e.beta = beta;
    e.flags = flags;
    return e;
  }
  Mat eval() const {
    switch (op) {
      case MAT:
        return a;
      case SCALE: {
        Mat m(a.rows, a.cols, CV_32F);
        const float s = (float)alpha;
        for (int r = 0; r < a.rows; r++)
          for (int k = 0; k < a.cols; k++) m.at<float>(r, k) = a.f(r, k) * s;
        return m;
      }
      case ADD: {
        Mat m(a.rows, a.cols, CV_32F);
        for (int r = 0; r < a.rows; r++)
          for (int k = 0; k < a.cols; k++)
            m.at<float>(r, k) = (float)((double)a.f(r, k) * alpha + (double)b.f(r, k) * beta);
        return m;
      }
      case T: {
        Mat m(a.cols, a.rows, CV_32F);
        const float s = (float)alpha;
        for (int r = 0; r < a.rows; r++)
          for (int k = 0; k < a.cols; k++) m.at<float>(k, r) = alpha == 1 ? a.f(r, k) : a.f(r, k) * s;
        return m;
      }
      case INV: {
        Mat A = a.clone(), m(3, 3, CV_32F);
        orc_inv3(A.data, m.data);
        return m;
      }
      case GEMM: {
        // op(a) transposed goes to orc_gemm, which accumulates in double as gemm does for a transposed operand; op(b)
        // transposed is only u*W.t() in DecomposeE, whose W holds 0 and +-1, so each sum has one exact term and the
        // materialised transpose gives the same result
        const Mat A = a.clone(), B = (flags & T2) ? MatExpr::make(T, b).eval() : b.clone();
        const int m = (flags & T1) ? A.cols : A.rows, k = (flags & T1) ? A.rows : A.cols, n = B.cols;
        const Mat C = c.empty() ? Mat() : c.clone();
        Mat D(m, n, CV_32F);
        orc_gemm(A.data, B.data, C.empty() ? nullptr : C.data, m, k, n, alpha, (flags & T1) ? 1 : 0, D.data);
        return D;
      }
    }
    return Mat();
  }
};

inline Mat::Mat(const MatExpr& e) { *this = e.eval().clone(); }
inline Mat& Mat::operator=(const MatExpr& e) {
  const Mat r = e.eval().clone();  // evaluated first: the destination may be an operand
  if (data && rows == r.rows && cols == r.cols) {
    for (int i = 0; i < rows; i++)
      for (int k = 0; k < cols; k++) data[i * step + k] = r.data[i * r.cols + k];
  } else {
    *this = r;
  }
  return *this;
}
inline MatExpr Mat::t() const { return MatExpr::make(MatExpr::T, *this); }
inline MatExpr Mat::inv() const { return MatExpr::make(MatExpr::INV, *this); }
inline MatExpr Mat::eye(int r, int c, int) {
  Mat m(r, c, CV_32F, Scalar(0));
  for (int i = 0; i < r && i < c; i++) m.at<float>(i, i) = 1.f;
  return MatExpr(m);
}
inline MatExpr Mat::zeros(int r, int c, int) { return MatExpr(Mat(r, c, CV_32F, Scalar(0))); }
inline MatExpr Mat::diag(const Mat& d) {
  const int n = d.rows * d.cols;
  Mat m(n, n, CV_32F, Scalar(0));
  for (int i = 0; i < n; i++) m.at<float>(i, i) = d.at<float>(i);
  return MatExpr(m);
}

// ---- the expression algebra (modules/core/src/matrix_expressions.cpp, for these forms)
inline MatExpr operator*(const Mat& a, const Mat& b) { return MatExpr::make(MatExpr::GEMM, a, 1, b); }
inline MatExpr operator*(const MatExpr& e, const Mat& m) {
  if (e.op == MatExpr::SCALE || e.op == MatExpr::MAT) return MatExpr::make(MatExpr::GEMM, e.a, e.alpha, m);
  if (e.op == MatExpr::T) return MatExpr::make(MatExpr::GEMM, e.a, e.alpha, m, 0, MatExpr::T1);
  return MatExpr::make(MatExpr::GEMM, e.eval(), 1, m);
}
inline MatExpr operator*(const Mat& m, const MatExpr& e) {
  if (e.op == MatExpr::SCALE || e.op == MatExpr::MAT) return MatExpr::make(MatExpr::GEMM, m, e.alpha, e.a);
  if (e.op == MatExpr::T) return MatExpr::make(MatExpr::GEMM, m, e.alpha, e.a, 0, MatExpr::T2);
  return MatExpr::make(MatExpr::GEMM, m, 1, e.eval());
}
inline MatExpr operator*(double s, const Mat& a) { return MatExpr::make(MatExpr::SCALE, a, s); }
inline MatExpr operator*(const Mat& a, double s) { return MatExpr::make(MatExpr::SCALE, a, s); }
inline MatExpr operator/(const Mat& a, double s) { return MatExpr::make(MatExpr::SCALE, a, 1. / s); }
inline MatExpr operator-(const Mat& a) { return MatExpr::make(MatExpr::SCALE, a, -1); }
inline MatExpr operator-(const MatExpr& e) {
  if (e.op == MatExpr::SCALE || e.op == MatExpr::T) {
    MatExpr r = e;
    r.alpha = -e.alpha;
    return r;
  }
  return MatExpr::make(MatExpr::SCALE, e.eval(), -1);
}
inline MatExpr operator+(const Mat& a, const Mat& b) { return MatExpr::make(MatExpr::ADD, a, 1, b, 1); }
inline MatExpr operator-(const Mat& a, const Mat& b) { return MatExpr::make(MatExpr::ADD, a, 1, b, -1); }
inline MatExpr operator-(const MatExpr& e, const Mat& b) {
  if (e.op == MatExpr::SCALE) return MatExpr::make(MatExpr::ADD, e.a, e.alpha, b, -1);
  return MatExpr::make(MatExpr::ADD, e.eval(), 1, b, -1);
}
inline MatExpr operator+(const MatExpr& e, const Mat& c) {
  if (e.op == MatExpr::GEMM && e.c.empty()) {
    MatExpr r = e;
    r.c = c;
    r.beta = 1;
    return r;
  }
  return MatExpr::make(MatExpr::ADD, e.eval(), 1, c, 1);
}
inline Mat& operator*=(Mat& a, double s) {  // convertTo(a, -1, s)
  a = MatExpr::make(MatExpr::SCALE, a, s);
  return a;
}

inline double norm(const Mat& a) {  // NORM_L2, double accumulator
  double s = 0;
  for (int r = 0; r < a.rows; r++)
    for (int c = 0; c < a.cols; c++) s += (double)a.f(r, c) * (double)a.f(r, c);
  return std::sqrt(s);
}
inline double determinant(const Mat& m) {
  const Mat M = m.clone();
  return orc_det3(M.data);
}

struct SVD {
  enum { MODIFY_A = 1, NO_UV = 2, FULL_UV = 4 };
  static void compute(const Mat& A, Mat& w, Mat& u, Mat& vt, int flags = 0) {
    const Mat a = A.clone();
    const int m = a.rows > a.cols ? a.rows : a.cols, n = a.rows < a.cols ? a.rows : a.cols;
    const int urows = (flags & FULL_UV) ? m : n;
    Mat W(n, 1, CV_32F), U, VT;
    if (a.rows >= a.cols) {
      U = Mat(a.rows, urows, CV_32F);
      VT = Mat(n, n, CV_32F);
    } else {
      U = Mat(n, n, CV_32F);
      VT = Mat(urows, a.cols, CV_32F);
    }
    orc_svd(a.data, a.rows, a.cols, (flags & FULL_UV) ? 1 : 0, W.data, U.data, VT.data);
    W.copyTo(w);
    U.copyTo(u);
    VT.copyTo(vt);
  }
};
inline void SVDecomp(const Mat& A, Mat& w, Mat& u, Mat& vt, int flags = 0) { SVD::compute(A, w, u, vt, flags); }

}  // namespace cv
