// oracle/refshim/refshim_cv_sim3solver.h — TEST INFRASTRUCTURE ONLY.
// The OpenCV C++ API as src/Sim3Solver.cc uses it, so that the reference's own file compiles in place
// (oracle/sim3solver.mk -> _ref/libref_sim3solver.so; the include directory refshim/sim3solver puts it behind
// <opencv2/opencv.hpp> and <opencv2/core/core.hpp>).  It extends refshim_cv_init.h, unchanged: that header's Mat is
// compiled under another name and cv::Mat derives from it, adding what Sim3Solver.cc needs beyond Initializer.cc:
//   - Size, Mat(Size, type), size(), create(rows, cols, type), Mat_<float> with its comma initialiser;
//   - Mat::dot as OpenCV's dotProd_ (double products, unrolled by 4) and cv::norm as OpenCV's two-lane double sum;
//   - reduce (REDUCE_SUM), eigen, Rodrigues and pow, from oracle/sim3solver.cpp's cv2-pinned primitives;
//   - the expression forms Sim3Solver.cc builds that Initializer.cc does not: Mat*Mat.t() (gemm with GEMM_2_T, double
//     sums), s*Mat.t() (a scaled transpose), (s*Mat)/x (one composed scale) and Mat - alpha*A*B (gemm with C).
#pragma once
#define Mat Mat_init_
#include "refshim_cv_init.h"
#undef Mat

#include "../sim3solver_oracle.h"

#define CV_REDUCE_SUM 0

namespace cv {

struct Size {
  int width, height;
  Size(int w = 0, int h = 0) : width(w), height(h) {}
};

class Mat : public Mat_init_ {
 public:
  Mat() {}
  Mat(int r, int c, int t) : Mat_init_(r, c, t) {}
  Mat(int r, int c, int t, Scalar s) : Mat_init_(r, c, t, s) {}
  Mat(int r, int c, int t, void* d) : Mat_init_(r, c, t, d) {}
  Mat(Size s, int t) : Mat_init_(s.height, s.width, t) {}
  Mat(const Mat_init_& m) : Mat_init_(m) {}
  Mat(const MatExpr& e) : Mat_init_(e) {}
  Mat& operator=(const MatExpr& e) {
    Mat_init_::operator=(e);
    return *this;
  }
  Mat& operator=(const Mat_init_& m) {
    Mat_init_::operator=(m);
    return *this;
  }
  Size size() const { return Size(cols, rows); }
  using Mat_init_::create;
  void create(int r, int c, int) { Mat_init_::create(r, c); }
  double dot(const Mat_init_& b) const {
    const Mat_init_ x = clone(), y = b.clone();
    return orc_s3s_dot(x.data, y.data, rows * cols);
  }
};

template <typename T>
class Mat_ : public Mat {
 public:
  Mat_(int r, int c) : Mat(r, c, CV_32F) {}
};

// Mat_<float>(r, c) << a, b, ...: each value stored as (float)
template <typename T>
struct MatCommaInitializer_ {
  Mat m;
  int i;
  template <typename V>
  MatCommaInitializer_& operator,(V v) {
    m.data[i++] = (float)v;
    return *this;
  }
  operator Mat() const { return m; }
};
template <typename T, typename V>
MatCommaInitializer_<T> operator<<(const Mat_<T>& m, V v) {
  MatCommaInitializer_<T> c;
  c.m = m;
  c.i = 0;
  c.m.data[c.i++] = (float)v;
  return c;
}

// Mat*Mat.t(): gemm(A, B, 1, noArray(), 0, D, GEMM_2_T), evaluated at once
inline MatExpr operator*(const Mat& a, const MatExpr& e) {
  if (e.op == MatExpr::T && e.alpha == 1) {
    const Mat_init_ A = a.clone(), B = e.a.clone();
    Mat D(A.rows, B.rows, CV_32F);
    orc_s3s_gemm_bt(A.data, B.data, A.rows, A.cols, B.rows, D.data);
    return MatExpr(D);
  }
  return static_cast<const Mat_init_&>(a) * e;
}
// s*Mat.t(): the transpose scaled by convertTo
inline MatExpr operator*(double s, const MatExpr& e) {
  if (e.op == MatExpr::T || e.op == MatExpr::SCALE) {
    MatExpr r = e;
    r.alpha = e.alpha * s;
    return r;
  }
  return MatExpr::make(MatExpr::SCALE, e.eval(), s);
}
// (s*Mat)/x: MatOp_AddEx::multiply by 1/x, one scale
inline MatExpr operator/(const MatExpr& e, double x) { return (1. / x) * e; }
// Mat - alpha*A*B: MatOp_GEMM::subtract, gemm(A, B, -alpha, Mat, 1)
inline MatExpr operator-(const Mat_init_& c, const MatExpr& e) {
  if (e.op == MatExpr::GEMM && e.c.empty() && !e.flags) {
    MatExpr r = e;
    r.alpha = -e.alpha;
    r.c = c;
    r.beta = 1;
    return r;
  }
  return MatExpr::make(MatExpr::ADD, c, 1, e.eval(), -1);
}

inline double norm(const Mat& a) {
  const Mat_init_ x = a.clone();
  return orc_s3s_norm(x.data, x.rows * x.cols);
}

inline void reduce(const Mat_init_& src, Mat_init_& dst, int dim, int) {
  const Mat_init_ s = src.clone();
  Mat_init_ d(s.rows, 1, CV_32F);
  if (dim != 1) return;  // Sim3Solver.cc reduces to a column only
  orc_s3s_reduce_sum_cols(s.data, s.rows, s.cols, d.data);
  d.copyTo(dst);
}

inline bool eigen(const Mat_init_& src, Mat_init_& evals, Mat_init_& evecs) {
  const Mat_init_ s = src.clone();
  Mat_init_ w(s.rows, 1, CV_32F), v(s.rows, s.rows, CV_32F);
  orc_s3s_eigen(s.data, s.rows, w.data, v.data);
  w.copyTo(evals);
  v.copyTo(evecs);
  return true;
}

inline void Rodrigues(const Mat_init_& src, Mat_init_& dst) {
  const Mat_init_ s = src.clone();
  Mat_init_ R(3, 3, CV_32F);
  orc_s3s_rodrigues(s.data, R.data);
  R.copyTo(dst);
}

inline void pow(const Mat_init_& src, double p, Mat_init_& dst) {
  const Mat_init_ s = src.clone();
  Mat_init_ d(s.rows, s.cols, CV_32F);
  if (p != 2) return;  // Sim3Solver.cc squares only
  orc_s3s_pow2(s.data, s.rows * s.cols, d.data);
  d.copyTo(dst);
}

}  // namespace cv
