// oracle/refshim/refshim_cv_pnpsolver.h — TEST INFRASTRUCTURE ONLY.
// The OpenCV API as src/PnPsolver.cc uses it, so that the reference's own file compiles in place
// (oracle/pnpsolver.mk -> _ref/libref_pnpsolver.so; the include directory refshim/pnpsolver puts it behind
// <opencv2/core/core.hpp>).  PnPsolver.cc's arithmetic is all in OpenCV's C API on CV_64F data, which the float-only
// cv::Mat of refshim_cv_init.h / refshim_cv_sim3solver.h cannot hold, so this stand-in is its own:
//   - Point2f, Point3f, KeyPoint (the members the constructor reads);
//   - Mat over float or double data (a header over external data, or owned), clone, convertTo(CV_32F), eye,
//     rowRange / colRange / col views, copyTo into a view, at<float>;
//   - the C API: CvMat, cvMat, cvCreateMat, cvReleaseMat, cvmSet, cvmGet, cvSetZero, cvMulTransposed, cvSVD, cvInvert,
//     cvSolve and the CV_SVD* constants, whose arithmetic is oracle/pnpsolver.cpp's cv2-pinned primitives.
#pragma once
#include <cstring>
#include <memory>
#include <vector>

#include "../pnpsolver_oracle.h"

#define CV_32F 5
#define CV_64F 6
#define CV_SVD 1
#define CV_SVD_MODIFY_A 1
#define CV_SVD_U_T 2
#define CV_SVD_V_T 4

namespace cv {

template <typename T>
struct Point_ {
  T x = 0, y = 0;
  Point_() {}
  Point_(T a, T b) : x(a), y(b) {}
};
typedef Point_<float> Point2f;
struct Point3f {
  float x = 0, y = 0, z = 0;
  Point3f() {}
  Point3f(float a, float b, float c) : x(a), y(b), z(c) {}
};
struct KeyPoint {
  Point2f pt;
  float size = 0, angle = -1, response = 0;
  int octave = 0, class_id = -1;
};

class Mat {
 public:
  int rows = 0, cols = 0, type = CV_32F, step = 0;  // step in elements
  unsigned char* data = nullptr;
  std::shared_ptr<std::vector<unsigned char>> own;

  Mat() {}
  Mat(int r, int c, int t) : rows(r), cols(c), type(t), step(c) {
    own = std::make_shared<std::vector<unsigned char>>((size_t)r * c * esz(), 0);
    data = own->data();
  }
  Mat(int r, int c, int t, void* d) : rows(r), cols(c), type(t), step(c), data((unsigned char*)d) {}
  size_t esz() const { return type == CV_64F ? 8 : 4; }
  bool empty() const { return !data || rows * cols == 0; }
  double get(int r, int c) const {
    const unsigned char* p = data + ((size_t)r * step + c) * esz();
    return type == CV_64F ? *(const double*)p : *(const float*)p;
  }
  void put(int r, int c, double v) {
    unsigned char* p = data + ((size_t)r * step + c) * esz();
    if (type == CV_64F)
      *(double*)p = v;
    else
      *(float*)p = (float)v;
  }
  template <typename T>
  T& at(int i) {
    return ((T*)data)[(size_t)(i / cols) * step + i % cols];
  }
  template <typename T>
  T& at(int r, int c) {
    return ((T*)data)[(size_t)r * step + c];
  }
  Mat clone() const {
    Mat m(rows, cols, type);
    for (int r = 0; r < rows; r++) std::memcpy(m.data + (size_t)r * cols * esz(), data + (size_t)r * step * esz(), cols * esz());
    return m;
  }
  // convertTo(dst, CV_32F): saturate_cast<float> of each element, i.e. (float)
  void convertTo(Mat& dst, int t) const {
    Mat m(rows, cols, t);
    for (int r = 0; r < rows; r++)
      for (int c = 0; c < cols; c++) m.put(r, c, t == CV_32F ? (double)(float)get(r, c) : get(r, c));
    dst = m;
  }
  static Mat eye(int r, int c, int t) {
    Mat m(r, c, t);
    for (int i = 0; i < r && i < c; i++) m.put(i, i, 1.0);
    return m;
  }
  Mat view(int r0, int c0, int nr, int nc) const {
    Mat m = *this;
    m.data = data + ((size_t)r0 * step + c0) * esz();
    m.rows = nr;
    m.cols = nc;
    return m;
  }
  Mat rowRange(int a, int b) const { return view(a, 0, b - a, cols); }
  Mat colRange(int a, int b) const { return view(0, a, rows, b - a); }
  Mat col(int c) const { return view(0, c, rows, 1); }
  // copyTo a destination of the same size and type fills it in place (a view included)
  void copyTo(Mat& dst) const {
    if (dst.rows != rows || dst.cols != cols || dst.type != type || !dst.data) dst = Mat(rows, cols, type);
    const Mat src = clone();
    for (int r = 0; r < rows; r++)
      for (int c = 0; c < cols; c++) dst.put(r, c, src.get(r, c));
  }
  void copyTo(Mat&& dst) const { copyTo(static_cast<Mat&>(dst)); }
};

}  // namespace cv

// ------------------------------------------------------------------------------------------------ the C API (CV_64F)
struct CvMat {
  int type, step, rows, cols;
  union {
    unsigned char* ptr;
    double* db;
    float* fl;
  } data;
};
inline CvMat cvMat(int rows, int cols, int type, void* data) {
  CvMat m;
  m.type = type;
  m.rows = rows;
  m.cols = cols;
  m.step = cols * 8;
  m.data.ptr = (unsigned char*)data;
  return m;
}
inline CvMat* cvCreateMat(int rows, int cols, int type) {
  CvMat* m = new CvMat(cvMat(rows, cols, type, nullptr));
  m->data.db = new double[(size_t)rows * cols > 0 ? (size_t)rows * cols : 1];
  return m;
}
inline void cvReleaseMat(CvMat** m) {
  if (m && *m) {
    delete[](*m)->data.db;
    delete *m;
    *m = nullptr;
  }
}
inline void cvmSet(CvMat* m, int r, int c, double v) { m->data.db[(size_t)r * m->cols + c] = v; }
inline double cvmGet(const CvMat* m, int r, int c) { return m->data.db[(size_t)r * m->cols + c]; }
inline void cvSetZero(CvMat* m) {
  for (int i = 0; i < m->rows * m->cols; i++) m->data.db[i] = 0;
}
// cvMulTransposed(A, D, 1): D = A^T A
inline void cvMulTransposed(const CvMat* A, CvMat* D, int order) {
  if (order == 1) orc_pnp_mul_transposed(A->data.db, A->rows, A->cols, D->data.db);
}
// cvSVD of a square matrix: W; U (transposed with CV_SVD_U_T); V (V itself unless CV_SVD_V_T)
inline void cvSVD(CvMat* A, CvMat* W, CvMat* U, CvMat* V, int flags) {
  const int n = A->rows;
  double w[12], u[144], vt[144];
  orc_pnp_svd(A->data.db, n, w, u, vt);
  for (int i = 0; i < n; i++) W->data.db[i] = w[i];
  for (int r = 0; r < n; r++)
    for (int c = 0; c < n; c++) {
      if (U) U->data.db[r * n + c] = (flags & CV_SVD_U_T) ? u[c * n + r] : u[r * n + c];
      if (V) V->data.db[r * n + c] = (flags & CV_SVD_V_T) ? vt[r * n + c] : vt[c * n + r];
    }
}
inline double cvInvert(const CvMat* A, CvMat* B, int) {
  orc_pnp_invert_svd(A->data.db, A->rows, B->data.db);
  return 0;
}
inline int cvSolve(const CvMat* A, const CvMat* b, CvMat* x, int) {
  orc_pnp_solve_svd(A->data.db, A->rows, A->cols, b->data.db, x->data.db);
  return 1;
}
