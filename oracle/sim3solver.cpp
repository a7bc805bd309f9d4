// TEST INFRASTRUCTURE — CPU restatement of Sim3Solver (src/Sim3Solver.cc), statement by statement, with the minimal
// sets as input (the reference draws them with DUtils::Random inside iterate).  Every cv::Mat is CV_32F; the OpenCV
// operations are restated from OpenCV 4.13 and tests/test_oracle_sim3solver.py pins them bit for bit against cv2 where
// cv2 exposes them (reduce, eigen, Rodrigues, norm, pow, gemm).  Mat::dot and the MatExpr scaling rules are read from
// OpenCV's source (cv2 binds neither); DESIGN §7 lists them.
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <vector>

#include "init_oracle.h"
#include "sim3solver_oracle.h"

extern "C" {

// cv::reduce(P, C, 1, REDUCE_SUM) over CV_32F: each row summed in float, left to right
void orc_s3s_reduce_sum_cols(const float* P, int rows, int cols, float* C) {
  for (int r = 0; r < rows; r++) {
    float a = P[(size_t)r * cols];
    for (int i = 1; i < cols; i++) a = a + P[(size_t)r * cols + i];
    C[r] = a;
  }
}

// lapack.cpp's own hypot template, in float (not glibc's hypotf: cv2.eigen agrees with this one bit for bit)
static inline float hypot_f(float a, float b) {
  a = std::fabs(a);
  b = std::fabs(b);
  if (a > b) {
    b /= a;
    return a * std::sqrt(1 + b * b);
  }
  if (b > 0) {
    a /= b;
    return b * std::sqrt(1 + a * a);
  }
  return 0;
}

// JacobiImpl_<float> (lapack.cpp) with V, then the descending sort
void orc_s3s_eigen(const float* Ain, int n, float* W, float* V) {
  float A[64];
  int indR[8], indC[8];
  memcpy(A, Ain, sizeof(float) * n * n);
  const float eps = FLT_EPSILON;
  for (int i = 0; i < n; i++) {
    for (int j = 0; j < n; j++) V[i * n + j] = 0.f;
    V[i * n + i] = 1.f;
  }
  int k, m, i, j;
  float mv;
  for (k = 0; k < n; k++) {
    W[k] = A[(n + 1) * k];
    if (k < n - 1) {
      for (m = k + 1, mv = std::fabs(A[n * k + m]), i = k + 2; i < n; i++) {
        const float val = std::fabs(A[n * k + i]);
        if (mv < val) mv = val, m = i;
      }
      indR[k] = m;
    }
    if (k > 0) {
      for (m = 0, mv = std::fabs(A[k]), i = 1; i < k; i++) {
        const float val = std::fabs(A[n * i + k]);
        if (mv < val) mv = val, m = i;
      }
      indC[k] = m;
    }
  }
  if (n > 1)
    for (int iters = 0, maxIters = n * n * 30; iters < maxIters; iters++) {
      for (k = 0, mv = std::fabs(A[indR[0]]), i = 1; i < n - 1; i++) {
        const float val = std::fabs(A[n * i + indR[i]]);
        if (mv < val) mv = val, k = i;
      }
      int l = indR[k];
      for (i = 1; i < n; i++) {
        const float val = std::fabs(A[n * indC[i] + i]);
        if (mv < val) mv = val, k = indC[i], l = i;
      }
      const float p = A[n * k + l];
      if (std::fabs(p) <= eps) break;
      const float y = (float)((W[l] - W[k]) * 0.5);
      float t = std::fabs(y) + hypot_f(p, y);
      float s = hypot_f(p, t);
      const float c = t / s;
      s = p / s;
      t = (p / t) * p;
      if (y < 0) s = -s, t = -t;
      A[n * k + l] = 0;
      W[k] -= t;
      W[l] += t;
      float a0, b0;
#define S3S_ROTATE(v0, v1) a0 = v0, b0 = v1, v0 = a0 * c - b0 * s, v1 = a0 * s + b0 * c
      for (i = 0; i < k; i++) S3S_ROTATE(A[n * i + k], A[n * i + l]);
      for (i = k + 1; i < l; i++) S3S_ROTATE(A[n * k + i], A[n * i + l]);
      for (i = l + 1; i < n; i++) S3S_ROTATE(A[n * k + i], A[n * l + i]);
      for (i = 0; i < n; i++) S3S_ROTATE(V[n * k + i], V[n * l + i]);
#undef S3S_ROTATE
      for (j = 0; j < 2; j++) {
        const int idx = j == 0 ? k : l;
        if (idx < n - 1) {
          for (m = idx + 1, mv = std::fabs(A[n * idx + m]), i = idx + 2; i < n; i++) {
            const float val = std::fabs(A[n * idx + i]);
            if (mv < val) mv = val, m = i;
          }
          indR[idx] = m;
        }
        if (idx > 0) {
          for (m = 0, mv = std::fabs(A[idx]), i = 1; i < idx; i++) {
            const float val = std::fabs(A[n * i + idx]);
            if (mv < val) mv = val, m = i;
          }
          indC[idx] = m;
        }
      }
    }
  for (k = 0; k < n - 1; k++) {
    m = k;
    for (i = k + 1; i < n; i++)
      if (W[m] < W[i]) m = i;
    if (k != m) {
      std::swap(W[m], W[k]);
      for (i = 0; i < n; i++) std::swap(V[n * m + i], V[n * k + i]);
    }
  }
}

// cvRodrigues2 (calibration.cpp), vector to matrix: Point3d r, theta = norm(r), R = c*I + c1*r*r^T + s*[r]_x in double
void orc_s3s_rodrigues(const float* v, float* R) {
  double rx = v[0], ry = v[1], rz = v[2];
  const double theta = std::sqrt(rx * rx + ry * ry + rz * rz);
  if (theta < DBL_EPSILON) {
    for (int i = 0; i < 9; i++) R[i] = (i % 4 == 0) ? 1.f : 0.f;
    return;
  }
  const double c = cos(theta), s = sin(theta), c1 = 1. - c;
  const double itheta = theta ? 1. / theta : 0.;
  rx *= itheta;
  ry *= itheta;
  rz *= itheta;
  const double rrt[9] = {rx * rx, rx * ry, rx * rz, rx * ry, ry * ry, ry * rz, rx * rz, ry * rz, rz * rz};
  const double r_x[9] = {0, -rz, ry, rz, 0, -rx, -ry, rx, 0};
  for (int i = 0; i < 9; i++) {
    const double e = (i % 4 == 0) ? 1. : 0.;
    R[i] = (float)((c * e + c1 * rrt[i]) + s * r_x[i]);
  }
}

// cv::norm(a) (NORM_L2) of CV_32F: squares in double accumulated in two lanes (even and odd entries), the lanes then
// added; for the 3-vector ComputeSim3 takes this is (x0^2 + x2^2) + x1^2, which cv2.norm gives bit for bit
double orc_s3s_norm(const float* a, int len) {
  double l0 = 0, l1 = 0;
  for (int i = 0; i < len; i++) {
    const double v = a[i];
    if (i % 2)
      l1 += v * v;
    else
      l0 += v * v;
  }
  return std::sqrt(l0 + l1);
}

// dotProd_<float> (matmul.simd.hpp), which dotProd_32f runs for fewer entries than one AVX-512 vector: double products,
// unrolled by 4
double orc_s3s_dot(const float* a, const float* b, int len) {
  double r = 0;
  int i = 0;
  for (; i <= len - 4; i += 4)
    r += (double)a[i] * b[i] + (double)a[i + 1] * b[i + 1] + (double)a[i + 2] * b[i + 2] + (double)a[i + 3] * b[i + 3];
  for (; i < len; i++) r += (double)a[i] * b[i];
  return r;
}

void orc_s3s_pow2(const float* a, int len, float* out) {
  for (int i = 0; i < len; i++) out[i] = a[i] * a[i];
}

void orc_s3s_gemm_bt(const float* A, const float* B, int m, int k, int n, float* D) {
  for (int r = 0; r < m; r++)
    for (int c = 0; c < n; c++) {
      double s = 0;
      for (int q = 0; q < k; q++) s += (double)A[r * k + q] * B[c * k + q];
      D[r * n + c] = (float)s;
    }
}

// :143-196.  The double -> int conversion of ceil() is x86's: NaN and out-of-range values become INT_MIN.
int orc_s3s_ransac_max_its(int N, double probability, int min_inliers, int max_iterations) {
  const float epsilon = (float)min_inliers / N;
  int nIterations;
  if (min_inliers == N) {
    nIterations = 1;
  } else {
    const double c = ceil(log(1 - probability) / log(1 - pow(epsilon, 3)));
    nIterations = (c >= (double)INT_MIN && c <= (double)INT_MAX) ? (int)c : INT_MIN;
  }
  return std::max(1, std::min(nIterations, max_iterations));
}

}  // extern "C"

namespace {

// ComputeCentroid (:295-305): reduce, C = C/P.cols (convertTo: times (float)(1./3)), Pr.col(i) = P.col(i) - C
void centroid(const float* P, float* Pr, float* C) {
  orc_s3s_reduce_sum_cols(P, 3, 3, C);
  const float sc = (float)(1. / 3);
  for (int r = 0; r < 3; r++) C[r] = C[r] * sc;
  for (int r = 0; r < 3; r++)
    for (int i = 0; i < 3; i++) Pr[r * 3 + i] = P[r * 3 + i] - C[r];
}

struct Hyp {
  float R[9], t[3], s, T12[16], T21[16];
};

// ComputeSim3 (:309-448)
void compute_sim3(const float* P1, const float* P2, bool fix, Hyp& h) {
  float Pr1[9], Pr2[9], O1[3], O2[3], M[9];
  centroid(P1, Pr1, O1);
  centroid(P2, Pr2, O2);
  orc_s3s_gemm_bt(Pr2, Pr1, 3, 3, 3, M);  // M = Pr2*Pr1.t()
#define m(r, c) M[(r) * 3 + (c)]
  // float sums, stored through double into Mat_<float>
  const double N11 = m(0, 0) + m(1, 1) + m(2, 2), N12 = m(1, 2) - m(2, 1), N13 = m(2, 0) - m(0, 2),
               N14 = m(0, 1) - m(1, 0), N22 = m(0, 0) - m(1, 1) - m(2, 2), N23 = m(0, 1) + m(1, 0),
               N24 = m(2, 0) + m(0, 2), N33 = -m(0, 0) + m(1, 1) - m(2, 2), N34 = m(1, 2) + m(2, 1),
               N44 = -m(0, 0) - m(1, 1) + m(2, 2);
#undef m
  const float N[16] = {(float)N11, (float)N12, (float)N13, (float)N14, (float)N12, (float)N22, (float)N23, (float)N24,
                       (float)N13, (float)N23, (float)N33, (float)N34, (float)N14, (float)N24, (float)N34, (float)N44};
  float eval[4], evec[16];
  orc_s3s_eigen(N, 4, eval, evec);
  float vec[3] = {evec[1], evec[2], evec[3]};
  const double nv = orc_s3s_norm(vec, 3);
  const double ang = atan2(nv, (double)evec[0]);
  // vec = 2*ang*vec/norm(vec): one MatExpr scale, alpha = (2*ang)*(1/norm), applied by convertTo as a float
  const float alpha = (float)((2 * ang) * (1. / nv));
  for (int i = 0; i < 3; i++) vec[i] = vec[i] * alpha;
  orc_s3s_rodrigues(vec, h.R);
  float P3[9];
  orc_gemm(h.R, Pr2, nullptr, 3, 3, 3, 1.0, 0, P3);
  if (!fix) {
    const double nom = orc_s3s_dot(Pr1, P3, 9);
    float aux[9];
    orc_s3s_pow2(P3, 9, aux);
    double den = 0;
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) den += aux[i * 3 + j];
    h.s = (float)(nom / den);
  } else {
    h.s = 1.0f;
  }
  // t = O1 - s*R*O2: gemm(R, O2, -s, O1, 1)
  orc_gemm(h.R, O2, O1, 3, 3, 1, -(double)h.s, 0, h.t);
  // T12 = [s*R | t]; T21 = [(1/s)*R.t() | -sRinv*t]
  const float sf = (float)(double)h.s, si = (float)(1.0 / h.s);
  float sRinv[9], tinv[3];
  for (int i = 0; i < 16; i++) h.T12[i] = h.T21[i] = (i % 5 == 0) ? 1.f : 0.f;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) {
      h.T12[r * 4 + c] = h.R[r * 3 + c] * sf;
      sRinv[r * 3 + c] = h.R[c * 3 + r] * si;
    }
  orc_gemm(sRinv, h.t, nullptr, 3, 3, 1, -1.0, 0, tinv);
  for (int r = 0; r < 3; r++) {
    h.T12[r * 4 + 3] = h.t[r];
    for (int c = 0; c < 3; c++) h.T21[r * 4 + c] = sRinv[r * 3 + c];
    h.T21[r * 4 + 3] = tinv[r];
  }
}

// FromCameraToImage (:526-545) of one point
void to_image(const float* X, const float* K, float* uv) {
  const float invz = 1 / X[2];
  const float x = X[0] * invz, y = X[1] * invz;
  uv[0] = K[0] * x + K[2];
  uv[1] = K[1] * y + K[3];
}

// Project (:499-523) of one point: Rcw*X + tcw as gemm(Rcw, X, 1, tcw, 1), then FromCameraToImage's arithmetic
void project(const float* T, const float* X, const float* K, float* uv) {
  const float R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]}, t[3] = {T[3], T[7], T[11]};
  float P[3];
  orc_gemm(R, X, t, 3, 3, 1, 1.0, 0, P);
  to_image(P, K, uv);
}

float threshold(float sigma2) { return (float)(size_t)(9.210 * sigma2); }

// CheckInliers (:451-479); returns mnInliersi
int check_inliers(const b2s_sim3solver_problem* p, const Hyp& h, std::vector<uint8_t>& inl, double* margin) {
  int n = 0;
  for (int i = 0; i < p->n; i++) {
    float p1im1[2], p2im2[2], p2im1[2], p1im2[2];
    to_image(p->X1c + 3 * i, p->K1, p1im1);
    to_image(p->X2c + 3 * i, p->K2, p2im2);
    project(h.T12, p->X2c + 3 * i, p->K1, p2im1);
    project(h.T21, p->X1c + 3 * i, p->K2, p1im2);
    const float d1[2] = {p1im1[0] - p2im1[0], p1im1[1] - p2im1[1]};
    const float d2[2] = {p1im2[0] - p2im2[0], p1im2[1] - p2im2[1]};
    const float err1 = (float)orc_s3s_dot(d1, d1, 2), err2 = (float)orc_s3s_dot(d2, d2, 2);
    const float th1 = threshold(p->sigma2_1[i]), th2 = threshold(p->sigma2_2[i]);
    if (margin) {
      if (std::isfinite(err1)) *margin = std::min(*margin, std::fabs((double)err1 - th1) / th1);
      if (std::isfinite(err2)) *margin = std::min(*margin, std::fabs((double)err2 - th2) / th2);
    }
    inl[(size_t)i] = (err1 < th1 && err2 < th2) ? 1 : 0;
    n += inl[(size_t)i];
  }
  return n;
}

}  // namespace

extern "C" {

void orc_s3s_compute_sim3(const float* P1, const float* P2, int fix_scale, float* hyp) {
  Hyp h;
  compute_sim3(P1, P2, fix_scale != 0, h);
  memcpy(hyp, h.R, 9 * sizeof(float));
  memcpy(hyp + 9, h.t, 3 * sizeof(float));
  hyp[12] = h.s;
  memcpy(hyp + 13, h.T12, 16 * sizeof(float));
  memcpy(hyp + 29, h.T21, 16 * sizeof(float));
}

// iterate (:199-285)
void orc_s3s_iterate(const b2s_sim3solver_problem* p, b2s_sim3solver_result* r, double* margin) {
  if (margin) *margin = INFINITY;
  r->returned = 0;
  r->best_changed = 0;
  r->n_inliers = 0;
  r->no_more = 0;
  r->iterations_used = 0;
  r->iterations_done = p->iterations_done;
  r->best_inliers = p->best_inliers;
  if (p->n > 0) memset(r->inliers, 0, (size_t)p->n);
  if (p->n < p->min_inliers) {
    r->no_more = 1;
    return;
  }
  std::vector<uint8_t> inl((size_t)p->n);
  int mnIterations = p->iterations_done, mnBestInliers = p->best_inliers, cur = 0;
  while (mnIterations < p->max_its && cur < p->k) {
    const int* set = p->sets + 3 * cur;
    cur++;
    mnIterations++;
    float P1[9], P2[9];
    for (int i = 0; i < 3; i++)
      for (int rr = 0; rr < 3; rr++) {
        P1[rr * 3 + i] = p->X1c[3 * set[i] + rr];
        P2[rr * 3 + i] = p->X2c[3 * set[i] + rr];
      }
    Hyp h;
    compute_sim3(P1, P2, p->fix_scale != 0, h);
    const int ni = check_inliers(p, h, inl, margin);
    if (ni >= mnBestInliers) {
      mnBestInliers = ni;
      r->best_changed = 1;
      memcpy(r->R, h.R, sizeof(r->R));
      memcpy(r->t, h.t, sizeof(r->t));
      r->s = h.s;
      if (ni > p->min_inliers) {
        r->returned = 1;
        r->n_inliers = ni;
        memcpy(r->inliers, inl.data(), (size_t)p->n);
        memcpy(r->T12, h.T12, sizeof(r->T12));
        r->iterations_used = cur;
        r->iterations_done = mnIterations;
        r->best_inliers = mnBestInliers;
        return;
      }
    }
  }
  r->no_more = mnIterations >= p->max_its;
  r->iterations_used = cur;
  r->iterations_done = mnIterations;
  r->best_inliers = mnBestInliers;
}

}  // extern "C"
