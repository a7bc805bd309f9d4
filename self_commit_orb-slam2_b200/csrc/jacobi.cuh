// jacobi.cuh — OpenCV's one-sided Jacobi SVD (JacobiSVDImpl_ in modules/core/src/lapack.cpp) on the device, one thread,
// for the element types SVD::compute instantiates it with: float (initializer.cu) and double (pnpsolver.cu).
#pragma once

#include <float.h>
#include <math.h>
#include <stdint.h>

namespace b2s {

// cv::RNG::next
__device__ __forceinline__ unsigned rng_next(uint64_t& state) {
  state = (uint64_t)(unsigned)state * 4164903690u + (unsigned)(state >> 32);
  return (unsigned)state;
}

// lapack.cpp's hypot template: a*sqrt(1 + (b/a)^2) with the larger magnitude outside, only + - * / sqrt
__device__ __forceinline__ double cv_hypot(double a, double b) {
  a = fabs(a);
  b = fabs(b);
  if (a > b) {
    b /= a;
    return a * sqrt(1 + b * b);
  }
  if (b > 0) {
    a /= b;
    return b * sqrt(1 + a * a);
  }
  return 0;
}

// The constants JacobiSVD passes per element type, and the rotation's hypot.  The float instantiation calls CUDA's
// double hypot where the initializer's restatement calls glibc's (DESIGN §7); the double one calls the template, as
// cv2 does (tests/test_oracle_pnpsolver.py pins it).
template <typename T>
struct JacobiTraits;
template <>
struct JacobiTraits<float> {
  static constexpr double minval = FLT_MIN;
  static constexpr float eps = FLT_EPSILON * 2;
  static __device__ __forceinline__ double rot_hypot(double p, double beta) { return hypot(p, beta); }
};
template <>
struct JacobiTraits<double> {
  static constexpr double minval = DBL_MIN;
  static constexpr double eps = DBL_EPSILON * 10;
  static __device__ __forceinline__ double rot_hypot(double p, double beta) { return cv_hypot(p, beta); }
};

// JacobiSVDImpl_<T> (oracle/init.cpp jacobi_svd for float, oracle/pnpsolver.cpp jacobi_svd for double): At n rows of m,
// W n, Vt n x n (row stride n), n1 rows of At normalised / completed from RNG(0x12345678).  NMAX bounds n.
template <int NMAX, typename T>
__device__ void jacobi_svd(T* At, int astep, T* Wout, T* Vt, int m, int n, int n1) {
  const double minval = JacobiTraits<T>::minval;
  const T eps = JacobiTraits<T>::eps;
  double W[NMAX];
  const int max_iter = m > 30 ? m : 30;
  for (int i = 0; i < n; i++) {
    double sd = 0;
    for (int k = 0; k < m; k++) {
      const T t = At[i * astep + k];
      sd += (double)t * t;
    }
    W[i] = sd;
    for (int k = 0; k < n; k++) Vt[i * n + k] = 0;
    Vt[i * n + i] = 1;
  }
  for (int iter = 0; iter < max_iter; iter++) {
    bool changed = false;
    for (int i = 0; i < n - 1; i++)
      for (int j = i + 1; j < n; j++) {
        T *Ai = At + i * astep, *Aj = At + j * astep;
        double a = W[i], p = 0, b = W[j];
        for (int k = 0; k < m; k++) p += (double)Ai[k] * Aj[k];
        if (fabs(p) <= eps * sqrt((double)a * b)) continue;
        p *= 2;
        const double beta = a - b, gamma = JacobiTraits<T>::rot_hypot(p, beta);
        T c, s;
        if (beta < 0) {
          const double delta = (gamma - beta) * 0.5;
          s = (T)sqrt(delta / gamma);
          c = (T)(p / (gamma * s * 2));
        } else {
          c = (T)sqrt((gamma + beta) / (gamma * 2));
          s = (T)(p / (gamma * c * 2));
        }
        a = b = 0;
        for (int k = 0; k < m; k++) {
          const T t0 = c * Ai[k] + s * Aj[k];
          const T t1 = -s * Ai[k] + c * Aj[k];
          Ai[k] = t0;
          Aj[k] = t1;
          a += (double)t0 * t0;
          b += (double)t1 * t1;
        }
        W[i] = a;
        W[j] = b;
        changed = true;
        T *Vi = Vt + i * n, *Vj = Vt + j * n;
        for (int k = 0; k < n; k++) {
          const T t0 = c * Vi[k] + s * Vj[k];
          const T t1 = -s * Vi[k] + c * Vj[k];
          Vi[k] = t0;
          Vj[k] = t1;
        }
      }
    if (!changed) break;
  }
  for (int i = 0; i < n; i++) {
    double sd = 0;
    for (int k = 0; k < m; k++) {
      const T t = At[i * astep + k];
      sd += (double)t * t;
    }
    W[i] = sqrt(sd);
  }
  for (int i = 0; i < n - 1; i++) {
    int j = i;
    for (int k = i + 1; k < n; k++)
      if (W[j] < W[k]) j = k;
    if (i != j) {
      const double w = W[i];
      W[i] = W[j];
      W[j] = w;
      for (int k = 0; k < m; k++) {
        const T x = At[i * astep + k];
        At[i * astep + k] = At[j * astep + k];
        At[j * astep + k] = x;
      }
      for (int k = 0; k < n; k++) {
        const T x = Vt[i * n + k];
        Vt[i * n + k] = Vt[j * n + k];
        Vt[j * n + k] = x;
      }
    }
  }
  for (int i = 0; i < n; i++) Wout[i] = (T)W[i];
  uint64_t rng = 0x12345678;
  for (int i = 0; i < n1; i++) {
    double sd = i < n ? W[i] : 0;
    for (int ii = 0; ii < 100 && sd <= minval; ii++) {
      const T val0 = (T)(1. / m);
      for (int k = 0; k < m; k++) At[i * astep + k] = (rng_next(rng) & 256) != 0 ? val0 : -val0;
      for (int it2 = 0; it2 < 2; it2++)
        for (int j = 0; j < i; j++) {
          sd = 0;
          for (int k = 0; k < m; k++) sd += At[i * astep + k] * At[j * astep + k];
          T asum = 0;
          for (int k = 0; k < m; k++) {
            const T t = (T)(At[i * astep + k] - sd * At[j * astep + k]);
            At[i * astep + k] = t;
            asum += fabs(t);
          }
          asum = asum > eps * 100 ? 1 / asum : 0;
          for (int k = 0; k < m; k++) At[i * astep + k] *= asum;
        }
      sd = 0;
      for (int k = 0; k < m; k++) {
        const T t = At[i * astep + k];
        sd += (double)t * t;
      }
      sd = sqrt(sd);
    }
    const T s = (T)(sd > minval ? 1 / sd : 0.);
    for (int k = 0; k < m; k++) At[i * astep + k] *= s;
  }
}

}  // namespace b2s
