// sim3.cuh — g2o::Sim3 (Thirdparty/g2o/g2o/types/sim3.h) on the device, FP64, 8 doubles per Sim3 in the layout of
// b2s_sim3 (qx qy qz qw tx ty tz s): product, inverse, map, the exponential map with its four sigma / theta branches and
// the log with W.lu().solve(t).  Shared by the essential graph (essential.cu) and OptimizeSim3 (sim3opt.cu); both are
// compiled without FMA contraction, because their numeric Jacobians amplify last-bit differences about 5e8 times.
#pragma once
#include <math.h>

#include "ba_math.cuh"

namespace b2s {

// quaternion product a * b (Eigen's formula)
__device__ __forceinline__ void q_mul(const double* a, const double* b, double* r) {
  r[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
  r[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  r[1] = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
  r[2] = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
}
// operator*: r = a.r * b.r, t = a.s (a.r * b.t) + a.t, s = a.s b.s
__device__ __forceinline__ void s3_mul(const double* a, const double* b, double* o) {
  double rt[3];
  quat_rotate(a, b + 4, rt);
  q_mul(a, b, o);
  for (int i = 0; i < 3; i++) o[4 + i] = a[7] * rt[i] + a[4 + i];
  o[7] = a[7] * b[7];
}
// inverse(): Sim3(r.conjugate(), r.conjugate() * ((-1 / s) t), 1 / s)
__device__ __forceinline__ void s3_inv(const double* a, double* o) {
  const double c[4] = {-a[0], -a[1], -a[2], a[3]};
  const double k = -1. / a[7];
  const double v[3] = {k * a[4], k * a[5], k * a[6]};
  double rt[3];
  quat_rotate(c, v, rt);
  for (int i = 0; i < 4; i++) o[i] = c[i];
  for (int i = 0; i < 3; i++) o[4 + i] = rt[i];
  o[7] = 1. / a[7];
}
// map(): s (r X) + t
__device__ __forceinline__ void s3_map(const double* a, const double* X, double* o) {
  double rt[3];
  quat_rotate(a, X, rt);
  for (int i = 0; i < 3; i++) o[i] = a[7] * rt[i] + a[4 + i];
}
__device__ __forceinline__ void skew(const double* v, double O[3][3]) {
  O[0][0] = 0; O[0][1] = -v[2]; O[0][2] = v[1];
  O[1][0] = v[2]; O[1][1] = 0; O[1][2] = -v[0];
  O[2][0] = -v[1]; O[2][1] = v[0]; O[2][2] = 0;
}
__device__ __forceinline__ void mat_mul3(const double A[3][3], const double B[3][3], double C[3][3]) {
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) C[i][j] = A[i][0] * B[0][j] + A[i][1] * B[1][j] + A[i][2] * B[2][j];
}
// Sim3(const Vector7d& update): the exponential map, all four sigma / theta branches
__device__ inline void s3_exp(const double* u, double* o) {
  const double omega[3] = {u[0], u[1], u[2]};
  const double sigma = u[6];
  const double theta = sqrt(omega[0] * omega[0] + omega[1] * omega[1] + omega[2] * omega[2]);
  double O[3][3], O2[3][3], R[3][3];
  skew(omega, O);
  const double s = exp(sigma);
  mat_mul3(O, O, O2);
  const double eps = 0.00001;
  double A, B, C;
  bool small = theta < eps;
  if (fabs(sigma) < eps) {
    C = 1;
    if (small) {
      A = 1. / 2.;
      B = 1. / 6.;
    } else {
      const double theta2 = theta * theta;
      A = (1 - cos(theta)) / (theta2);
      B = (theta - sin(theta)) / (theta2 * theta);
    }
  } else {
    C = (s - 1) / sigma;
    if (small) {
      const double sigma2 = sigma * sigma;
      A = ((sigma - 1) * s + 1) / sigma2;
      B = ((0.5 * sigma2 - sigma + 1) * s) / (sigma2 * sigma);
    } else {
      const double a = s * sin(theta), b = s * cos(theta);
      const double theta2 = theta * theta, sigma2 = sigma * sigma;
      const double c = theta2 + sigma2;
      A = (a * sigma + (1 - b) * theta) / (theta * c);
      B = (C - ((b - 1) * sigma + a * theta) / (c)) * 1. / (theta2);
    }
  }
  if (small) {
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) R[i][j] = ((i == j ? 1.0 : 0.0) + O[i][j]) + O2[i][j];
  } else {
    const double k1 = sin(theta) / theta, k2 = (1 - cos(theta)) / (theta * theta);
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) R[i][j] = ((i == j ? 1.0 : 0.0) + k1 * O[i][j]) + k2 * O2[i][j];
  }
  quat_from_R(R, o);
  double W[3][3];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) W[i][j] = (A * O[i][j] + B * O2[i][j]) + C * (i == j ? 1.0 : 0.0);
  for (int i = 0; i < 3; i++) o[4 + i] = W[i][0] * u[3] + W[i][1] * u[4] + W[i][2] * u[5];
  o[7] = s;
}
// log(): omega, upsilon = W^-1 t (partial-pivoting LU), sigma
__device__ inline void s3_log(const double* a, double* res) {
  const double s = a[7];
  const double sigma = log(s);
  double R[3][3];
  quat_to_R(a, R);
  const double d = 0.5 * (R[0][0] + R[1][1] + R[2][2] - 1);
  const double dR[3] = {R[2][1] - R[1][2], R[0][2] - R[2][0], R[1][0] - R[0][1]};
  const double eps = 0.00001;
  double omega[3], A, B, C;
  if (fabs(sigma) < eps) {
    C = 1;
    if (d > 1 - eps) {
      for (int i = 0; i < 3; i++) omega[i] = 0.5 * dR[i];
      A = 1. / 2.;
      B = 1. / 6.;
    } else {
      const double theta = acos(d);
      const double theta2 = theta * theta;
      const double k = theta / (2 * sqrt(1 - d * d));
      for (int i = 0; i < 3; i++) omega[i] = k * dR[i];
      A = (1 - cos(theta)) / (theta2);
      B = (theta - sin(theta)) / (theta2 * theta);
    }
  } else {
    C = (s - 1) / sigma;
    if (d > 1 - eps) {
      const double sigma2 = sigma * sigma;
      for (int i = 0; i < 3; i++) omega[i] = 0.5 * dR[i];
      A = ((sigma - 1) * s + 1) / (sigma2);
      B = ((0.5 * sigma2 - sigma + 1) * s) / (sigma2 * sigma);
    } else {
      const double theta = acos(d);
      const double k = theta / (2 * sqrt(1 - d * d));
      for (int i = 0; i < 3; i++) omega[i] = k * dR[i];
      const double theta2 = theta * theta;
      const double aa = s * sin(theta), bb = s * cos(theta);
      const double c = theta2 + sigma * sigma;
      A = (aa * sigma + (1 - bb) * theta) / (theta * c);
      B = (C - ((bb - 1) * sigma + aa * theta) / (c)) * 1. / (theta2);
    }
  }
  double O[3][3], BO[3][3], BOO[3][3], W[3][3];
  skew(omega, O);
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) BO[i][j] = B * O[i][j];
  mat_mul3(BO, O, BOO);  // B*Omega*Omega evaluates left to right
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) W[i][j] = (A * O[i][j] + BOO[i][j]) + C * (i == j ? 1.0 : 0.0);
  // W.lu().solve(t): row pivoting on the largest |entry| (first one on ties), L unit lower, U upper
  int perm[3] = {0, 1, 2};
  for (int k = 0; k < 3; k++) {
    int p = k;
    double best = fabs(W[k][k]);
    for (int i = k + 1; i < 3; i++)
      if (fabs(W[i][k]) > best) {
        best = fabs(W[i][k]);
        p = i;
      }
    if (p != k) {
      for (int j = 0; j < 3; j++) {
        const double tmp = W[k][j];
        W[k][j] = W[p][j];
        W[p][j] = tmp;
      }
      const int tp = perm[k];
      perm[k] = perm[p];
      perm[p] = tp;
    }
    if (W[k][k] == 0.0) continue;
    for (int i = k + 1; i < 3; i++) {
      W[i][k] /= W[k][k];
      for (int j = k + 1; j < 3; j++) W[i][j] -= W[i][k] * W[k][j];
    }
  }
  double x[3];
  for (int i = 0; i < 3; i++) {
    double v = a[4 + perm[i]];
    for (int k = 0; k < i; k++) v -= W[i][k] * x[k];
    x[i] = v;
  }
  for (int i = 2; i >= 0; i--) {
    double v = x[i];
    for (int k = i + 1; k < 3; k++) v -= W[i][k] * x[k];
    x[i] = v / W[i][i];
  }
  for (int i = 0; i < 3; i++) res[i] = omega[i];
  for (int i = 0; i < 3; i++) res[3 + i] = x[i];
  res[6] = sigma;
}

}  // namespace b2s
