// ba_math.cuh — FP64 SE3 / projection helpers shared by the bundle adjusters (localba.cu: LocalBA and
// PoseOptimization; gba.cu: global bundle adjustment).
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace b2s {

constexpr int POSE_STRIDE = 8;  // doubles per SE3Quat pose: q(x,y,z,w), t(x,y,z), pad

// ---------------------------------------------------------------- small FP64 helpers
__device__ __forceinline__ void quat_rotate(const double* q, const double* v, double* o) {
  double uvx = q[1] * v[2] - q[2] * v[1], uvy = q[2] * v[0] - q[0] * v[2], uvz = q[0] * v[1] - q[1] * v[0];
  uvx += uvx; uvy += uvy; uvz += uvz;
  o[0] = v[0] + q[3] * uvx + (q[1] * uvz - q[2] * uvy);
  o[1] = v[1] + q[3] * uvy + (q[2] * uvx - q[0] * uvz);
  o[2] = v[2] + q[3] * uvz + (q[0] * uvy - q[1] * uvx);
}
__device__ __forceinline__ void pose_map(const double* P, const double* X, double* o) {
  quat_rotate(P, X, o);
  o[0] += P[4]; o[1] += P[5]; o[2] += P[6];
}
__host__ __device__ __forceinline__ void quat_to_R(const double* q, double R[3][3]) {
  const double tx = 2 * q[0], ty = 2 * q[1], tz = 2 * q[2];
  const double twx = tx * q[3], twy = ty * q[3], twz = tz * q[3];
  const double txx = tx * q[0], txy = ty * q[0], txz = tz * q[0];
  const double tyy = ty * q[1], tyz = tz * q[1], tzz = tz * q[2];
  R[0][0] = 1 - (tyy + tzz); R[0][1] = txy - twz; R[0][2] = txz + twy;
  R[1][0] = txy + twz; R[1][1] = 1 - (txx + tzz); R[1][2] = tyz - twx;
  R[2][0] = txz - twy; R[2][1] = tyz + twx; R[2][2] = 1 - (txx + tyy);
}
__host__ __device__ __forceinline__ void quat_from_R(const double m[3][3], double* q) {  // Eigen::Quaterniond(Matrix3d)
  double t = m[0][0] + m[1][1] + m[2][2];
  if (t > 0.0) {
    t = sqrt(t + 1.0);
    q[3] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (m[2][1] - m[1][2]) * t;
    q[1] = (m[0][2] - m[2][0]) * t;
    q[2] = (m[1][0] - m[0][1]) * t;
  } else {
    int i = 0;
    if (m[1][1] > m[0][0]) i = 1;
    if (m[2][2] > m[i][i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = sqrt(m[i][i] - m[j][j] - m[k][k] + 1.0);
    double v[3];
    v[i] = 0.5 * t;
    t = 0.5 / t;
    q[3] = (m[k][j] - m[j][k]) * t;
    v[j] = (m[j][i] + m[i][j]) * t;
    v[k] = (m[k][i] + m[i][k]) * t;
    q[0] = v[0]; q[1] = v[1]; q[2] = v[2];
  }
}
__host__ __device__ __forceinline__ void normalize_rot(double* q) {  // SE3Quat::normalizeRotation
  if (q[3] < 0) {
    q[0] = -q[0]; q[1] = -q[1]; q[2] = -q[2]; q[3] = -q[3];
  }
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n;
}

// Converter::toSE3Quat (src/Converter.cc:57-66): row-major float 4x4 Tcw -> pose P (POSE_STRIDE doubles)
__host__ __device__ __forceinline__ void se3quat_from_Tcw(const float* T, double* P) {
  double R[3][3];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) R[i][j] = T[i * 4 + j];
  quat_from_R(R, P);
  normalize_rot(P);
  P[4] = T[3]; P[5] = T[7]; P[6] = T[11]; P[7] = 0;
}
// Converter::toCvMat(SE3Quat) (src/Converter.cc:96-107): pose P -> row-major float 4x4 Tcw
__host__ __device__ __forceinline__ void se3quat_to_Tcw(const double* P, float* T) {
  double R[3][3];
  quat_to_R(P, R);
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) T[r * 4 + c] = (float)R[r][c];
    T[r * 4 + 3] = (float)P[4 + r];
  }
  T[12] = 0.f; T[13] = 0.f; T[14] = 0.f; T[15] = 1.f;
}

// SE3Quat::exp(update) * estimate  (se3quat.h:223-257, :103-109)
static __device__ void pose_oplus(double* P, const double* upd) {
  const double wx = upd[0], wy = upd[1], wz = upd[2];
  const double theta = sqrt(wx * wx + wy * wy + wz * wz);
  const double O[3][3] = {{0, -wz, wy}, {wz, 0, -wx}, {-wy, wx, 0}};
  double O2[3][3];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) O2[i][j] = O[i][0] * O[0][j] + O[i][1] * O[1][j] + O[i][2] * O[2][j];
  double R[3][3], V[3][3];
  if (theta < 0.00001) {
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) {
        R[i][j] = (i == j ? 1.0 : 0.0) + O[i][j] + O2[i][j];
        V[i][j] = R[i][j];
      }
  } else {
    const double a = sin(theta) / theta;
    const double bb = (1 - cos(theta)) / (theta * theta);
    const double c = (theta - sin(theta)) / (theta * theta * theta);
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) {
        R[i][j] = (i == j ? 1.0 : 0.0) + a * O[i][j] + bb * O2[i][j];
        V[i][j] = (i == j ? 1.0 : 0.0) + bb * O[i][j] + c * O2[i][j];
      }
  }
  double eq[4], et[3];
  quat_from_R(R, eq);
  normalize_rot(eq);
  for (int i = 0; i < 3; i++) et[i] = V[i][0] * upd[3] + V[i][1] * upd[4] + V[i][2] * upd[5];
  double rt[3];
  quat_rotate(eq, P + 4, rt);
  const double a0 = eq[0], a1 = eq[1], a2 = eq[2], a3 = eq[3];
  const double b0 = P[0], b1 = P[1], b2 = P[2], b3 = P[3];
  double r[4];
  r[3] = a3 * b3 - a0 * b0 - a1 * b1 - a2 * b2;
  r[0] = a3 * b0 + a0 * b3 + a1 * b2 - a2 * b1;
  r[1] = a3 * b1 + a1 * b3 + a2 * b0 - a0 * b2;
  r[2] = a3 * b2 + a2 * b3 + a0 * b1 - a1 * b0;
  normalize_rot(r);
  P[0] = r[0]; P[1] = r[1]; P[2] = r[2]; P[3] = r[3];
  P[4] = et[0] + rt[0]; P[5] = et[1] + rt[1]; P[6] = et[2] + rt[2];
}

__device__ __forceinline__ void huber(double e, double delta, double& rho0, double& rho1) {
  const double dsqr = delta * delta;
  if (e <= dsqr) {
    rho0 = e;
    rho1 = 1.;
  } else {
    const double s = sqrt(e);
    rho0 = 2 * s * delta - dsqr;
    rho1 = delta / s;
  }
}

struct EdgeJac {
  double A[3][3], B[3][6];  // a monocular edge has an all-zero third row (adds exact zeros to every product)
  double Xc[3];
};
// linearizeOplus (types_six_dof_expmap.cpp:103-139 mono, :188-234 stereo).  The reference divides by z and z^2 in
// every entry; here 1/z is formed once (differences ~1 ulp, far inside the 1e-5 bar).
__device__ __forceinline__ void edge_jacobians(const double* P, const double* X, bool st, double fx, double fy, double bf,
                                               EdgeJac& J) {
  double R[3][3];
  pose_map(P, X, J.Xc);
  quat_to_R(P, R);
  const double x = J.Xc[0], y = J.Xc[1], z = J.Xc[2];
  const double iz = 1.0 / z, iz2 = iz * iz;
  const double fxz = fx * iz, fyz = fy * iz, fxx = fx * x * iz2, fyy = fy * y * iz2;
  const double bz = st ? bf * iz2 : 0.0;
#pragma unroll
  for (int c = 0; c < 3; c++) {
    J.A[0][c] = -fxz * R[0][c] + fxx * R[2][c];
    J.A[1][c] = -fyz * R[1][c] + fyy * R[2][c];
    J.A[2][c] = st ? (J.A[0][c] - bz * R[2][c]) : 0.0;
  }
  J.B[0][0] = x * y * iz2 * fx;
  J.B[0][1] = -(1 + (x * x * iz2)) * fx;
  J.B[0][2] = y * iz * fx;
  J.B[0][3] = -iz * fx;
  J.B[0][4] = 0;
  J.B[0][5] = x * iz2 * fx;
  J.B[1][0] = (1 + y * y * iz2) * fy;
  J.B[1][1] = -x * y * iz2 * fy;
  J.B[1][2] = -x * iz * fy;
  J.B[1][3] = 0;
  J.B[1][4] = -iz * fy;
  J.B[1][5] = y * iz2 * fy;
  J.B[2][0] = st ? (J.B[0][0] - bz * y) : 0.0;
  J.B[2][1] = st ? (J.B[0][1] + bz * x) : 0.0;
  J.B[2][2] = st ? J.B[0][2] : 0.0;
  J.B[2][3] = st ? J.B[0][3] : 0.0;
  J.B[2][4] = 0;
  J.B[2][5] = st ? (J.B[0][5] - bz) : 0.0;
}

}  // namespace b2s
