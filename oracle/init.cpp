// TEST INFRASTRUCTURE — CPU restatement of Initializer::Initialize (src/Initializer.cc), statement by statement, with
// the cv::Mat expressions it evaluates written out as OpenCV evaluates them (see init_oracle.h and DESIGN §7):
//   - storage is float (CV_32F); gemm without transposition and with an inner size of 2 to 4 that equals one of the
//     outer sizes (every product here but K.t()*F) sums float products in float, otherwise it accumulates in double;
//     either way alpha (s*U*Rp) and C (R*x + t) are applied in double before the one rounding to float; Mat::dot and
//     cv::norm accumulate in double;
//   - a scaled matrix (m * a, m / a, -m, m *= a) is Mat::convertTo: each element times (float)a, in float;
//   - a.row(i) = x*P.row(2) - P.row(0) is addWeighted: x*P2k - P0k in double, rounded once;
//   - SVD::compute / SVDecomp is JacobiSVDImpl_<float> (modules/core/src/lapack.cpp), including the completion of the
//     basis beyond the rank from RNG(0x12345678) that gives ComputeF21 its 9th row of vt;
//   - Mat::inv of a 3 x 3 matrix is invert's closed form with a double determinant; cv::determinant is the double det3.
// Compiled with -ffp-contract=off (oracle/Makefile), like the reference's float code on x86-64.
#include "init_oracle.h"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <utility>
#include <vector>

namespace {

struct Rng {  // cv::RNG
  uint64_t state;
  explicit Rng(uint64_t s) : state(s ? s : 0xffffffffu) {}
  unsigned next() {
    state = (uint64_t)(unsigned)state * 4164903690u + (unsigned)(state >> 32);
    return (unsigned)state;
  }
};

// JacobiSVDImpl_<float>(At, astep, W, Vt, vstep, m, n, n1, FLT_MIN, FLT_EPSILON*2): At holds n rows of length m (the
// columns of the decomposed matrix), afterwards the left singular vectors (n1 of them, the rows beyond the rank completed
// to an orthonormal basis); W the n singular values in descending order; Vt the n x n right singular vectors.
void jacobi_svd(float* At, int astep, float* Wout, float* Vt, int vstep, int m, int n, int n1) {
  const double minval = FLT_MIN;
  const float eps = FLT_EPSILON * 2;
  std::vector<double> W((size_t)n);
  const int max_iter = std::max(m, 30);
  for (int i = 0; i < n; i++) {
    double sd = 0;
    for (int k = 0; k < m; k++) {
      const float t = At[i * astep + k];
      sd += (double)t * t;
    }
    W[i] = sd;
    for (int k = 0; k < n; k++) Vt[i * vstep + k] = 0;
    Vt[i * vstep + i] = 1;
  }
  for (int iter = 0; iter < max_iter; iter++) {
    bool changed = false;
    for (int i = 0; i < n - 1; i++)
      for (int j = i + 1; j < n; j++) {
        float *Ai = At + i * astep, *Aj = At + j * astep;
        double a = W[i], p = 0, b = W[j];
        for (int k = 0; k < m; k++) p += (double)Ai[k] * Aj[k];
        if (std::abs(p) <= eps * std::sqrt((double)a * b)) continue;
        p *= 2;
        const double beta = a - b, gamma = std::hypot(p, beta);
        float c, s;
        if (beta < 0) {
          const double delta = (gamma - beta) * 0.5;
          s = (float)std::sqrt(delta / gamma);
          c = (float)(p / (gamma * s * 2));
        } else {
          c = (float)std::sqrt((gamma + beta) / (gamma * 2));
          s = (float)(p / (gamma * c * 2));
        }
        a = b = 0;
        for (int k = 0; k < m; k++) {
          const float t0 = c * Ai[k] + s * Aj[k];
          const float t1 = -s * Ai[k] + c * Aj[k];
          Ai[k] = t0;
          Aj[k] = t1;
          a += (double)t0 * t0;
          b += (double)t1 * t1;
        }
        W[i] = a;
        W[j] = b;
        changed = true;
        float *Vi = Vt + i * vstep, *Vj = Vt + j * vstep;
        for (int k = 0; k < n; k++) {
          const float t0 = c * Vi[k] + s * Vj[k];
          const float t1 = -s * Vi[k] + c * Vj[k];
          Vi[k] = t0;
          Vj[k] = t1;
        }
      }
    if (!changed) break;
  }
  for (int i = 0; i < n; i++) {
    double sd = 0;
    for (int k = 0; k < m; k++) {
      const float t = At[i * astep + k];
      sd += (double)t * t;
    }
    W[i] = std::sqrt(sd);
  }
  for (int i = 0; i < n - 1; i++) {
    int j = i;
    for (int k = i + 1; k < n; k++)
      if (W[j] < W[k]) j = k;
    if (i != j) {
      std::swap(W[i], W[j]);
      for (int k = 0; k < m; k++) std::swap(At[i * astep + k], At[j * astep + k]);
      for (int k = 0; k < n; k++) std::swap(Vt[i * vstep + k], Vt[j * vstep + k]);
    }
  }
  for (int i = 0; i < n; i++) Wout[i] = (float)W[i];
  Rng rng(0x12345678);
  for (int i = 0; i < n1; i++) {
    double sd = i < n ? W[i] : 0;
    for (int ii = 0; ii < 100 && sd <= minval; ii++) {
      const float val0 = (float)(1. / m);
      for (int k = 0; k < m; k++) At[i * astep + k] = (rng.next() & 256) != 0 ? val0 : -val0;
      for (int it2 = 0; it2 < 2; it2++)
        for (int j = 0; j < i; j++) {
          sd = 0;
          for (int k = 0; k < m; k++) sd += At[i * astep + k] * At[j * astep + k];
          float asum = 0;
          for (int k = 0; k < m; k++) {
            const float t = (float)(At[i * astep + k] - sd * At[j * astep + k]);
            At[i * astep + k] = t;
            asum += std::abs(t);
          }
          asum = asum > eps * 100 ? 1 / asum : 0;
          for (int k = 0; k < m; k++) At[i * astep + k] *= asum;
        }
      sd = 0;
      for (int k = 0; k < m; k++) {
        const float t = At[i * astep + k];
        sd += (double)t * t;
      }
      sd = std::sqrt(sd);
    }
    const float s = (float)(sd > minval ? 1 / sd : 0.);
    for (int k = 0; k < m; k++) At[i * astep + k] *= s;
  }
}

// 3 x 3 helpers (row-major)
void mul(const float* A, const float* B, int m, int k, int n, float* D, double alpha = 1.0, const float* C = nullptr) {
  orc_gemm(A, B, C, m, k, n, alpha, 0, D);
}
void scale(float* v, int n, double alpha) {  // Mat::convertTo(dst, -1, alpha)
  const float a = (float)alpha;
  for (int i = 0; i < n; i++) v[i] = v[i] * a;
}
double norm(const float* v, int n) {
  double s = 0;
  for (int i = 0; i < n; i++) s += (double)v[i] * v[i];
  return std::sqrt(s);
}
void eye3(float* T) {
  for (int i = 0; i < 9; i++) T[i] = (i % 4 == 0) ? 1.f : 0.f;
}

struct Init {
  const b2s_init_problem* p;
  std::vector<std::pair<int, int> > M;  // mvMatches12
  float sigma2;
  const float* kp1() const { return p->kp1; }
  const float* kp2() const { return p->kp2; }

  // Normalize (:1501-1575)
  static void normalize(const float* kp, int N, std::vector<float>& pn, float* T) {
    float meanX = 0, meanY = 0;
    pn.resize((size_t)N * 2);
    for (int i = 0; i < N; i++) {
      meanX += kp[2 * i];
      meanY += kp[2 * i + 1];
    }
    meanX = meanX / N;
    meanY = meanY / N;
    float meanDevX = 0, meanDevY = 0;
    for (int i = 0; i < N; i++) {
      pn[2 * i] = kp[2 * i] - meanX;
      pn[2 * i + 1] = kp[2 * i + 1] - meanY;
      meanDevX += std::fabs(pn[2 * i]);
      meanDevY += std::fabs(pn[2 * i + 1]);
    }
    meanDevX = meanDevX / N;
    meanDevY = meanDevY / N;
    const float sX = 1.0 / meanDevX;
    const float sY = 1.0 / meanDevY;
    for (int i = 0; i < N; i++) {
      pn[2 * i] = pn[2 * i] * sX;
      pn[2 * i + 1] = pn[2 * i + 1] * sY;
    }
    eye3(T);
    T[0] = sX;
    T[4] = sY;
    T[2] = -meanX * sX;
    T[5] = -meanY * sY;
  }

  // ComputeH21 (:419-522): vt.row(8) of the 16 x 9 system
  static void computeH21(const float* P1, const float* P2, float* H) {
    float A[16 * 9];
    for (int i = 0; i < 8; i++) {
      const float u1 = P1[2 * i], v1 = P1[2 * i + 1], u2 = P2[2 * i], v2 = P2[2 * i + 1];
      float* r0 = A + (2 * i) * 9;
      float* r1 = A + (2 * i + 1) * 9;
      r0[0] = 0; r0[1] = 0; r0[2] = 0; r0[3] = -u1; r0[4] = -v1; r0[5] = -1; r0[6] = v2 * u1; r0[7] = v2 * v1; r0[8] = v2;
      r1[0] = u1; r1[1] = v1; r1[2] = 1; r1[3] = 0; r1[4] = 0; r1[5] = 0; r1[6] = -u2 * u1; r1[7] = -u2 * v1; r1[8] = -u2;
    }
    float w[9], u[16 * 16], vt[81];
    orc_svd(A, 16, 9, 1, w, u, vt);
    std::memcpy(H, vt + 8 * 9, 9 * sizeof(float));
  }

  // ComputeF21 (:532-613)
  static void computeF21(const float* P1, const float* P2, float* F) {
    float A[8 * 9];
    for (int i = 0; i < 8; i++) {
      const float u1 = P1[2 * i], v1 = P1[2 * i + 1], u2 = P2[2 * i], v2 = P2[2 * i + 1];
      float* r = A + i * 9;
      r[0] = u2 * u1; r[1] = u2 * v1; r[2] = u2; r[3] = v2 * u1; r[4] = v2 * v1; r[5] = v2; r[6] = u1; r[7] = v1; r[8] = 1;
    }
    float w[9], u[64], vt[81];
    orc_svd(A, 8, 9, 1, w, u, vt);
    float Fpre[9];
    std::memcpy(Fpre, vt + 8 * 9, 9 * sizeof(float));
    float w3[3], u3[9], vt3[9];
    orc_svd(Fpre, 3, 3, 1, w3, u3, vt3);
    w3[2] = 0;
    float D[9] = {w3[0], 0, 0, 0, w3[1], 0, 0, 0, w3[2]}, UD[9];
    mul(u3, D, 3, 3, 3, UD);
    mul(UD, vt3, 3, 3, 3, F);
  }

  float checkHomography(const float* H21, const float* H12, std::vector<uint8_t>& in, float sigma) const {
    const int N = (int)M.size();
    float score = 0;
    const float th = 5.991;
    const float invSigmaSquare = 1.0 / (sigma * sigma);
    for (int i = 0; i < N; i++) {
      bool bIn = true;
      const float u1 = kp1()[2 * M[i].first], v1 = kp1()[2 * M[i].first + 1];
      const float u2 = kp2()[2 * M[i].second], v2 = kp2()[2 * M[i].second + 1];
      const float w2in1inv = 1.0 / (H12[6] * u2 + H12[7] * v2 + H12[8]);
      const float u2in1 = (H12[0] * u2 + H12[1] * v2 + H12[2]) * w2in1inv;
      const float v2in1 = (H12[3] * u2 + H12[4] * v2 + H12[5]) * w2in1inv;
      const float squareDist1 = (u1 - u2in1) * (u1 - u2in1) + (v1 - v2in1) * (v1 - v2in1);
      const float chiSquare1 = squareDist1 * invSigmaSquare;
      if (chiSquare1 > th)
        bIn = false;
      else
        score += th - chiSquare1;
      const float w1in2inv = 1.0 / (H21[6] * u1 + H21[7] * v1 + H21[8]);
      const float u1in2 = (H21[0] * u1 + H21[1] * v1 + H21[2]) * w1in2inv;
      const float v1in2 = (H21[3] * u1 + H21[4] * v1 + H21[5]) * w1in2inv;
      const float squareDist2 = (u2 - u1in2) * (u2 - u1in2) + (v2 - v1in2) * (v2 - v1in2);
      const float chiSquare2 = squareDist2 * invSigmaSquare;
      if (chiSquare2 > th)
        bIn = false;
      else
        score += th - chiSquare2;
      in[i] = bIn;
    }
    return score;
  }

  float checkFundamental(const float* F, std::vector<uint8_t>& in, float sigma) const {
    const int N = (int)M.size();
    float score = 0;
    const float th = 3.841;
    const float thScore = 5.991;
    const float invSigmaSquare = 1.0 / (sigma * sigma);
    for (int i = 0; i < N; i++) {
      bool bIn = true;
      const float u1 = kp1()[2 * M[i].first], v1 = kp1()[2 * M[i].first + 1];
      const float u2 = kp2()[2 * M[i].second], v2 = kp2()[2 * M[i].second + 1];
      const float a2 = F[0] * u1 + F[1] * v1 + F[2];
      const float b2 = F[3] * u1 + F[4] * v1 + F[5];
      const float c2 = F[6] * u1 + F[7] * v1 + F[8];
      const float num2 = a2 * u2 + b2 * v2 + c2;
      const float squareDist1 = num2 * num2 / (a2 * a2 + b2 * b2);
      const float chiSquare1 = squareDist1 * invSigmaSquare;
      if (chiSquare1 > th)
        bIn = false;
      else
        score += thScore - chiSquare1;
      const float a1 = F[0] * u2 + F[3] * v2 + F[6];
      const float b1 = F[1] * u2 + F[4] * v2 + F[7];
      const float c1 = F[2] * u2 + F[5] * v2 + F[8];
      const float num1 = a1 * u1 + b1 * v1 + c1;
      const float squareDist2 = num1 * num1 / (a1 * a1 + b1 * b1);
      const float chiSquare2 = squareDist2 * invSigmaSquare;
      if (chiSquare2 > th)
        bIn = false;
      else
        score += thScore - chiSquare2;
      in[i] = bIn;
    }
    return score;
  }

  // FindHomography (:234-331) / FindFundamental (:334-401); returns the best iteration or -1
  int find(bool homography, const std::vector<float>& pn1, const std::vector<float>& pn2, const float* T1,
           const float* T2, std::vector<uint8_t>& inl, float& score, float* best) const {
    const int N = (int)M.size();
    float T2x[9];
    if (homography)
      orc_inv3(T2, T2x);
    else
      for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) T2x[3 * r + c] = T2[3 * c + r];
    score = 0.0;
    inl.assign((size_t)N, 0);
    std::vector<uint8_t> cur((size_t)N, 0);
    int bestIt = -1;
    std::memset(best, 0, 9 * sizeof(float));
    for (int it = 0; it < p->iterations; it++) {
      float P1[16], P2[16];
      for (int j = 0; j < 8; j++) {
        const int idx = p->sets[8 * it + j];
        P1[2 * j] = pn1[2 * M[idx].first];
        P1[2 * j + 1] = pn1[2 * M[idx].first + 1];
        P2[2 * j] = pn2[2 * M[idx].second];
        P2[2 * j + 1] = pn2[2 * M[idx].second + 1];
      }
      float Xn[9], tmp[9], X[9], Xinv[9];
      if (homography)
        computeH21(P1, P2, Xn);
      else
        computeF21(P1, P2, Xn);
      mul(T2x, Xn, 3, 3, 3, tmp);
      mul(tmp, T1, 3, 3, 3, X);
      float currentScore;
      if (homography) {
        orc_inv3(X, Xinv);
        currentScore = checkHomography(X, Xinv, cur, p->sigma);
      } else {
        currentScore = checkFundamental(X, cur, p->sigma);
      }
      if (currentScore > score) {
        std::memcpy(best, X, 9 * sizeof(float));
        inl = cur;
        score = currentScore;
        bestIt = it;
      }
    }
    return bestIt;
  }

  // Triangulate (:1461-1498)
  static void triangulate(const float* k1, const float* k2, const float* P1, const float* P2, float* x3D) {
    float A[16];
    for (int c = 0; c < 4; c++) {
      A[c] = (float)((double)k1[0] * P1[8 + c] - P1[c]);
      A[4 + c] = (float)((double)k1[1] * P1[8 + c] - P1[4 + c]);
      A[8 + c] = (float)((double)k2[0] * P2[8 + c] - P2[c]);
      A[12 + c] = (float)((double)k2[1] * P2[8 + c] - P2[4 + c]);
    }
    float w[4], u[16], vt[16];
    orc_svd(A, 4, 4, 1, w, u, vt);
    std::memcpy(x3D, vt + 12, 3 * sizeof(float));
    scale(x3D, 3, 1. / vt[15]);
  }

  // CheckRT (:1578-1785)
  int checkRT(const float* R, const float* t, const std::vector<uint8_t>& inl, const float* K, std::vector<float>& p3d,
              float th2, std::vector<uint8_t>& good, float& parallax) const {
    const float fx = K[0], fy = K[4], cx = K[2], cy = K[5];
    good.assign((size_t)p->n1, 0);
    p3d.assign((size_t)p->n1 * 3, 0.f);
    std::vector<float> vCosParallax;
    float P1[12] = {0};
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 3; c++) P1[4 * r + c] = K[3 * r + c];
    float Rt[12], P2[12];
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) Rt[4 * r + c] = R[3 * r + c];
      Rt[4 * r + 3] = t[r];
    }
    mul(K, Rt, 3, 3, 4, P2);
    float O2[3];
    orc_gemm(R, t, nullptr, 3, 3, 1, -1.0, 1, O2);
    int nGood = 0;
    for (size_t i = 0; i < M.size(); i++) {
      if (!inl[i]) continue;
      const float* k1 = kp1() + 2 * M[i].first;
      const float* k2 = kp2() + 2 * M[i].second;
      float X[3];
      triangulate(k1, k2, P1, P2, X);
      if (!std::isfinite(X[0]) || !std::isfinite(X[1]) || !std::isfinite(X[2])) {
        good[M[i].first] = 0;
        continue;
      }
      const float n2[3] = {X[0] - O2[0], X[1] - O2[1], X[2] - O2[2]};
      const float dist1 = norm(X, 3);
      const float dist2 = norm(n2, 3);
      const double dot = (double)X[0] * n2[0] + (double)X[1] * n2[1] + (double)X[2] * n2[2];
      const float cosParallax = dot / (dist1 * dist2);
      if (X[2] <= 0 && cosParallax < 0.99998) continue;
      float X2[3];
      mul(R, X, 3, 3, 1, X2, 1.0, t);
      if (X2[2] <= 0 && cosParallax < 0.99998) continue;
      const float invZ1 = 1.0 / X[2];
      const float im1x = fx * X[0] * invZ1 + cx;
      const float im1y = fy * X[1] * invZ1 + cy;
      const float squareError1 = (im1x - k1[0]) * (im1x - k1[0]) + (im1y - k1[1]) * (im1y - k1[1]);
      if (squareError1 > th2) continue;
      const float invZ2 = 1.0 / X2[2];
      const float im2x = fx * X2[0] * invZ2 + cx;
      const float im2y = fy * X2[1] * invZ2 + cy;
      const float squareError2 = (im2x - k2[0]) * (im2x - k2[0]) + (im2y - k2[1]) * (im2y - k2[1]);
      if (squareError2 > th2) continue;
      vCosParallax.push_back(cosParallax);
      for (int k = 0; k < 3; k++) p3d[3 * M[i].first + k] = X[k];
      nGood++;
      if (cosParallax < 0.99998) good[M[i].first] = 1;
    }
    if (nGood > 0) {
      std::sort(vCosParallax.begin(), vCosParallax.end());
      const size_t idx = std::min(50, int(vCosParallax.size() - 1));
      parallax = std::acos(vCosParallax[idx]) * 180 / 3.1415926535897932384626433832795;
    } else {
      parallax = 0;
    }
    return nGood;
  }

  void take(b2s_init_result* r, const std::vector<float>& p3d, const std::vector<uint8_t>& tri) const {
    std::memcpy(r->p3d, p3d.data(), p3d.size() * sizeof(float));
    std::memcpy(r->triangulated, tri.data(), tri.size());
  }

  // ReconstructH (:1135-1433)
  bool reconstructH(const std::vector<uint8_t>& inl, const float* H21, const float* K, b2s_init_result* r) const {
    int N = 0;
    for (uint8_t b : inl) N += b ? 1 : 0;
    float invK[9], tmp[9], A[9];
    orc_inv3(K, invK);
    mul(invK, H21, 3, 3, 3, tmp);
    mul(tmp, K, 3, 3, 3, A);
    float w[3], U[9], Vt[9];
    orc_svd(A, 3, 3, 1, w, U, Vt);
    const float s = orc_det3(U) * orc_det3(Vt);
    const float d1 = w[0], d2 = w[1], d3 = w[2];
    r->n_hyp = 0;
    if (d1 / d2 < 1.00001 || d2 / d3 < 1.00001) return false;
    float vR[8][9], vt[8][3];
    const float aux1 = std::sqrt((d1 * d1 - d2 * d2) / (d1 * d1 - d3 * d3));
    const float aux3 = std::sqrt((d2 * d2 - d3 * d3) / (d1 * d1 - d3 * d3));
    const float x1[] = {aux1, aux1, -aux1, -aux1};
    const float x3[] = {aux3, -aux3, aux3, -aux3};
    const float aux_stheta = std::sqrt((d1 * d1 - d2 * d2) * (d2 * d2 - d3 * d3)) / ((d1 + d3) * d2);
    const float ctheta = (d2 * d2 + d1 * d3) / ((d1 + d3) * d2);
    const float stheta[] = {aux_stheta, -aux_stheta, -aux_stheta, aux_stheta};
    for (int i = 0; i < 4; i++) {
      float Rp[9];
      eye3(Rp);
      Rp[0] = ctheta;
      Rp[2] = -stheta[i];
      Rp[6] = stheta[i];
      Rp[8] = ctheta;
      float URp[9];
      mul(U, Rp, 3, 3, 3, URp, (double)s);
      mul(URp, Vt, 3, 3, 3, vR[i]);
      float tp[3] = {x1[i], 0, -x3[i]};
      scale(tp, 3, d1 - d3);
      float t[3];
      mul(U, tp, 3, 3, 1, t);
      scale(t, 3, 1. / norm(t, 3));
      std::memcpy(vt[i], t, sizeof(t));
    }
    const float aux_sphi = std::sqrt((d1 * d1 - d2 * d2) * (d2 * d2 - d3 * d3)) / ((d1 - d3) * d2);
    const float cphi = (d1 * d3 - d2 * d2) / ((d1 - d3) * d2);
    const float sphi[] = {aux_sphi, -aux_sphi, -aux_sphi, aux_sphi};
    for (int i = 0; i < 4; i++) {
      float Rp[9];
      eye3(Rp);
      Rp[0] = cphi;
      Rp[2] = sphi[i];
      Rp[4] = -1;
      Rp[6] = sphi[i];
      Rp[8] = -cphi;
      float URp[9];
      mul(U, Rp, 3, 3, 3, URp, (double)s);
      mul(URp, Vt, 3, 3, 3, vR[4 + i]);
      float tp[3] = {x1[i], 0, x3[i]};
      scale(tp, 3, d1 + d3);
      float t[3];
      mul(U, tp, 3, 3, 1, t);
      scale(t, 3, 1. / norm(t, 3));
      std::memcpy(vt[4 + i], t, sizeof(t));
    }
    int bestGood = 0, secondBestGood = 0, bestSolutionIdx = -1;
    float bestParallax = -1;
    std::vector<float> bestP3D;
    std::vector<uint8_t> bestTriangulated;
    r->n_hyp = 8;
    for (int i = 0; i < 8; i++) {
      float parallaxi;
      std::vector<float> vP3Di;
      std::vector<uint8_t> vbTriangulatedi;
      const int nGood = checkRT(vR[i], vt[i], inl, K, vP3Di, 4.0 * sigma2, vbTriangulatedi, parallaxi);
      r->n_good[i] = nGood;
      r->parallax[i] = parallaxi;
      if (nGood > bestGood) {
        secondBestGood = bestGood;
        bestGood = nGood;
        bestSolutionIdx = i;
        bestParallax = parallaxi;
        bestP3D = vP3Di;
        bestTriangulated = vbTriangulatedi;
      } else if (nGood > secondBestGood) {
        secondBestGood = nGood;
      }
    }
    const float minParallax = 1.0;
    const int minTriangulated = 50;
    if (secondBestGood < 0.75 * bestGood && bestParallax >= minParallax && bestGood > minTriangulated &&
        bestGood > 0.9 * N) {
      std::memcpy(r->R21, vR[bestSolutionIdx], sizeof(r->R21));
      std::memcpy(r->t21, vt[bestSolutionIdx], sizeof(r->t21));
      r->rt_state = 1;
      take(r, bestP3D, bestTriangulated);
      return true;
    }
    return false;
  }

  // ReconstructF (:956-1127) with DecomposeE (:1798-1843)
  bool reconstructF(const std::vector<uint8_t>& inl, const float* F21, const float* K, b2s_init_result* r) const {
    int N = 0;
    for (uint8_t b : inl) N += b ? 1 : 0;
    float KtF[9], E[9];
    orc_gemm(K, F21, nullptr, 3, 3, 3, 1.0, 1, KtF);
    mul(KtF, K, 3, 3, 3, E);
    float w[3], u[9], vt[9];
    orc_svd(E, 3, 3, 0, w, u, vt);
    float t[3] = {u[2], u[5], u[8]};
    scale(t, 3, 1. / norm(t, 3));
    const float W[9] = {0, -1, 0, 1, 0, 0, 0, 0, 1};
    const float Wt[9] = {0, 1, 0, -1, 0, 0, 0, 0, 1};
    float uW[9], R1[9], R2[9];
    mul(u, W, 3, 3, 3, uW);
    mul(uW, vt, 3, 3, 3, R1);
    if (orc_det3(R1) < 0) scale(R1, 9, -1.0);
    mul(u, Wt, 3, 3, 3, uW);
    mul(uW, vt, 3, 3, 3, R2);
    if (orc_det3(R2) < 0) scale(R2, 9, -1.0);
    float t1[3], t2[3];
    std::memcpy(t1, t, sizeof(t));
    std::memcpy(t2, t, sizeof(t));
    scale(t2, 3, -1.0);
    const float* Rs[4] = {R1, R2, R1, R2};
    const float* ts[4] = {t1, t1, t2, t2};
    std::vector<float> vP3D[4];
    std::vector<uint8_t> vbTri[4];
    int nGood[4];
    float parallax[4];
    r->n_hyp = 4;
    for (int i = 0; i < 4; i++) {
      nGood[i] = checkRT(Rs[i], ts[i], inl, K, vP3D[i], 4.0 * sigma2, vbTri[i], parallax[i]);
      r->n_good[i] = nGood[i];
      r->parallax[i] = parallax[i];
    }
    const int maxGood = std::max(nGood[0], std::max(nGood[1], std::max(nGood[2], nGood[3])));
    r->rt_state = -1;  // R21 = cv::Mat(); t21 = cv::Mat();
    const float minParallax = 1.0;
    const int minTriangulated = 50;
    const int nMinGood = std::max(static_cast<int>(0.9 * N), minTriangulated);
    int nsimilar = 0;
    for (int i = 0; i < 4; i++)
      if (nGood[i] > 0.7 * maxGood) nsimilar++;
    if (maxGood < nMinGood || nsimilar > 1) return false;
    for (int i = 0; i < 4; i++)
      if (maxGood == nGood[i]) {
        if (parallax[i] > minParallax) {
          take(r, vP3D[i], vbTri[i]);
          std::memcpy(r->R21, Rs[i], sizeof(r->R21));
          std::memcpy(r->t21, ts[i], sizeof(r->t21));
          r->rt_state = 1;
          return true;
        }
        break;  // the if / else if chain stops at the first hypothesis with maxGood
      }
    return false;
  }
};

}  // namespace

extern "C" {

void orc_svd(const float* A, int rows, int cols, int full_uv, float* w, float* u, float* vt) {
  int m = rows, n = cols;
  const bool at = m < n;
  if (at) std::swap(m, n);
  const int urows = full_uv ? m : n;
  std::vector<float> tu((size_t)urows * m, 0.f), tv((size_t)n * n);
  for (int i = 0; i < n; i++)
    for (int k = 0; k < m; k++) tu[(size_t)i * m + k] = at ? A[i * cols + k] : A[k * cols + i];
  jacobi_svd(tu.data(), m, w, tv.data(), n, m, n, urows);
  if (!at) {
    for (int k = 0; k < m; k++)
      for (int i = 0; i < urows; i++) u[k * urows + i] = tu[(size_t)i * m + k];
    std::memcpy(vt, tv.data(), tv.size() * sizeof(float));
  } else {
    for (int k = 0; k < n; k++)
      for (int i = 0; i < n; i++) u[k * n + i] = tv[(size_t)i * n + k];
    std::memcpy(vt, tu.data(), tu.size() * sizeof(float));
  }
}

double orc_det3(const float* m) {
#define M3(r, c) m[3 * (r) + (c)]
  return M3(0, 0) * ((double)M3(1, 1) * M3(2, 2) - (double)M3(1, 2) * M3(2, 1)) -
         M3(0, 1) * ((double)M3(1, 0) * M3(2, 2) - (double)M3(1, 2) * M3(2, 0)) +
         M3(0, 2) * ((double)M3(1, 0) * M3(2, 1) - (double)M3(1, 1) * M3(2, 0));
}

int orc_inv3(const float* m, float* o) {
  double d = orc_det3(m);
  if (d == 0.) {
    for (int i = 0; i < 9; i++) o[i] = 0.f;
    return 0;
  }
  d = 1. / d;
  double t[9];
  t[0] = ((double)M3(1, 1) * M3(2, 2) - (double)M3(1, 2) * M3(2, 1)) * d;
  t[1] = ((double)M3(0, 2) * M3(2, 1) - (double)M3(0, 1) * M3(2, 2)) * d;
  t[2] = ((double)M3(0, 1) * M3(1, 2) - (double)M3(0, 2) * M3(1, 1)) * d;
  t[3] = ((double)M3(1, 2) * M3(2, 0) - (double)M3(1, 0) * M3(2, 2)) * d;
  t[4] = ((double)M3(0, 0) * M3(2, 2) - (double)M3(0, 2) * M3(2, 0)) * d;
  t[5] = ((double)M3(0, 2) * M3(1, 0) - (double)M3(0, 0) * M3(1, 2)) * d;
  t[6] = ((double)M3(1, 0) * M3(2, 1) - (double)M3(1, 1) * M3(2, 0)) * d;
  t[7] = ((double)M3(0, 1) * M3(2, 0) - (double)M3(0, 0) * M3(2, 1)) * d;
  t[8] = ((double)M3(0, 0) * M3(1, 1) - (double)M3(0, 1) * M3(1, 0)) * d;
#undef M3
  for (int i = 0; i < 9; i++) o[i] = (float)t[i];
  return 1;
}

void orc_gemm(const float* A, const float* B, const float* C, int m, int k, int n, double alpha, int tA, float* D) {
  const bool small = !tA && k >= 2 && k <= 4 && (k == n || k == m);
  for (int r = 0; r < m; r++)
    for (int c = 0; c < n; c++) {
      double s = 0;
      if (small) {  // gemm's path for 2 <= k <= 4: float products summed in float, in k order
        float f = 0;
        for (int q = 0; q < k; q++) f = f + A[r * k + q] * B[q * n + c];
        s = f;
      } else {
        for (int q = 0; q < k; q++) s += (double)(tA ? A[q * m + r] : A[r * k + q]) * B[q * n + c];
      }
      double v = s * alpha;
      if (C) v += (double)C[r * n + c];
      D[r * n + c] = (float)v;
    }
}

static void compact(Init& I, const b2s_init_problem* p) {
  I.p = p;
  I.sigma2 = p->sigma * p->sigma;
  for (int i = 0; i < p->n1; i++)
    if (p->matches12[i] >= 0) I.M.push_back(std::make_pair(i, p->matches12[i]));
}

int orc_find(const b2s_init_problem* p, int homography, float* score, float* X, uint8_t* inl) {
  Init I;
  compact(I, p);
  std::vector<float> pn1, pn2;
  float T1[9], T2[9];
  Init::normalize(p->kp1, p->n1, pn1, T1);
  Init::normalize(p->kp2, p->n2, pn2, T2);
  std::vector<uint8_t> v;
  const int best = I.find(homography != 0, pn1, pn2, T1, T2, v, *score, X);
  std::memcpy(inl, v.data(), v.size());
  return best;
}

int orc_reconstruct(const b2s_init_problem* p, int homography, const uint8_t* inl, const float* X, b2s_init_result* r) {
  Init I;
  compact(I, p);
  const std::vector<uint8_t> v(inl, inl + I.M.size());
  r->rt_state = 0;
  r->n_hyp = 0;
  for (int i = 0; i < 8; i++) {
    r->n_good[i] = 0;
    r->parallax[i] = 0.f;
  }
  r->ret = homography ? I.reconstructH(v, X, p->K, r) : I.reconstructF(v, X, p->K, r);
  return r->ret;
}

int orc_initialize(const b2s_init_problem* p, b2s_init_result* r) {
  Init I;
  compact(I, p);
  const int N = (int)I.M.size();
  r->n_matches = N;
  r->ret = 0;
  r->rt_state = 0;
  r->n_hyp = 0;
  for (int i = 0; i < 8; i++) {
    r->n_good[i] = 0;
    r->parallax[i] = 0.f;
  }
  std::vector<float> pn1, pn2;
  float T1[9], T2[9];
  Init::normalize(p->kp1, p->n1, pn1, T1);
  Init::normalize(p->kp2, p->n2, pn2, T2);
  std::vector<uint8_t> inlH, inlF;
  float SH, SF;
  r->best_h_iter = I.find(true, pn1, pn2, T1, T2, inlH, SH, r->H21);
  r->best_f_iter = I.find(false, pn1, pn2, T1, T2, inlF, SF, r->F21);
  if (r->inliers_h) std::memcpy(r->inliers_h, inlH.data(), (size_t)N);
  if (r->inliers_f) std::memcpy(r->inliers_f, inlF.data(), (size_t)N);
  const float RH = SH / (SH + SF);
  r->SH = SH;
  r->SF = SF;
  r->RH = RH;
  if (RH > 0.40) {
    r->model = 1;
    r->ret = I.reconstructH(inlH, r->H21, p->K, r);
  } else {
    r->model = 2;
    if (r->best_f_iter >= 0) r->ret = I.reconstructF(inlF, r->F21, p->K, r);
  }
  return 0;
}

}  // extern "C"
