// TEST INFRASTRUCTURE — CPU restatement of PnPsolver (src/PnPsolver.cc), statement by statement, with the minimal sets as
// input and the OpenCV C API calls written out as OpenCV 4 evaluates them on CV_64F data (see pnpsolver_oracle.h and
// DESIGN §7):
//   - cvMulTransposed(A, D, 1) is MulTransposedR: D[i][j] = sum over rows k of A[k][i]*A[k][j], one double accumulator
//     per entry from 0 in row order, the upper triangle mirrored;
//   - cvSVD is SVD::compute: JacobiSVDImpl_<double> (DBL_MIN, DBL_EPSILON*10, lapack.cpp's hypot template, the basis
//     beyond the rank completed from RNG(0x12345678)); CV_SVD_U_T leaves U transposed, and without CV_SVD_V_T the V
//     argument receives V;
//   - cvInvert / cvSolve with CV_SVD are SVBkSb: singular values at most DBL_EPSILON*2 * sum(w) are skipped, the rest
//     accumulated in order of decreasing singular value;
//   - qr_solve returns with X unwritten where a column's eta is 0; gauss_newton's x is then the previous step's
//     increment, and 0 at the first step (the reference reads uninitialised memory there).
// Compiled with -ffp-contract=off (oracle/Makefile), like the reference's double code on x86-64.
#include "pnpsolver_oracle.h"

#include <algorithm>
#include <cfloat>
#include <climits>
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

double cv_hypot(double a, double b) {  // lapack.cpp's hypot template
  a = std::abs(a);
  b = std::abs(b);
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

// JacobiSVDImpl_<double>(At, astep, W, Vt, vstep, m, n, n1, DBL_MIN, DBL_EPSILON*10)
void jacobi_svd(double* At, int astep, double* Wout, double* Vt, int vstep, int m, int n, int n1) {
  const double minval = DBL_MIN;
  const double eps = DBL_EPSILON * 10;
  std::vector<double> W((size_t)n);
  const int max_iter = std::max(m, 30);
  for (int i = 0; i < n; i++) {
    double sd = 0;
    for (int k = 0; k < m; k++) {
      const double t = At[i * astep + k];
      sd += t * t;
    }
    W[i] = sd;
    for (int k = 0; k < n; k++) Vt[i * vstep + k] = 0;
    Vt[i * vstep + i] = 1;
  }
  for (int iter = 0; iter < max_iter; iter++) {
    bool changed = false;
    for (int i = 0; i < n - 1; i++)
      for (int j = i + 1; j < n; j++) {
        double *Ai = At + i * astep, *Aj = At + j * astep;
        double a = W[i], p = 0, b = W[j];
        for (int k = 0; k < m; k++) p += Ai[k] * Aj[k];
        if (std::abs(p) <= eps * std::sqrt(a * b)) continue;
        p *= 2;
        const double beta = a - b, gamma = cv_hypot(p, beta);
        double c, s;
        if (beta < 0) {
          const double delta = (gamma - beta) * 0.5;
          s = std::sqrt(delta / gamma);
          c = p / (gamma * s * 2);
        } else {
          c = std::sqrt((gamma + beta) / (gamma * 2));
          s = p / (gamma * c * 2);
        }
        a = b = 0;
        for (int k = 0; k < m; k++) {
          const double t0 = c * Ai[k] + s * Aj[k];
          const double t1 = -s * Ai[k] + c * Aj[k];
          Ai[k] = t0;
          Aj[k] = t1;
          a += t0 * t0;
          b += t1 * t1;
        }
        W[i] = a;
        W[j] = b;
        changed = true;
        double *Vi = Vt + i * vstep, *Vj = Vt + j * vstep;
        for (int k = 0; k < n; k++) {
          const double t0 = c * Vi[k] + s * Vj[k];
          const double t1 = -s * Vi[k] + c * Vj[k];
          Vi[k] = t0;
          Vj[k] = t1;
        }
      }
    if (!changed) break;
  }
  for (int i = 0; i < n; i++) {
    double sd = 0;
    for (int k = 0; k < m; k++) {
      const double t = At[i * astep + k];
      sd += t * t;
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
  for (int i = 0; i < n; i++) Wout[i] = W[i];
  Rng rng(0x12345678);
  for (int i = 0; i < n1; i++) {
    double sd = i < n ? W[i] : 0;
    for (int ii = 0; ii < 100 && sd <= minval; ii++) {
      const double val0 = 1. / m;
      for (int k = 0; k < m; k++) At[i * astep + k] = (rng.next() & 256) != 0 ? val0 : -val0;
      for (int it2 = 0; it2 < 2; it2++)
        for (int j = 0; j < i; j++) {
          sd = 0;
          for (int k = 0; k < m; k++) sd += At[i * astep + k] * At[j * astep + k];
          double asum = 0;
          for (int k = 0; k < m; k++) {
            const double t = At[i * astep + k] - sd * At[j * astep + k];
            At[i * astep + k] = t;
            asum += std::abs(t);
          }
          asum = asum > eps * 100 ? 1 / asum : 0;
          for (int k = 0; k < m; k++) At[i * astep + k] *= asum;
        }
      sd = 0;
      for (int k = 0; k < m; k++) {
        const double t = At[i * astep + k];
        sd += t * t;
      }
      sd = std::sqrt(sd);
    }
    const double s = sd > minval ? 1 / sd : 0.;
    for (int k = 0; k < m; k++) At[i * astep + k] *= s;
  }
}

// SVD::compute of a square n x n matrix: At = rows of U^T (the transposed input, rotated), W, Vt
void svd_at(const double* A, int n, double* At, double* w, double* Vt) {
  for (int i = 0; i < n; i++)
    for (int k = 0; k < n; k++) At[i * n + k] = A[k * n + i];
  jacobi_svd(At, n, w, Vt, n, n, n, n);
}

// MulTransposedR without delta, scale 1
void mul_transposed(const double* A, int rows, int cols, double* D) {
  for (int i = 0; i < cols; i++)
    for (int j = i; j < cols; j++) {
      double s = 0;
      for (int k = 0; k < rows; k++) s += A[k * cols + i] * A[k * cols + j];
      D[i * cols + j] = D[j * cols + i] = s;
    }
}

// cv::invert(DECOMP_SVD): SVD::compute, then SVBkSbImpl_ with b = null (u not transposed, one column per output)
void invert_svd(const double* A, int n, double* D) {
  double At[144], w[12], Vt[144];
  svd_at(A, n, At, w, Vt);
  double threshold = 0;
  for (int i = 0; i < n; i++) threshold += w[i];
  threshold *= DBL_EPSILON * 2;
  for (int i = 0; i < n * n; i++) D[i] = 0;
  for (int i = 0; i < n; i++) {
    double wi = w[i];
    if (std::abs(wi) <= threshold) continue;
    wi = 1 / wi;
    double buf[12];
    for (int j = 0; j < n; j++) buf[j] = At[i * n + j] * wi;  // u[j][i] * wi
    for (int r = 0; r < n; r++) {
      const double s = Vt[i * n + r];
      for (int j = 0; j < n; j++) D[r * n + j] = D[r * n + j] + s * buf[j];
    }
  }
}

// cv::solve(DECOMP_SVD): JacobiSVD of A^T, then SVBkSbImpl_ with u transposed and one right-hand side
void solve_svd(const double* A, int rows, int cols, const double* b, double* x) {
  const int m = rows, n = cols;
  std::vector<double> At((size_t)n * m);
  double w[12], Vt[144];
  for (int i = 0; i < n; i++)
    for (int k = 0; k < m; k++) At[(size_t)i * m + k] = A[k * n + i];
  jacobi_svd(At.data(), m, w, Vt, n, m, n, n);
  double threshold = 0;
  for (int i = 0; i < n; i++) threshold += w[i];
  threshold *= DBL_EPSILON * 2;
  for (int j = 0; j < n; j++) x[j] = 0;
  for (int i = 0; i < n; i++) {
    double wi = w[i];
    if (std::abs(wi) <= threshold) continue;
    wi = 1 / wi;
    double s = 0;
    for (int j = 0; j < m; j++) s += At[(size_t)i * m + j] * b[j];
    s *= wi;
    for (int j = 0; j < n; j++) x[j] = x[j] + s * Vt[i * n + j];
  }
}

// The EPnP part of PnPsolver (:466-1385): the members it reads and writes, the same names and statements
struct Epnp {
  double uc, vc, fu, fv;
  int number_of_correspondences = 0;
  std::vector<double> pws, us, alphas, pcs;
  double cws[4][3], ccs[4][3];

  Epnp(const float* cam, int m) : uc(cam[2]), vc(cam[3]), fu(cam[0]), fv(cam[1]) {
    pws.resize(3 * (size_t)m);
    us.resize(2 * (size_t)m);
    alphas.resize(4 * (size_t)m);
    pcs.resize(3 * (size_t)m);
  }
  void add_correspondence(double X, double Y, double Z, double u, double v) {
    pws[3 * number_of_correspondences] = X;
    pws[3 * number_of_correspondences + 1] = Y;
    pws[3 * number_of_correspondences + 2] = Z;
    us[2 * number_of_correspondences] = u;
    us[2 * number_of_correspondences + 1] = v;
    number_of_correspondences++;
  }
  void choose_control_points() {
    cws[0][0] = cws[0][1] = cws[0][2] = 0;
    for (int i = 0; i < number_of_correspondences; i++)
      for (int j = 0; j < 3; j++) cws[0][j] += pws[3 * i + j];
    for (int j = 0; j < 3; j++) cws[0][j] /= number_of_correspondences;
    std::vector<double> PW0(3 * (size_t)number_of_correspondences);
    double pw0tpw0[9], dc[3], uct[9], vt[9];
    for (int i = 0; i < number_of_correspondences; i++)
      for (int j = 0; j < 3; j++) PW0[3 * i + j] = pws[3 * i + j] - cws[0][j];
    mul_transposed(PW0.data(), number_of_correspondences, 3, pw0tpw0);
    svd_at(pw0tpw0, 3, uct, dc, vt);  // cvSVD(.., CV_SVD_MODIFY_A | CV_SVD_U_T): UCt = the rows of At
    for (int i = 1; i < 4; i++) {
      const double k = std::sqrt(dc[i - 1] / number_of_correspondences);
      for (int j = 0; j < 3; j++) cws[i][j] = cws[0][j] + k * uct[3 * (i - 1) + j];
    }
  }
  void compute_barycentric_coordinates() {
    double cc[9], cc_inv[9];
    for (int i = 0; i < 3; i++)
      for (int j = 1; j < 4; j++) cc[3 * i + j - 1] = cws[j][i] - cws[0][i];
    invert_svd(cc, 3, cc_inv);
    const double* ci = cc_inv;
    for (int i = 0; i < number_of_correspondences; i++) {
      const double* pi = &pws[3 * i];
      double* a = &alphas[4 * i];
      for (int j = 0; j < 3; j++)
        a[1 + j] = ci[3 * j] * (pi[0] - cws[0][0]) + ci[3 * j + 1] * (pi[1] - cws[0][1]) +
                   ci[3 * j + 2] * (pi[2] - cws[0][2]);
      a[0] = 1.0f - a[1] - a[2] - a[3];
    }
  }
  void fill_M(double* M, int row, const double* as, double u, double v) {
    double* M1 = M + row * 12;
    double* M2 = M1 + 12;
    for (int i = 0; i < 4; i++) {
      M1[3 * i] = as[i] * fu;
      M1[3 * i + 1] = 0.0;
      M1[3 * i + 2] = as[i] * (uc - u);
      M2[3 * i] = 0.0;
      M2[3 * i + 1] = as[i] * fv;
      M2[3 * i + 2] = as[i] * (vc - v);
    }
  }
  void compute_ccs(const double* betas, const double* ut) {
    for (int i = 0; i < 4; i++) ccs[i][0] = ccs[i][1] = ccs[i][2] = 0.0f;
    for (int i = 0; i < 4; i++) {
      const double* v = ut + 12 * (11 - i);
      for (int j = 0; j < 4; j++)
        for (int k = 0; k < 3; k++) ccs[j][k] += betas[i] * v[3 * j + k];
    }
  }
  void compute_pcs() {
    for (int i = 0; i < number_of_correspondences; i++) {
      const double* a = &alphas[4 * i];
      double* pc = &pcs[3 * i];
      for (int j = 0; j < 3; j++) pc[j] = a[0] * ccs[0][j] + a[1] * ccs[1][j] + a[2] * ccs[2][j] + a[3] * ccs[3][j];
    }
  }
  static double dist2(const double* p1, const double* p2) {
    return (p1[0] - p2[0]) * (p1[0] - p2[0]) + (p1[1] - p2[1]) * (p1[1] - p2[1]) + (p1[2] - p2[2]) * (p1[2] - p2[2]);
  }
  static double dot(const double* v1, const double* v2) { return v1[0] * v2[0] + v1[1] * v2[1] + v1[2] * v2[2]; }
  double reprojection_error(const double R[3][3], const double t[3]) {
    double sum2 = 0.0;
    for (int i = 0; i < number_of_correspondences; i++) {
      const double* pw = &pws[3 * i];
      const double Xc = dot(R[0], pw) + t[0];
      const double Yc = dot(R[1], pw) + t[1];
      const double inv_Zc = 1.0 / (dot(R[2], pw) + t[2]);
      const double ue = uc + fu * Xc * inv_Zc;
      const double ve = vc + fv * Yc * inv_Zc;
      const double u = us[2 * i], v = us[2 * i + 1];
      sum2 += std::sqrt((u - ue) * (u - ue) + (v - ve) * (v - ve));
    }
    return sum2 / number_of_correspondences;
  }
  void estimate_R_and_t(double R[3][3], double t[3]) {
    double pc0[3], pw0[3];
    pc0[0] = pc0[1] = pc0[2] = 0.0;
    pw0[0] = pw0[1] = pw0[2] = 0.0;
    for (int i = 0; i < number_of_correspondences; i++) {
      const double* pc = &pcs[3 * i];
      const double* pw = &pws[3 * i];
      for (int j = 0; j < 3; j++) {
        pc0[j] += pc[j];
        pw0[j] += pw[j];
      }
    }
    for (int j = 0; j < 3; j++) {
      pc0[j] /= number_of_correspondences;
      pw0[j] /= number_of_correspondences;
    }
    double abt[9], abt_d[3], abt_u[9], abt_v[9], At[9], Vt[9];
    for (int i = 0; i < 9; i++) abt[i] = 0;
    for (int i = 0; i < number_of_correspondences; i++) {
      const double* pc = &pcs[3 * i];
      const double* pw = &pws[3 * i];
      for (int j = 0; j < 3; j++) {
        abt[3 * j] += (pc[j] - pc0[j]) * (pw[0] - pw0[0]);
        abt[3 * j + 1] += (pc[j] - pc0[j]) * (pw[1] - pw0[1]);
        abt[3 * j + 2] += (pc[j] - pc0[j]) * (pw[2] - pw0[2]);
      }
    }
    svd_at(abt, 3, At, abt_d, Vt);  // cvSVD(ABt, D, U, V, CV_SVD_MODIFY_A): U = At^T, V = Vt^T
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) {
        abt_u[3 * i + j] = At[3 * j + i];
        abt_v[3 * i + j] = Vt[3 * j + i];
      }
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) R[i][j] = dot(abt_u + 3 * i, abt_v + 3 * j);
    const double det = R[0][0] * R[1][1] * R[2][2] + R[0][1] * R[1][2] * R[2][0] + R[0][2] * R[1][0] * R[2][1] -
                       R[0][2] * R[1][1] * R[2][0] - R[0][1] * R[1][0] * R[2][2] - R[0][0] * R[1][2] * R[2][1];
    if (det < 0) {
      R[2][0] = -R[2][0];
      R[2][1] = -R[2][1];
      R[2][2] = -R[2][2];
    }
    t[0] = pc0[0] - dot(R[0], pw0);
    t[1] = pc0[1] - dot(R[1], pw0);
    t[2] = pc0[2] - dot(R[2], pw0);
  }
  void solve_for_sign() {
    if (pcs[2] < 0.0) {
      for (int i = 0; i < 4; i++)
        for (int j = 0; j < 3; j++) ccs[i][j] = -ccs[i][j];
      for (int i = 0; i < number_of_correspondences; i++) {
        pcs[3 * i] = -pcs[3 * i];
        pcs[3 * i + 1] = -pcs[3 * i + 1];
        pcs[3 * i + 2] = -pcs[3 * i + 2];
      }
    }
  }
  double compute_R_and_t(const double* ut, const double* betas, double R[3][3], double t[3]) {
    compute_ccs(betas, ut);
    compute_pcs();
    solve_for_sign();
    estimate_R_and_t(R, t);
    return reprojection_error(R, t);
  }
  static void find_betas_approx_1(const double* L_6x10, const double* Rho, double* betas) {
    double l_6x4[6 * 4], b4[4];
    for (int i = 0; i < 6; i++) {
      l_6x4[4 * i] = L_6x10[10 * i];
      l_6x4[4 * i + 1] = L_6x10[10 * i + 1];
      l_6x4[4 * i + 2] = L_6x10[10 * i + 3];
      l_6x4[4 * i + 3] = L_6x10[10 * i + 6];
    }
    solve_svd(l_6x4, 6, 4, Rho, b4);
    if (b4[0] < 0) {
      betas[0] = std::sqrt(-b4[0]);
      betas[1] = -b4[1] / betas[0];
      betas[2] = -b4[2] / betas[0];
      betas[3] = -b4[3] / betas[0];
    } else {
      betas[0] = std::sqrt(b4[0]);
      betas[1] = b4[1] / betas[0];
      betas[2] = b4[2] / betas[0];
      betas[3] = b4[3] / betas[0];
    }
  }
  static void find_betas_approx_2(const double* L_6x10, const double* Rho, double* betas) {
    double l_6x3[6 * 3], b3[3];
    for (int i = 0; i < 6; i++)
      for (int j = 0; j < 3; j++) l_6x3[3 * i + j] = L_6x10[10 * i + j];
    solve_svd(l_6x3, 6, 3, Rho, b3);
    if (b3[0] < 0) {
      betas[0] = std::sqrt(-b3[0]);
      betas[1] = (b3[2] < 0) ? std::sqrt(-b3[2]) : 0.0;
    } else {
      betas[0] = std::sqrt(b3[0]);
      betas[1] = (b3[2] > 0) ? std::sqrt(b3[2]) : 0.0;
    }
    if (b3[1] < 0) betas[0] = -betas[0];
    betas[2] = 0.0;
    betas[3] = 0.0;
  }
  static void find_betas_approx_3(const double* L_6x10, const double* Rho, double* betas) {
    double l_6x5[6 * 5], b5[5];
    for (int i = 0; i < 6; i++)
      for (int j = 0; j < 5; j++) l_6x5[5 * i + j] = L_6x10[10 * i + j];
    solve_svd(l_6x5, 6, 5, Rho, b5);
    if (b5[0] < 0) {
      betas[0] = std::sqrt(-b5[0]);
      betas[1] = (b5[2] < 0) ? std::sqrt(-b5[2]) : 0.0;
    } else {
      betas[0] = std::sqrt(b5[0]);
      betas[1] = (b5[2] > 0) ? std::sqrt(b5[2]) : 0.0;
    }
    if (b5[1] < 0) betas[0] = -betas[0];
    betas[2] = b5[3] / betas[0];
    betas[3] = 0.0;
  }
  static void compute_L_6x10(const double* ut, double* l_6x10) {
    const double* v[4];
    v[0] = ut + 12 * 11;
    v[1] = ut + 12 * 10;
    v[2] = ut + 12 * 9;
    v[3] = ut + 12 * 8;
    double dv[4][6][3];
    for (int i = 0; i < 4; i++) {
      int a = 0, b = 1;
      for (int j = 0; j < 6; j++) {
        dv[i][j][0] = v[i][3 * a] - v[i][3 * b];
        dv[i][j][1] = v[i][3 * a + 1] - v[i][3 * b + 1];
        dv[i][j][2] = v[i][3 * a + 2] - v[i][3 * b + 2];
        b++;
        if (b > 3) {
          a++;
          b = a + 1;
        }
      }
    }
    for (int i = 0; i < 6; i++) {
      double* row = l_6x10 + 10 * i;
      row[0] = dot(dv[0][i], dv[0][i]);
      row[1] = 2.0f * dot(dv[0][i], dv[1][i]);
      row[2] = dot(dv[1][i], dv[1][i]);
      row[3] = 2.0f * dot(dv[0][i], dv[2][i]);
      row[4] = 2.0f * dot(dv[1][i], dv[2][i]);
      row[5] = dot(dv[2][i], dv[2][i]);
      row[6] = 2.0f * dot(dv[0][i], dv[3][i]);
      row[7] = 2.0f * dot(dv[1][i], dv[3][i]);
      row[8] = 2.0f * dot(dv[2][i], dv[3][i]);
      row[9] = dot(dv[3][i], dv[3][i]);
    }
  }
  void compute_rho(double* rho) {
    rho[0] = dist2(cws[0], cws[1]);
    rho[1] = dist2(cws[0], cws[2]);
    rho[2] = dist2(cws[0], cws[3]);
    rho[3] = dist2(cws[1], cws[2]);
    rho[4] = dist2(cws[1], cws[3]);
    rho[5] = dist2(cws[2], cws[3]);
  }
  static void compute_A_and_b_gauss_newton(const double* l_6x10, const double* rho, const double betas[4], double* A,
                                           double* b) {
    for (int i = 0; i < 6; i++) {
      const double* rowL = l_6x10 + i * 10;
      double* rowA = A + i * 4;
      rowA[0] = 2 * rowL[0] * betas[0] + rowL[1] * betas[1] + rowL[3] * betas[2] + rowL[6] * betas[3];
      rowA[1] = rowL[1] * betas[0] + 2 * rowL[2] * betas[1] + rowL[4] * betas[2] + rowL[7] * betas[3];
      rowA[2] = rowL[3] * betas[0] + rowL[4] * betas[1] + 2 * rowL[5] * betas[2] + rowL[8] * betas[3];
      rowA[3] = rowL[6] * betas[0] + rowL[7] * betas[1] + rowL[8] * betas[2] + 2 * rowL[9] * betas[3];
      b[i] = rho[i] - (rowL[0] * betas[0] * betas[0] + rowL[1] * betas[0] * betas[1] + rowL[2] * betas[1] * betas[1] +
                       rowL[3] * betas[0] * betas[2] + rowL[4] * betas[1] * betas[2] + rowL[5] * betas[2] * betas[2] +
                       rowL[6] * betas[0] * betas[3] + rowL[7] * betas[1] * betas[3] + rowL[8] * betas[2] * betas[3] +
                       rowL[9] * betas[3] * betas[3]);
    }
  }
  // qr_solve for the 6 x 4 Gauss-Newton system; X is left as it is where a column's eta is 0
  static void qr_solve(double* pA, double* pb, double* pX) {
    const int nr = 6, nc = 4;
    double A1[6], A2[6];
    double* ppAkk = pA;
    for (int k = 0; k < nc; k++) {
      double *ppAik = ppAkk, eta = std::fabs(*ppAik);
      for (int i = k + 1; i < nr; i++) {
        const double elt = std::fabs(*ppAik);
        if (eta < elt) eta = elt;
        ppAik += nc;
      }
      if (eta == 0) return;
      {
        double *ppAik = ppAkk, sum = 0.0, inv_eta = 1. / eta;
        for (int i = k; i < nr; i++) {
          *ppAik *= inv_eta;
          sum += *ppAik * *ppAik;
          ppAik += nc;
        }
        double sigma = std::sqrt(sum);
        if (*ppAkk < 0) sigma = -sigma;
        *ppAkk += sigma;
        A1[k] = sigma * *ppAkk;
        A2[k] = -eta * sigma;
        for (int j = k + 1; j < nc; j++) {
          double *ppAik = ppAkk, sum = 0;
          for (int i = k; i < nr; i++) {
            sum += *ppAik * ppAik[j - k];
            ppAik += nc;
          }
          const double tau = sum / A1[k];
          ppAik = ppAkk;
          for (int i = k; i < nr; i++) {
            ppAik[j - k] -= tau * *ppAik;
            ppAik += nc;
          }
        }
      }
      ppAkk += nc + 1;
    }
    double *ppAjj = pA, *b = pb;
    for (int j = 0; j < nc; j++) {
      double *ppAij = ppAjj, tau = 0;
      for (int i = j; i < nr; i++) {
        tau += *ppAij * b[i];
        ppAij += nc;
      }
      tau /= A1[j];
      ppAij = ppAjj;
      for (int i = j; i < nr; i++) {
        b[i] -= tau * *ppAij;
        ppAij += nc;
      }
      ppAjj += nc + 1;
    }
    pX[nc - 1] = b[nc - 1] / A2[nc - 1];
    for (int i = nc - 2; i >= 0; i--) {
      double *ppAij = pA + i * nc + (i + 1), sum = 0;
      for (int j = i + 1; j < nc; j++) {
        sum += *ppAij * pX[j];
        ppAij++;
      }
      pX[i] = (b[i] - sum) / A2[i];
    }
  }
  static void gauss_newton(const double* L_6x10, const double* Rho, double betas[4]) {
    const int iterations_number = 5;
    double a[6 * 4], b[6], x[4] = {0, 0, 0, 0};
    for (int k = 0; k < iterations_number; k++) {
      compute_A_and_b_gauss_newton(L_6x10, Rho, betas, a, b);
      qr_solve(a, b, x);
      for (int i = 0; i < 4; i++) betas[i] += x[i];
    }
  }
  double compute_pose(double R[3][3], double t[3]) {
    choose_control_points();
    compute_barycentric_coordinates();
    std::vector<double> M(2 * (size_t)number_of_correspondences * 12);
    for (int i = 0; i < number_of_correspondences; i++) fill_M(M.data(), 2 * i, &alphas[4 * i], us[2 * i], us[2 * i + 1]);
    double mtm[12 * 12], d[12], ut[12 * 12], vt[12 * 12];
    mul_transposed(M.data(), 2 * number_of_correspondences, 12, mtm);
    svd_at(mtm, 12, ut, d, vt);  // cvSVD(.., CV_SVD_MODIFY_A | CV_SVD_U_T)
    double l_6x10[6 * 10], rho[6];
    compute_L_6x10(ut, l_6x10);
    compute_rho(rho);
    double Betas[4][4], rep_errors[4];
    double Rs[4][3][3], ts[4][3];
    find_betas_approx_1(l_6x10, rho, Betas[1]);
    gauss_newton(l_6x10, rho, Betas[1]);
    rep_errors[1] = compute_R_and_t(ut, Betas[1], Rs[1], ts[1]);
    find_betas_approx_2(l_6x10, rho, Betas[2]);
    gauss_newton(l_6x10, rho, Betas[2]);
    rep_errors[2] = compute_R_and_t(ut, Betas[2], Rs[2], ts[2]);
    find_betas_approx_3(l_6x10, rho, Betas[3]);
    gauss_newton(l_6x10, rho, Betas[3]);
    rep_errors[3] = compute_R_and_t(ut, Betas[3], Rs[3], ts[3]);
    int N = 1;
    if (rep_errors[2] < rep_errors[1]) N = 2;
    if (rep_errors[3] < rep_errors[N]) N = 3;
    for (int i = 0; i < 3; i++) {
      for (int j = 0; j < 3; j++) R[i][j] = Rs[N][i][j];
      t[i] = ts[N][i];
    }
    return rep_errors[N];
  }
};

double pose_of(const float* P3Dw, const float* P2D, const int* idx, int m, const float* cam, double R[3][3],
               double t[3]) {
  Epnp e(cam, m);
  for (int i = 0; i < m; i++) {
    const int j = idx[i];
    e.add_correspondence(P3Dw[3 * j], P3Dw[3 * j + 1], P3Dw[3 * j + 2], P2D[2 * j], P2D[2 * j + 1]);
  }
  return e.compute_pose(R, t);
}

// CheckInliers (:421-458); margin: the smallest |error2 - max_error| / max_error seen
int check_inliers(const b2s_pnpsolver_problem* p, const double R[3][3], const double t[3], uint8_t* inl,
                  double* margin) {
  const double uc = p->uc, vc = p->vc, fu = p->fu, fv = p->fv;
  int n = 0;
  for (int i = 0; i < p->n; i++) {
    const float x = p->P3Dw[3 * i], y = p->P3Dw[3 * i + 1], z = p->P3Dw[3 * i + 2];
    const float Xc = R[0][0] * x + R[0][1] * y + R[0][2] * z + t[0];
    const float Yc = R[1][0] * x + R[1][1] * y + R[1][2] * z + t[1];
    const float invZc = 1 / (R[2][0] * x + R[2][1] * y + R[2][2] * z + t[2]);
    const double ue = uc + fu * Xc * invZc;
    const double ve = vc + fv * Yc * invZc;
    const float distX = p->P2D[2 * i] - ue;
    const float distY = p->P2D[2 * i + 1] - ve;
    const float error2 = distX * distX + distY * distY;
    const float maxError = p->sigma2[i] * p->th2;
    inl[i] = error2 < maxError;
    n += inl[i];
    if (margin && maxError > 0 && std::isfinite(error2))
      *margin = std::min(*margin, std::abs((double)error2 - maxError) / maxError);
  }
  return n;
}

void to_Tcw(const double R[3][3], const double t[3], float* T) {
  for (int i = 0; i < 16; i++) T[i] = (i % 5 == 0) ? 1.f : 0.f;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) T[4 * r + c] = (float)R[r][c];
    T[4 * r + 3] = (float)t[r];
  }
}

}  // namespace

extern "C" {

void orc_pnp_mul_transposed(const double* A, int rows, int cols, double* D) { mul_transposed(A, rows, cols, D); }

void orc_pnp_svd(const double* A, int n, double* w, double* u, double* vt) {
  double At[144];
  svd_at(A, n, At, w, vt);
  for (int k = 0; k < n; k++)
    for (int i = 0; i < n; i++) u[k * n + i] = At[i * n + k];
}

void orc_pnp_invert_svd(const double* A, int n, double* D) { invert_svd(A, n, D); }

void orc_pnp_solve_svd(const double* A, int rows, int cols, const double* b, double* x) {
  solve_svd(A, rows, cols, b, x);
}

void orc_pnp_ransac_parameters(int N, double probability, int min_inliers, int max_iterations, int min_set,
                               float epsilon, int* min_inliers_out, int* max_its_out) {
  float mRansacEpsilon = epsilon;
  int nMinInliers = N * mRansacEpsilon;
  if (nMinInliers < min_inliers) nMinInliers = min_inliers;
  if (nMinInliers < min_set) nMinInliers = min_set;
  const int mRansacMinInliers = nMinInliers;
  if (mRansacEpsilon < (float)mRansacMinInliers / N) mRansacEpsilon = (float)mRansacMinInliers / N;
  int nIterations;
  if (mRansacMinInliers == N)
    nIterations = 1;
  else
    nIterations = std::ceil(std::log(1 - probability) / std::log(1 - std::pow(mRansacEpsilon, 3)));
  *min_inliers_out = mRansacMinInliers;
  *max_its_out = std::max(1, std::min(nIterations, max_iterations));
}

double orc_pnp_compute_pose(const float* P3Dw, const float* P2D, const int* idx, int m, const float* cam, double* R,
                            double* t) {
  double Rm[3][3];
  const double e = pose_of(P3Dw, P2D, idx, m, cam, Rm, t);
  std::memcpy(R, Rm, sizeof(Rm));
  return e;
}

void orc_pnp_iterate(const b2s_pnpsolver_problem* p, b2s_pnpsolver_result* r, double* margin, double* hyp) {
  const int N = p->n;
  const float cam[4] = {p->fu, p->fv, p->uc, p->vc};
  if (margin) *margin = INFINITY;
  int mnIterations = p->iterations_done, mnBestInliers = p->best_inliers;
  std::vector<uint8_t> mvbBestInliers(p->best_mask, p->best_mask + N), mvbInliersi((size_t)N), refined((size_t)N);
  float mBestTcw[16];
  std::memcpy(mBestTcw, p->best_Tcw, sizeof(mBestTcw));
  r->returned = 0;
  r->n_inliers = 0;
  r->no_more = 0;
  r->best_changed = 0;
  if (N > 0) std::memset(r->inliers, 0, (size_t)N);
  int nCurrentIterations = 0;
  if (N < p->min_inliers) {
    r->no_more = 1;
  } else {
    // while (mnIterations < mRansacMaxIts || nCurrentIterations < nIterations): k = max(nIterations, mRansacMaxIts -
    // mnIterations) iterations
    while (nCurrentIterations < p->k) {
      nCurrentIterations++;
      mnIterations++;
      double Ri[3][3], ti[3];
      const double err = pose_of(p->P3Dw, p->P2D, p->sets + 4 * (nCurrentIterations - 1), 4, cam, Ri, ti);
      double* h = hyp ? hyp + 15 * (nCurrentIterations - 1) : nullptr;
      const int mnInliersi = check_inliers(p, Ri, ti, mvbInliersi.data(), margin);
      if (h) {
        std::memcpy(h, Ri, sizeof(Ri));
        std::memcpy(h + 9, ti, sizeof(ti));
        h[12] = err;
        h[13] = mnInliersi;
        h[14] = -1;
      }
      if (mnInliersi >= p->min_inliers) {
        if (mnInliersi > mnBestInliers) {
          mvbBestInliers = mvbInliersi;
          mnBestInliers = mnInliersi;
          to_Tcw(Ri, ti, mBestTcw);
          r->best_changed = 1;
        }
        // Refine (:366-418)
        std::vector<int> vIndices;
        for (int i = 0; i < N; i++)
          if (mvbBestInliers[i]) vIndices.push_back(i);
        double Rr[3][3], tr[3];
        pose_of(p->P3Dw, p->P2D, vIndices.data(), (int)vIndices.size(), cam, Rr, tr);
        const int mnRefinedInliers = check_inliers(p, Rr, tr, refined.data(), margin);
        if (h) h[14] = mnRefinedInliers;
        if (mnRefinedInliers > p->min_inliers) {
          r->returned = 1;
          r->n_inliers = mnRefinedInliers;
          std::memcpy(r->inliers, refined.data(), (size_t)N);
          to_Tcw(Rr, tr, r->Tcw);
          break;
        }
      }
    }
    if (!r->returned && mnIterations >= p->max_its) {
      r->no_more = 1;
      if (mnBestInliers >= p->min_inliers) {
        r->returned = 1;
        r->n_inliers = mnBestInliers;
        if (N > 0) std::memcpy(r->inliers, mvbBestInliers.data(), (size_t)N);
        std::memcpy(r->Tcw, mBestTcw, sizeof(mBestTcw));
      }
    }
  }
  r->iterations_used = nCurrentIterations;
  r->iterations_done = mnIterations;
  r->best_inliers = mnBestInliers;
  std::memcpy(r->best_Tcw, mBestTcw, sizeof(mBestTcw));
  if (N > 0) std::memcpy(r->best_mask, mvbBestInliers.data(), (size_t)N);
}

}  // extern "C"
