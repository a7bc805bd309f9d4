/*
 * oracle/essential.cpp — CPU restatement of Optimizer::OptimizeEssentialGraph (src/Optimizer.cc:1017-1339) from the
 * point where the graph is built (TEST INFRASTRUCTURE, see orb_oracle.h).
 *
 *   - g2o::Sim3 (types/sim3.h): exp with its four sigma / theta branches, log with W.lu().solve(t), product, inverse,
 *     map; quaternion <-> matrix with Eigen's formulas;
 *   - EdgeSim3::computeError = log(S_ji * S_i * S_j^-1); identity information;
 *   - BaseBinaryEdge::linearizeOplus: central differences, delta = 1e-9, oplus = Sim3(update) * estimate with
 *     update[6] = 0 under fix_scale (which also zeroes the solver's x entry);
 *   - H and b summed per block in edge order; vertices without an edge and the fixed vertex are not in the system;
 *   - the system (7 scalars per free vertex) is factorised by a skyline Cholesky over its envelope;
 *   - OptimizationAlgorithmLevenberg::solve (core/optimization_algorithm_levenberg.cpp:61-164), 20 iterations, user
 *     lambda 1e-16, computeScale over x and b in index order;
 *   - write-back: [R t/s; 0 1] of every keyframe, every point through its reference keyframe (ref_kf = -1: unchanged).
 */
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <utility>
#include <vector>

#include "essential_oracle.h"

namespace {

struct S3 {
  double v[8];  // qx qy qz qw tx ty tz s
};

void qrot(const double* q, const double* v, double* o) {
  double uv[3] = {q[1] * v[2] - q[2] * v[1], q[2] * v[0] - q[0] * v[2], q[0] * v[1] - q[1] * v[0]};
  for (int i = 0; i < 3; i++) uv[i] += uv[i];
  const double uuv[3] = {q[1] * uv[2] - q[2] * uv[1], q[2] * uv[0] - q[0] * uv[2], q[0] * uv[1] - q[1] * uv[0]};
  for (int i = 0; i < 3; i++) o[i] = v[i] + q[3] * uv[i] + uuv[i];
}
S3 mul(const S3& a, const S3& b) {
  S3 o;
  const double* x = a.v;
  const double* y = b.v;
  o.v[3] = x[3] * y[3] - x[0] * y[0] - x[1] * y[1] - x[2] * y[2];
  o.v[0] = x[3] * y[0] + x[0] * y[3] + x[1] * y[2] - x[2] * y[1];
  o.v[1] = x[3] * y[1] + x[1] * y[3] + x[2] * y[0] - x[0] * y[2];
  o.v[2] = x[3] * y[2] + x[2] * y[3] + x[0] * y[1] - x[1] * y[0];
  double rt[3];
  qrot(x, y + 4, rt);
  for (int i = 0; i < 3; i++) o.v[4 + i] = x[7] * rt[i] + x[4 + i];
  o.v[7] = x[7] * y[7];
  return o;
}
S3 inv(const S3& a) {
  S3 o;
  o.v[0] = -a.v[0]; o.v[1] = -a.v[1]; o.v[2] = -a.v[2]; o.v[3] = a.v[3];
  const double k = -1. / a.v[7];
  const double t[3] = {k * a.v[4], k * a.v[5], k * a.v[6]};
  qrot(o.v, t, o.v + 4);
  o.v[7] = 1. / a.v[7];
  return o;
}
void map3(const S3& a, const double* X, double* o) {
  double rt[3];
  qrot(a.v, X, rt);
  for (int i = 0; i < 3; i++) o[i] = a.v[7] * rt[i] + a.v[4 + i];
}
void quat_from_R(const double m[3][3], double* q) {
  double t = m[0][0] + m[1][1] + m[2][2];
  if (t > 0.0) {
    t = std::sqrt(t + 1.0);
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
    t = std::sqrt(m[i][i] - m[j][j] - m[k][k] + 1.0);
    q[i] = 0.5 * t;
    t = 0.5 / t;
    q[3] = (m[k][j] - m[j][k]) * t;
    q[j] = (m[j][i] + m[i][j]) * t;
    q[k] = (m[k][i] + m[i][k]) * t;
  }
}
void quat_to_R(const double* q, double R[3][3]) {
  const double tx = 2 * q[0], ty = 2 * q[1], tz = 2 * q[2];
  const double twx = tx * q[3], twy = ty * q[3], twz = tz * q[3];
  const double txx = tx * q[0], txy = ty * q[0], txz = tz * q[0];
  const double tyy = ty * q[1], tyz = tz * q[1], tzz = tz * q[2];
  R[0][0] = 1 - (tyy + tzz); R[0][1] = txy - twz; R[0][2] = txz + twy;
  R[1][0] = txy + twz; R[1][1] = 1 - (txx + tzz); R[1][2] = tyz - twx;
  R[2][0] = txz - twy; R[2][1] = tyz + twx; R[2][2] = 1 - (txx + tyy);
}
void skew(const double* w, double O[3][3]) {
  O[0][0] = 0; O[0][1] = -w[2]; O[0][2] = w[1];
  O[1][0] = w[2]; O[1][1] = 0; O[1][2] = -w[0];
  O[2][0] = -w[1]; O[2][1] = w[0]; O[2][2] = 0;
}
void mm3(const double A[3][3], const double B[3][3], double C[3][3]) {
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) C[i][j] = A[i][0] * B[0][j] + A[i][1] * B[1][j] + A[i][2] * B[2][j];
}
S3 expmap(const double* u) {
  const double w[3] = {u[0], u[1], u[2]};
  const double sigma = u[6];
  const double theta = std::sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  double O[3][3], O2[3][3], R[3][3];
  skew(w, O);
  const double s = std::exp(sigma);
  mm3(O, O, O2);
  const double eps = 0.00001;
  double A, B, C;
  const bool small = theta < eps;
  if (std::fabs(sigma) < eps) {
    C = 1;
    if (small) {
      A = 1. / 2.;
      B = 1. / 6.;
    } else {
      const double theta2 = theta * theta;
      A = (1 - std::cos(theta)) / theta2;
      B = (theta - std::sin(theta)) / (theta2 * theta);
    }
  } else {
    C = (s - 1) / sigma;
    if (small) {
      const double sigma2 = sigma * sigma;
      A = ((sigma - 1) * s + 1) / sigma2;
      B = ((0.5 * sigma2 - sigma + 1) * s) / (sigma2 * sigma);
    } else {
      const double a = s * std::sin(theta), b = s * std::cos(theta);
      const double theta2 = theta * theta, sigma2 = sigma * sigma, c = theta2 + sigma2;
      A = (a * sigma + (1 - b) * theta) / (theta * c);
      B = (C - ((b - 1) * sigma + a * theta) / c) * 1. / theta2;
    }
  }
  const double k1 = small ? 1.0 : std::sin(theta) / theta, k2 = small ? 1.0 : (1 - std::cos(theta)) / (theta * theta);
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      R[i][j] = small ? ((i == j ? 1.0 : 0.0) + O[i][j]) + O2[i][j] : ((i == j ? 1.0 : 0.0) + k1 * O[i][j]) + k2 * O2[i][j];
  S3 o;
  quat_from_R(R, o.v);
  double W[3][3];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) W[i][j] = (A * O[i][j] + B * O2[i][j]) + C * (i == j ? 1.0 : 0.0);
  for (int i = 0; i < 3; i++) o.v[4 + i] = W[i][0] * u[3] + W[i][1] * u[4] + W[i][2] * u[5];
  o.v[7] = s;
  return o;
}
void logmap(const S3& a, double* res) {
  const double s = a.v[7], sigma = std::log(s);
  double R[3][3];
  quat_to_R(a.v, R);
  const double d = 0.5 * (R[0][0] + R[1][1] + R[2][2] - 1);
  const double dR[3] = {R[2][1] - R[1][2], R[0][2] - R[2][0], R[1][0] - R[0][1]};
  const double eps = 0.00001;
  double w[3], A, B, C;
  const bool small = d > 1 - eps;
  double theta = 0;
  if (small) {
    for (int i = 0; i < 3; i++) w[i] = 0.5 * dR[i];
  } else {
    theta = std::acos(d);
    const double k = theta / (2 * std::sqrt(1 - d * d));
    for (int i = 0; i < 3; i++) w[i] = k * dR[i];
  }
  if (std::fabs(sigma) < eps) {
    C = 1;
    if (small) {
      A = 1. / 2.;
      B = 1. / 6.;
    } else {
      const double theta2 = theta * theta;
      A = (1 - std::cos(theta)) / theta2;
      B = (theta - std::sin(theta)) / (theta2 * theta);
    }
  } else {
    C = (s - 1) / sigma;
    if (small) {
      const double sigma2 = sigma * sigma;
      A = ((sigma - 1) * s + 1) / sigma2;
      B = ((0.5 * sigma2 - sigma + 1) * s) / (sigma2 * sigma);
    } else {
      const double theta2 = theta * theta;
      const double aa = s * std::sin(theta), bb = s * std::cos(theta), c = theta2 + sigma * sigma;
      A = (aa * sigma + (1 - bb) * theta) / (theta * c);
      B = (C - ((bb - 1) * sigma + aa * theta) / c) * 1. / theta2;
    }
  }
  double O[3][3], BO[3][3], BOO[3][3], W[3][3];
  skew(w, O);
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) BO[i][j] = B * O[i][j];
  mm3(BO, O, BOO);
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) W[i][j] = (A * O[i][j] + BOO[i][j]) + C * (i == j ? 1.0 : 0.0);
  int perm[3] = {0, 1, 2};
  for (int k = 0; k < 3; k++) {
    int p = k;
    double best = std::fabs(W[k][k]);
    for (int i = k + 1; i < 3; i++)
      if (std::fabs(W[i][k]) > best) {
        best = std::fabs(W[i][k]);
        p = i;
      }
    if (p != k) {
      for (int j = 0; j < 3; j++) std::swap(W[k][j], W[p][j]);
      std::swap(perm[k], perm[p]);
    }
    if (W[k][k] == 0.0) continue;
    for (int i = k + 1; i < 3; i++) {
      W[i][k] /= W[k][k];
      for (int j = k + 1; j < 3; j++) W[i][j] -= W[i][k] * W[k][j];
    }
  }
  double x[3];
  for (int i = 0; i < 3; i++) {
    double v = a.v[4 + perm[i]];
    for (int k = 0; k < i; k++) v -= W[i][k] * x[k];
    x[i] = v;
  }
  for (int i = 2; i >= 0; i--) {
    double v = x[i];
    for (int k = i + 1; k < 3; k++) v -= W[i][k] * x[k];
    x[i] = v / W[i][i];
  }
  for (int i = 0; i < 3; i++) res[i] = w[i];
  for (int i = 0; i < 3; i++) res[3 + i] = x[i];
  res[6] = sigma;
}

S3 from(const orc_sim3& s) {
  S3 o;
  memcpy(o.v, &s, sizeof(o.v));
  return o;
}
void to(const S3& s, orc_sim3* o) { memcpy(o, s.v, sizeof(s.v)); }

void edge_error(const S3& C, const S3& Si, const S3& Sj, double* e) { logmap(mul(mul(C, Si), inv(Sj)), e); }
S3 oplus(const S3& est, const double* upd, bool fixScale) {
  double u[7];
  for (int k = 0; k < 7; k++) u[k] = upd[k];
  if (fixScale) u[6] = 0;
  return mul(expmap(u), est);
}

}  // namespace

extern "C" {

void orc_sim3_exp(const double* u, orc_sim3* o) { to(expmap(u), o); }
void orc_sim3_log(const orc_sim3* a, double* o) { logmap(from(*a), o); }
void orc_sim3_mul(const orc_sim3* a, const orc_sim3* b, orc_sim3* o) { to(mul(from(*a), from(*b)), o); }
void orc_sim3_inverse(const orc_sim3* a, orc_sim3* o) { to(inv(from(*a)), o); }
void orc_sim3_map(const orc_sim3* a, const double* X, double* o) { map3(from(*a), X, o); }
void orc_sim3_from_Rt(const double* R9, const double* t, double s, orc_sim3* o) {
  double R[3][3];
  for (int i = 0; i < 9; i++) R[i / 3][i % 3] = R9[i];
  S3 r;
  quat_from_R(R, r.v);
  for (int i = 0; i < 3; i++) r.v[4 + i] = t[i];
  r.v[7] = s;
  to(r, o);
}

int orc_optimize_essential_graph(const orc_eg_problem* p, orc_eg_result* r) {
  const int nKf = p->n_kf, nE = p->n_edges;
  const bool fixScale = p->fix_scale != 0;
  std::vector<S3> est((size_t)nKf), est0((size_t)nKf);
  for (int k = 0; k < nKf; k++) est[(size_t)k] = est0[(size_t)k] = from(p->Siw[k]);
  std::vector<int> pidx((size_t)nKf, -1);
  std::vector<uint8_t> active((size_t)nKf, 0);
  for (int e = 0; e < nE; e++) active[(size_t)p->edges[e].i] = active[(size_t)p->edges[e].j] = 1;
  int nFree = 0;
  for (int k = 0; k < nKf; k++)
    if (active[(size_t)k] && k != p->fixed_kf) pidx[(size_t)k] = nFree++;
  const int n = nFree * 7;
  // skyline: row i stores columns [first[i], i]
  std::vector<int> first((size_t)n);
  for (int i = 0; i < n; i++) first[(size_t)i] = i / 7 * 7;
  for (int e = 0; e < nE; e++) {
    const int a = pidx[(size_t)p->edges[e].i], b = pidx[(size_t)p->edges[e].j];
    if (a < 0 || b < 0) continue;
    const int R = std::max(a, b), C = std::min(a, b);
    for (int k = 0; k < 7; k++) first[(size_t)R * 7 + k] = std::min(first[(size_t)R * 7 + k], C * 7);
  }
  std::vector<size_t> rowOff((size_t)n + 1, 0);
  for (int i = 0; i < n; i++) rowOff[(size_t)i + 1] = rowOff[(size_t)i] + (size_t)(i - first[(size_t)i] + 1);
  auto at = [&](std::vector<double>& M, int i, int j) -> double& { return M[rowOff[(size_t)i] + (size_t)(j - first[(size_t)i])]; };

  std::vector<double> err((size_t)nE * 7), J((size_t)nE * 98), H(rowOff[(size_t)n]), L, b((size_t)n), x((size_t)n);
  auto chi2_of = [&](const std::vector<S3>& S, bool keep) {
    double chi = 0;
    for (int e = 0; e < nE; e++) {
      double er[7];
      edge_error(from(p->edges[e].meas), S[(size_t)p->edges[e].i], S[(size_t)p->edges[e].j], er);
      double c = 0;
      for (int k = 0; k < 7; k++) c += er[k] * er[k];
      chi += c;
      if (keep)
        for (int k = 0; k < 7; k++) err[(size_t)e * 7 + k] = er[k];
    }
    return chi;
  };

  std::vector<int32_t> trace;
  int nTrials = 0;
  double chi2Initial = 0, lambda = 1e-16, ni = 2;
  int nBad = 0;
  bool ok = nE > 0;
  for (int it = 0; it < 20 && ok; it++) {
    double currentChi = chi2_of(est, true);
    const double iniChi = currentChi;
    if (it == 0) chi2Initial = currentChi;
    // linearise
    const double delta = 1e-9, scalar = 1.0 / (2 * delta);
    for (int e = 0; e < nE; e++) {
      const int vi = p->edges[e].i, vj = p->edges[e].j;
      const S3 C = from(p->edges[e].meas);
      for (int side = 0; side < 2; side++) {
        const int v = side ? vj : vi;
        if (pidx[(size_t)v] < 0) continue;
        for (int d = 0; d < 7; d++) {
          double upd[7] = {0, 0, 0, 0, 0, 0, 0}, ep[7], em[7];
          upd[d] = delta;
          S3 P = oplus(est[(size_t)v], upd, fixScale);
          edge_error(C, side ? est[(size_t)vi] : P, side ? P : est[(size_t)vj], ep);
          upd[d] = -delta;
          P = oplus(est[(size_t)v], upd, fixScale);
          edge_error(C, side ? est[(size_t)vi] : P, side ? P : est[(size_t)vj], em);
          for (int k = 0; k < 7; k++) J[(size_t)e * 98 + side * 49 + k * 7 + d] = scalar * (ep[k] - em[k]);
        }
      }
    }
    // H, b in edge order
    std::fill(H.begin(), H.end(), 0.0);
    std::fill(b.begin(), b.end(), 0.0);
    for (int e = 0; e < nE; e++) {
      const int pv[2] = {pidx[(size_t)p->edges[e].i], pidx[(size_t)p->edges[e].j]};
      const double* Jv[2] = {&J[(size_t)e * 98], &J[(size_t)e * 98 + 49]};
      for (int s = 0; s < 2; s++) {
        if (pv[s] < 0) continue;
        for (int rr = 0; rr < 7; rr++) {
          double h = 0;
          for (int k = 0; k < 7; k++) h += Jv[s][k * 7 + rr] * -err[(size_t)e * 7 + k];
          b[(size_t)pv[s] * 7 + rr] += h;
          for (int c = 0; c <= rr; c++) {
            double hh = 0;
            for (int k = 0; k < 7; k++) hh += Jv[s][k * 7 + rr] * Jv[s][k * 7 + c];
            at(H, pv[s] * 7 + rr, pv[s] * 7 + c) += hh;
          }
        }
      }
      if (pv[0] >= 0 && pv[1] >= 0) {
        const int rs = pv[0] > pv[1] ? 0 : 1;  // row vertex: the larger index
        for (int rr = 0; rr < 7; rr++)
          for (int c = 0; c < 7; c++) {
            double hh = 0;
            for (int k = 0; k < 7; k++) hh += Jv[rs][k * 7 + rr] * Jv[1 - rs][k * 7 + c];
            at(H, pv[rs] * 7 + rr, pv[1 - rs] * 7 + c) += hh;
          }
      }
    }
    double rho = 0;
    int qmax = 0;
    do {
      // (H + lambda I) x = b by a skyline Cholesky
      L = H;
      for (int i = 0; i < n; i++) at(L, i, i) += lambda;
      bool solved = true;
      for (int i = 0; i < n && solved; i++)
        for (int j = first[(size_t)i]; j <= i; j++) {
          double s = at(L, i, j);
          for (int k = std::max(first[(size_t)i], first[(size_t)j]); k < j; k++) s -= at(L, i, k) * at(L, j, k);
          if (i == j) {
            if (!(s > 0.0) || !std::isfinite(s)) {
              solved = false;
              break;
            }
            at(L, i, i) = std::sqrt(s);
          } else {
            at(L, i, j) = s / at(L, j, j);
          }
        }
      std::vector<S3> estT = est;
      double scale = 0, tempChi = DBL_MAX;
      if (solved) {
        std::vector<double> y = b;
        for (int i = 0; i < n; i++) {
          double s = y[(size_t)i];
          for (int k = first[(size_t)i]; k < i; k++) s -= at(L, i, k) * y[(size_t)k];
          y[(size_t)i] = s / at(L, i, i);
        }
        for (int i = n - 1; i >= 0; i--) {
          x[(size_t)i] = y[(size_t)i] / at(L, i, i);
          for (int k = first[(size_t)i]; k < i; k++) y[(size_t)k] -= at(L, i, k) * x[(size_t)i];
        }
        for (int k = 0; k < nKf; k++) {
          const int pv = pidx[(size_t)k];
          if (pv < 0) continue;
          if (fixScale) x[(size_t)pv * 7 + 6] = 0;
          estT[(size_t)k] = oplus(est[(size_t)k], &x[(size_t)pv * 7], false);
        }
        tempChi = chi2_of(estT, false);
        for (int j = 0; j < n; j++) scale += x[(size_t)j] * (lambda * x[(size_t)j] + b[(size_t)j]);
      }
      rho = currentChi - tempChi;
      scale += 1e-3;
      rho /= scale;
      if (!solved) rho = -1;
      const bool good = rho > 0 && std::isfinite(tempChi);
      if (trace.size() < 255) trace.push_back(good ? 1 : 0);
      nTrials++;
      if (good) {
        double alpha = 1. - std::pow((2 * rho - 1), 3);
        alpha = std::min(alpha, 2. / 3.);
        lambda *= std::max(1. / 3., alpha);
        ni = 2;
        currentChi = tempChi;
        est = estT;
      } else {
        lambda *= ni;
        ni *= 2;
      }
      qmax++;
    } while (rho < 0 && qmax < 10);
    if (qmax == 10 || rho == 0) break;
    if ((iniChi - currentChi) * 1e3 < iniChi) nBad++;
    else nBad = 0;
    if (nBad >= 3) break;
  }
  // write-back
  for (int k = 0; k < nKf; k++) {
    const S3& S = est[(size_t)k];
    double R[3][3];
    quat_to_R(S.v, R);
    const double is = 1. / S.v[7];
    float* T = r->Tcw_out + (size_t)k * 16;
    for (int i = 0; i < 3; i++) {
      for (int j = 0; j < 3; j++) T[i * 4 + j] = (float)R[i][j];
      T[i * 4 + 3] = (float)(S.v[4 + i] * is);
    }
    T[12] = 0.f; T[13] = 0.f; T[14] = 0.f; T[15] = 1.f;
  }
  for (int m = 0; m < p->n_mp; m++) {
    const int rk = p->ref_kf[m];
    if (rk < 0) {
      for (int c = 0; c < 3; c++) r->points_out[(size_t)m * 3 + c] = p->points[(size_t)m * 3 + c];
      continue;
    }
    const double X[3] = {p->points[(size_t)m * 3], p->points[(size_t)m * 3 + 1], p->points[(size_t)m * 3 + 2]};
    double Y[3], Z[3];
    map3(est0[(size_t)rk], X, Y);
    map3(inv(est[(size_t)rk]), Y, Z);
    for (int c = 0; c < 3; c++) r->points_out[(size_t)m * 3 + c] = (float)Z[c];
  }
  r->chi2_initial = chi2Initial;
  r->chi2_final = nE ? chi2_of(est, false) : 0.0;
  r->n_trials = nTrials;
  if (r->trace) {
    for (size_t i = 0; i < trace.size(); i++) r->trace[i] = trace[i];
    r->trace[trace.size()] = -1;
  }
  return 0;
}

}  // extern "C"
