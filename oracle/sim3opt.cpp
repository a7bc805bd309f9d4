/*
 * oracle/sim3opt.cpp — CPU restatement of Optimizer::OptimizeSim3 (src/Optimizer.cc:1364-1590) from the point where the
 * graph is built (TEST INFRASTRUCTURE, see orb_oracle.h).  The g2o::Sim3 operations are the essential graph oracle's
 * (orc_sim3_*, oracle/essential.cpp, linked into the same library).
 *
 *   - EdgeSim3ProjectXYZ = obs1 - cam_map1(project(S X2c)), EdgeInverseSim3ProjectXYZ = obs2 - cam_map2(project(S^-1
 *     X1c)), information I * invSigma2, Huber with delta = (float)sqrt(th2), chi2 = e^T Omega e;
 *   - BaseBinaryEdge::linearizeOplus of the Sim3 vertex only (the points are fixed): central differences,
 *     delta = 1e-9, oplus = Sim3(update) * estimate with update[6] = 0 under fix_scale (which also zeroes the solver's
 *     x entry);
 *   - constructQuadraticForm of a robust edge (rho' Omega, -rho' Omega e), H and b summed in edge order, the 7 x 7
 *     system solved by Cholesky, computeLambdaInit = 1e-5 max |H_jj| at each optimize();
 *   - optimize(5), drop the pairs with an edge chi2 > th2, return early below 10 pairs, optimize(nBad ? 10 : 5),
 *     classify again.
 */
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

#include "sim3opt_oracle.h"

namespace {

struct S3 {
  orc_sim3 s;
};
S3 from(const orc_sim3& s) { return S3{s}; }
void to(const S3& a, orc_sim3* o) { *o = a.s; }
S3 mul(const S3& a, const S3& b) {
  S3 o;
  orc_sim3_mul(&a.s, &b.s, &o.s);
  return o;
}
S3 inv(const S3& a) {
  S3 o;
  orc_sim3_inverse(&a.s, &o.s);
  return o;
}
void map3(const S3& a, const double* X, double* o) { orc_sim3_map(&a.s, X, o); }
// VertexSim3Expmap::oplusImpl: Sim3(update) * estimate, update[6] = 0 under fix_scale
S3 oplus(const S3& est, const double* upd, bool fixScale) {
  double u[7];
  for (int k = 0; k < 7; k++) u[k] = upd[k];
  if (fixScale) u[6] = 0;
  S3 e;
  orc_sim3_exp(u, &e.s);
  return mul(e, est);
}

}  // namespace

namespace {

// Optimizer::OptimizeSim3 after the graph is built: edge e = 2 m + side (e12, then e21) of correspondence m
struct Sim3Opt {
  const orc_sim3_problem* p;
  double K[8], th2, delta, dsqr;
  std::vector<uint8_t> active;
  std::vector<double> err, chi, J, W, omr;  // per edge: error, chi2, Jacobian (2 x 7), rho' w, -rho' w e
  std::vector<int32_t> trace;
  int nTrials = 0;

  void proj(const S3& S, const float* X, const float* obs, const double* k, double* e) const {
    const double x[3] = {X[0], X[1], X[2]};
    double y[3];
    map3(S, x, y);
    const double u = y[0] / y[2], v = y[1] / y[2];
    e[0] = (double)obs[0] - (u * k[0] + k[2]);
    e[1] = (double)obs[1] - (v * k[1] + k[3]);
  }
  void edge(const S3& S, const S3& Si, int m, int side, double* e) const {
    if (side == 0) proj(S, p->X2c + 3 * m, p->obs1 + 2 * m, K, e);
    else proj(Si, p->X1c + 3 * m, p->obs2 + 2 * m, K + 4, e);
  }
  double info(int m, int side) const { return (double)(side ? p->inv_sigma2_2[m] : p->inv_sigma2_1[m]); }
  // computeActiveErrors + activeRobustChi2
  double evaluate(const S3& S) {
    const S3 Si = inv(S);
    double sum = 0;
    for (int m = 0; m < p->n; m++) {
      if (!active[(size_t)m]) continue;
      for (int side = 0; side < 2; side++) {
        const size_t e = (size_t)m * 2 + side;
        const double w = info(m, side);
        edge(S, Si, m, side, &err[e * 2]);
        const double c = err[e * 2] * (w * err[e * 2]) + err[e * 2 + 1] * (w * err[e * 2 + 1]);
        chi[e] = c;
        sum += c <= dsqr ? c : 2 * std::sqrt(c) * delta - dsqr;
      }
    }
    return sum;
  }
  // linearizeOplus + constructQuadraticForm of every active edge, summed in edge order
  void build(const S3& S, double* H, double* b) {
    const bool fixScale = p->fix_scale != 0;
    const double dl = 1e-9, scalar = 1.0 / (2 * dl);
    for (int m = 0; m < p->n; m++) {
      if (!active[(size_t)m]) continue;
      for (int side = 0; side < 2; side++) {
        const size_t e = (size_t)m * 2 + side;
        for (int d = 0; d < 7; d++) {
          double upd[7] = {0, 0, 0, 0, 0, 0, 0}, ep[2], em[2];
          upd[d] = dl;
          S3 P = oplus(S, upd, fixScale);
          edge(P, inv(P), m, side, ep);
          upd[d] = -dl;
          P = oplus(S, upd, fixScale);
          edge(P, inv(P), m, side, em);
          J[e * 14 + d] = scalar * (ep[0] - em[0]);
          J[e * 14 + 7 + d] = scalar * (ep[1] - em[1]);
        }
        const double w = info(m, side), c = chi[e];
        const double rho1 = c <= dsqr ? 1. : delta / std::sqrt(c);
        W[e] = rho1 * w;
        omr[e * 2] = -(w * err[e * 2]) * rho1;
        omr[e * 2 + 1] = -(w * err[e * 2 + 1]) * rho1;
      }
    }
    for (int r = 0; r < 7; r++) {
      for (int c = r; c < 7; c++) {
        double acc = 0;
        for (int m = 0; m < p->n; m++) {
          if (!active[(size_t)m]) continue;
          for (size_t e = (size_t)m * 2; e < (size_t)m * 2 + 2; e++) {
            const double* Je = &J[e * 14];
            acc += (Je[r] * W[e]) * Je[c] + (Je[7 + r] * W[e]) * Je[7 + c];
          }
        }
        H[r * 7 + c] = H[c * 7 + r] = acc;
      }
      double acc = 0;
      for (int m = 0; m < p->n; m++) {
        if (!active[(size_t)m]) continue;
        for (size_t e = (size_t)m * 2; e < (size_t)m * 2 + 2; e++)
          acc += J[e * 14 + r] * omr[e * 2] + J[e * 14 + 7 + r] * omr[e * 2 + 1];
      }
      b[r] = acc;
    }
  }
  // SparseOptimizer::optimize(iterations) with OptimizationAlgorithmLevenberg::solve
  void optimize(S3& S, int iterations) {
    const bool fixScale = p->fix_scale != 0;
    double lambda = 0, ni = 2;
    int nBad = 0;
    for (int it = 0; it < iterations; it++) {
      double currentChi = evaluate(S);
      const double iniChi = currentChi;
      double H[49], b[7];
      build(S, H, b);
      if (it == 0) {  // computeLambdaInit
        double maxDiag = 0;
        for (int j = 0; j < 7; j++) maxDiag = std::max(std::fabs(H[j * 7 + j]), maxDiag);
        lambda = 1e-5 * maxDiag;
        ni = 2;
        nBad = 0;
      }
      double rho = 0;
      int qmax = 0;
      do {
        double A[49], x[7], y[7];
        for (int i = 0; i < 49; i++) A[i] = (i % 8 == 0) ? H[i] + lambda : H[i];
        bool solved = true;
        for (int k = 0; k < 7 && solved; k++) {
          double s = A[k * 7 + k];
          for (int j = 0; j < k; j++) s -= A[k * 7 + j] * A[k * 7 + j];
          if (!(s > 0.0) || !std::isfinite(s)) {
            solved = false;
            break;
          }
          A[k * 7 + k] = std::sqrt(s);
          for (int i = k + 1; i < 7; i++) {
            double t = A[i * 7 + k];
            for (int j = 0; j < k; j++) t -= A[i * 7 + j] * A[k * 7 + j];
            A[i * 7 + k] = t / A[k * 7 + k];
          }
        }
        double tempChi = DBL_MAX, scale = 0;
        S3 ST = S;
        if (solved) {  // a failed solve leaves the state and the edges' errors as they were
          for (int i = 0; i < 7; i++) {
            double s = b[i];
            for (int k = 0; k < i; k++) s -= A[i * 7 + k] * y[k];
            y[i] = s / A[i * 7 + i];
          }
          for (int i = 6; i >= 0; i--) {
            double s = y[i];
            for (int k = i + 1; k < 7; k++) s -= A[k * 7 + i] * x[k];
            x[i] = s / A[i * 7 + i];
          }
          if (fixScale) x[6] = 0;
          ST = oplus(S, x, false);
          for (int j = 0; j < 7; j++) scale += x[j] * (lambda * x[j] + b[j]);
          tempChi = evaluate(ST);
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
          S = ST;
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
  }
  bool bad(size_t m) const { return chi[m * 2] > th2 || chi[m * 2 + 1] > th2; }
};

}  // namespace

extern "C" int orc_optimize_sim3(const orc_sim3_problem* p, orc_sim3_result* r, double* chi2_out) {
  Sim3Opt o;
  o.p = p;
  const float K[8] = {p->fx1, p->fy1, p->cx1, p->cy1, p->fx2, p->fy2, p->cx2, p->cy2};
  for (int k = 0; k < 8; k++) o.K[k] = (double)K[k];
  o.th2 = (double)p->th2;
  const float deltaHuber = std::sqrt(p->th2);
  o.delta = (double)deltaHuber;
  o.dsqr = o.delta * o.delta;
  const size_t n = (size_t)std::max(p->n, 0);
  o.active.assign(n, 1);
  o.err.assign(n * 4, 0.0);
  o.chi.assign(n * 2, 0.0);
  o.J.assign(n * 28, 0.0);
  o.W.assign(n * 2, 0.0);
  o.omr.assign(n * 4, 0.0);
  S3 S = from(p->S12);
  if (n) o.optimize(S, 5);  // initializeOptimization refuses an empty graph, and optimize() then does nothing
  int nBad = 0;
  for (size_t m = 0; m < n; m++)
    if (o.bad(m)) {
      o.active[m] = 0;
      nBad++;
    }
  int nIn = 0;
  const bool early = (int)n - nBad < 10;
  if (!early) {
    o.optimize(S, nBad > 0 ? 10 : 5);
    for (size_t m = 0; m < n; m++) {
      if (!o.active[m]) continue;
      if (o.bad(m)) o.active[m] = 0;
      else nIn++;
    }
  }
  for (size_t m = 0; m < n; m++) r->keep[m] = o.active[m];
  to(early ? from(p->S12) : S, &r->S12_out);
  r->n_inliers = early ? 0 : nIn;
  r->n_trials = o.nTrials;
  if (r->trace) {
    for (size_t i = 0; i < o.trace.size(); i++) r->trace[i] = o.trace[i];
    r->trace[o.trace.size()] = -1;
  }
  if (chi2_out)
    for (size_t e = 0; e < n * 2; e++) chi2_out[e] = o.chi[e];
  return 0;
}
