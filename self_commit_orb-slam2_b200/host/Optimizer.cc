#include "Optimizer.h"

#include <mutex>

#include "b2s_host.h"

namespace ORB_SLAM2 {
namespace {

using b2s_host::fail;

int create_ba(const int* cap, b2s_ba_solver** h) {
  return b2s_ba_create(cap[0], cap[1], cap[2], 1, b2s_host::device(), h);
}

// LocalBA runs on the LocalMapping thread only (src/LocalMapping.cc:123): one solver, grown on demand.
b2s_host::Slot<b2s_ba_solver, 3, b2s_ba_destroy> g_localBA;
// PoseOptimization runs on the Tracking thread: its own solver handle (handles are not shared between threads)
b2s_host::Slot<b2s_ba_solver, 3, b2s_ba_destroy> g_pose;
// Global BA runs on LoopClosing's GBA thread (and once for the monocular initial map): its own handle, grown on demand
b2s_host::Slot<b2s_gba_solver, 3, b2s_gba_destroy> g_gba;
// The essential graph runs on LoopClosing's thread: its own handle, grown on demand
b2s_host::Slot<b2s_eg_solver, 3, b2s_eg_destroy> g_eg;
// OptimizeSim3 runs on LoopClosing's thread: its own handle, grown on demand
b2s_host::Slot<b2s_sim3opt_solver, 1, b2s_sim3opt_destroy> g_sim3;

}  // namespace

void Optimizer::LocalBundleAdjustment(const LocalBAWindow& w, bool* pbStopFlag, LocalBAResult& out) {
  std::lock_guard<std::mutex> lock(g_localBA.mutex);
  const int nKF = (int)w.fixed.size(), nMP = (int)w.points.size() / 3, nE = (int)w.edges.size();
  int rc = g_localBA.get({nKF, nMP, nE}, {64, 8192, 65536}, create_ba);
  if (rc != B2S_OK) fail("Optimizer::LocalBundleAdjustment", rc);
  b2s_ba_problem p;
  p.n_kf = nKF;
  p.n_local = w.nLocal;
  p.Tcw = w.Tcw.data();
  p.fixed = w.fixed.data();
  p.n_mp = nMP;
  p.points = w.points.data();
  p.n_edges = nE;
  p.edges = w.edges.data();
  p.fx = w.fx; p.fy = w.fy; p.cx = w.cx; p.cy = w.cy; p.bf = w.bf;
  p.its1 = 5;   // optimizer.optimize(5)  :864
  p.its2 = 10;  // optimizer.optimize(10) :917
  out.Tcw.assign((size_t)w.nLocal * 16, 0.f);
  out.points.assign((size_t)nMP * 3, 0.f);
  out.outlier.assign(nE, 0);
  out.aborted = false;
  b2s_ba_result r;
  r.Tcw_out = out.Tcw.data();
  r.points_out = out.points.data();
  r.edge_outlier = out.outlier.data();
  r.trace = nullptr;
  r.chi2_final = 0;
  r.n_trials = 0;
  static_assert(sizeof(bool) == 1, "bool stop flag is read as a byte");
  rc = b2s_local_ba(g_localBA.h, &p, (const volatile uint8_t*)pbStopFlag, &r);
  if (rc == B2S_ERR_ABORTED) {
    out.aborted = true;
    return;
  }
  if (rc != B2S_OK) fail("Optimizer::LocalBundleAdjustment", rc);
}

int Optimizer::PoseOptimization(const PoseProblem& f, float TcwOut[16], std::vector<uint8_t>& outlier) {
  std::lock_guard<std::mutex> lock(g_pose.mutex);
  int rc = g_pose.get({0, 0, 0}, {4, 16, 64}, create_ba);
  if (rc != B2S_OK) fail("Optimizer::PoseOptimization", rc);
  const int N = (int)f.hasMapPoint.size();
  outlier.assign(N > 0 ? N : 1, 0);
  b2s_pose_problem p;
  p.Tcw = f.Tcw; p.n = N; p.has_mp = f.hasMapPoint.data(); p.Xw = f.Xw.data(); p.kpx = f.kpx.data(); p.kpy = f.kpy.data();
  p.uright = f.uRight.data(); p.inv_sigma2 = f.invSigma2.data();
  p.fx = f.fx; p.fy = f.fy; p.cx = f.cx; p.cy = f.cy; p.bf = f.bf;
  b2s_pose_result r;
  r.Tcw_out = TcwOut; r.outlier = outlier.data(); r.trace = nullptr; r.n_inliers = 0; r.n_trials = 0;
  rc = b2s_pose_optimization(g_pose.h, &p, &r);
  if (rc != B2S_OK) fail("Optimizer::PoseOptimization", rc);
  outlier.resize(N);
  return r.n_inliers;
}

void Optimizer::BundleAdjustment(const GlobalBAMap& m, int nIterations, bool* pbStopFlag, bool bRobust,
                                 GlobalBAResult& out) {
  std::lock_guard<std::mutex> lock(g_gba.mutex);
  const int nKF = (int)m.fixed.size(), nMP = (int)m.points.size() / 3, nE = (int)m.edges.size();
  int rc = g_gba.get({nKF, nMP, nE}, {256, 32768, 262144}, [](const int* c, b2s_gba_solver** h) {
    return b2s_gba_create(c[0], c[1], c[2], b2s_host::device(), h);
  });
  if (rc != B2S_OK) fail("Optimizer::BundleAdjustment", rc);
  b2s_gba_problem p;
  p.n_kf = nKF; p.Tcw = m.Tcw.data(); p.fixed = m.fixed.data();
  p.n_mp = nMP; p.points = m.points.data();
  p.n_edges = nE; p.edges = m.edges.data();
  p.fx = m.fx; p.fy = m.fy; p.cx = m.cx; p.cy = m.cy; p.bf = m.bf;
  p.iterations = nIterations;
  p.robust = bRobust ? 1 : 0;
  out.Tcw.assign((size_t)nKF * 16, 0.f);
  out.points = m.points;
  out.included.assign((size_t)(nMP > 0 ? nMP : 1), 0);
  b2s_gba_result r;
  r.Tcw_out = out.Tcw.data(); r.points_out = out.points.data(); r.point_included = out.included.data();
  r.trace = nullptr; r.chi2_final = 0; r.n_trials = 0;
  static_assert(sizeof(bool) == 1, "bool stop flag is read as a byte");
  rc = b2s_global_ba(g_gba.h, &p, (const volatile uint8_t*)pbStopFlag, &r);
  if (rc != B2S_OK) fail("Optimizer::BundleAdjustment", rc);
  out.included.resize(nMP);
}

void Optimizer::OptimizeEssentialGraph(const EssentialGraph& g, EssentialGraphResult& out) {
  std::lock_guard<std::mutex> lock(g_eg.mutex);
  const int nKF = (int)g.Siw.size(), nE = (int)g.edges.size(), nMP = (int)g.refKF.size();
  int rc = g_eg.get({nKF, nE, nMP}, {1024, 16384, 65536}, [](const int* c, b2s_eg_solver** h) {
    return b2s_eg_create(c[0], c[1], c[2], b2s_host::device(), h);
  });
  if (rc != B2S_OK) fail("Optimizer::OptimizeEssentialGraph", rc);
  b2s_eg_problem p;
  p.n_kf = nKF; p.Siw = g.Siw.data(); p.fixed_kf = g.fixedKF; p.fix_scale = g.fixScale ? 1 : 0;
  p.n_edges = nE; p.edges = g.edges.data();
  p.n_mp = nMP; p.points = g.points.data(); p.ref_kf = g.refKF.data();
  out.Tcw.assign((size_t)(nKF > 0 ? nKF : 1) * 16, 0.f);
  out.points.assign((size_t)(nMP > 0 ? nMP : 1) * 3, 0.f);
  b2s_eg_result r;
  r.Tcw_out = out.Tcw.data(); r.points_out = out.points.data(); r.trace = nullptr;
  r.chi2_initial = r.chi2_final = 0; r.n_trials = 0;
  rc = b2s_optimize_essential_graph(g_eg.h, &p, &r);
  if (rc != B2S_OK) fail("Optimizer::OptimizeEssentialGraph", rc);
  out.Tcw.resize((size_t)nKF * 16);
  out.points.resize((size_t)nMP * 3);
}

int Optimizer::OptimizeSim3(const Sim3Problem& p, Sim3Result& out) {
  std::lock_guard<std::mutex> lock(g_sim3.mutex);
  const int n = (int)p.invSigma2_1.size();
  int rc = g_sim3.get({n}, {4096}, [](const int* c, b2s_sim3opt_solver** h) {
    return b2s_sim3opt_create(c[0], 1, b2s_host::device(), h);
  });
  if (rc != B2S_OK) fail("Optimizer::OptimizeSim3", rc);
  b2s_sim3_problem q;
  q.n = n;
  q.X1c = p.X1c.data(); q.X2c = p.X2c.data(); q.obs1 = p.obs1.data(); q.obs2 = p.obs2.data();
  q.inv_sigma2_1 = p.invSigma2_1.data(); q.inv_sigma2_2 = p.invSigma2_2.data();
  q.fx1 = p.K1[0]; q.fy1 = p.K1[1]; q.cx1 = p.K1[2]; q.cy1 = p.K1[3];
  q.fx2 = p.K2[0]; q.fy2 = p.K2[1]; q.cx2 = p.K2[2]; q.cy2 = p.K2[3];
  q.S12 = p.S12; q.th2 = p.th2; q.fix_scale = p.fixScale ? 1 : 0;
  out.keep.assign((size_t)(n > 0 ? n : 1), 0);
  b2s_sim3_result r;
  r.keep = out.keep.data(); r.trace = nullptr; r.n_inliers = r.n_trials = 0;
  rc = b2s_optimize_sim3(g_sim3.h, 1, &q, &r);
  if (rc != B2S_OK) fail("Optimizer::OptimizeSim3", rc);
  out.keep.resize((size_t)n);
  out.S12 = r.S12_out;
  out.nInliers = r.n_inliers;
  return r.n_inliers;
}

}  // namespace ORB_SLAM2
