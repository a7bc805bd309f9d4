#include "Optimizer.h"

#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <stdexcept>

namespace ORB_SLAM2 {

// LocalBA runs on the LocalMapping thread only (src/LocalMapping.cc:123): one solver, grown on demand.
static b2s_ba_solver* g_solver = nullptr;
static int g_kf = 0, g_mp = 0, g_e = 0;
static std::mutex g_mutex;

void Optimizer::LocalBundleAdjustment(const LocalBAWindow& w, bool* pbStopFlag, LocalBAResult& out) {
  std::lock_guard<std::mutex> lock(g_mutex);
  const int nKF = (int)w.fixed.size(), nMP = (int)w.points.size() / 3, nE = (int)w.edges.size();
  if (!g_solver || nKF > g_kf || nMP > g_mp || nE > g_e) {
    b2s_ba_destroy(g_solver);
    g_solver = nullptr;
    g_kf = nKF > 64 ? nKF : 64;
    g_mp = nMP > 8192 ? nMP : 8192;
    g_e = nE > 65536 ? nE : 65536;
    const char* e = getenv("B2S_DEVICE");
    int rc = b2s_ba_create(g_kf, g_mp, g_e, 1, e ? atoi(e) : 0, &g_solver);
    if (rc != B2S_OK) {
      fprintf(stderr, "Optimizer::LocalBundleAdjustment: libb200slam error %d: %s\n", rc, b2s_last_error());
      throw std::runtime_error(b2s_last_error());
    }
  }
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
  int rc = b2s_local_ba(g_solver, &p, (const volatile uint8_t*)pbStopFlag, &r);
  if (rc == B2S_ERR_ABORTED) {
    out.aborted = true;
    return;
  }
  if (rc != B2S_OK) {
    fprintf(stderr, "Optimizer::LocalBundleAdjustment: libb200slam error %d: %s\n", rc, b2s_last_error());
    throw std::runtime_error(b2s_last_error());
  }
}

// PoseOptimization runs on the Tracking thread: its own solver handle (handles are not shared between threads)
static b2s_ba_solver* g_poseSolver = nullptr;
static std::mutex g_poseMutex;

int Optimizer::PoseOptimization(const PoseProblem& f, float TcwOut[16], std::vector<uint8_t>& outlier) {
  std::lock_guard<std::mutex> lock(g_poseMutex);
  if (!g_poseSolver) {
    const char* e = getenv("B2S_DEVICE");
    int rc = b2s_ba_create(4, 16, 64, 1, e ? atoi(e) : 0, &g_poseSolver);
    if (rc != B2S_OK) {
      fprintf(stderr, "Optimizer::PoseOptimization: libb200slam error %d: %s\n", rc, b2s_last_error());
      throw std::runtime_error(b2s_last_error());
    }
  }
  const int N = (int)f.hasMapPoint.size();
  outlier.assign(N > 0 ? N : 1, 0);
  b2s_pose_problem p;
  p.Tcw = f.Tcw; p.n = N; p.has_mp = f.hasMapPoint.data(); p.Xw = f.Xw.data(); p.kpx = f.kpx.data(); p.kpy = f.kpy.data();
  p.uright = f.uRight.data(); p.inv_sigma2 = f.invSigma2.data();
  p.fx = f.fx; p.fy = f.fy; p.cx = f.cx; p.cy = f.cy; p.bf = f.bf;
  b2s_pose_result r;
  r.Tcw_out = TcwOut; r.outlier = outlier.data(); r.trace = nullptr; r.n_inliers = 0; r.n_trials = 0;
  int rc = b2s_pose_optimization(g_poseSolver, &p, &r);
  if (rc != B2S_OK) {
    fprintf(stderr, "Optimizer::PoseOptimization: libb200slam error %d: %s\n", rc, b2s_last_error());
    throw std::runtime_error(b2s_last_error());
  }
  outlier.resize(N);
  return r.n_inliers;
}

// Global BA runs on LoopClosing's GBA thread (and once for the monocular initial map): its own handle, grown on demand
static b2s_gba_solver* g_gbaSolver = nullptr;
static int g_gkf = 0, g_gmp = 0, g_ge = 0;
static std::mutex g_gbaMutex;

void Optimizer::BundleAdjustment(const GlobalBAMap& m, int nIterations, bool* pbStopFlag, bool bRobust,
                                 GlobalBAResult& out) {
  std::lock_guard<std::mutex> lock(g_gbaMutex);
  const int nKF = (int)m.fixed.size(), nMP = (int)m.points.size() / 3, nE = (int)m.edges.size();
  if (!g_gbaSolver || nKF > g_gkf || nMP > g_gmp || nE > g_ge) {
    b2s_gba_destroy(g_gbaSolver);
    g_gbaSolver = nullptr;
    g_gkf = nKF > 256 ? nKF : 256;
    g_gmp = nMP > 32768 ? nMP : 32768;
    g_ge = nE > 262144 ? nE : 262144;
    const char* e = getenv("B2S_DEVICE");
    int rc = b2s_gba_create(g_gkf, g_gmp, g_ge, e ? atoi(e) : 0, &g_gbaSolver);
    if (rc != B2S_OK) {
      fprintf(stderr, "Optimizer::BundleAdjustment: libb200slam error %d: %s\n", rc, b2s_last_error());
      throw std::runtime_error(b2s_last_error());
    }
  }
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
  int rc = b2s_global_ba(g_gbaSolver, &p, (const volatile uint8_t*)pbStopFlag, &r);
  if (rc != B2S_OK) {
    fprintf(stderr, "Optimizer::BundleAdjustment: libb200slam error %d: %s\n", rc, b2s_last_error());
    throw std::runtime_error(b2s_last_error());
  }
  out.included.resize(nMP);
}

// The essential graph runs on LoopClosing's thread: its own handle, grown on demand
static b2s_eg_solver* g_egSolver = nullptr;
static int g_ekf = 0, g_ee = 0, g_emp = 0;
static std::mutex g_egMutex;

void Optimizer::OptimizeEssentialGraph(const EssentialGraph& g, EssentialGraphResult& out) {
  std::lock_guard<std::mutex> lock(g_egMutex);
  const int nKF = (int)g.Siw.size(), nE = (int)g.edges.size(), nMP = (int)g.refKF.size();
  if (!g_egSolver || nKF > g_ekf || nE > g_ee || nMP > g_emp) {
    b2s_eg_destroy(g_egSolver);
    g_egSolver = nullptr;
    g_ekf = nKF > 1024 ? nKF : 1024;
    g_ee = nE > 16384 ? nE : 16384;
    g_emp = nMP > 65536 ? nMP : 65536;
    const char* e = getenv("B2S_DEVICE");
    int rc = b2s_eg_create(g_ekf, g_ee, g_emp, e ? atoi(e) : 0, &g_egSolver);
    if (rc != B2S_OK) {
      fprintf(stderr, "Optimizer::OptimizeEssentialGraph: libb200slam error %d: %s\n", rc, b2s_last_error());
      throw std::runtime_error(b2s_last_error());
    }
  }
  b2s_eg_problem p;
  p.n_kf = nKF; p.Siw = g.Siw.data(); p.fixed_kf = g.fixedKF; p.fix_scale = g.fixScale ? 1 : 0;
  p.n_edges = nE; p.edges = g.edges.data();
  p.n_mp = nMP; p.points = g.points.data(); p.ref_kf = g.refKF.data();
  out.Tcw.assign((size_t)(nKF > 0 ? nKF : 1) * 16, 0.f);
  out.points.assign((size_t)(nMP > 0 ? nMP : 1) * 3, 0.f);
  b2s_eg_result r;
  r.Tcw_out = out.Tcw.data(); r.points_out = out.points.data(); r.trace = nullptr;
  r.chi2_initial = r.chi2_final = 0; r.n_trials = 0;
  int rc = b2s_optimize_essential_graph(g_egSolver, &p, &r);
  if (rc != B2S_OK) {
    fprintf(stderr, "Optimizer::OptimizeEssentialGraph: libb200slam error %d: %s\n", rc, b2s_last_error());
    throw std::runtime_error(b2s_last_error());
  }
  out.Tcw.resize((size_t)nKF * 16);
  out.points.resize((size_t)nMP * 3);
}

// OptimizeSim3 runs on LoopClosing's thread: its own handle, grown on demand
static b2s_sim3opt_solver* g_s3Solver = nullptr;
static int g_s3n = 0;
static std::mutex g_s3Mutex;

int Optimizer::OptimizeSim3(const Sim3Problem& p, Sim3Result& out) {
  std::lock_guard<std::mutex> lock(g_s3Mutex);
  const int n = (int)p.invSigma2_1.size();
  if (!g_s3Solver || n > g_s3n) {
    b2s_sim3opt_destroy(g_s3Solver);
    g_s3Solver = nullptr;
    g_s3n = n > 4096 ? n : 4096;
    const char* e = getenv("B2S_DEVICE");
    int rc = b2s_sim3opt_create(g_s3n, 1, e ? atoi(e) : 0, &g_s3Solver);
    if (rc != B2S_OK) {
      fprintf(stderr, "Optimizer::OptimizeSim3: libb200slam error %d: %s\n", rc, b2s_last_error());
      throw std::runtime_error(b2s_last_error());
    }
  }
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
  int rc = b2s_optimize_sim3(g_s3Solver, 1, &q, &r);
  if (rc != B2S_OK) {
    fprintf(stderr, "Optimizer::OptimizeSim3: libb200slam error %d: %s\n", rc, b2s_last_error());
    throw std::runtime_error(b2s_last_error());
  }
  out.keep.resize((size_t)n);
  out.S12 = r.S12_out;
  out.nInliers = r.n_inliers;
  return r.n_inliers;
}

}  // namespace ORB_SLAM2
