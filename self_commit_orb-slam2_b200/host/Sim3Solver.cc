#include "Sim3Solver.h"

#include <cstdio>
#include <cstdlib>
#include <mutex>

namespace ORB_SLAM2 {

// LoopClosing's thread: one handle for the process, grown on demand
static b2s_sim3solver* g_sim3Ransac = nullptr;
static int g_sim3RansacMatches = 0, g_sim3RansacSets = 0;
static std::mutex g_sim3RansacMutex;

int Sim3Ransac::Iterate(const Sim3RansacProblem& p, Sim3RansacResult& out) {
  std::lock_guard<std::mutex> lock(g_sim3RansacMutex);
  const int n = (int)(p.X1c.size() / 3), k = (int)(p.sets.size() / 3);
  if (!g_sim3Ransac || n > g_sim3RansacMatches || k > g_sim3RansacSets) {
    b2s_sim3solver_destroy(g_sim3Ransac);
    g_sim3Ransac = nullptr;
    g_sim3RansacMatches = n > 1024 ? n : 1024;
    g_sim3RansacSets = k > 300 ? k : 300;
    const char* e = getenv("B2S_DEVICE");
    const int rc = b2s_sim3solver_create(g_sim3RansacMatches, g_sim3RansacSets, 1, e ? atoi(e) : 0, &g_sim3Ransac);
    if (rc != B2S_OK) {
      fprintf(stderr, "Sim3Ransac::Iterate: libb200slam error %d: %s\n", rc, b2s_last_error());
      g_sim3Ransac = nullptr;
      return rc;
    }
  }
  b2s_sim3solver_problem q;
  q.n = n;
  q.X1c = p.X1c.data();
  q.X2c = p.X2c.data();
  q.sigma2_1 = p.sigma2_1.data();
  q.sigma2_2 = p.sigma2_2.data();
  for (int i = 0; i < 4; i++) {
    q.K1[i] = p.K1[i];
    q.K2[i] = p.K2[i];
  }
  q.fix_scale = p.fixScale ? 1 : 0;
  q.min_inliers = p.minInliers;
  q.max_its = p.maxIts;
  q.iterations_done = p.iterations;
  q.best_inliers = p.bestInliers;
  q.k = k;
  q.sets = p.sets.data();
  out.inliers.assign((size_t)(n > 0 ? n : 1), 0);
  b2s_sim3solver_result r;
  r.inliers = out.inliers.data();
  const int rc = b2s_sim3solver_iterate(g_sim3Ransac, 1, &q, &r);
  if (rc != B2S_OK) {
    fprintf(stderr, "Sim3Ransac::Iterate: libb200slam error %d: %s\n", rc, b2s_last_error());
    return rc;
  }
  out.inliers.resize((size_t)n);
  out.returned = r.returned != 0;
  for (int i = 0; i < 16; i++) out.T12[i] = r.T12[i];
  out.bestChanged = r.best_changed != 0;
  if (out.bestChanged) {
    for (int i = 0; i < 9; i++) out.R[i] = r.R[i];
    for (int i = 0; i < 3; i++) out.t[i] = r.t[i];
    out.s = r.s;
  }
  out.nInliers = r.n_inliers;
  out.noMore = r.no_more != 0;
  out.iterationsUsed = r.iterations_used;
  out.iterations = r.iterations_done;
  out.bestInliers = r.best_inliers;
  return B2S_OK;
}

}  // namespace ORB_SLAM2
