#include "PnPsolver.h"

#include <cstdio>
#include <cstdlib>
#include <mutex>

namespace ORB_SLAM2 {

// Tracking's thread: one handle for the process, grown on demand
static b2s_pnpsolver* g_pnpRansac = nullptr;
static int g_pnpRansacMatches = 0, g_pnpRansacSets = 0;
static std::mutex g_pnpRansacMutex;

int PnPRansac::Iterate(const PnPRansacProblem& p, PnPRansacResult& out) {
  std::lock_guard<std::mutex> lock(g_pnpRansacMutex);
  const int n = (int)(p.P3Dw.size() / 3), k = (int)(p.sets.size() / 4);
  if (!g_pnpRansac || n > g_pnpRansacMatches || k > g_pnpRansacSets) {
    b2s_pnpsolver_destroy(g_pnpRansac);
    g_pnpRansac = nullptr;
    g_pnpRansacMatches = n > 1024 ? n : 1024;
    g_pnpRansacSets = k > 300 ? k : 300;
    const char* e = getenv("B2S_DEVICE");
    const int rc = b2s_pnpsolver_create(g_pnpRansacMatches, g_pnpRansacSets, 1, e ? atoi(e) : 0, &g_pnpRansac);
    if (rc != B2S_OK) {
      fprintf(stderr, "PnPRansac::Iterate: libb200slam error %d: %s\n", rc, b2s_last_error());
      g_pnpRansac = nullptr;
      return rc;
    }
  }
  std::vector<uint8_t> bestIn((size_t)(n > 0 ? n : 1), 0);
  for (int i = 0; i < n && i < (int)p.bestMask.size(); i++) bestIn[(size_t)i] = p.bestMask[(size_t)i];
  b2s_pnpsolver_problem q;
  q.n = n;
  q.P3Dw = p.P3Dw.data();
  q.P2D = p.P2D.data();
  q.sigma2 = p.sigma2.data();
  q.fu = p.K[0];
  q.fv = p.K[1];
  q.uc = p.K[2];
  q.vc = p.K[3];
  q.th2 = p.th2;
  q.min_inliers = p.minInliers;
  q.max_its = p.maxIts;
  q.min_set = 4;
  q.iterations_done = p.iterations;
  q.best_inliers = p.bestInliers;
  q.best_Tcw = p.bestTcw;
  q.best_mask = bestIn.data();
  q.k = k;
  q.sets = p.sets.data();
  out.inliers.assign((size_t)(n > 0 ? n : 1), 0);
  out.bestMask.assign((size_t)(n > 0 ? n : 1), 0);
  b2s_pnpsolver_result r;
  r.inliers = out.inliers.data();
  r.best_mask = out.bestMask.data();
  const int rc = b2s_pnpsolver_iterate(g_pnpRansac, 1, &q, &r);
  if (rc != B2S_OK) {
    fprintf(stderr, "PnPRansac::Iterate: libb200slam error %d: %s\n", rc, b2s_last_error());
    return rc;
  }
  out.inliers.resize((size_t)n);
  out.bestMask.resize((size_t)n);
  out.returned = r.returned != 0;
  for (int i = 0; i < 16; i++) {
    out.Tcw[i] = r.Tcw[i];
    out.bestTcw[i] = r.best_Tcw[i];
  }
  out.nInliers = r.n_inliers;
  out.noMore = r.no_more != 0;
  out.iterationsUsed = r.iterations_used;
  out.iterations = r.iterations_done;
  out.bestInliers = r.best_inliers;
  out.bestChanged = r.best_changed != 0;
  return B2S_OK;
}

}  // namespace ORB_SLAM2
