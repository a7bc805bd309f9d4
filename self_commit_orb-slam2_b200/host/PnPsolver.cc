#include "PnPsolver.h"

#include <mutex>

#include "b2s_host.h"

namespace ORB_SLAM2 {

// Tracking's thread: one handle for the process, grown on demand
static b2s_host::Slot<b2s_pnpsolver, 2, b2s_pnpsolver_destroy> g_pnpRansac;

int PnPRansac::Iterate(const PnPRansacProblem& p, PnPRansacResult& out) {
  std::lock_guard<std::mutex> lock(g_pnpRansac.mutex);
  const int n = (int)(p.P3Dw.size() / 3), k = (int)(p.sets.size() / 4);
  int rc = g_pnpRansac.get({n, k}, {1024, 300}, [](const int* c, b2s_pnpsolver** h) {
    return b2s_pnpsolver_create(c[0], c[1], 1, b2s_host::device(), h);
  });
  if (rc != B2S_OK) {
    b2s_host::report("PnPRansac::Iterate", rc);
    return rc;
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
  rc = b2s_pnpsolver_iterate(g_pnpRansac.h, 1, &q, &r);
  if (rc != B2S_OK) {
    b2s_host::report("PnPRansac::Iterate", rc);
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
