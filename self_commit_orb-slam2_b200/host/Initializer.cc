#include "Initializer.h"

#include <cstdio>
#include <cstdlib>
#include <mutex>

namespace ORB_SLAM2 {

// Tracking's thread: one handle for the process, grown on demand
static b2s_init_solver* g_initSolver = nullptr;
static int g_initKeys = 0, g_initIterations = 0;
static std::mutex g_initMutex;

int MonoInitializer::Initialize(const InitProblem& p, InitResult& out) {
  std::lock_guard<std::mutex> lock(g_initMutex);
  const int n1 = (int)p.matches12.size(), n2 = (int)(p.kp2.size() / 2), it = (int)(p.sets.size() / 8);
  const int keys = n1 > n2 ? n1 : n2;
  if (!g_initSolver || keys > g_initKeys || it > g_initIterations) {
    b2s_init_destroy(g_initSolver);
    g_initSolver = nullptr;
    g_initKeys = keys > 4096 ? keys : 4096;
    g_initIterations = it > 200 ? it : 200;
    const char* e = getenv("B2S_DEVICE");
    const int rc = b2s_init_create(g_initKeys, g_initIterations, 1, e ? atoi(e) : 0, &g_initSolver);
    if (rc != B2S_OK) {
      fprintf(stderr, "MonoInitializer::Initialize: libb200slam error %d: %s\n", rc, b2s_last_error());
      g_initSolver = nullptr;
      return rc;
    }
  }
  b2s_init_problem q;
  q.n1 = n1;
  q.n2 = n2;
  q.kp1 = p.kp1.data();
  q.kp2 = p.kp2.data();
  q.matches12 = p.matches12.data();
  for (int i = 0; i < 9; i++) q.K[i] = p.K[i];
  q.sigma = p.sigma;
  q.iterations = it;
  q.sets = p.sets.data();
  out.p3d.assign((size_t)n1 * 3, 0.f);
  out.triangulated.assign((size_t)n1, 0);
  b2s_init_result r;
  r.p3d = out.p3d.data();
  r.triangulated = out.triangulated.data();
  r.inliers_h = r.inliers_f = nullptr;
  const int rc = b2s_initialize(g_initSolver, 1, &q, &r);
  if (rc != B2S_OK) {
    fprintf(stderr, "MonoInitializer::Initialize: libb200slam error %d: %s\n", rc, b2s_last_error());
    return rc;
  }
  out.ret = r.ret != 0;
  out.model = r.model;
  out.rtState = r.rt_state;
  for (int i = 0; i < 9; i++) out.R21[i] = r.R21[i];
  for (int i = 0; i < 3; i++) out.t21[i] = r.t21[i];
  if (!out.ret) {
    out.p3d.clear();
    out.triangulated.clear();
  }
  return B2S_OK;
}

}  // namespace ORB_SLAM2
