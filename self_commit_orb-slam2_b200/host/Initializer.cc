#include "Initializer.h"

#include <mutex>

#include "b2s_host.h"

namespace ORB_SLAM2 {

// Tracking's thread: one handle for the process, grown on demand
static b2s_host::Slot<b2s_init_solver, 2, b2s_init_destroy> g_init;

int MonoInitializer::Initialize(const InitProblem& p, InitResult& out) {
  std::lock_guard<std::mutex> lock(g_init.mutex);
  const int n1 = (int)p.matches12.size(), n2 = (int)(p.kp2.size() / 2), it = (int)(p.sets.size() / 8);
  int rc = g_init.get({n1 > n2 ? n1 : n2, it}, {4096, 200}, [](const int* c, b2s_init_solver** h) {
    return b2s_init_create(c[0], c[1], 1, b2s_host::device(), h);
  });
  if (rc != B2S_OK) {
    b2s_host::report("MonoInitializer::Initialize", rc);
    return rc;
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
  rc = b2s_initialize(g_init.h, 1, &q, &r);
  if (rc != B2S_OK) {
    b2s_host::report("MonoInitializer::Initialize", rc);
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
