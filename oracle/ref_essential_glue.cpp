// TEST INFRASTRUCTURE — drives the reference's OWN Optimizer::OptimizeEssentialGraph (src/Optimizer.cc:1017-1339,
// compiled in place, unmodified, with the vendored g2o and src/Converter.cc: the objects oracle/Makefile builds for
// libref_optimizer.so) on an object graph built from oracle/essential_oracle.h's orc_eg_map.  Built by
// `make -f essential.mk` into _ref/libref_essential.so; with -DB2S_ADAPTER_BUILD and the product's
// host/adapters/Optimizer_b200.cc instead of the reference's Optimizer.cc it is _ref/libadapter_essential.so
// (adp_essential_graph).  Also exports g2o::Sim3 of the reference's header (ref_sim3_*).
//
// Mapping: keyframe k -> KeyFrame with mnId = k and map point m -> MapPoint with mnId = m, each allocated in one array,
// so that std::map<KeyFrame*, ...> and std::set<KeyFrame*> (LoopConnections, CorrectedSim3, children, loop edges) iterate
// in keyframe index order.  The Map lists the non-bad keyframes (bad ones are reachable only as covisible neighbours)
// and every map point, in index order.
#include <cstdint>
#include <cstring>
#include <vector>

#include "Optimizer.h"
#include "essential_oracle.h"

namespace ORB_SLAM2 {
std::mutex MapPoint::mGlobalMutex;
float Frame::fx = 0, Frame::fy = 0, Frame::cx = 0, Frame::cy = 0;
}  // namespace ORB_SLAM2

using namespace ORB_SLAM2;

#ifdef B2S_ADAPTER_BUILD
#define ref_essential_graph adp_essential_graph
#endif

static g2o::Sim3 to_g2o(const orc_sim3& s) {
  g2o::Sim3 r;
  for (int i = 0; i < 8; i++) r[i] = (&s.q[0])[i];
  return r;
}
static void from_g2o(const g2o::Sim3& s, orc_sim3* o) {
  for (int i = 0; i < 8; i++) (&o->q[0])[i] = s[i];
}

extern "C" {

void ref_sim3_exp(const double* u, orc_sim3* o) {
  g2o::Vector7d v;
  for (int i = 0; i < 7; i++) v[i] = u[i];
  from_g2o(g2o::Sim3(v), o);
}
void ref_sim3_log(const orc_sim3* a, double* o) {
  const g2o::Vector7d v = to_g2o(*a).log();
  for (int i = 0; i < 7; i++) o[i] = v[i];
}
void ref_sim3_mul(const orc_sim3* a, const orc_sim3* b, orc_sim3* o) { from_g2o(to_g2o(*a) * to_g2o(*b), o); }
void ref_sim3_inverse(const orc_sim3* a, orc_sim3* o) { from_g2o(to_g2o(*a).inverse(), o); }
void ref_sim3_map(const orc_sim3* a, const double* X, double* o) {
  Eigen::Vector3d x(X[0], X[1], X[2]);
  const Eigen::Vector3d y = to_g2o(*a).map(x);
  for (int i = 0; i < 3; i++) o[i] = y[i];
}

int ref_essential_graph(const orc_eg_map* p, orc_eg_map_result* r) {
  const int nk = p->n_kf, nm = p->n_mp;
  std::vector<KeyFrame> kfs((size_t)nk);
  std::vector<MapPoint> mps((size_t)nm);
  Map map;
  auto kf = [&](int k) -> KeyFrame* { return (k >= 0 && k < nk) ? &kfs[(size_t)k] : nullptr; };
  for (int k = 0; k < nk; k++) {
    KeyFrame& K = kfs[(size_t)k];
    K.mnId = (unsigned long)k;
    K.Tcw = cv::Mat(4, 4, CV_32F);
    for (int i = 0; i < 16; i++) K.Tcw.at<float>(i / 4, i % 4) = p->Tcw[16 * k + i];
    K.mbBad = p->kf_bad[k] != 0;
    if (!K.mbBad) map.mvKFs.push_back(&K);
  }
  for (int k = 0; k < nk; k++) {
    if (p->parent[k] < -1 || p->parent[k] >= nk) return -2;
    KeyFrame* par = kf(p->parent[k]);
    kfs[(size_t)k].mpParent = par;
    if (par && !kfs[(size_t)k].mbBad) par->mspChildren.insert(&kfs[(size_t)k]);
  }
  for (int i = 0; i < p->n_loop; i++) {
    KeyFrame *a = kf(p->loop_edges[2 * i]), *b = kf(p->loop_edges[2 * i + 1]);
    if (!a || !b) return -3;
    a->mspLoopEdges.insert(b);
  }
  for (int i = 0; i < p->n_cov; i++) {
    KeyFrame *a = kf(p->cov[3 * i]), *b = kf(p->cov[3 * i + 1]);
    if (!a || !b) return -4;
    a->mvCovisible.push_back(b);
    a->mWeights[b] = p->cov[3 * i + 2];
  }
  LoopClosing::KeyFrameAndPose corrected, noncorrected;
  for (int i = 0; i < p->n_corr; i++) {
    KeyFrame* a = kf(p->corr_kf[i]);
    if (!a) return -5;
    corrected[a] = to_g2o(p->corr_S[i]);
    noncorrected[a] = to_g2o(p->noncorr_S[i]);
  }
  std::map<KeyFrame*, std::set<KeyFrame*> > connections;
  for (int i = 0; i < p->n_conn; i++) {
    KeyFrame *a = kf(p->conn[2 * i]), *b = kf(p->conn[2 * i + 1]);
    if (!a || !b) return -6;
    connections[a].insert(b);
  }
  for (int m = 0; m < nm; m++) {
    MapPoint& M = mps[(size_t)m];
    M.mnId = (unsigned long)m;
    M.mWorldPos = cv::Mat(3, 1, CV_32F);
    for (int i = 0; i < 3; i++) M.mWorldPos.at<float>(i) = p->points[3 * m + i];
    M.mbBad = p->mp_bad[m] != 0;
    M.mpRefKF = kf(p->mp_ref[m]);
    M.mnCorrectedByKF = (unsigned long)p->mp_corrected_by[m];
    M.mnCorrectedReference = (unsigned long)p->mp_corrected_ref[m];
    map.mvMPs.push_back(&M);
  }
  KeyFrame *loop = kf(p->loop_kf), *cur = kf(p->cur_kf);
  if (!loop || !cur) return -7;
  g2o::b2s_lm_trace().clear();

  const bool fixScale = p->fix_scale != 0;
  Optimizer::OptimizeEssentialGraph(&map, loop, cur, noncorrected, corrected, connections, fixScale);

  for (int k = 0; k < nk; k++)
    for (int i = 0; i < 16; i++) r->Tcw_out[16 * k + i] = kfs[(size_t)k].Tcw.at<float>(i / 4, i % 4);
  for (int m = 0; m < nm; m++) {
    for (int i = 0; i < 3; i++) r->points_out[3 * m + i] = mps[(size_t)m].mWorldPos.at<float>(i);
    r->mp_updates[m] = mps[(size_t)m].nUpdates;
  }
  std::vector<g2o::B2sLmIteration>& it = g2o::b2s_lm_trace();
  int n = 0;
  for (size_t i = 0; i < it.size(); i++)
    for (int k = 0; k < it[i].trials; k++) {
      const int acc = (k == it[i].trials - 1) ? it[i].last_accepted : 0;
      if (r->trace && n < 255) r->trace[n] = acc;
      n++;
    }
  if (r->trace) r->trace[n < 255 ? n : 255] = -1;
  r->n_trials = n;
  return 0;
}

}  // extern "C"
