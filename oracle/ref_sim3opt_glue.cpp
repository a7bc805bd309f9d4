// TEST INFRASTRUCTURE — drives the reference's OWN Optimizer::OptimizeSim3 (src/Optimizer.cc:1364-1590, compiled in
// place, unmodified, with the vendored g2o and src/Converter.cc: the objects oracle/Makefile builds for
// libref_optimizer.so) on two stub keyframes and their map points, built from oracle/sim3opt_oracle.h's orc_sim3_graph.
// Built by `make -f sim3opt.mk` into _ref/libref_sim3opt.so; with -DB2S_ADAPTER_BUILD and the product's
// host/adapters/Optimizer_b200.cc instead of the reference's Optimizer.cc it is _ref/libadapter_sim3opt.so
// (adp_optimize_sim3).
//
// Mapping: pKF1 has mnId 0, pKF2 mnId 1; map point m has mnId m and, if mp_idx2[m] >= 0, one observation in pKF2.
#include <cstdint>
#include <cstring>
#include <vector>

#include "Optimizer.h"
#include "sim3opt_oracle.h"

namespace ORB_SLAM2 {
std::mutex MapPoint::mGlobalMutex;
float Frame::fx = 0, Frame::fy = 0, Frame::cx = 0, Frame::cy = 0;
}  // namespace ORB_SLAM2

using namespace ORB_SLAM2;

#ifdef B2S_ADAPTER_BUILD
#define ref_optimize_sim3 adp_optimize_sim3
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

int ref_optimize_sim3(const orc_sim3_graph* g, orc_sim3_graph_result* r) {
  KeyFrame kf[2];
  std::vector<MapPoint> mps((size_t)g->n_mp);
  const float* T[2] = {g->Tcw1, g->Tcw2};
  const float* K[2] = {g->K1, g->K2};
  const int nk[2] = {g->n1, g->n2};
  const float* kp[2] = {g->kp1, g->kp2};
  const int32_t* oct[2] = {g->oct1, g->oct2};
  const float* isg[2] = {g->inv_sigma2_1, g->inv_sigma2_2};
  for (int k = 0; k < 2; k++) {
    KeyFrame& F = kf[k];
    F.mnId = (unsigned long)k;
    F.Tcw = cv::Mat(4, 4, CV_32F);
    for (int i = 0; i < 16; i++) F.Tcw.at<float>(i / 4, i % 4) = T[k][i];
    F.mK = cv::Mat::eye(3, 3, CV_32F);
    F.mK.at<float>(0, 0) = K[k][0];
    F.mK.at<float>(1, 1) = K[k][1];
    F.mK.at<float>(0, 2) = K[k][2];
    F.mK.at<float>(1, 2) = K[k][3];
    F.mvKeysUn.resize((size_t)nk[k]);
    for (int i = 0; i < nk[k]; i++) {
      F.mvKeysUn[(size_t)i].pt.x = kp[k][2 * i];
      F.mvKeysUn[(size_t)i].pt.y = kp[k][2 * i + 1];
      if (oct[k][i] < 0 || oct[k][i] >= g->n_levels) return -2;
      F.mvKeysUn[(size_t)i].octave = oct[k][i];
    }
    F.mvInvLevelSigma2.assign(isg[k], isg[k] + g->n_levels);
  }
  for (int m = 0; m < g->n_mp; m++) {
    MapPoint& M = mps[(size_t)m];
    M.mnId = (unsigned long)m;
    M.mWorldPos = cv::Mat(3, 1, CV_32F);
    for (int i = 0; i < 3; i++) M.mWorldPos.at<float>(i) = g->points[3 * m + i];
    M.mbBad = g->mp_bad[m] != 0;
    if (g->mp_idx2[m] >= g->n2) return -3;
    if (g->mp_idx2[m] >= 0) M.mObservations[&kf[1]] = (size_t)g->mp_idx2[m];
  }
  auto mp = [&](int32_t i) -> MapPoint* { return (i >= 0 && i < g->n_mp) ? &mps[(size_t)i] : nullptr; };
  kf[0].mvpMapPoints.resize((size_t)g->n1);
  std::vector<MapPoint*> vpMatches1((size_t)g->n1);
  for (int i = 0; i < g->n1; i++) {
    kf[0].mvpMapPoints[(size_t)i] = mp(g->mp1[i]);
    vpMatches1[(size_t)i] = mp(g->matches1[i]);
  }
  g2o::Sim3 S12 = to_g2o(g->S12);
  g2o::b2s_lm_trace().clear();

  r->ret = Optimizer::OptimizeSim3(&kf[0], &kf[1], vpMatches1, S12, g->th2, g->fix_scale != 0);

  for (int i = 0; i < g->n1; i++) r->match_kept[i] = vpMatches1[(size_t)i] != nullptr;
  from_g2o(S12, &r->S12_out);
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
