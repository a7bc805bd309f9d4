// TEST INFRASTRUCTURE — drives the reference's OWN Optimizer::GlobalBundleAdjustemnt / BundleAdjustment
// (src/Optimizer.cc:55-341, compiled in place, unmodified, with the vendored g2o and src/Converter.cc: the objects
// oracle/Makefile builds for libref_optimizer.so) on an object graph built from oracle/gba_oracle.h's orc_gba_map.
// Built by `make -f gba.mk` into _ref/libref_gba.so; with -DB2S_ADAPTER_BUILD and the product's
// host/adapters/Optimizer_b200.cc instead of the reference's Optimizer.cc it is _ref/libadapter_gba.so (adp_global_ba).
//
// Mapping: keyframe k -> KeyFrame with mnId = k and map point m -> MapPoint with mnId = m, each allocated in one array, so
// that std::map<KeyFrame*, size_t> (a point's observations) iterates in keyframe index order.  The Map lists every
// keyframe and point, bad ones included, in index order.  Observation o of keyframe k is that keyframe's keypoint number
// o (octave = o), so mvInvLevelSigma2[kpUn.octave] returns the observation's inv_sigma2.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <set>
#include <utility>
#include <vector>

#include "Optimizer.h"
#include "gba_oracle.h"

namespace ORB_SLAM2 {
std::mutex MapPoint::mGlobalMutex;
float Frame::fx = 0, Frame::fy = 0, Frame::cx = 0, Frame::cy = 0;
}  // namespace ORB_SLAM2

using namespace ORB_SLAM2;

#ifdef B2S_ADAPTER_BUILD
#define ref_global_ba adp_global_ba
#endif

static cv::Mat mat44(const float* T) {
  cv::Mat m(4, 4, CV_32F);
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) m.at<float>(i, j) = T[i * 4 + j];
  return m;
}

extern "C" int ref_global_ba(const orc_gba_map* p, const volatile uint8_t* stop, orc_gba_map_result* r) {
  std::vector<KeyFrame> kfs((size_t)p->n_kf);
  std::vector<MapPoint> mps((size_t)p->n_mp);
  Map map;
  for (int k = 0; k < p->n_kf; k++) {
    KeyFrame& kf = kfs[(size_t)k];
    kf.mnId = (unsigned long)k;
    kf.fx = p->fx;
    kf.fy = p->fy;
    kf.cx = p->cx;
    kf.cy = p->cy;
    kf.mbf = p->bf;
    kf.Tcw = mat44(p->Tcw + 16 * k);
    kf.mbBad = p->kf_bad[k] != 0;
    map.mvKFs.push_back(&kf);
  }
  for (int m = 0; m < p->n_mp; m++) {
    MapPoint& mp = mps[(size_t)m];
    mp.mnId = (unsigned long)m;
    mp.mWorldPos = cv::Mat(3, 1, CV_32F);
    for (int i = 0; i < 3; i++) mp.mWorldPos.at<float>(i) = p->points[3 * m + i];
    mp.mbBad = p->mp_bad[m] != 0;
    map.mvMPs.push_back(&mp);
  }
  std::set<std::pair<int, int> > seen;
  for (int e = 0; e < p->n_obs; e++) {
    const orc_ba_edge& ob = p->obs[e];
    if (ob.kf < 0 || ob.kf >= p->n_kf || ob.mp < 0 || ob.mp >= p->n_mp) return -4;
    if (e > 0 && ob.mp < p->obs[e - 1].mp) return -5;
    if (!seen.insert(std::make_pair(ob.kf, ob.mp)).second) return -6;
    KeyFrame& kf = kfs[(size_t)ob.kf];
    const size_t idx = kf.mvKeysUn.size();
    cv::KeyPoint kp(ob.obs[0], ob.obs[1], 31.f);
    kp.octave = (int)idx;
    kf.mvKeysUn.push_back(kp);
    kf.mvuRight.push_back(ob.obs[2]);
    kf.mvInvLevelSigma2.push_back(ob.inv_sigma2);
    mps[(size_t)ob.mp].mObservations[&kf] = idx;
  }
  g2o::b2s_lm_trace().clear();

  Optimizer::GlobalBundleAdjustemnt(&map, p->iterations, (bool*)const_cast<uint8_t*>(stop), (unsigned long)p->loop_kf,
                                    p->robust != 0);

  for (int k = 0; k < p->n_kf; k++) {
    KeyFrame& kf = kfs[(size_t)k];
    r->kf_gba[k] = kf.mTcwGBA.empty() ? 0 : 1;
    const cv::Mat& T = r->kf_gba[k] ? kf.mTcwGBA : kf.Tcw;
    for (int i = 0; i < 4; i++)
      for (int j = 0; j < 4; j++) r->Tcw_out[16 * k + 4 * i + j] = T.at<float>(i, j);
    r->kf_ba_global[k] = kf.mnBAGlobalForKF;
  }
  for (int m = 0; m < p->n_mp; m++) {
    MapPoint& mp = mps[(size_t)m];
    r->mp_gba[m] = mp.mPosGBA.empty() ? 0 : 1;
    const cv::Mat& X = r->mp_gba[m] ? mp.mPosGBA : mp.mWorldPos;
    for (int i = 0; i < 3; i++) r->points_out[3 * m + i] = X.at<float>(i);
    r->mp_ba_global[m] = mp.mnBAGlobalForKF;
    r->mp_updates[m] = mp.nUpdates;
  }
  // LM iterations of this thread -> accept(1) / reject(0) per trial, -1 terminated (empty for the adapter build)
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
