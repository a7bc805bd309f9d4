// TEST INFRASTRUCTURE — C entry points around the reference's own MapPoint::UpdateNormalAndDepth and
// LocalMapping::ProcessNewKeyFrame + MapPointCulling (src/LocalMapping.cc, src/KeyFrame.cc and src/MapPoint.cc compiled
// in place, unmodified, against the stand-ins of refshim/slam_stubs_kfinsert.h and the pinned OpenCV forms of
// refshim/refshim_cv_kfinsert.h).  Built into oracle/_ref/libref_kfinsert.so (git-ignored).
//
// One call builds an object graph from a problem of include/b200slam.h: the keyframes are constructed by the
// reference's constructor from a Frame holding each one's octaves, right coordinates (+1 / -1 from the stereo flags)
// and descriptors (a row of 8 floats holding the 32 bytes), with placement new into one buffer in table order, so that
// their address order is their table order; the camera centre Ow, mbBad and the current keyframe's slots are written
// through member pointers.  Every keyframe starts without connections; the current one as a new keyframe
// (mbFirstConnection).  The map points are built by the reference's constructor (mnFirstKFid comes from the keyframe
// it is given, whose mnId is set for the call), with their observations, nObs, mnFound, mnVisible, bad flag, reference
// keyframe and a given initial descriptor.  Map::EraseMapPoint (stubbed) records the points SetBadFlag sets bad.
//
// Built with -DB2S_ADAPTER_BUILD into _ref/libadapter_kfinsert.so, the entry point is adp_process_new_keyframe and the
// association and culling go through the product's b200::ProcessNewKeyFrame (host/adapters/LocalMapping_b200.cc).
#ifdef B2S_ADAPTER_BUILD
#define KFI_FN(name) adp_##name
#include "adapters/LocalMapping_b200.h"
#else
#define KFI_FN(name) ref_##name
#endif
#include <algorithm>
#include <chrono>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <list>
#include <memory>
#include <new>
#include <unordered_map>
#include <vector>

#include "LocalMapping.h"
#include "b200slam.h"

namespace ORB_SLAM2 {
// the reference's Frame.cc is not compiled: the default constructor and the statics the KeyFrame constructor reads
Frame::Frame() {}
long unsigned int Frame::nNextId = 0;
bool Frame::mbInitialComputations = true;
float Frame::cx, Frame::cy, Frame::fx, Frame::fy, Frame::invfx, Frame::invfy;
float Frame::mnMinX, Frame::mnMinY, Frame::mnMaxX, Frame::mnMaxY;
float Frame::mfGridElementWidthInv, Frame::mfGridElementHeightInv;
}  // namespace ORB_SLAM2

using namespace ORB_SLAM2;

namespace {

// member pointers to the protected state (include/KeyFrame.h:386-432, include/MapPoint.h:278-316)
struct KfAccess : KeyFrame {
  static std::map<KeyFrame*, int> KeyFrame::*conn() { return &KfAccess::mConnectedKeyFrameWeights; }
  static bool KeyFrame::*bad() { return &KfAccess::mbBad; }
  static cv::Mat KeyFrame::*center() { return &KfAccess::Ow; }
  static std::vector<MapPoint*> KeyFrame::*points() { return &KfAccess::mvpMapPoints; }
};
struct MpAccess : MapPoint {
  static std::map<KeyFrame*, size_t> MapPoint::*obs() { return &MpAccess::mObservations; }
  static bool MapPoint::*bad() { return &MpAccess::mbBad; }
  static KeyFrame* MapPoint::*refKF() { return &MpAccess::mpRefKF; }
  static int MapPoint::*found() { return &MpAccess::mnFound; }
  static int MapPoint::*visible() { return &MpAccess::mnVisible; }
  static cv::Mat MapPoint::*normal() { return &MpAccess::mNormalVector; }
  static cv::Mat MapPoint::*descriptor() { return &MpAccess::mDescriptor; }
  static float MapPoint::*minD() { return &MpAccess::mfMinDistance; }
  static float MapPoint::*maxD() { return &MpAccess::mfMaxDistance; }
};

struct Mapper : LocalMapping {
  Mapper(Map* pMap, bool mono) : LocalMapping(pMap, mono) {}
  void run(KeyFrame* pKF, const std::vector<MapPoint*>& recent) {
    mlpRecentAddedMapPoints.assign(recent.begin(), recent.end());
#ifdef B2S_ADAPTER_BUILD
    mpCurrentKeyFrame = pKF;
    pKF->ComputeBoW();
    rc = b200::ProcessNewKeyFrame(pKF, mpMap, mlpRecentAddedMapPoints, mbMonocular);
#else
    mlNewKeyFrames.push_back(pKF);
    ProcessNewKeyFrame();
    MapPointCulling();
#endif
  }
  std::list<MapPoint*>& recent() { return mlpRecentAddedMapPoints; }
  int rc = 0;
};

struct Graph {
  Map map;
  KeyFrameDatabase db;
  ORBVocabulary voc;
  unsigned char* buf = nullptr;
  int n = 0;
  std::vector<std::unique_ptr<MapPoint> > mps;
  std::unordered_map<const MapPoint*, int> mpIndex;
  KeyFrame* kf(int i) { return reinterpret_cast<KeyFrame*>(buf + (size_t)i * sizeof(KeyFrame)); }
  int index(const KeyFrame* k) const {
    return (int)((reinterpret_cast<const unsigned char*>(k) - buf) / sizeof(KeyFrame));
  }
  ~Graph() {
    mps.clear();
    for (int i = 0; i < n; i++) kf(i)->~KeyFrame();
    free(buf);
  }

  // keyframes: per-index arrays of length len[k]; octave / stereo / descriptor of each index
  void keyframes(int nkf, const float* centers, const uint8_t* bad, const std::vector<std::vector<int> >& oct,
                 const std::vector<std::vector<float> >& right, const std::vector<std::vector<uint8_t> >& desc,
                 const float* sf, int nlev) {
    buf = static_cast<unsigned char*>(aligned_alloc(alignof(KeyFrame), ((size_t)nkf * sizeof(KeyFrame) + 63) / 64 * 64));
    for (int i = 0; i < nkf; i++) {
      Frame F;
      F.mTcw = cv::Mat::eye(4, 4, CV_32F);
      F.N = (int)oct[(size_t)i].size();
      F.mvKeysUn.assign((size_t)F.N, cv::KeyPoint());
      for (int j = 0; j < F.N; j++) F.mvKeysUn[(size_t)j].octave = oct[(size_t)i][(size_t)j];
      F.mvuRight = right[(size_t)i];
      F.mvDepth.assign((size_t)F.N, -1.f);
      F.mDescriptors = cv::Mat(std::max(F.N, 1), 8, CV_32F);
      if (F.N) memcpy(F.mDescriptors.data, desc[(size_t)i].data(), 32 * (size_t)F.N);
      F.mvpMapPoints.assign((size_t)F.N, nullptr);
      F.mnScaleLevels = nlev;
      F.mvScaleFactors.assign(sf, sf + nlev);
      F.mpORBvocabulary = &voc;
      KeyFrame::nNextId = (long unsigned int)i;
      new (kf(i)) KeyFrame(F, &map, &db);
      n = i + 1;
      cv::Mat Ow(3, 1, CV_32F);
      for (int c = 0; c < 3; c++) Ow.at<float>(c) = centers[3 * i + c];
      kf(i)->*KfAccess::center() = Ow;
      kf(i)->*KfAccess::bad() = bad && bad[i];
    }
  }
  MapPoint* point(const float* pos, int64_t firstKf) {
    KeyFrame* k = kf(0);
    const long unsigned int id = k->mnId;
    k->mnId = (long unsigned int)firstKf;  // the constructor takes mnFirstKFid = pRefKF->mnId
    cv::Mat P(3, 1, CV_32F);
    for (int c = 0; c < 3; c++) P.at<float>(c) = pos[c];
    MapPoint* mp = new MapPoint(P, k, &map);
    k->mnId = id;
    mpIndex[mp] = (int)mps.size();
    mps.emplace_back(mp);
    return mp;
  }
};

}  // namespace

extern "C" {

#ifndef B2S_ADAPTER_BUILD
/* MapPoint::UpdateNormalAndDepth on every point of the problem (each observation gets its own index in its keyframe). */
int ref_update_normal_and_depth(const b2s_normal_depth_problem* p, b2s_normal_depth_result* r) {
  const int n = p->n_kf, O = p->obs_off[p->n_mp];
  std::vector<std::vector<int> > oct((size_t)n);
  std::vector<std::vector<float> > right((size_t)n);
  std::vector<std::vector<uint8_t> > desc((size_t)n);
  std::vector<int> idx((size_t)O);
  for (int o = 0; o < O; o++) {
    std::vector<int>& v = oct[(size_t)p->obs_kf[o]];
    idx[(size_t)o] = (int)v.size();
    v.push_back(p->obs_octave[o]);
  }
  for (int i = 0; i < n; i++) {
    right[(size_t)i].assign(oct[(size_t)i].size(), -1.f);
    desc[(size_t)i].assign(32 * oct[(size_t)i].size(), 0);
  }
  Graph g;
  g.keyframes(n, p->kf_center, nullptr, oct, right, desc, p->scale_factors, p->n_levels);
  for (int m = 0; m < p->n_mp; m++) {
    MapPoint* mp = g.point(p->mp_pos + 3 * (size_t)m, 0);
    mp->*MpAccess::bad() = p->mp_bad[m] != 0;
    mp->*MpAccess::refKF() = p->mp_ref[m] >= 0 && p->mp_ref[m] < n ? g.kf(p->mp_ref[m]) : nullptr;
    for (int o = p->obs_off[m]; o < p->obs_off[m + 1]; o++)
      (mp->*MpAccess::obs())[g.kf(p->obs_kf[o])] = (size_t)idx[(size_t)o];
    mp->UpdateNormalAndDepth();
    const cv::Mat& nv = mp->*MpAccess::normal();
    for (int c = 0; c < 3; c++) r->normal[3 * m + c] = nv.at<float>(c);
    r->min_dist[m] = mp->*MpAccess::minD();
    r->max_dist[m] = mp->*MpAccess::maxD();
    r->updated[m] = !p->mp_bad[m] && p->obs_off[m + 1] > p->obs_off[m];
  }
  return B2S_OK;
}
#endif

/* ProcessNewKeyFrame (BoW, connections and the map insertion stubbed or the reference's own) and MapPointCulling on the
 * graph of problem p; mp_desc_in (32 * n_mp): each point's mDescriptor on entry.  Outputs after the call: mp_nobs,
 * mp_bad, obs_alive (the entry observations), cur_idx (n_mp: the current keyframe's index in mObservations, -1), normal
 * (3 * n_mp), min_dist, max_dist, desc_out (32 * n_mp), slot_out (n_slots), recent_out / *n_recent (n_recent +
 * n_slots), erased / *n_erased (the points set bad, in SetBadFlag order), conn_* (CSR over n_kf, conn_cap: every
 * keyframe's mConnectedKeyFrameWeights).  *wall_ns (optional): the host wall time of the association and culling.
 * Returns B2S_OK, B2S_ERR_CAPACITY, or the adapter's error. */
int KFI_FN(process_new_keyframe)(const b2s_kfinsert_problem* p, const uint8_t* mp_desc_in, int32_t* mp_nobs,
                                 uint8_t* mp_bad, uint8_t* obs_alive, int32_t* cur_idx, float* normal, float* min_dist,
                                 float* max_dist, uint8_t* desc_out, int32_t* slot_out, int32_t* recent_out,
                                 int32_t* n_recent, int32_t* erased, int32_t* n_erased, int32_t* conn_off,
                                 int32_t* conn_kf, int32_t* conn_w, int conn_cap, double* wall_ns) {
  const int n = p->n_kf, O = p->obs_off[p->n_mp];
  std::vector<int> len((size_t)n, 0);
  len[(size_t)p->cur] = p->n_slots;
  for (int o = 0; o < O; o++) len[(size_t)p->obs_kf[o]] = std::max(len[(size_t)p->obs_kf[o]], p->obs_idx[o] + 1);
  std::vector<std::vector<int> > oct((size_t)n);
  std::vector<std::vector<float> > right((size_t)n);
  std::vector<std::vector<uint8_t> > desc((size_t)n);
  for (int i = 0; i < n; i++) {
    oct[(size_t)i].assign((size_t)len[(size_t)i], 0);
    right[(size_t)i].assign((size_t)len[(size_t)i], -1.f);
    desc[(size_t)i].assign(32 * (size_t)len[(size_t)i], 0);
  }
  for (int s = 0; s < p->n_slots; s++) {
    right[(size_t)p->cur][(size_t)s] = p->slot_stereo[s] ? 1.f : -1.f;
    memcpy(&desc[(size_t)p->cur][32 * (size_t)s], p->slot_desc + 32 * (size_t)s, 32);
  }
  for (int o = 0; o < O; o++) {
    const int k = p->obs_kf[o], i = p->obs_idx[o];
    oct[(size_t)k][(size_t)i] = p->obs_octave[o];
    if (k != p->cur) memcpy(&desc[(size_t)k][32 * (size_t)i], p->obs_desc + 32 * (size_t)o, 32);
  }
  Graph g;
  g.keyframes(n, p->kf_center, p->kf_bad, oct, right, desc, p->scale_factors, p->n_levels);
  for (int m = 0; m < p->n_mp; m++) {
    MapPoint* mp = g.point(p->mp_pos + 3 * (size_t)m, p->mp_first_kf[m]);
    mp->*MpAccess::bad() = p->mp_bad[m] != 0;
    mp->*MpAccess::refKF() = p->mp_ref[m] >= 0 && p->mp_ref[m] < n ? g.kf(p->mp_ref[m]) : nullptr;
    mp->nObs = p->mp_nobs[m];
    mp->*MpAccess::found() = p->mp_found[m];
    mp->*MpAccess::visible() = p->mp_visible[m];
    cv::Mat d(1, 8, CV_32F);
    memcpy(d.data, mp_desc_in + 32 * (size_t)m, 32);
    mp->*MpAccess::descriptor() = d;
    for (int o = p->obs_off[m]; o < p->obs_off[m + 1]; o++)
      (mp->*MpAccess::obs())[g.kf(p->obs_kf[o])] = (size_t)p->obs_idx[o];
  }
  KeyFrame* cur = g.kf(p->cur);
  KeyFrame::nNextId = (long unsigned int)n;
  cur->mnId = (long unsigned int)p->cur_id;
  std::vector<MapPoint*>& pts = cur->*KfAccess::points();
  for (int s = 0; s < p->n_slots; s++) pts[(size_t)s] = p->slot_mp[s] >= 0 ? g.mps[(size_t)p->slot_mp[s]].get() : nullptr;
  std::vector<MapPoint*> recent;
  for (int e = 0; e < p->n_recent; e++) recent.push_back(g.mps[(size_t)p->recent[e]].get());

  Mapper lm(&g.map, p->monocular != 0);
  const auto t0 = std::chrono::steady_clock::now();
  lm.run(cur, recent);
  if (wall_ns) *wall_ns = std::chrono::duration<double, std::nano>(std::chrono::steady_clock::now() - t0).count();
  if (lm.rc != 0) return lm.rc;

  int needConn = 0;
  for (int i = 0; i < n; i++) needConn += (int)(g.kf(i)->*KfAccess::conn()).size();
  if (needConn > conn_cap) return B2S_ERR_CAPACITY;
  for (int m = 0; m < p->n_mp; m++) {
    MapPoint* mp = g.mps[(size_t)m].get();
    mp_nobs[m] = mp->nObs;
    mp_bad[m] = mp->*MpAccess::bad();
    const std::map<KeyFrame*, size_t>& obs = mp->*MpAccess::obs();
    for (int o = p->obs_off[m]; o < p->obs_off[m + 1]; o++) obs_alive[o] = obs.count(g.kf(p->obs_kf[o])) != 0;
    const auto it = obs.find(cur);
    cur_idx[m] = it == obs.end() ? -1 : (int)it->second;
    const cv::Mat& nv = mp->*MpAccess::normal();
    for (int c = 0; c < 3; c++) normal[3 * m + c] = nv.at<float>(c);
    min_dist[m] = mp->*MpAccess::minD();
    max_dist[m] = mp->*MpAccess::maxD();
    memcpy(desc_out + 32 * (size_t)m, (mp->*MpAccess::descriptor()).data, 32);
  }
  for (int s = 0; s < p->n_slots; s++) slot_out[s] = pts[(size_t)s] ? g.mpIndex[pts[(size_t)s]] : -1;
  int nr = 0;
  for (MapPoint* mp : lm.recent()) recent_out[nr++] = g.mpIndex[mp];
  *n_recent = nr;
  *n_erased = (int)g.map.erasedPoints.size();
  for (size_t j = 0; j < g.map.erasedPoints.size(); j++) erased[j] = g.mpIndex[g.map.erasedPoints[j]];
  int cc = 0;
  conn_off[0] = 0;
  for (int i = 0; i < n; i++) {
    for (auto& kv : g.kf(i)->*KfAccess::conn()) {
      conn_kf[cc] = g.index(kv.first);
      conn_w[cc++] = kv.second;
    }
    conn_off[i + 1] = cc;
  }
  return B2S_OK;
}
}
