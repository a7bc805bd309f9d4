// TEST INFRASTRUCTURE — C entry point around the reference's own LocalMapping::KeyFrameCulling (src/LocalMapping.cc,
// src/KeyFrame.cc and src/MapPoint.cc compiled in place, unmodified, against the stand-ins of
// refshim/slam_stubs_localmapping.h).  Built into oracle/_ref/libref_localmapping.so (git-ignored).
//
// One call builds an object graph from a b2s_culling_problem plus a spanning tree and connection maps: the keyframes
// are constructed by the reference's constructor from a Frame holding each one's slots, octaves, right coordinates
// (+1 / -1 from obs_stereo) and depths, with placement new into one buffer in table order (so that their address order
// is their table order); the map points by the reference's constructor, with the problem's observations, nObs and bad
// flags, and no reference keyframe (EraseObservation's re-pointing of mpRefKF is then never taken).  The per-index
// arrays are the union of what the slots and the observations say, which the caller keeps consistent.  Protected state
// is written and read through member pointers taken in derived classes.  Then LocalMapping::KeyFrameCulling runs with
// the given current keyframe, whose ordered covisibility list is set to local_kf.  Map::EraseKeyFrame (stubbed) records
// the culls in the order SetBadFlag makes them.
//
// Built with -DB2S_ADAPTER_BUILD into _ref/libadapter_culling.so, the entry point is adp_keyframe_culling and the call
// goes through the product's b200::KeyFrameCulling (host/adapters/LocalMapping_b200.cc).
#ifdef B2S_ADAPTER_BUILD
#define CULL_FN(name) adp_##name
#include "adapters/LocalMapping_b200.h"
#else
#define CULL_FN(name) ref_##name
#endif
#include <algorithm>
#include <chrono>
#include <cstdint>
#include <cstdlib>
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
  static std::vector<KeyFrame*> KeyFrame::*ordKf() { return &KfAccess::mvpOrderedConnectedKeyFrames; }
  static std::vector<int> KeyFrame::*ordW() { return &KfAccess::mvOrderedWeights; }
  static KeyFrame* KeyFrame::*parent() { return &KfAccess::mpParent; }
  static std::set<KeyFrame*> KeyFrame::*children() { return &KfAccess::mspChildrens; }
  static bool KeyFrame::*first() { return &KfAccess::mbFirstConnection; }
  static bool KeyFrame::*notErase() { return &KfAccess::mbNotErase; }
  static bool KeyFrame::*toBeErased() { return &KfAccess::mbToBeErased; }
  static bool KeyFrame::*bad() { return &KfAccess::mbBad; }
  static std::vector<MapPoint*> KeyFrame::*points() { return &KfAccess::mvpMapPoints; }
};
struct MpAccess : MapPoint {
  static std::map<KeyFrame*, size_t> MapPoint::*obs() { return &MpAccess::mObservations; }
  static bool MapPoint::*bad() { return &MpAccess::mbBad; }
  static KeyFrame* MapPoint::*refKF() { return &MpAccess::mpRefKF; }
};

struct Culler : LocalMapping {
  Culler(Map* pMap, bool mono) : LocalMapping(pMap, mono) {}
  void cull(KeyFrame* pKF) {
    mpCurrentKeyFrame = pKF;
    KeyFrameCulling();
  }
};

struct Graph {
  Map map;
  KeyFrameDatabase db;
  unsigned char* buf = nullptr;
  int n = 0;
  std::vector<std::unique_ptr<MapPoint> > mps;
  KeyFrame* kf(int i) { return reinterpret_cast<KeyFrame*>(buf + (size_t)i * sizeof(KeyFrame)); }
  int index(const KeyFrame* k) const {
    return (int)((reinterpret_cast<const unsigned char*>(k) - buf) / sizeof(KeyFrame));
  }
  ~Graph() {
    mps.clear();
    for (int i = 0; i < n; i++) kf(i)->~KeyFrame();
    free(buf);
  }
};

}  // namespace

extern "C" {

/* cur: the current keyframe (a table index, not in local_kf); parent (n_kf): mpParent's index, -1 for NULL; conn_off /
 * conn_kf / conn_w (CSR over n_kf, keyframe indices ascending): mConnectedKeyFrameWeights (each keyframe's ordered list
 * is UpdateBestCovisibles of it, cur's is local_kf).  The result's n_mps and n_redundant are -1 (the reference keeps no
 * counts).  Outputs after the call: kf_bad / kf_to_be_erased (n_kf), parent_out (n_kf), erased (n_kf) with *n_erased:
 * the culled keyframes in SetBadFlag order, conn_out_* (CSR, conn_cap) and child_out_* (CSR, child_cap).  *wall_ns
 * (optional): the host wall time of the culling alone.  Returns B2S_OK or B2S_ERR_CAPACITY. */
int CULL_FN(keyframe_culling)(const b2s_culling_problem* p, int cur, const int32_t* parent, const int32_t* conn_off,
                              const int32_t* conn_kf, const int32_t* conn_w, b2s_culling_result* r, uint8_t* kf_bad,
                              uint8_t* kf_to_be_erased, int32_t* parent_out, int32_t* erased, int32_t* n_erased,
                              int32_t* conn_out_off, int32_t* conn_out_kf, int32_t* conn_out_w, int conn_cap,
                              int32_t* child_out_off, int32_t* child_out_kf, int child_cap, double* wall_ns) {
  const int n = p->n_kf;
  std::vector<int> localPos((size_t)n, -1), len((size_t)n, 0);
  for (int l = 0; l < p->n_local; l++) {
    localPos[(size_t)p->local_kf[l]] = l;
    len[(size_t)p->local_kf[l]] = p->slot_off[l + 1] - p->slot_off[l];
  }
  for (int o = 0; o < p->obs_off[p->n_mp]; o++)
    len[(size_t)p->obs_kf[o]] = std::max(len[(size_t)p->obs_kf[o]], p->obs_idx[o] + 1);
  // each keyframe's per-index arrays: octave, mvuRight, mvDepth
  std::vector<std::vector<int> > oct((size_t)n);
  std::vector<std::vector<float> > right((size_t)n), depth((size_t)n);
  for (int i = 0; i < n; i++) {
    oct[(size_t)i].assign((size_t)len[(size_t)i], 0);
    right[(size_t)i].assign((size_t)len[(size_t)i], -1.f);
    depth[(size_t)i].assign((size_t)len[(size_t)i], -1.f);
  }
  for (int l = 0; l < p->n_local; l++)
    for (int s = p->slot_off[l]; s < p->slot_off[l + 1]; s++) {
      oct[(size_t)p->local_kf[l]][(size_t)(s - p->slot_off[l])] = p->slot_octave[s];
      if (!p->monocular) depth[(size_t)p->local_kf[l]][(size_t)(s - p->slot_off[l])] = p->slot_depth[s];
    }
  for (int o = 0; o < p->obs_off[p->n_mp]; o++) {
    oct[(size_t)p->obs_kf[o]][(size_t)p->obs_idx[o]] = p->obs_octave[o];
    right[(size_t)p->obs_kf[o]][(size_t)p->obs_idx[o]] = p->obs_stereo[o] ? 1.f : -1.f;
  }
  Graph g;
  g.buf = static_cast<unsigned char*>(aligned_alloc(alignof(KeyFrame), ((size_t)n * sizeof(KeyFrame) + 63) / 64 * 64));
  for (int i = 0; i < n; i++) {
    Frame F;
    F.mTcw = cv::Mat::eye(4, 4, CV_32F);
    F.mThDepth = p->th_depth[i];
    F.N = len[(size_t)i];
    F.mvKeysUn.assign((size_t)F.N, cv::KeyPoint());
    for (int j = 0; j < F.N; j++) F.mvKeysUn[(size_t)j].octave = oct[(size_t)i][(size_t)j];
    F.mvuRight = right[(size_t)i];
    F.mvDepth = depth[(size_t)i];
    F.mvpMapPoints.assign((size_t)F.N, nullptr);
    KeyFrame::nNextId = (long unsigned int)p->kf_id[i];  // the constructor takes mnId = nNextId++
    new (g.kf(i)) KeyFrame(F, &g.map, &g.db);
    g.n = i + 1;
  }
  for (int m = 0; m < p->n_mp; m++) {
    MapPoint* mp = new MapPoint(cv::Mat::zeros(3, 1, CV_32F), g.kf(0), &g.map);
    g.mps.emplace_back(mp);
    mp->*MpAccess::refKF() = nullptr;
    mp->*MpAccess::bad() = p->mp_bad[m] != 0;
    mp->nObs = p->mp_nobs[m];
    for (int o = p->obs_off[m]; o < p->obs_off[m + 1]; o++) (mp->*MpAccess::obs())[g.kf(p->obs_kf[o])] = (size_t)p->obs_idx[o];
  }
  std::unordered_map<const MapPoint*, int> mpIndex;
  for (int m = 0; m < p->n_mp; m++) mpIndex[g.mps[(size_t)m].get()] = m;
  for (int l = 0; l < p->n_local; l++) {
    std::vector<MapPoint*>& pts = g.kf(p->local_kf[l])->*KfAccess::points();
    for (int s = p->slot_off[l]; s < p->slot_off[l + 1]; s++)
      pts[(size_t)(s - p->slot_off[l])] = p->slot_mp[s] >= 0 ? g.mps[(size_t)p->slot_mp[s]].get() : nullptr;
  }
  for (int i = 0; i < n; i++) {
    KeyFrame* k = g.kf(i);
    std::map<KeyFrame*, int>& conn = k->*KfAccess::conn();
    for (int j = conn_off[i]; j < conn_off[i + 1]; j++) conn[g.kf(conn_kf[j])] = conn_w[j];
    k->UpdateBestCovisibles();
    k->*KfAccess::first() = false;
    k->*KfAccess::notErase() = p->not_erase[i] != 0;
    k->*KfAccess::parent() = parent[i] >= 0 ? g.kf(parent[i]) : nullptr;
  }
  for (int i = 0; i < n; i++)
    if (parent[i] >= 0) g.kf(parent[i])->AddChild(g.kf(i));
  {
    KeyFrame* c = g.kf(cur);
    std::vector<KeyFrame*>& ok = c->*KfAccess::ordKf();
    std::vector<int>& ow = c->*KfAccess::ordW();
    ok.clear();
    ow.clear();
    for (int l = 0; l < p->n_local; l++) {
      ok.push_back(g.kf(p->local_kf[l]));
      ow.push_back(c->GetWeight(ok.back()));
    }
  }

  const auto t0 = std::chrono::steady_clock::now();
#ifdef B2S_ADAPTER_BUILD
  if (b200::KeyFrameCulling(g.kf(cur), p->monocular != 0) != 0) return -1;
#else
  Culler lm(&g.map, p->monocular != 0);
  lm.cull(g.kf(cur));
#endif
  if (wall_ns) *wall_ns = std::chrono::duration<double, std::nano>(std::chrono::steady_clock::now() - t0).count();

  int needConn = 0, needChild = 0;
  for (int i = 0; i < n; i++) {
    needConn += (int)(g.kf(i)->*KfAccess::conn()).size();
    needChild += (int)(g.kf(i)->*KfAccess::children()).size();
  }
  if (needConn > conn_cap || needChild > child_cap) return B2S_ERR_CAPACITY;
  int culled = 0;
  for (int l = 0; l < p->n_local; l++) {
    KeyFrame* k = g.kf(p->local_kf[l]);
    r->n_mps[l] = r->n_redundant[l] = -1;
    if (k->mnId == 0)
      r->verdict[l] = B2S_CULL_SKIPPED;
    else if (std::find(g.map.erased.begin(), g.map.erased.end(), k) != g.map.erased.end())
      r->verdict[l] = B2S_CULL_CULLED;
    else if (k->*KfAccess::toBeErased())
      r->verdict[l] = B2S_CULL_DEFERRED;
    else
      r->verdict[l] = B2S_CULL_KEPT;
    culled += r->verdict[l] == B2S_CULL_CULLED;
    const std::vector<MapPoint*>& pts = k->*KfAccess::points();
    for (int s = p->slot_off[l]; s < p->slot_off[l + 1]; s++) {
      const MapPoint* mp = pts[(size_t)(s - p->slot_off[l])];
      r->slot_mp[s] = mp ? mpIndex[mp] : -1;
    }
  }
  r->n_culled = culled;
  *n_erased = (int)g.map.erased.size();
  for (size_t j = 0; j < g.map.erased.size(); j++) erased[j] = g.index(g.map.erased[j]);
  for (int m = 0; m < p->n_mp; m++) {
    MapPoint* mp = g.mps[(size_t)m].get();
    r->mp_bad[m] = mp->*MpAccess::bad();
    r->mp_nobs[m] = mp->nObs;
    const std::map<KeyFrame*, size_t>& obs = mp->*MpAccess::obs();
    for (int o = p->obs_off[m]; o < p->obs_off[m + 1]; o++) r->obs_alive[o] = obs.count(g.kf(p->obs_kf[o])) != 0;
  }
  int cc = 0, ch = 0;
  conn_out_off[0] = child_out_off[0] = 0;
  for (int i = 0; i < n; i++) {
    KeyFrame* k = g.kf(i);
    kf_bad[i] = k->*KfAccess::bad();
    kf_to_be_erased[i] = k->*KfAccess::toBeErased();
    parent_out[i] = k->*KfAccess::parent() ? g.index(k->*KfAccess::parent()) : -1;
    for (auto& kv : k->*KfAccess::conn()) {
      conn_out_kf[cc] = g.index(kv.first);
      conn_out_w[cc++] = kv.second;
    }
    for (KeyFrame* c : k->*KfAccess::children()) child_out_kf[ch++] = g.index(c);
    conn_out_off[i + 1] = cc;
    child_out_off[i + 1] = ch;
  }
  return B2S_OK;
}
}
