// TEST INFRASTRUCTURE — C entry point around the reference's own KeyFrame (src/KeyFrame.cc compiled in place, unmodified,
// with its include/KeyFrame.h and include/Frame.h, against the stand-ins of refshim/slam_stubs_keyframe.h).  Built into
// oracle/_ref/libref_keyframe.so (git-ignored).
//
// One call builds an object graph from a b2s_covis_problem: the keyframes are constructed by the reference's constructor
// from a minimal Frame, with placement new into one buffer in table order (ascending mnId), so that their address order
// is their mnId order; map points are stand-ins with the problem's observers and bad flags.  The protected connection
// state is written and read through member pointers taken in a derived class.  Then KeyFrame::UpdateConnections runs on
// the members one after another, and the glue records GetVectorCovisibleKeyFrames() before each call and the connection
// map after it.  The result holds the final state of every keyframe (changed = 1 for all) and its children.
//
// Built with -DB2S_ADAPTER_BUILD into _ref/libadapter_covis.so, the entry point is adp_update_connections and the calls
// go through the product's b200::UpdateConnections (host/adapters/Covisibility_b200.cc) as one batch.
#ifdef B2S_ADAPTER_BUILD
#define COVIS_FN(name) adp_##name
#include "adapters/Covisibility_b200.h"
#else
#define COVIS_FN(name) ref_##name
#endif
#include <chrono>
#include <cstdint>
#include <cstdlib>
#include <new>
#include <vector>

#include "KeyFrame.h"
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

// member pointers to KeyFrame's protected state (include/KeyFrame.h:386-432)
struct Access : KeyFrame {
  static std::map<KeyFrame*, int> KeyFrame::*conn() { return &Access::mConnectedKeyFrameWeights; }
  static std::vector<KeyFrame*> KeyFrame::*ordKf() { return &Access::mvpOrderedConnectedKeyFrames; }
  static std::vector<int> KeyFrame::*ordW() { return &Access::mvOrderedWeights; }
  static bool KeyFrame::*first() { return &Access::mbFirstConnection; }
  static KeyFrame* KeyFrame::*parent() { return &Access::mpParent; }
  static std::set<KeyFrame*> KeyFrame::*children() { return &Access::mspChildrens; }
  static std::vector<MapPoint*> KeyFrame::*points() { return &Access::mvpMapPoints; }
  static bool KeyFrame::*bad() { return &Access::mbBad; }
};

struct Graph {
  Map map;
  KeyFrameDatabase db;
  unsigned char* buf = nullptr;
  int n = 0;
  std::vector<MapPoint> mps;
  KeyFrame* kf(int i) { return reinterpret_cast<KeyFrame*>(buf + (size_t)i * sizeof(KeyFrame)); }
  int index(const KeyFrame* k) const {
    return (int)((reinterpret_cast<const unsigned char*>(k) - buf) / sizeof(KeyFrame));
  }
  ~Graph() {
    for (int i = 0; i < n; i++) kf(i)->~KeyFrame();
    free(buf);
  }
};

}  // namespace

extern "C" {

/* kf_bad (optional, n_kf): KeyFrame::mbBad; child_off / child_kf (optional, CSR over n_kf): mspChildrens on entry.
 * out_child_off (n_kf + 1) / out_child_kf (child_cap): mspChildrens after the batch.  *wall_ns (optional): the host wall
 * time of the calls alone, without building or reading the graph.  Returns B2S_OK or B2S_ERR_CAPACITY. */
int COVIS_FN(update_connections)(const b2s_covis_problem* p, const uint8_t* kf_bad, const int32_t* child_off,
                                 const int32_t* child_kf, b2s_covis_result* r, int32_t* out_child_off,
                                 int32_t* out_child_kf, int child_cap, double* wall_ns) {
  const int n = p->n_kf, B = p->batch;
  Graph g;
  g.buf = static_cast<unsigned char*>(aligned_alloc(alignof(KeyFrame), ((size_t)n * sizeof(KeyFrame) + 63) / 64 * 64));
  Frame F;
  F.mTcw = cv::Mat::eye(4, 4, CV_32F);
  F.N = 0;
  for (int i = 0; i < n; i++) {
    KeyFrame::nNextId = (long unsigned int)p->kf_id[i];  // the constructor takes mnId = nNextId++
    new (g.kf(i)) KeyFrame(F, &g.map, &g.db);
    g.n = i + 1;
  }
  g.mps.resize((size_t)p->n_mp);
  for (int m = 0; m < p->n_mp; m++) {
    g.mps[(size_t)m].mbBad = p->mp_bad[m] != 0;
    for (int o = p->obs_off[m]; o < p->obs_off[m + 1]; o++) g.mps[(size_t)m].mObservations[g.kf(p->obs_kf[o])] = 0;
  }
  for (int i = 0; i < n; i++) {
    KeyFrame* k = g.kf(i);
    std::map<KeyFrame*, int>& conn = k->*Access::conn();
    for (int j = p->map_off[i]; j < p->map_off[i + 1]; j++) conn[g.kf(p->map_kf[j])] = p->map_w[j];
    for (int j = p->list_off[i]; j < p->list_off[i + 1]; j++) {
      (k->*Access::ordKf()).push_back(g.kf(p->list_kf[j]));
      (k->*Access::ordW()).push_back(p->list_w[j]);
    }
    k->*Access::first() = p->first_connection[i] != 0;
    k->*Access::parent() = p->parent[i] >= 0 ? g.kf(p->parent[i]) : nullptr;
    if (kf_bad) k->*Access::bad() = kf_bad[i] != 0;
    if (child_off)
      for (int j = child_off[i]; j < child_off[i + 1]; j++) (k->*Access::children()).insert(g.kf(child_kf[j]));
  }
  std::vector<bool> seen((size_t)n, false);
  for (int b = 0; b < B; b++) {  // each member's slots: its first call's
    const int m = p->member[b];
    if (seen[(size_t)m]) continue;
    seen[(size_t)m] = true;
    std::vector<MapPoint*>& pts = g.kf(m)->*Access::points();
    pts.clear();
    for (int s = p->slot_off[b]; s < p->slot_off[b + 1]; s++)
      pts.push_back(p->slot_mp[s] >= 0 ? &g.mps[(size_t)p->slot_mp[s]] : nullptr);
  }

  std::vector<std::vector<KeyFrame*> > before((size_t)B);
  std::vector<std::map<KeyFrame*, int> > after((size_t)B);
  const auto t0 = std::chrono::steady_clock::now();
#ifdef B2S_ADAPTER_BUILD
  std::vector<KeyFrame*> members;
  for (int b = 0; b < B; b++) members.push_back(g.kf(p->member[b]));
  b200::CovisibilityReads reads;
  if (b200::UpdateConnections(members, &reads) != 0) return -1;
  for (int b = 0; b < B; b++) {
    before[(size_t)b] = reads.before[(size_t)b];
    after[(size_t)b] = reads.after[(size_t)b];
  }
#else
  for (int b = 0; b < B; b++) {
    KeyFrame* k = g.kf(p->member[b]);
    before[(size_t)b] = k->GetVectorCovisibleKeyFrames();
    k->UpdateConnections();
    after[(size_t)b] = k->*Access::conn();
  }
#endif
  if (wall_ns) *wall_ns = std::chrono::duration<double, std::nano>(std::chrono::steady_clock::now() - t0).count();

  int needMap = 0, needList = 0, needStart = 0, needAfter = 0, needChild = 0;
  for (int i = 0; i < n; i++) {
    needMap += (int)(g.kf(i)->*Access::conn()).size();
    needList += (int)(g.kf(i)->*Access::ordKf()).size();
    needChild += (int)(g.kf(i)->*Access::children()).size();
  }
  for (int b = 0; b < B; b++) {
    needStart += (int)before[(size_t)b].size();
    needAfter += (int)after[(size_t)b].size();
  }
  r->map_need = needMap;
  r->list_need = needList;
  r->start_need = needStart;
  r->after_need = needAfter;
  if (needMap > r->map_cap || needList > r->list_cap || needStart > r->start_cap || needAfter > r->after_cap ||
      needChild > child_cap)
    return B2S_ERR_CAPACITY;
  int cm = 0, cl = 0, cc = 0;
  r->map_off[0] = r->list_off[0] = out_child_off[0] = 0;
  for (int i = 0; i < n; i++) {
    KeyFrame* k = g.kf(i);
    r->changed[i] = 1;
    r->parent[i] = k->*Access::parent() ? g.index(k->*Access::parent()) : -1;
    r->first_connection[i] = k->*Access::first();
    for (auto& kv : k->*Access::conn()) {
      r->map_kf[cm] = g.index(kv.first);
      r->map_w[cm++] = kv.second;
    }
    const std::vector<KeyFrame*>& ok = k->*Access::ordKf();
    const std::vector<int>& ow = k->*Access::ordW();
    for (size_t j = 0; j < ok.size(); j++) {
      r->list_kf[cl] = g.index(ok[j]);
      r->list_w[cl++] = ow[j];
    }
    for (KeyFrame* c : k->*Access::children()) out_child_kf[cc++] = g.index(c);
    r->map_off[i + 1] = cm;
    r->list_off[i + 1] = cl;
    out_child_off[i + 1] = cc;
  }
  int cs = 0, ca = 0;
  r->start_off[0] = r->after_off[0] = 0;
  for (int b = 0; b < B; b++) {
    for (KeyFrame* k : before[(size_t)b]) r->start_kf[cs++] = g.index(k);
    for (auto& kv : after[(size_t)b]) {
      r->after_kf[ca] = g.index(kv.first);
      r->after_w[ca++] = kv.second;
    }
    r->start_off[b + 1] = cs;
    r->after_off[b + 1] = ca;
  }
  r->n_pairs = 0;  // the children carry AddChild's effect
  return B2S_OK;
}
}
