// Batched KeyFrame::UpdateConnections (src/KeyFrame.cc:386-507) over b2s_update_connections, against the reference's
// unchanged include/KeyFrame.h.  The call gathers the tables from the object graph, makes one device call and scatters the
// result back.  KeyFrame's connection state is protected; it is read and written through member pointers taken in a
// derived class, under the locks the reference takes: mMutexFeatures to read the slots (GetMapPointMatches),
// mMutexConnections to read and write the connection state.
//
// The table holds the members, every keyframe that observes one of their non-bad points, and the keyframes those name
// in their connection maps, ordered lists and parents (so that every index resolves); the last ring's own state is
// never read and goes in empty.  On a library error the call prints to stderr and returns its code; the graph is
// unchanged then.
#include "adapters/Covisibility_b200.h"

#include <algorithm>
#include <mutex>
#include <set>
#include <unordered_map>

#include "MapPoint.h"
#include "b200slam.h"
#include "../b2s_host.h"

namespace ORB_SLAM2 {
namespace b200 {
namespace {

struct Access : KeyFrame {
  static std::map<KeyFrame*, int> KeyFrame::*conn() { return &Access::mConnectedKeyFrameWeights; }
  static std::vector<KeyFrame*> KeyFrame::*ordKf() { return &Access::mvpOrderedConnectedKeyFrames; }
  static std::vector<int> KeyFrame::*ordW() { return &Access::mvOrderedWeights; }
  static bool KeyFrame::*first() { return &Access::mbFirstConnection; }
  static KeyFrame* KeyFrame::*parent() { return &Access::mpParent; }
  static std::mutex KeyFrame::*mutexConnections() { return &Access::mMutexConnections; }
};

// One handle for the process (LocalMapping and LoopClosing call it in turn), grown on demand.
// capacities: keyframes, points, observations, slots, connections, batch
b2s_host::Slot<b2s_covis, 6, b2s_covis_destroy> g_covis;
const int kCovisFloor[6] = {256, 8192, 65536, 8192, 65536, 1};

int create_covis(const int* c, b2s_covis** h) {
  return b2s_covis_create(c[0], c[1], c[2], c[3], c[4], c[5], b2s_host::device(), h);
}

bool by_id(const KeyFrame* a, const KeyFrame* b) { return a->mnId < b->mnId; }

}  // namespace

int UpdateConnections(const std::vector<KeyFrame*>& vpKFs, CovisibilityReads* reads) {
  const int B = (int)vpKFs.size();
  if (B < 1) return B2S_ERR_BAD_ARG;
  // slots and points
  std::vector<std::vector<MapPoint*> > slots((size_t)B);
  std::unordered_map<MapPoint*, int> mpIndex;
  std::vector<MapPoint*> mps;
  std::unordered_map<KeyFrame*, std::vector<MapPoint*> > slotsOf;
  for (int b = 0; b < B; b++) {
    auto it = slotsOf.find(vpKFs[(size_t)b]);
    if (it == slotsOf.end()) it = slotsOf.emplace(vpKFs[(size_t)b], vpKFs[(size_t)b]->GetMapPointMatches()).first;
    slots[(size_t)b] = it->second;
    for (MapPoint* pMP : it->second)
      if (pMP && mpIndex.emplace(pMP, (int)mps.size()).second) mps.push_back(pMP);
  }
  std::vector<uint8_t> mpBad(mps.size());
  std::vector<std::map<KeyFrame*, size_t> > obs(mps.size());
  std::set<KeyFrame*> core(vpKFs.begin(), vpKFs.end());
  for (size_t m = 0; m < mps.size(); m++) {
    mpBad[m] = mps[m]->isBad();
    if (mpBad[m]) continue;
    obs[m] = mps[m]->GetObservations();
    for (auto& kv : obs[m]) core.insert(kv.first);
  }
  // the entry state of the members and observers; the keyframes it names join the table
  struct Entry {
    std::map<KeyFrame*, int> conn;
    std::vector<KeyFrame*> ordKf;
    std::vector<int> ordW;
    bool first;
    KeyFrame* parent;
  };
  std::unordered_map<KeyFrame*, Entry> entry;
  std::set<KeyFrame*> all(core);
  for (KeyFrame* k : core) {
    std::unique_lock<std::mutex> lock(k->*Access::mutexConnections());
    Entry e{k->*Access::conn(), k->*Access::ordKf(), k->*Access::ordW(), k->*Access::first(), k->*Access::parent()};
    for (auto& kv : e.conn) all.insert(kv.first);
    all.insert(e.ordKf.begin(), e.ordKf.end());
    if (e.parent) all.insert(e.parent);
    entry.emplace(k, std::move(e));
  }
  std::vector<KeyFrame*> table(all.begin(), all.end());
  std::sort(table.begin(), table.end(), by_id);
  std::unordered_map<KeyFrame*, int> idx;
  for (size_t i = 0; i < table.size(); i++) idx[table[i]] = (int)i;

  const int n = (int)table.size(), nmp = (int)mps.size();
  std::vector<uint64_t> ids((size_t)n);
  std::vector<int32_t> mapOff(1, 0), mapKf, mapW, listOff(1, 0), listKf, listW, parent((size_t)n, -1);
  std::vector<uint8_t> first((size_t)n, 0);
  for (int i = 0; i < n; i++) {
    KeyFrame* k = table[(size_t)i];
    ids[(size_t)i] = k->mnId;
    auto it = entry.find(k);
    if (it != entry.end()) {
      const Entry& e = it->second;
      for (auto& kv : e.conn) {  // std::map order is pointer order; the table's is mnId order
        mapKf.push_back(idx[kv.first]);
        mapW.push_back(kv.second);
      }
      std::sort(mapKf.begin() + mapOff.back(), mapKf.end());
      for (size_t j = mapOff.back(); j < mapKf.size(); j++) mapW[j] = e.conn.at(table[(size_t)mapKf[j]]);
      for (size_t j = 0; j < e.ordKf.size(); j++) {
        listKf.push_back(idx[e.ordKf[j]]);
        listW.push_back(e.ordW[j]);
      }
      first[(size_t)i] = e.first;
      parent[(size_t)i] = e.parent ? idx[e.parent] : -1;
    }
    mapOff.push_back((int32_t)mapKf.size());
    listOff.push_back((int32_t)listKf.size());
  }
  std::vector<int32_t> obsOff(1, 0), obsKf;
  for (int m = 0; m < nmp; m++) {
    const size_t s = obsKf.size();
    for (auto& kv : obs[(size_t)m]) obsKf.push_back(idx[kv.first]);
    std::sort(obsKf.begin() + s, obsKf.end());
    obsOff.push_back((int32_t)obsKf.size());
  }
  std::vector<int32_t> member((size_t)B), slotOff(1, 0), slotMp;
  for (int b = 0; b < B; b++) {
    member[(size_t)b] = idx[vpKFs[(size_t)b]];
    for (MapPoint* pMP : slots[(size_t)b]) slotMp.push_back(pMP ? mpIndex[pMP] : -1);
    slotOff.push_back((int32_t)slotMp.size());
  }

  b2s_covis_problem p;
  p.n_kf = n;
  p.kf_id = ids.data();
  p.map_off = mapOff.data();
  p.map_kf = mapKf.data();
  p.map_w = mapW.data();
  p.list_off = listOff.data();
  p.list_kf = listKf.data();
  p.list_w = listW.data();
  p.first_connection = first.data();
  p.parent = parent.data();
  p.n_mp = nmp;
  p.mp_bad = mpBad.data();
  p.obs_off = obsOff.data();
  p.obs_kf = obsKf.data();
  p.batch = B;
  p.member = member.data();
  p.slot_off = slotOff.data();
  p.slot_mp = slotMp.data();

  std::vector<uint8_t> rChanged((size_t)n), rFirst((size_t)n);
  std::vector<int32_t> rParent((size_t)n), rMapOff((size_t)n + 1), rListOff((size_t)n + 1), pairs(2 * (size_t)B),
      startOff((size_t)B + 1), afterOff((size_t)B + 1);
  std::vector<int32_t> rMapKf, rMapW, rListKf, rListW, startKf, afterKf, afterW;
  b2s_covis_result r;
  int rc;
  {
    std::lock_guard<std::mutex> lock(g_covis.mutex);
    rc = g_covis.get({n, nmp, (int)obsKf.size(), (int)slotMp.size(), (int)std::max(mapKf.size(), listKf.size()), B},
                     kCovisFloor, create_covis);
    size_t cap = 4096;
    if (rc == B2S_OK) for (;;) {
      rMapKf.resize(cap);
      rMapW.resize(cap);
      rListKf.resize(cap);
      rListW.resize(cap);
      startKf.resize(cap);
      afterKf.resize(cap);
      afterW.resize(cap);
      r = b2s_covis_result{rChanged.data(), rParent.data(), rFirst.data(), rMapOff.data(), rMapKf.data(), rMapW.data(),
                           (int)cap, rListOff.data(), rListKf.data(), rListW.data(), (int)cap, pairs.data(), 0,
                           startOff.data(), startKf.data(), (int)cap, afterOff.data(), afterKf.data(), afterW.data(),
                           (int)cap, 0, 0, 0, 0};
      rc = b2s_update_connections(g_covis.h, &p, &r);
      const int need = std::max({r.map_need, r.list_need, r.start_need, r.after_need});
      if (rc == B2S_ERR_CAPACITY && need > (int)cap) {
        cap = (size_t)need;
        continue;
      }
      if (rc == B2S_ERR_CAPACITY) {  // the handle's output areas: grow them
        rc = g_covis.get({n, nmp, (int)obsKf.size(), (int)slotMp.size(), 2 * std::max(g_covis.cap[4], 1), B},
                         kCovisFloor, create_covis);
        if (rc == B2S_OK) continue;
      }
      break;
    }
  }
  if (rc != B2S_OK) {
    b2s_host::report("UpdateConnections", rc);
    return rc;
  }
  for (int i = 0; i < n; i++) {
    if (!r.changed[i]) continue;
    KeyFrame* k = table[(size_t)i];
    std::unique_lock<std::mutex> lock(k->*Access::mutexConnections());
    std::map<KeyFrame*, int>& conn = k->*Access::conn();
    conn.clear();
    for (int j = r.map_off[i]; j < r.map_off[i + 1]; j++) conn[table[(size_t)r.map_kf[j]]] = r.map_w[j];
    std::vector<KeyFrame*>& ok = k->*Access::ordKf();
    std::vector<int>& ow = k->*Access::ordW();
    ok.clear();
    ow.clear();
    for (int j = r.list_off[i]; j < r.list_off[i + 1]; j++) {
      ok.push_back(table[(size_t)r.list_kf[j]]);
      ow.push_back(r.list_w[j]);
    }
    k->*Access::first() = r.first_connection[i] != 0;
    k->*Access::parent() = r.parent[i] >= 0 ? table[(size_t)r.parent[i]] : nullptr;
  }
  for (int q = 0; q < r.n_pairs; q++) table[(size_t)pairs[2 * q]]->AddChild(table[(size_t)pairs[2 * q + 1]]);
  if (reads) {
    reads->before.assign((size_t)B, std::vector<KeyFrame*>());
    reads->after.assign((size_t)B, std::map<KeyFrame*, int>());
    for (int b = 0; b < B; b++) {
      for (int j = r.start_off[b]; j < r.start_off[b + 1]; j++) reads->before[(size_t)b].push_back(table[(size_t)startKf[j]]);
      for (int j = r.after_off[b]; j < r.after_off[b + 1]; j++)
        reads->after[(size_t)b][table[(size_t)afterKf[j]]] = afterW[j];
    }
  }
  return B2S_OK;
}

}  // namespace b200
}  // namespace ORB_SLAM2
