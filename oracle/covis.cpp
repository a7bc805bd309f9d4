// TEST INFRASTRUCTURE — CPU restatement of KeyFrame::UpdateConnections (src/KeyFrame.cc:386-507), AddConnection
// (:159-178) and UpdateBestCovisibles (:185-209) over the flattened tables of b2s_covis_problem, one call after another in
// batch order.  Keyframes are table indices; index order stands for the reference's pointer order (DESIGN §2), so
// std::map<int, int> iterates as std::map<KeyFrame*, int> does and the pair sort breaks ties the same way.  Built into
// oracle/liborb_covis.so by covis.mk.
#include <algorithm>
#include <cstring>
#include <list>
#include <map>
#include <utility>
#include <vector>

#include "../include/b200slam.h"

namespace {

struct KF {
  std::map<int, int> conn;                   // mConnectedKeyFrameWeights
  std::vector<int> ordKf, ordW;              // mvpOrderedConnectedKeyFrames, mvOrderedWeights
  bool first = true;                         // mbFirstConnection
  int parent = -1;                           // mpParent
  bool changed = false;
};

// :185-209
void UpdateBestCovisibles(KF& k) {
  std::vector<std::pair<int, int> > vPairs;
  vPairs.reserve(k.conn.size());
  for (auto mit = k.conn.begin(); mit != k.conn.end(); mit++) vPairs.push_back(std::make_pair(mit->second, mit->first));
  std::sort(vPairs.begin(), vPairs.end());
  std::list<int> lKFs, lWs;
  for (size_t i = 0; i < vPairs.size(); i++) {
    lKFs.push_front(vPairs[i].second);
    lWs.push_front(vPairs[i].first);
  }
  k.ordKf.assign(lKFs.begin(), lKFs.end());
  k.ordW.assign(lWs.begin(), lWs.end());
}

// :159-178, called on partner `k` with pKF = the calling keyframe
void AddConnection(KF& k, int pKF, int weight) {
  if (!k.conn.count(pKF))
    k.conn[pKF] = weight;
  else if (k.conn[pKF] != weight)
    k.conn[pKF] = weight;
  else
    return;
  k.changed = true;
  UpdateBestCovisibles(k);
}

}  // namespace

extern "C" int orc_update_connections(const b2s_covis_problem* p, b2s_covis_result* r) {
  const int n = p->n_kf, B = p->batch;
  std::vector<KF> kfs((size_t)n);
  for (int i = 0; i < n; i++) {
    KF& k = kfs[(size_t)i];
    for (int j = p->map_off[i]; j < p->map_off[i + 1]; j++) k.conn[p->map_kf[j]] = p->map_w[j];
    k.ordKf.assign(p->list_kf + p->list_off[i], p->list_kf + p->list_off[i + 1]);
    k.ordW.assign(p->list_w + p->list_off[i], p->list_w + p->list_off[i + 1]);
    k.first = p->first_connection[i] != 0;
    k.parent = p->parent[i];
  }
  std::vector<std::vector<int> > startKf((size_t)B), afterKf((size_t)B), afterW((size_t)B);
  std::vector<int> pairs;
  const int th = 15;  // :438
  for (int b = 0; b < B; b++) {
    const int self = p->member[b];
    KF& K = kfs[(size_t)self];
    startKf[(size_t)b] = K.ordKf;  // GetVectorCovisibleKeyFrames() before the call
    // :391-427
    std::map<int, int> KFcounter;
    for (int s = p->slot_off[b]; s < p->slot_off[b + 1]; s++) {
      const int pMP = p->slot_mp[s];
      if (pMP < 0) continue;
      if (p->mp_bad[pMP]) continue;
      for (int o = p->obs_off[pMP]; o < p->obs_off[pMP + 1]; o++) {
        const int kf = p->obs_kf[o];
        if (p->kf_id[kf] == p->kf_id[self]) continue;
        KFcounter[kf]++;
      }
    }
    if (!KFcounter.empty()) {  // :430-431
      // :436-474
      int nmax = 0;
      int pKFmax = -1;
      std::vector<std::pair<int, int> > vPairs;
      vPairs.reserve(KFcounter.size());
      for (auto mit = KFcounter.begin(); mit != KFcounter.end(); mit++) {
        if (mit->second > nmax) {
          nmax = mit->second;
          pKFmax = mit->first;
        }
        if (mit->second >= th) {
          vPairs.push_back(std::make_pair(mit->second, mit->first));
          AddConnection(kfs[(size_t)mit->first], self, mit->second);
        }
      }
      if (vPairs.empty()) {
        vPairs.push_back(std::make_pair(nmax, pKFmax));
        AddConnection(kfs[(size_t)pKFmax], self, nmax);
      }
      // :477-485
      std::sort(vPairs.begin(), vPairs.end());
      std::list<int> lKFs, lWs;
      for (size_t i = 0; i < vPairs.size(); i++) {
        lKFs.push_front(vPairs[i].second);
        lWs.push_front(vPairs[i].first);
      }
      // :488-505
      K.conn = KFcounter;
      K.ordKf.assign(lKFs.begin(), lKFs.end());
      K.ordW.assign(lWs.begin(), lWs.end());
      K.changed = true;
      if (K.first && p->kf_id[self] != 0) {
        K.parent = K.ordKf.front();
        pairs.push_back(K.parent);
        pairs.push_back(self);
        K.first = false;
      }
    }
    for (auto& kv : K.conn) {  // the connection map right after the call
      afterKf[(size_t)b].push_back(kv.first);
      afterW[(size_t)b].push_back(kv.second);
    }
  }

  int needMap = 0, needList = 0, needStart = 0, needAfter = 0;
  for (const KF& k : kfs)
    if (k.changed) {
      needMap += (int)k.conn.size();
      needList += (int)k.ordKf.size();
    }
  for (int b = 0; b < B; b++) {
    needStart += (int)startKf[(size_t)b].size();
    needAfter += (int)afterKf[(size_t)b].size();
  }
  r->map_need = needMap;
  r->list_need = needList;
  r->start_need = needStart;
  r->after_need = needAfter;
  if (needMap > r->map_cap || needList > r->list_cap || needStart > r->start_cap || needAfter > r->after_cap)
    return B2S_ERR_CAPACITY;
  int cm = 0, cl = 0;
  r->map_off[0] = r->list_off[0] = 0;
  for (int i = 0; i < n; i++) {
    const KF& k = kfs[(size_t)i];
    r->changed[i] = k.changed;
    r->parent[i] = k.parent;
    r->first_connection[i] = k.first;
    if (k.changed) {
      for (auto& kv : k.conn) {
        r->map_kf[cm] = kv.first;
        r->map_w[cm++] = kv.second;
      }
      for (size_t j = 0; j < k.ordKf.size(); j++) {
        r->list_kf[cl] = k.ordKf[j];
        r->list_w[cl++] = k.ordW[j];
      }
    }
    r->map_off[i + 1] = cm;
    r->list_off[i + 1] = cl;
  }
  int cs = 0, ca = 0;
  r->start_off[0] = r->after_off[0] = 0;
  for (int b = 0; b < B; b++) {
    for (int v : startKf[(size_t)b]) r->start_kf[cs++] = v;
    for (size_t j = 0; j < afterKf[(size_t)b].size(); j++) {
      r->after_kf[ca] = afterKf[(size_t)b][j];
      r->after_w[ca++] = afterW[(size_t)b][j];
    }
    r->start_off[b + 1] = cs;
    r->after_off[b + 1] = ca;
  }
  r->n_pairs = (int)pairs.size() / 2;
  if (!pairs.empty()) memcpy(r->child_pairs, pairs.data(), pairs.size() * sizeof(int));
  return B2S_OK;
}
