// LocalMapping::KeyFrameCulling (src/LocalMapping.cc:873-956) over b2s_keyframe_culling, against the reference's
// unchanged include/KeyFrame.h and include/MapPoint.h.  The call gathers the tables from the object graph, makes one
// device call for the verdicts, and calls the reference's KeyFrame::SetBadFlag on the culled and deferred keyframes in
// list order: SetBadFlag applies to the points exactly the effects the device modelled, and keeps the spanning tree,
// EraseConnection and the map / database erasure the reference's own.
//
// The reads take the reference's locks: GetVectorCovisibleKeyFrames and mbNotErase under mMutexConnections (the flag is
// protected and read through a member pointer taken in a derived class), GetMapPointMatches under mMutexFeatures, and
// isBad / Observations / GetObservations under the points' own locks.  mvKeysUn, mvuRight, mvDepth and mThDepth are
// constant after construction.  The table holds the local keyframes and every observer of their points, in mnId order.
// On a library error the call prints to stderr and returns its code; the graph is unchanged then.
#include "adapters/LocalMapping_b200.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <set>
#include <unordered_map>
#include <vector>

#include "MapPoint.h"
#include "b200slam.h"

namespace ORB_SLAM2 {
namespace b200 {
namespace {

struct Access : KeyFrame {
  static bool KeyFrame::*notErase() { return &Access::mbNotErase; }
  static std::mutex KeyFrame::*mutexConnections() { return &Access::mMutexConnections; }
};

// One handle for the process, grown on demand.
struct CullingSlot {
  b2s_culling* h = nullptr;
  int kf = 0, mp = 0, obs = 0, local = 0, slots = 0;
  std::mutex m;
  b2s_culling* get(int nkf, int nmp, int nobs, int nlocal, int nslots) {
    if (h && nkf <= kf && nmp <= mp && nobs <= obs && nlocal <= local && nslots <= slots) return h;
    b2s_culling_destroy(h);
    h = nullptr;
    kf = std::max({nkf, kf, 256});
    mp = std::max({nmp, mp, 8192});
    obs = std::max({nobs, obs, 65536});
    local = std::max({nlocal, local, 256});
    slots = std::max({nslots, slots, 65536});
    const char* e = getenv("B2S_DEVICE");
    if (b2s_culling_create(kf, mp, obs, local, slots, 1, e ? atoi(e) : 0, &h) != B2S_OK) {
      fprintf(stderr, "KeyFrameCulling (b200): %s\n", b2s_last_error());
      h = nullptr;
      kf = mp = obs = local = slots = 0;
    }
    return h;
  }
} g_culling;

bool by_id(const KeyFrame* a, const KeyFrame* b) { return a->mnId < b->mnId; }

}  // namespace

int KeyFrameCulling(KeyFrame* pCurrentKF, bool bMonocular) {
  const std::vector<KeyFrame*> vpLocal = pCurrentKF->GetVectorCovisibleKeyFrames();
  const int L = (int)vpLocal.size();
  if (L == 0) return B2S_OK;
  std::vector<std::vector<MapPoint*> > slots((size_t)L);
  std::unordered_map<MapPoint*, int> mpIndex;
  std::vector<MapPoint*> mps;
  for (int l = 0; l < L; l++) {
    slots[(size_t)l] = vpLocal[(size_t)l]->GetMapPointMatches();
    for (MapPoint* pMP : slots[(size_t)l])
      if (pMP && mpIndex.emplace(pMP, (int)mps.size()).second) mps.push_back(pMP);
  }
  const int nmp = (int)mps.size();
  std::vector<uint8_t> mpBad((size_t)nmp);
  std::vector<int32_t> mpNobs((size_t)nmp);
  std::vector<std::map<KeyFrame*, size_t> > obs((size_t)nmp);
  std::set<KeyFrame*> all(vpLocal.begin(), vpLocal.end());
  for (int m = 0; m < nmp; m++) {
    mpBad[(size_t)m] = mps[(size_t)m]->isBad();
    mpNobs[(size_t)m] = mps[(size_t)m]->Observations();
    obs[(size_t)m] = mps[(size_t)m]->GetObservations();
    for (auto& kv : obs[(size_t)m]) all.insert(kv.first);
  }
  std::vector<KeyFrame*> table(all.begin(), all.end());
  std::sort(table.begin(), table.end(), by_id);
  std::unordered_map<KeyFrame*, int> idx;
  for (size_t i = 0; i < table.size(); i++) idx[table[i]] = (int)i;
  const int n = (int)table.size();

  std::vector<uint64_t> ids((size_t)n);
  std::vector<uint8_t> notErase((size_t)n);
  std::vector<float> thDepth((size_t)n);
  for (int i = 0; i < n; i++) {
    KeyFrame* k = table[(size_t)i];
    ids[(size_t)i] = k->mnId;
    thDepth[(size_t)i] = k->mThDepth;
    std::unique_lock<std::mutex> lock(k->*Access::mutexConnections());
    notErase[(size_t)i] = k->*Access::notErase();
  }
  std::vector<int32_t> obsOff(1, 0), obsKf, obsIdx, obsOct;
  std::vector<uint8_t> obsStereo;
  for (int m = 0; m < nmp; m++) {
    std::vector<std::pair<int, size_t> > row;
    for (auto& kv : obs[(size_t)m]) row.push_back(std::make_pair(idx[kv.first], kv.second));
    std::sort(row.begin(), row.end());
    for (auto& e : row) {
      KeyFrame* k = table[(size_t)e.first];
      if (e.second >= k->mvKeysUn.size() || e.second >= k->mvuRight.size()) {
        fprintf(stderr, "KeyFrameCulling (b200): an observation's index lies outside its keyframe's keypoints\n");
        return B2S_ERR_BAD_ARG;
      }
      obsKf.push_back(e.first);
      obsIdx.push_back((int32_t)e.second);
      obsOct.push_back(k->mvKeysUn[e.second].octave);
      obsStereo.push_back(k->mvuRight[e.second] >= 0);
    }
    obsOff.push_back((int32_t)obsKf.size());
  }
  std::vector<int32_t> localKf((size_t)L), slotOff(1, 0), slotMp, slotOct;
  std::vector<float> slotDepth;
  for (int l = 0; l < L; l++) {
    KeyFrame* k = vpLocal[(size_t)l];
    localKf[(size_t)l] = idx[k];
    const std::vector<MapPoint*>& sl = slots[(size_t)l];
    for (size_t i = 0; i < sl.size(); i++) {
      slotMp.push_back(sl[i] ? mpIndex[sl[i]] : -1);
      slotOct.push_back(i < k->mvKeysUn.size() ? k->mvKeysUn[i].octave : 0);
      slotDepth.push_back(i < k->mvDepth.size() ? k->mvDepth[i] : 0.f);
    }
    slotOff.push_back((int32_t)slotMp.size());
  }

  b2s_culling_problem p;
  p.n_kf = n;
  p.kf_id = ids.data();
  p.not_erase = notErase.data();
  p.th_depth = thDepth.data();
  p.n_mp = nmp;
  p.mp_bad = mpBad.data();
  p.mp_nobs = mpNobs.data();
  p.obs_off = obsOff.data();
  p.obs_kf = obsKf.data();
  p.obs_idx = obsIdx.data();
  p.obs_octave = obsOct.data();
  p.obs_stereo = obsStereo.data();
  p.n_local = L;
  p.local_kf = localKf.data();
  p.slot_off = slotOff.data();
  p.slot_mp = slotMp.data();
  p.slot_octave = slotOct.data();
  p.slot_depth = slotDepth.data();
  p.monocular = bMonocular ? 1 : 0;

  std::vector<uint8_t> verdict((size_t)L), rBad((size_t)nmp), rAlive(obsKf.size());
  std::vector<int32_t> nMps((size_t)L), nRed((size_t)L), rNobs((size_t)nmp), rSlot(slotMp.size());
  b2s_culling_result r{verdict.data(), nMps.data(), nRed.data(), rBad.data(), rNobs.data(), rAlive.data(), rSlot.data(),
                       0};
  int rc;
  {
    std::lock_guard<std::mutex> lock(g_culling.m);
    b2s_culling* h = g_culling.get(n, nmp, (int)obsKf.size(), L, (int)slotMp.size());
    if (!h) return B2S_ERR_CUDA;
    rc = b2s_keyframe_culling(h, 1, &p, &r);
  }
  if (rc != B2S_OK) {
    fprintf(stderr, "KeyFrameCulling (b200): %s\n", b2s_last_error());
    return rc;
  }
  for (int l = 0; l < L; l++)
    if (verdict[(size_t)l] == B2S_CULL_CULLED || verdict[(size_t)l] == B2S_CULL_DEFERRED) vpLocal[(size_t)l]->SetBadFlag();
  return B2S_OK;
}

}  // namespace b200
}  // namespace ORB_SLAM2
