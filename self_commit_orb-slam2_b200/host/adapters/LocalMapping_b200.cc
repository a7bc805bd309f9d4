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
//
// ProcessNewKeyFrame's association and MapPointCulling over b2s_process_new_keyframe (one matcher handle for the
// process).  The reads take the reference's locks: GetMapPointMatches, and isBad / GetObservations / Observations /
// GetWorldPos / GetReferenceKeyFrame / GetFound, and mnVisible under the point's mMutexFeatures (protected, through
// member pointers); GetCameraCenter and isBad of the keyframes.  The keyframe table is the current keyframe and every
// observer of the points in std::less<KeyFrame*> order, the order of the reference's std::map, so the device sums
// UpdateNormalAndDepth's terms in the reference's order.  The writes: the reference's AddObservation, then the normal,
// the distances (under mMutexPos) and the descriptor (under mMutexFeatures) through member pointers; then the
// reference's UpdateConnections, Map::AddKeyFrame and, in list order, MapPoint::SetBadFlag.
#include "adapters/LocalMapping_b200.h"

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <iterator>
#include <list>
#include <map>
#include <mutex>
#include <set>
#include <unordered_map>
#include <vector>

#include "MapPoint.h"
#include "b200slam.h"
#include "../b2s_host.h"

namespace ORB_SLAM2 {
namespace b200 {
namespace {

struct Access : KeyFrame {
  static bool KeyFrame::*notErase() { return &Access::mbNotErase; }
  static std::mutex KeyFrame::*mutexConnections() { return &Access::mMutexConnections; }
};
struct MpAccess : MapPoint {
  static int MapPoint::*visible() { return &MpAccess::mnVisible; }
  static std::mutex MapPoint::*mutexFeatures() { return &MpAccess::mMutexFeatures; }
  static std::mutex MapPoint::*mutexPos() { return &MpAccess::mMutexPos; }
  static cv::Mat MapPoint::*normal() { return &MpAccess::mNormalVector; }
  static cv::Mat MapPoint::*descriptor() { return &MpAccess::mDescriptor; }
  static float MapPoint::*minD() { return &MpAccess::mfMinDistance; }
  static float MapPoint::*maxD() { return &MpAccess::mfMaxDistance; }
};

// One handle for the process, grown on demand; capacities: keyframes, points, observations, local keyframes, slots.
b2s_host::Slot<b2s_culling, 5, b2s_culling_destroy> g_culling;

bool by_id(const KeyFrame* a, const KeyFrame* b) { return a->mnId < b->mnId; }

// One matcher handle for the process (its buffers grow on demand).
b2s_host::Slot<b2s_matcher, 1, b2s_matcher_destroy> g_matcher;

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
    std::lock_guard<std::mutex> lock(g_culling.mutex);
    rc = g_culling.get({n, nmp, (int)obsKf.size(), L, (int)slotMp.size()}, {256, 8192, 65536, 256, 65536},
                       [](const int* c, b2s_culling** h) {
                         return b2s_culling_create(c[0], c[1], c[2], c[3], c[4], 1, b2s_host::device(), h);
                       });
    if (rc == B2S_OK) rc = b2s_keyframe_culling(g_culling.h, 1, &p, &r);
  }
  if (rc != B2S_OK) {
    b2s_host::report("KeyFrameCulling", rc);
    return rc;
  }
  for (int l = 0; l < L; l++)
    if (verdict[(size_t)l] == B2S_CULL_CULLED || verdict[(size_t)l] == B2S_CULL_DEFERRED) vpLocal[(size_t)l]->SetBadFlag();
  return B2S_OK;
}

int ProcessNewKeyFrame(KeyFrame* pKF, Map* pMap, std::list<MapPoint*>& lRecent, bool bMonocular) {
  // 1. the tables, under the reference's locks
  const std::vector<MapPoint*> slots = pKF->GetMapPointMatches();
  std::unordered_map<MapPoint*, int> mpIndex;
  std::vector<MapPoint*> mps;
  for (MapPoint* pMP : slots)
    if (pMP && mpIndex.emplace(pMP, (int)mps.size()).second) mps.push_back(pMP);
  for (MapPoint* pMP : lRecent)
    if (mpIndex.emplace(pMP, (int)mps.size()).second) mps.push_back(pMP);
  const int nmp = (int)mps.size();
  std::vector<uint8_t> mpBad((size_t)nmp);
  std::vector<int32_t> mpNobs((size_t)nmp), mpFound((size_t)nmp), mpVisible((size_t)nmp), mpRef((size_t)nmp, -1);
  std::vector<int64_t> mpFirst((size_t)nmp);
  std::vector<float> mpPos(3 * (size_t)nmp);
  std::vector<KeyFrame*> refKf((size_t)nmp);
  std::vector<std::map<KeyFrame*, size_t> > obs((size_t)nmp);
  std::set<KeyFrame*> all;  // std::less<KeyFrame*>: the order of the points' std::map
  all.insert(pKF);
  for (int m = 0; m < nmp; m++) {
    MapPoint* pMP = mps[(size_t)m];
    mpBad[(size_t)m] = pMP->isBad();
    obs[(size_t)m] = pMP->GetObservations();
    mpNobs[(size_t)m] = pMP->Observations();
    mpFound[(size_t)m] = pMP->GetFound();
    {
      std::unique_lock<std::mutex> lock(pMP->*MpAccess::mutexFeatures());
      mpVisible[(size_t)m] = pMP->*MpAccess::visible();
    }
    mpFirst[(size_t)m] = pMP->mnFirstKFid;
    const cv::Mat P = pMP->GetWorldPos();
    for (int c = 0; c < 3; c++) mpPos[3 * (size_t)m + c] = P.at<float>(c);
    refKf[(size_t)m] = pMP->GetReferenceKeyFrame();
    for (auto& kv : obs[(size_t)m]) all.insert(kv.first);
  }
  const std::vector<KeyFrame*> table(all.begin(), all.end());
  std::unordered_map<KeyFrame*, int> idx;
  for (size_t i = 0; i < table.size(); i++) idx[table[i]] = (int)i;
  const int n = (int)table.size();
  std::vector<float> centers(3 * (size_t)n);
  std::vector<uint8_t> kfBad((size_t)n);
  for (int i = 0; i < n; i++) {
    const cv::Mat Ow = table[(size_t)i]->GetCameraCenter();
    for (int c = 0; c < 3; c++) centers[3 * (size_t)i + c] = Ow.at<float>(c);
    kfBad[(size_t)i] = table[(size_t)i]->isBad();
  }
  for (int m = 0; m < nmp; m++) {
    const auto it = idx.find(refKf[(size_t)m]);
    if (it != idx.end()) mpRef[(size_t)m] = it->second;
  }
  std::vector<int32_t> obsOff(1, 0), obsKf, obsIdx, obsOct;
  std::vector<uint8_t> obsDesc;
  for (int m = 0; m < nmp; m++) {
    for (auto& kv : obs[(size_t)m]) {  // already in table order
      KeyFrame* k = kv.first;
      if (kv.second >= k->mvKeysUn.size() || (int)kv.second >= k->mDescriptors.rows) {
        fprintf(stderr, "ProcessNewKeyFrame (b200): an observation's index lies outside its keyframe's keypoints\n");
        return B2S_ERR_BAD_ARG;
      }
      obsKf.push_back(idx[k]);
      obsIdx.push_back((int32_t)kv.second);
      obsOct.push_back(k->mvKeysUn[kv.second].octave);
      const unsigned char* d = reinterpret_cast<const unsigned char*>(k->mDescriptors.row((int)kv.second).data);
      obsDesc.insert(obsDesc.end(), d, d + 32);
    }
    obsOff.push_back((int32_t)obsKf.size());
  }
  const int S = (int)slots.size();
  std::vector<int32_t> slotMp((size_t)S);
  std::vector<uint8_t> slotStereo((size_t)S), slotDesc(32 * (size_t)S);
  for (int s = 0; s < S; s++) {
    slotMp[(size_t)s] = slots[(size_t)s] ? mpIndex[slots[(size_t)s]] : -1;
    slotStereo[(size_t)s] = pKF->mvuRight[(size_t)s] >= 0;
    memcpy(&slotDesc[32 * (size_t)s], reinterpret_cast<const unsigned char*>(pKF->mDescriptors.row(s).data), 32);
  }
  std::vector<int32_t> recent;
  for (MapPoint* pMP : lRecent) recent.push_back(mpIndex[pMP]);

  b2s_kfinsert_problem p;
  p.n_kf = n;
  p.kf_center = centers.data();
  p.kf_bad = kfBad.data();
  p.cur = idx[pKF];
  p.cur_id = pKF->mnId;
  p.n_slots = S;
  p.slot_mp = slotMp.data();
  p.slot_stereo = slotStereo.data();
  p.slot_desc = slotDesc.data();
  p.n_mp = nmp;
  p.mp_pos = mpPos.data();
  p.mp_bad = mpBad.data();
  p.mp_ref = mpRef.data();
  p.mp_nobs = mpNobs.data();
  p.mp_found = mpFound.data();
  p.mp_visible = mpVisible.data();
  p.mp_first_kf = mpFirst.data();
  p.obs_off = obsOff.data();
  p.obs_kf = obsKf.data();
  p.obs_idx = obsIdx.data();
  p.obs_octave = obsOct.data();
  p.obs_desc = obsDesc.data();
  p.n_recent = (int)recent.size();
  p.recent = recent.data();
  p.scale_factors = pKF->mvScaleFactors.data();
  p.n_levels = pKF->mnScaleLevels;
  p.monocular = bMonocular ? 1 : 0;

  // 2. one device call
  const size_t L = recent.size() + (size_t)S;
  std::vector<int32_t> rNobs((size_t)nmp), rAdded((size_t)nmp), rDesc((size_t)nmp), rSlot((size_t)S), rList(L);
  std::vector<uint8_t> rBad((size_t)nmp), rAlive(obsKf.size()), rUpdated((size_t)nmp), rVerdict(L);
  std::vector<float> rNormal(3 * (size_t)nmp), rMin((size_t)nmp), rMax((size_t)nmp);
  b2s_kfinsert_result r{rNobs.data(), rBad.data(),    rAdded.data(), rAlive.data(), rUpdated.data(),
                        rNormal.data(), rMin.data(),  rMax.data(),   rDesc.data(),  rSlot.data(),
                        rList.data(),  rVerdict.data(), 0,           0};
  int rc;
  {
    std::lock_guard<std::mutex> lock(g_matcher.mutex);
    rc = g_matcher.get({4096}, {4096}, [](const int* c, b2s_matcher** h) {
      return b2s_matcher_create(c[0], 1, b2s_host::device(), h);
    });
    if (rc == B2S_OK) rc = b2s_process_new_keyframe(g_matcher.h, 1, &p, &r);
  }
  if (rc != B2S_OK) {
    b2s_host::report("ProcessNewKeyFrame", rc);
    return rc;
  }

  // 3. the association (:229-237): AddObservation, then the normal, distances and descriptor the device computed
  for (int m = 0; m < nmp; m++) {
    if (rAdded[(size_t)m] < 0) continue;
    MapPoint* pMP = mps[(size_t)m];
    pMP->AddObservation(pKF, (size_t)rAdded[(size_t)m]);
    {
      std::unique_lock<std::mutex> lock(pMP->*MpAccess::mutexPos());
      cv::Mat nv(3, 1, CV_32F);
      for (int c = 0; c < 3; c++) nv.at<float>(c) = rNormal[3 * (size_t)m + c];
      pMP->*MpAccess::normal() = nv;
      pMP->*MpAccess::minD() = rMin[(size_t)m];
      pMP->*MpAccess::maxD() = rMax[(size_t)m];
    }
    const int j = rDesc[(size_t)m];
    if (j < 0) continue;
    // position j of the row with the new observation inserted: the j-th observer in map order
    const std::map<KeyFrame*, size_t> o = pMP->GetObservations();
    auto it = o.begin();
    std::advance(it, j);
    std::unique_lock<std::mutex> lock(pMP->*MpAccess::mutexFeatures());
    pMP->*MpAccess::descriptor() = it->first->mDescriptors.row((int)it->second).clone();
  }
  // 4. the rest of ProcessNewKeyFrame (:250-253)
  pKF->UpdateConnections();
  pMap->AddKeyFrame(pKF);
  // 5. MapPointCulling's SetBadFlag calls, in list order, and 6. the list it leaves
  lRecent.clear();
  for (int e = 0; e < r.n_list; e++) {
    MapPoint* pMP = mps[(size_t)rList[(size_t)e]];
    if (rVerdict[(size_t)e] == B2S_KFI_CULLED_RATIO || rVerdict[(size_t)e] == B2S_KFI_CULLED_OBS) pMP->SetBadFlag();
    if (rVerdict[(size_t)e] == B2S_KFI_KEPT) lRecent.push_back(pMP);
  }
  return B2S_OK;
}

}  // namespace b200
}  // namespace ORB_SLAM2
