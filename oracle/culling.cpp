// TEST INFRASTRUCTURE — CPU restatement of LocalMapping::KeyFrameCulling (src/LocalMapping.cc:873-956) over the flattened
// tables of one b2s_culling_problem, statement by statement, with the point-side effects of the KeyFrame::SetBadFlag it
// calls (src/KeyFrame.cc:599-722): MapPoint::EraseObservation (src/MapPoint.cc:170-200) and MapPoint::SetBadFlag
// (:217-234) with KeyFrame::EraseMapPointMatch(idx) on the observers.  Keyframes are table indices; the observations of
// a point are a std::map<int, size_t> in index order.  Slots of keyframes outside the local list are not part of the
// problem: EraseMapPointMatch on them changes nothing the result holds.  Built into oracle/liborb_culling.so by
// culling.mk.
#include <map>
#include <vector>

#include "../include/b200slam.h"

namespace {

struct Point {
  bool mbBad;
  int nObs;
  std::map<int, size_t> mObservations;  // keyframe -> idx
};

struct State {
  const b2s_culling_problem* p;
  std::vector<Point> mps;
  std::vector<std::vector<int> > slots;  // mvpMapPoints of each local keyframe
  std::vector<int> localPos;             // table index -> position in the local list, -1 outside it

  int obsEntry(int m, int k) const {
    for (int o = p->obs_off[m]; o < p->obs_off[m + 1]; o++)
      if (p->obs_kf[o] == k) return o;
    return -1;
  }
  // KeyFrame::EraseMapPointMatch(const size_t& idx) (src/KeyFrame.cc)
  void EraseMapPointMatch(int k, size_t idx) {
    const int l = localPos[(size_t)k];
    if (l >= 0) slots[(size_t)l][idx] = -1;
  }
  // MapPoint::SetBadFlag (src/MapPoint.cc:217-234)
  void SetBadFlag(int m) {
    std::map<int, size_t> obs;
    {
      mps[(size_t)m].mbBad = true;
      obs = mps[(size_t)m].mObservations;
      mps[(size_t)m].mObservations.clear();
    }
    for (std::map<int, size_t>::iterator mit = obs.begin(), mend = obs.end(); mit != mend; mit++)
      EraseMapPointMatch(mit->first, mit->second);
  }
  // MapPoint::EraseObservation (src/MapPoint.cc:170-200)
  void EraseObservation(int m, int k) {
    bool bBad = false;
    Point& P = mps[(size_t)m];
    if (P.mObservations.count(k)) {
      const int o = obsEntry(m, k);  // the observation's idx is P.mObservations[k]; its stereo flag sits beside it
      if (p->obs_stereo[o])
        P.nObs -= 2;
      else
        P.nObs--;
      P.mObservations.erase(k);
      if (P.nObs <= 2) bBad = true;
    }
    if (bBad) SetBadFlag(m);
  }
  // KeyFrame::SetBadFlag (src/KeyFrame.cc:599-722), its effects on points
  void KeyFrameSetBadFlag(int l, uint8_t* verdict) {
    const int k = p->local_kf[l];
    if (p->kf_id[k] == 0) return;
    if (p->not_erase[k]) {  // mbToBeErased = true
      verdict[l] = B2S_CULL_DEFERRED;
      return;
    }
    verdict[l] = B2S_CULL_CULLED;
    std::vector<int>& mv = slots[(size_t)l];
    for (size_t i = 0; i < mv.size(); i++)
      if (mv[i] >= 0) EraseObservation(mv[i], k);
  }
};

}  // namespace

extern "C" int orc_keyframe_culling(const b2s_culling_problem* p, b2s_culling_result* r) {
  State st;
  st.p = p;
  st.mps.resize((size_t)p->n_mp);
  for (int m = 0; m < p->n_mp; m++) {
    st.mps[(size_t)m].mbBad = p->mp_bad[m] != 0;
    st.mps[(size_t)m].nObs = p->mp_nobs[m];
    for (int o = p->obs_off[m]; o < p->obs_off[m + 1]; o++)
      st.mps[(size_t)m].mObservations[p->obs_kf[o]] = (size_t)p->obs_idx[o];
  }
  st.localPos.assign((size_t)p->n_kf, -1);
  st.slots.resize((size_t)p->n_local);
  for (int l = 0; l < p->n_local; l++) {
    st.localPos[(size_t)p->local_kf[l]] = l;
    st.slots[(size_t)l].assign(p->slot_mp + p->slot_off[l], p->slot_mp + p->slot_off[l + 1]);
  }
  const bool mbMonocular = p->monocular != 0;

  // :881-955
  for (int l = 0; l < p->n_local; l++) {
    const int pKF = p->local_kf[l];
    r->verdict[l] = B2S_CULL_SKIPPED;
    r->n_mps[l] = r->n_redundant[l] = 0;
    if (p->kf_id[pKF] == 0) continue;
    const std::vector<int> vpMapPoints = st.slots[(size_t)l];
    const int so = p->slot_off[l];

    int nObs = 3;
    const int thObs = nObs;
    int nRedundantObservations = 0;
    int nMPs = 0;
    for (size_t i = 0, iend = vpMapPoints.size(); i < iend; i++) {
      const int pMP = vpMapPoints[i];
      if (pMP >= 0) {
        if (!st.mps[(size_t)pMP].mbBad) {
          if (!mbMonocular) {
            const float d = p->slot_depth[so + i];
            if (d > p->th_depth[pKF] || d < 0) continue;
          }
          nMPs++;
          if (st.mps[(size_t)pMP].nObs > thObs) {
            const int& scaleLevel = p->slot_octave[so + i];
            const std::map<int, size_t> observations = st.mps[(size_t)pMP].mObservations;
            int nObs = 0;
            for (std::map<int, size_t>::const_iterator mit = observations.begin(), mend = observations.end();
                 mit != mend; mit++) {
              const int pKFi = mit->first;
              if (pKFi == pKF) continue;
              const int scaleLeveli = p->obs_octave[st.obsEntry(pMP, pKFi)];
              if ((long long)scaleLeveli <= (long long)scaleLevel + 1) {
                nObs++;
                if (nObs >= thObs) break;
              }
            }
            if (nObs >= thObs) nRedundantObservations++;
          }
        }
      }
    }
    r->n_mps[l] = nMPs;
    r->n_redundant[l] = nRedundantObservations;
    r->verdict[l] = B2S_CULL_KEPT;
    if (nRedundantObservations > 0.9 * nMPs) st.KeyFrameSetBadFlag(l, r->verdict);
  }

  int culled = 0;
  for (int l = 0; l < p->n_local; l++) culled += r->verdict[l] == B2S_CULL_CULLED;
  r->n_culled = culled;
  for (int m = 0; m < p->n_mp; m++) {
    r->mp_bad[m] = st.mps[(size_t)m].mbBad;
    r->mp_nobs[m] = st.mps[(size_t)m].nObs;
    for (int o = p->obs_off[m]; o < p->obs_off[m + 1]; o++)
      r->obs_alive[o] = st.mps[(size_t)m].mObservations.count(p->obs_kf[o]) != 0;
  }
  for (int l = 0; l < p->n_local; l++)
    for (int s = p->slot_off[l]; s < p->slot_off[l + 1]; s++) r->slot_mp[s] = st.slots[(size_t)l][(size_t)(s - p->slot_off[l])];
  return B2S_OK;
}
