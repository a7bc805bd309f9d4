// TEST INFRASTRUCTURE — CPU restatement, statement by statement, of
//   MapPoint::UpdateNormalAndDepth (src/MapPoint.cc:477-521)                 orc_update_normal_and_depth
//   the association loop of LocalMapping::ProcessNewKeyFrame (src/LocalMapping.cc:217-249), with the AddObservation
//   (src/MapPoint.cc:138-152), UpdateNormalAndDepth and ComputeDistinctiveDescriptors (:359-440) it calls, then
//   LocalMapping::MapPointCulling (:261-308) with MapPoint::SetBadFlag (:217-234)  orc_process_new_keyframe
// over the flattened tables of include/b200slam.h.  It runs the reference's serial loops on a std::map / std::list
// model, not the device's parallel passes, so the two can be compared.  Keyframes are table indices in address order,
// so a std::map<int, size_t> iterates a point's observers in the reference's order.  The OpenCV forms (DESIGN.md §7):
// Mat - Mat is a float subtraction; cv::norm of a float 3 x 1 column sums the squares in double in order; `normal +
// normali/s` is scaleAdd with alpha (float)(1./s), fused and rounded once; `normal/n` is convertTo with (float)(1./n).
// Built into oracle/liborb_kfinsert.so by kfinsert.mk.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <list>
#include <map>
#include <vector>

#include "../include/b200slam.h"

namespace {

double norm3(const float* v) {  // cv::norm (NORM_L2) of a CV_32F 3 x 1 column: double squares in order
  const double x = v[0], y = v[1], z = v[2];
  return std::sqrt((x * x + y * y) + z * z);
}

// The normal and distances of one good, observed point: obs are its observers (table index -> octave) in map order
void normal_and_depth(const float* pos, const std::vector<int>& kfs, int refOctave, int ref, const float* centers,
                      const float* sf, int nlev, float* normal, float* minD, float* maxD) {
  float nrm[3] = {0.f, 0.f, 0.f};
  int n = 0;
  for (int k : kfs) {
    const float* Owi = centers + 3 * (size_t)k;
    float normali[3];
    for (int i = 0; i < 3; i++) normali[i] = pos[i] - Owi[i];
    const float alpha = (float)(1. / norm3(normali));
    for (int i = 0; i < 3; i++) nrm[i] = std::fmaf(normali[i], alpha, nrm[i]);
    n++;
  }
  float PC[3];
  for (int i = 0; i < 3; i++) PC[i] = pos[i] - centers[3 * (size_t)ref + i];
  const float dist = (float)norm3(PC);
  const float levelScaleFactor = sf[refOctave];
  *maxD = dist * levelScaleFactor;
  *minD = *maxD / sf[nlev - 1];
  const float inv = (float)(1. / n);
  for (int i = 0; i < 3; i++) {
    normal[i] = nrm[i] * inv + 0.f;  // convertTo: src * alpha + beta, beta = 0
  }
}

int hamming(const uint8_t* a, const uint8_t* b) {
  int d = 0;
  for (int i = 0; i < 32; i++) d += __builtin_popcount((unsigned)(a[i] ^ b[i]));
  return d;
}

struct Point {
  bool mbBad;
  int nObs;
  std::map<int, size_t> mObservations;  // keyframe -> idx
};

}  // namespace

extern "C" {

int orc_update_normal_and_depth(const b2s_normal_depth_problem* p, b2s_normal_depth_result* r) {
  for (int m = 0; m < p->n_mp; m++) {
    r->updated[m] = 0;
    if (p->mp_bad[m] || p->obs_off[m + 1] == p->obs_off[m]) continue;
    std::vector<int> kfs;
    int refOct = -1;
    for (int o = p->obs_off[m]; o < p->obs_off[m + 1]; o++) {
      kfs.push_back(p->obs_kf[o]);
      if (p->obs_kf[o] == p->mp_ref[m]) refOct = p->obs_octave[o];
    }
    if (refOct < 0) return B2S_ERR_BAD_ARG;
    normal_and_depth(p->mp_pos + 3 * (size_t)m, kfs, refOct, p->mp_ref[m], p->kf_center, p->scale_factors,
                     p->n_levels, r->normal + 3 * (size_t)m, r->min_dist + m, r->max_dist + m);
    r->updated[m] = 1;
  }
  return B2S_OK;
}

int orc_process_new_keyframe(const b2s_kfinsert_problem* p, b2s_kfinsert_result* r) {
  const int cur = p->cur;
  std::vector<Point> mps((size_t)p->n_mp);
  std::map<std::pair<int, size_t>, int> obsEntry;  // (point, keyframe) of an entry observation -> its index
  for (int m = 0; m < p->n_mp; m++) {
    mps[(size_t)m].mbBad = p->mp_bad[m] != 0;
    mps[(size_t)m].nObs = p->mp_nobs[m];
    for (int o = p->obs_off[m]; o < p->obs_off[m + 1]; o++) {
      mps[(size_t)m].mObservations[p->obs_kf[o]] = (size_t)p->obs_idx[o];
      obsEntry[{m, (size_t)p->obs_kf[o]}] = o;
    }
    r->mp_added[m] = -1;
    r->mp_updated[m] = 0;
    r->mp_desc[m] = -1;
  }
  std::vector<int> slots(p->slot_mp, p->slot_mp + p->n_slots);
  std::list<int> recent(p->recent, p->recent + p->n_recent);

  // ProcessNewKeyFrame (:217-249)
  for (int i = 0; i < p->n_slots; i++) {
    const int m = slots[(size_t)i];
    if (m < 0) continue;
    Point& mp = mps[(size_t)m];
    if (mp.mbBad) continue;
    if (!mp.mObservations.count(cur)) {
      // AddObservation(mpCurrentKeyFrame, i)
      mp.mObservations[cur] = (size_t)i;
      mp.nObs += p->slot_stereo[i] ? 2 : 1;
      r->mp_added[m] = i;
      // UpdateNormalAndDepth
      std::vector<int> kfs;
      for (auto& kv : mp.mObservations) kfs.push_back(kv.first);
      int refOct = -1;
      for (int o = p->obs_off[m]; o < p->obs_off[m + 1]; o++)
        if (p->obs_kf[o] == p->mp_ref[m]) refOct = p->obs_octave[o];
      if (refOct < 0) return B2S_ERR_BAD_ARG;
      normal_and_depth(p->mp_pos + 3 * (size_t)m, kfs, refOct, p->mp_ref[m], p->kf_center, p->scale_factors,
                       p->n_levels, r->mp_normal + 3 * (size_t)m, r->mp_min_dist + m, r->mp_max_dist + m);
      r->mp_updated[m] = 1;
      // ComputeDistinctiveDescriptors
      std::vector<const uint8_t*> desc;
      std::vector<int> rowPos;
      int j = 0;
      for (auto& kv : mp.mObservations) {
        if (!p->kf_bad[kv.first])
          desc.push_back(kv.first == cur ? p->slot_desc + 32 * kv.second
                                         : p->obs_desc + 32 * (size_t)obsEntry[{m, (size_t)kv.first}]),
              rowPos.push_back(j);
        j++;
      }
      if (desc.empty()) continue;
      const size_t N = desc.size();
      std::vector<std::vector<int> > D(N, std::vector<int>(N, 0));
      for (size_t a = 0; a < N; a++)
        for (size_t b = a + 1; b < N; b++) D[a][b] = D[b][a] = hamming(desc[a], desc[b]);
      int BestMedian = INT_MAX, BestIdx = 0;
      for (size_t a = 0; a < N; a++) {
        std::vector<int> v = D[a];
        std::sort(v.begin(), v.end());
        const int median = v[(size_t)(0.5 * (N - 1))];
        if (median < BestMedian) {
          BestMedian = median;
          BestIdx = (int)a;
        }
      }
      r->mp_desc[m] = rowPos[(size_t)BestIdx];
    } else {
      recent.push_back(m);
    }
  }
  int n = 0;
  for (int m : recent) r->list_mp[n++] = m;
  r->n_list = n;

  // MapPointCulling (:261-308)
  const int nThObs = p->monocular ? 2 : 3;
  const int nCurrentKFid = (int)(uint32_t)p->cur_id;
  int e = 0, culled = 0;
  for (auto lit = recent.begin(); lit != recent.end(); e++) {
    const int m = *lit;
    Point& mp = mps[(size_t)m];
    const float ratio = static_cast<float>(p->mp_found[m]) / p->mp_visible[m];
    const int age = (int)((uint32_t)nCurrentKFid - (uint32_t)(int)(uint32_t)(uint64_t)p->mp_first_kf[m]);
    int v;
    if (mp.mbBad) {
      v = B2S_KFI_BAD;
    } else if (ratio < 0.25f) {
      v = B2S_KFI_CULLED_RATIO;
    } else if (age >= 2 && mp.nObs <= nThObs) {
      v = B2S_KFI_CULLED_OBS;
    } else if (age >= 3) {
      v = B2S_KFI_RETIRED;
    } else {
      v = B2S_KFI_KEPT;
    }
    r->list_verdict[e] = (uint8_t)v;
    if (v == B2S_KFI_CULLED_RATIO || v == B2S_KFI_CULLED_OBS) {  // SetBadFlag: EraseMapPointMatch on every observer
      culled++;
      mp.mbBad = true;
      for (auto& kv : mp.mObservations)
        if (kv.first == cur) slots[kv.second] = -1;
      mp.mObservations.clear();
    }
    if (v == B2S_KFI_KEPT)
      ++lit;
    else
      lit = recent.erase(lit);
  }
  r->n_culled = culled;

  for (int m = 0; m < p->n_mp; m++) {
    const Point& mp = mps[(size_t)m];
    r->mp_nobs[m] = mp.nObs;
    r->mp_bad[m] = mp.mbBad;
    for (int o = p->obs_off[m]; o < p->obs_off[m + 1]; o++) r->obs_alive[o] = mp.mObservations.count(p->obs_kf[o]) != 0;
  }
  if (p->n_slots) memcpy(r->slot_mp, slots.data(), sizeof(int) * (size_t)p->n_slots);
  return B2S_OK;
}
}
