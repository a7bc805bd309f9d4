// ORBmatcher_b200.cc — drop-in implementation of the reference's ORBmatcher class (include/ORBmatcher.h:57-215) on top of
// libb200slam.so: the constructor, DescriptorDistance and the eleven Search* / Fuse methods keep their exact signatures on
// Frame& / KeyFrame* / MapPoint*, so Tracking, LocalMapping and LoopClosing call them unchanged
// (src/Tracking.cc:937, 1189, 1355, 1817, 2048, 2102; src/LocalMapping.cc:323, 668; src/LoopClosing.cc:345, 453, 533, 812).
// Compile this file INSIDE the reference tree in place of src/ORBmatcher.cc (it includes the reference's own
// include/ORBmatcher.h) and link libb200slam.so.
//
// Every method is gather -> one C-ABI call -> scatter:
//   * gather: what only the object graph knows — which features hold usable map points, the DBoW2 node of every feature,
//     the projection of a map point with the caller's pose (float cv::Mat algebra, same expression order as the
//     reference so the windows are the same floats), the visibility / distance / normal gates that come before the
//     descriptor search;
//   * search on the GPU: candidate enumeration on the 64 x 48 feature grid, Hamming distances, best / second-best, ratio
//     tests, greedy occupancy, the rotation-histogram cull (csrc/matcher.cu);
//   * scatter: the assignments and the map bookkeeping (AddObservation / AddMapPoint / Replace / vpReplacePoint), in the
//     reference's iteration order.
// One difference in evaluation order is inherent to batching: inside Fuse the gates of map point i are evaluated before
// the bookkeeping of points < i is applied (the reference interleaves them); the stand-in objects of the parity tests
// only log that bookkeeping, like the reference's own data flow within one call does not depend on it.
//
// tests: oracle/ref_matcher_glue.cpp drives this file (oracle/_ref/libadapter_matcher.so) and the reference's own
// src/ORBmatcher.cc (libref_matcher.so) on the same stand-in objects; tests/test_adapters_gpu.py requires identical
// match arrays and counts for all eleven methods.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <set>
#include <string>
#include <vector>

#include "ORBmatcher.h"

#include "b200slam.h"
#include "../b2s_host.h"

using namespace std;

namespace ORB_SLAM2 {

const int ORBmatcher::TH_HIGH = 100;
const int ORBmatcher::TH_LOW = 50;
const int ORBmatcher::HISTO_LENGTH = 30;

namespace {

// ORBmatcher objects are stack temporaries (one per call site); the device handle they use is per THREAD, grown on demand
// and destroyed at thread exit: creating one costs a stream and ~30 cudaMalloc, destroying one synchronises the device.
struct ThreadHandle : b2s_host::Slot<b2s_matcher, 1, b2s_matcher_destroy> {
  ~ThreadHandle() { b2s_matcher_destroy(h); }
};
b2s_matcher* handle_for(int n) {
  static thread_local ThreadHandle slot;
  const int rc = slot.get({n}, {4096}, [](const int* c, b2s_matcher** h) {
    return b2s_matcher_create(c[0], 1, b2s_host::device(), h);
  });
  if (rc != B2S_OK) b2s_host::report("ORBmatcher", rc);
  return slot.h;
}
bool ok(int rc, const char* where) {
  if (rc == B2S_OK) return true;
  b2s_host::report(("ORBmatcher::" + std::string(where)).c_str(), rc);
  return false;
}

// flat views of a Frame / KeyFrame
struct Flat {
  vector<float> x, y, angle, uright;
  vector<int32_t> octave;
  vector<uint8_t> descCopy;
  const uint8_t* desc = nullptr;
  int n = 0;
};
template <class H>
void flatten(const H& f, Flat& o) {
  o.n = (int)f.mvKeysUn.size();
  o.x.resize(o.n);
  o.y.resize(o.n);
  o.angle.resize(o.n);
  o.octave.resize(o.n);
  o.uright.assign(o.n, -1.f);
  for (int i = 0; i < o.n; i++) {
    const cv::KeyPoint& kp = f.mvKeysUn[i];
    o.x[i] = kp.pt.x;
    o.y[i] = kp.pt.y;
    o.angle[i] = kp.angle;
    o.octave[i] = kp.octave;
    if (i < (int)f.mvuRight.size()) o.uright[i] = f.mvuRight[i];
  }
  if ((size_t)f.mDescriptors.step == 32 || o.n == 0) {
    o.desc = f.mDescriptors.data;
  } else {  // rows are not contiguous: pack them
    o.descCopy.resize((size_t)o.n * 32);
    for (int i = 0; i < o.n; i++) memcpy(&o.descCopy[(size_t)i * 32], f.mDescriptors.ptr(i), 32);
    o.desc = o.descCopy.data();
  }
}
template <class H>
vector<int32_t> nodes_of(const H& f, int n) {
  vector<int32_t> node(n, -1);  // features without a node never match
  int32_t fill = -2;
  (void)fill;
  for (DBoW2::FeatureVector::const_iterator it = f.mFeatVec.begin(); it != f.mFeatVec.end(); ++it)
    for (size_t k = 0; k < it->second.size(); k++)
      if ((int)it->second[k] < n) node[it->second[k]] = (int32_t)it->first;
  return node;
}
b2s_frame_geom geom_of(const Frame& F) {
  b2s_frame_geom g;
  g.mnMinX = Frame::mnMinX;
  g.mnMinY = Frame::mnMinY;
  g.mnMaxX = Frame::mnMaxX;
  g.mnMaxY = Frame::mnMaxY;
  g.bf = F.mbf;
  g.scale_factors = F.mvScaleFactors.data();
  g.nlevels = (int)F.mvScaleFactors.size();
  return g;
}
b2s_frame_geom geom_of(const KeyFrame& K) {
  b2s_frame_geom g;
  g.mnMinX = (float)K.mnMinX;
  g.mnMinY = (float)K.mnMinY;
  g.mnMaxX = (float)K.mnMaxX;
  g.mnMaxY = (float)K.mnMaxY;
  g.bf = K.mbf;
  g.scale_factors = K.mvScaleFactors.data();
  g.nlevels = (int)K.mvScaleFactors.size();
  return g;
}
void put_desc(uint8_t* dst, MapPoint* p) {
  const cv::Mat d = p->GetDescriptor();
  memcpy(dst, d.data, 32);
}

// the window a map point opens in a keyframe after projection with (Rcw, tcw) seen from Ow: the gates of
// src/ORBmatcher.cc:424-466 / 1046-1092 / 1214-1262 in the reference's expression order
void window_query(MapPoint* pMP, KeyFrame* pKF, const cv::Mat& Rcw, const cv::Mat& tcw, const cv::Mat& Ow, float th,
                  bool withRight, b2s_win_query& q) {
  memset(&q, 0, sizeof(q));
  put_desc(q.desc, pMP);
  cv::Mat p3Dw = pMP->GetWorldPos();
  cv::Mat p3Dc = Rcw * p3Dw + tcw;
  if (p3Dc.at<float>(2) < 0.0f) return;
  const float invz = 1.0 / p3Dc.at<float>(2);
  const float x = p3Dc.at<float>(0) * invz;
  const float y = p3Dc.at<float>(1) * invz;
  const float u = pKF->fx * x + pKF->cx;
  const float v = pKF->fy * y + pKF->cy;
  if (!pKF->IsInImage(u, v)) return;
  const float ur = u - pKF->mbf * invz;
  const float maxDistance = pMP->GetMaxDistanceInvariance();
  const float minDistance = pMP->GetMinDistanceInvariance();
  cv::Mat PO = p3Dw - Ow;
  const float dist3D = cv::norm(PO);
  if (dist3D < minDistance || dist3D > maxDistance) return;
  cv::Mat Pn = pMP->GetNormal();
  if (PO.dot(Pn) < 0.5 * dist3D) return;
  const int level = pMP->PredictScale(dist3D, pKF);
  q.u = u;
  q.v = v;
  q.ur = withRight ? ur : 0.f;
  q.radius = th * pKF->mvScaleFactors[level];
  q.min_level = level - 1;
  q.max_level = level;
  q.valid = 1;
}

void sim3_parts(const cv::Mat& Scw, cv::Mat& Rcw, cv::Mat& tcw, cv::Mat& Ow) {
  cv::Mat sRcw = Scw.rowRange(0, 3).colRange(0, 3);
  const float scw = sqrt(sRcw.row(0).dot(sRcw.row(0)));
  Rcw = sRcw / scw;
  tcw = Scw.rowRange(0, 3).col(3) / scw;
  Ow = -Rcw.t() * tcw;
}

int run_windows(KeyFrame* pKF, const vector<b2s_win_query>& q, const uint8_t* occupied, int flags, int thDist,
                vector<int32_t>& best, const char* where) {
  Flat k;
  flatten(*pKF, k);
  best.assign(q.size(), -1);
  if (q.empty() || k.n == 0) return 0;
  b2s_matcher* h = handle_for(std::max(k.n, (int)q.size()));
  if (!h) return 0;
  const b2s_frame_geom g = geom_of(*pKF);
  int n = 0;
  if (!ok(b2s_search_windows(h, q.data(), (int)q.size(), k.x.data(), k.y.data(), k.octave.data(), k.uright.data(),
                             pKF->mvInvLevelSigma2.data(), occupied, k.desc, k.n, &g, flags, thDist, best.data(), nullptr, &n),
          where)) {
    best.assign(q.size(), -1);
    return 0;
  }
  return n;
}

}  // namespace

ORBmatcher::ORBmatcher(float nnratio, bool checkOri) : mfNNratio(nnratio), mbCheckOrientation(checkOri) {}

int ORBmatcher::DescriptorDistance(const cv::Mat& a, const cv::Mat& b) {
  // one pair is not worth a launch (batches: b2s_descriptor_distance); 4 x 64-bit popcount
  int d = 0;
  for (int i = 0; i < 4; i++) {
    uint64_t x, y;
    memcpy(&x, a.data + 8 * i, 8);
    memcpy(&y, b.data + 8 * i, 8);
    d += __builtin_popcountll(x ^ y);
  }
  return d;
}

// ---- Tracking::SearchLocalPoints (src/ORBmatcher.cc:70-175)
int ORBmatcher::SearchByProjection(Frame& F, const vector<MapPoint*>& vpMapPoints, const float th) {
  const int nq = (int)vpMapPoints.size();
  if (nq == 0 || F.N == 0) return 0;
  vector<b2s_map_query> q((size_t)nq);
  for (int i = 0; i < nq; i++) {
    MapPoint* p = vpMapPoints[i];
    b2s_map_query& m = q[i];
    memset(&m, 0, sizeof(m));
    if (!p->mbTrackInView || p->isBad()) continue;
    m.u = p->mTrackProjX;
    m.v = p->mTrackProjY;
    m.ur = p->mTrackProjXR;
    m.view_cos = p->mTrackViewCos;
    m.level = p->mnTrackScaleLevel;
    m.in_view = 1;
    m.has_obs = p->Observations() > 0;
    put_desc(m.desc, p);
  }
  Flat f;
  flatten(F, f);
  vector<uint8_t> occupied((size_t)f.n, 0);
  for (int j = 0; j < f.n; j++) occupied[j] = F.mvpMapPoints[j] && F.mvpMapPoints[j]->Observations() > 0;
  b2s_matcher* h = handle_for(std::max(f.n, nq));
  if (!h) return 0;
  const b2s_frame_geom g = geom_of(F);
  vector<int32_t> match((size_t)f.n, -1);
  int n = 0;
  if (!ok(b2s_search_by_projection_map(h, q.data(), nq, f.x.data(), f.y.data(), f.octave.data(), f.uright.data(), occupied.data(),
                                       f.desc, f.n, &g, th, TH_HIGH, mfNNratio, match.data(), &n),
          "SearchByProjection(Frame, MapPoints)"))
    return 0;
  for (int j = 0; j < f.n; j++)
    if (match[j] >= 0) F.mvpMapPoints[j] = vpMapPoints[match[j]];
  return n;
}

// ---- Tracking::TrackReferenceKeyFrame / Relocalization (:230-382)
int ORBmatcher::SearchByBoW(KeyFrame* pKF, Frame& F, vector<MapPoint*>& vpMapPointMatches) {
  const vector<MapPoint*> vpMapPointsKF = pKF->GetMapPointMatches();
  vpMapPointMatches = vector<MapPoint*>(F.N, static_cast<MapPoint*>(NULL));
  Flat k, f;
  flatten(*pKF, k);
  flatten(F, f);
  if (k.n == 0 || f.n == 0) return 0;
  const vector<int32_t> nodeK = nodes_of(*pKF, k.n), nodeF = nodes_of(F, f.n);
  vector<uint8_t> valid((size_t)k.n, 0);
  for (int i = 0; i < k.n; i++) valid[i] = vpMapPointsKF[i] && !vpMapPointsKF[i]->isBad();
  vector<float> angF((size_t)f.n);
  for (int j = 0; j < f.n; j++) angF[j] = F.mvKeys[j].angle;  // (:325 reads F.mvKeys, not mvKeysUn)
  b2s_matcher* h = handle_for(std::max(k.n, f.n));
  if (!h) return 0;
  vector<int32_t> matchF((size_t)f.n, -1);
  int n = 0;
  if (!ok(b2s_search_by_bow(h, k.desc, nodeK.data(), valid.data(), k.angle.data(), k.n, f.desc, nodeF.data(), nullptr, angF.data(),
                            f.n, TH_LOW, mfNNratio, /*strict_lt=*/0, mbCheckOrientation, matchF.data(), &n),
          "SearchByBoW(KeyFrame, Frame)"))
    return 0;
  for (int j = 0; j < f.n; j++)
    if (matchF[j] >= 0) vpMapPointMatches[j] = vpMapPointsKF[matchF[j]];
  return n;
}

// ---- LoopClosing::ComputeSim3 (:388-512)
int ORBmatcher::SearchByProjection(KeyFrame* pKF, cv::Mat Scw, const vector<MapPoint*>& vpPoints, vector<MapPoint*>& vpMatched,
                                   int th) {
  cv::Mat Rcw, tcw, Ow;
  sim3_parts(Scw, Rcw, tcw, Ow);
  set<MapPoint*> spAlreadyFound(vpMatched.begin(), vpMatched.end());
  spAlreadyFound.erase(static_cast<MapPoint*>(NULL));
  vector<b2s_win_query> q(vpPoints.size());
  for (size_t i = 0; i < vpPoints.size(); i++) {
    memset(&q[i], 0, sizeof(b2s_win_query));
    MapPoint* p = vpPoints[i];
    if (p->isBad() || spAlreadyFound.count(p)) continue;
    window_query(p, pKF, Rcw, tcw, Ow, (float)th, false, q[i]);
  }
  vector<uint8_t> occupied(vpMatched.size(), 0);
  for (size_t j = 0; j < vpMatched.size(); j++) occupied[j] = vpMatched[j] != NULL;
  vector<int32_t> best;
  const int n = run_windows(pKF, q, occupied.data(), B2S_WIN_GREEDY, TH_LOW, best, "SearchByProjection(KeyFrame, Scw)");
  for (size_t i = 0; i < best.size(); i++)
    if (best[i] >= 0) vpMatched[best[i]] = vpPoints[i];
  return n;
}

// ---- Tracking::MonocularInitialization (:515-643)
int ORBmatcher::SearchForInitialization(Frame& F1, Frame& F2, vector<cv::Point2f>& vbPrevMatched, vector<int>& vnMatches12,
                                        int windowSize) {
  Flat a, b;
  flatten(F1, a);
  flatten(F2, b);
  vnMatches12 = vector<int>(a.n, -1);
  if (a.n == 0 || b.n == 0) return 0;
  vector<float> px((size_t)a.n), py((size_t)a.n);
  for (int i = 0; i < a.n; i++) {
    px[i] = vbPrevMatched[i].x;
    py[i] = vbPrevMatched[i].y;
  }
  b2s_matcher* h = handle_for(std::max(a.n, b.n));
  if (!h) return 0;
  const b2s_frame_geom g = geom_of(F2);
  vector<int32_t> m12((size_t)a.n, -1);
  int n = 0;
  if (!ok(b2s_search_for_initialization(h, px.data(), py.data(), a.octave.data(), a.angle.data(), a.desc, a.n, b.x.data(),
                                        b.y.data(), b.octave.data(), b.angle.data(), b.desc, b.n, &g, windowSize, TH_LOW,
                                        mfNNratio, mbCheckOrientation, m12.data(), &n),
          "SearchForInitialization"))
    return 0;
  for (int i = 0; i < a.n; i++) {
    vnMatches12[i] = m12[i];
    if (m12[i] >= 0) vbPrevMatched[i] = F2.mvKeysUn[m12[i]].pt;  // :636-638
  }
  return n;
}

// ---- LoopClosing::ComputeSim3 (:656-799): strict '<' TH_LOW, both sides need map points
int ORBmatcher::SearchByBoW(KeyFrame* pKF1, KeyFrame* pKF2, vector<MapPoint*>& vpMatches12) {
  const vector<MapPoint*> vpMapPoints1 = pKF1->GetMapPointMatches();
  const vector<MapPoint*> vpMapPoints2 = pKF2->GetMapPointMatches();
  vpMatches12 = vector<MapPoint*>(vpMapPoints1.size(), static_cast<MapPoint*>(NULL));
  Flat a, b;
  flatten(*pKF1, a);
  flatten(*pKF2, b);
  if (a.n == 0 || b.n == 0) return 0;
  const vector<int32_t> nodeA = nodes_of(*pKF1, a.n), nodeB = nodes_of(*pKF2, b.n);
  vector<uint8_t> validA((size_t)a.n, 0), validB((size_t)b.n, 0);
  for (int i = 0; i < a.n; i++) validA[i] = vpMapPoints1[i] && !vpMapPoints1[i]->isBad();
  for (int j = 0; j < b.n; j++) validB[j] = vpMapPoints2[j] && !vpMapPoints2[j]->isBad();
  b2s_matcher* h = handle_for(std::max(a.n, b.n));
  if (!h) return 0;
  vector<int32_t> match2((size_t)b.n, -1);
  int n = 0;
  if (!ok(b2s_search_by_bow(h, a.desc, nodeA.data(), validA.data(), a.angle.data(), a.n, b.desc, nodeB.data(), validB.data(),
                            b.angle.data(), b.n, TH_LOW, mfNNratio, /*strict_lt=*/1, mbCheckOrientation, match2.data(), &n),
          "SearchByBoW(KeyFrame, KeyFrame)"))
    return 0;
  for (int j = 0; j < b.n; j++)
    if (match2[j] >= 0) vpMatches12[match2[j]] = vpMapPoints2[j];
  return n;
}

// ---- LocalMapping::CreateNewMapPoints (:810-1009)
int ORBmatcher::SearchForTriangulation(KeyFrame* pKF1, KeyFrame* pKF2, cv::Mat F12, vector<pair<size_t, size_t> >& vMatchedPairs,
                                       const bool bOnlyStereo) {
  // epipole of camera 1 in image 2 (:815-823)
  cv::Mat Cw = pKF1->GetCameraCenter();
  cv::Mat R2w = pKF2->GetRotation();
  cv::Mat t2w = pKF2->GetTranslation();
  cv::Mat C2 = R2w * Cw + t2w;
  const float invz = 1.0f / C2.at<float>(2);
  const float ex = pKF2->fx * C2.at<float>(0) * invz + pKF2->cx;
  const float ey = pKF2->fy * C2.at<float>(1) * invz + pKF2->cy;
  Flat a, b;
  flatten(*pKF1, a);
  flatten(*pKF2, b);
  vMatchedPairs.clear();
  if (a.n == 0 || b.n == 0) return 0;
  const vector<int32_t> nodeA = nodes_of(*pKF1, a.n), nodeB = nodes_of(*pKF2, b.n);
  vector<uint8_t> hasA((size_t)a.n), stA((size_t)a.n), hasB((size_t)b.n), stB((size_t)b.n);
  for (int i = 0; i < a.n; i++) {
    hasA[i] = pKF1->GetMapPoint(i) != NULL;
    stA[i] = pKF1->mvuRight[i] >= 0;
  }
  for (int j = 0; j < b.n; j++) {
    hasB[j] = pKF2->GetMapPoint(j) != NULL;
    stB[j] = pKF2->mvuRight[j] >= 0;
  }
  b2s_kf_features fa = {a.desc, nodeA.data(), hasA.data(), stA.data(), a.x.data(), a.y.data(), a.octave.data(), a.angle.data(), a.n};
  b2s_kf_features fb = {b.desc, nodeB.data(), hasB.data(), stB.data(), b.x.data(), b.y.data(), b.octave.data(), b.angle.data(), b.n};
  float F[9];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) F[3 * r + c] = F12.at<float>(r, c);
  b2s_matcher* h = handle_for(std::max(a.n, b.n));
  if (!h) return 0;
  vector<int32_t> m12((size_t)a.n, -1);
  int n = 0;
  if (!ok(b2s_search_for_triangulation(h, &fa, &fb, F, ex, ey, pKF2->mvScaleFactors.data(), pKF2->mvLevelSigma2.data(),
                                       (int)pKF2->mvScaleFactors.size(), bOnlyStereo, mbCheckOrientation, m12.data(), &n),
          "SearchForTriangulation"))
    return 0;
  vMatchedPairs.reserve(n);
  for (int i = 0; i < a.n; i++)
    if (m12[i] >= 0) vMatchedPairs.push_back(make_pair((size_t)i, (size_t)m12[i]));
  return n;
}

// ---- LocalMapping::SearchInNeighbors (:1020-1174)
int ORBmatcher::Fuse(KeyFrame* pKF, const vector<MapPoint*>& vpMapPoints, const float th) {
  cv::Mat Rcw = pKF->GetRotation();
  cv::Mat tcw = pKF->GetTranslation();
  cv::Mat Ow = pKF->GetCameraCenter();
  vector<b2s_win_query> q(vpMapPoints.size());
  for (size_t i = 0; i < vpMapPoints.size(); i++) {
    memset(&q[i], 0, sizeof(b2s_win_query));
    MapPoint* p = vpMapPoints[i];
    if (!p || p->isBad() || p->IsInKeyFrame(pKF)) continue;
    window_query(p, pKF, Rcw, tcw, Ow, th, true, q[i]);
  }
  vector<int32_t> best;
  run_windows(pKF, q, nullptr, B2S_WIN_CHI2, TH_LOW, best, "Fuse(KeyFrame, MapPoints)");
  int nFused = 0;
  for (size_t i = 0; i < best.size(); i++) {
    if (best[i] < 0) continue;
    MapPoint* pMP = vpMapPoints[i];
    MapPoint* pMPinKF = pKF->GetMapPoint(best[i]);
    if (pMPinKF) {
      if (!pMPinKF->isBad()) {
        if (pMPinKF->Observations() > pMP->Observations())
          pMP->Replace(pMPinKF);
        else
          pMPinKF->Replace(pMP);
      }
    } else {
      pMP->AddObservation(pKF, best[i]);
      pKF->AddMapPoint(pMP, best[i]);
    }
    nFused++;
  }
  return nFused;
}

// ---- LoopClosing::SearchAndFuse (:1179-1310)
int ORBmatcher::Fuse(KeyFrame* pKF, cv::Mat Scw, const vector<MapPoint*>& vpPoints, float th, vector<MapPoint*>& vpReplacePoint) {
  cv::Mat Rcw, tcw, Ow;
  sim3_parts(Scw, Rcw, tcw, Ow);
  const set<MapPoint*> spAlreadyFound = pKF->GetMapPoints();
  vector<b2s_win_query> q(vpPoints.size());
  for (size_t i = 0; i < vpPoints.size(); i++) {
    memset(&q[i], 0, sizeof(b2s_win_query));
    MapPoint* p = vpPoints[i];
    if (p->isBad() || spAlreadyFound.count(p)) continue;
    window_query(p, pKF, Rcw, tcw, Ow, th, false, q[i]);
  }
  vector<int32_t> best;
  run_windows(pKF, q, nullptr, 0, TH_LOW, best, "Fuse(KeyFrame, Scw)");
  int nFused = 0;
  for (size_t i = 0; i < best.size(); i++) {
    if (best[i] < 0) continue;
    MapPoint* pMP = vpPoints[i];
    MapPoint* pMPinKF = pKF->GetMapPoint(best[i]);
    if (pMPinKF) {
      if (!pMPinKF->isBad()) vpReplacePoint[i] = pMPinKF;
    } else {
      pMP->AddObservation(pKF, best[i]);
      pKF->AddMapPoint(pMP, best[i]);
    }
    nFused++;
  }
  return nFused;
}

// ---- LoopClosing::ComputeSim3 (:1314-1555): two window searches + the mutual-consistency check
int ORBmatcher::SearchBySim3(KeyFrame* pKF1, KeyFrame* pKF2, vector<MapPoint*>& vpMatches12, const float& s12, const cv::Mat& R12,
                             const cv::Mat& t12, const float th) {
  cv::Mat R1w = pKF1->GetRotation(), t1w = pKF1->GetTranslation();
  cv::Mat R2w = pKF2->GetRotation(), t2w = pKF2->GetTranslation();
  cv::Mat sR12 = s12 * R12;
  cv::Mat sR21 = (1.0 / s12) * R12.t();
  cv::Mat t21 = -sR21 * t12;
  const vector<MapPoint*> vpMapPoints1 = pKF1->GetMapPointMatches();
  const vector<MapPoint*> vpMapPoints2 = pKF2->GetMapPointMatches();
  const int N1 = (int)vpMapPoints1.size(), N2 = (int)vpMapPoints2.size();
  vector<bool> done1(N1, false), done2(N2, false);
  for (int i = 0; i < N1; i++) {
    MapPoint* p = vpMatches12[i];
    if (!p) continue;
    done1[i] = true;
    const int idx2 = p->GetIndexInKeyFrame(pKF2);
    if (idx2 >= 0 && idx2 < N2) done2[idx2] = true;
  }
  vector<int32_t> match1, match2;
  for (int dir = 0; dir < 2; dir++) {
    KeyFrame* dst = dir ? pKF1 : pKF2;
    const vector<MapPoint*>& src = dir ? vpMapPoints2 : vpMapPoints1;
    vector<b2s_win_query> q(src.size());
    for (size_t i = 0; i < src.size(); i++) {
      b2s_win_query& w = q[i];
      memset(&w, 0, sizeof(w));
      MapPoint* pMP = src[i];
      if (!pMP || (dir ? done2[i] : done1[i]) || pMP->isBad()) continue;
      put_desc(w.desc, pMP);
      cv::Mat p3Dw = pMP->GetWorldPos();
      cv::Mat pd;
      if (!dir) {
        cv::Mat p3Dc1 = R1w * p3Dw + t1w;
        pd = sR21 * p3Dc1 + t21;
      } else {
        cv::Mat p3Dc2 = R2w * p3Dw + t2w;
        pd = sR12 * p3Dc2 + t12;
      }
      if (pd.at<float>(2) < 0.0) continue;
      const float invz = 1.0 / pd.at<float>(2);
      const float x = pd.at<float>(0) * invz;
      const float y = pd.at<float>(1) * invz;
      const float u = pKF1->fx * x + pKF1->cx;  // (both directions use pKF1's intrinsics, :1320-1323)
      const float v = pKF1->fy * y + pKF1->cy;
      if (!dst->IsInImage(u, v)) continue;
      const float maxDistance = pMP->GetMaxDistanceInvariance();
      const float minDistance = pMP->GetMinDistanceInvariance();
      const float dist3D = cv::norm(pd);
      if (dist3D < minDistance || dist3D > maxDistance) continue;
      const int level = pMP->PredictScale(dist3D, dst);
      w.u = u;
      w.v = v;
      w.radius = th * dst->mvScaleFactors[level];
      w.min_level = level - 1;
      w.max_level = level;
      w.valid = 1;
    }
    run_windows(dst, q, nullptr, 0, TH_HIGH, dir ? match2 : match1, "SearchBySim3");
  }
  int nFound = 0;
  for (int i1 = 0; i1 < N1; i1++) {
    const int idx2 = i1 < (int)match1.size() ? match1[i1] : -1;
    if (idx2 < 0) continue;
    if (idx2 < (int)match2.size() && match2[idx2] == i1) {
      vpMatches12[i1] = vpMapPoints2[idx2];
      nFound++;
    }
  }
  return nFound;
}

// ---- Tracking::TrackWithMotionModel (:1569-1728)
int ORBmatcher::SearchByProjection(Frame& CurrentFrame, const Frame& LastFrame, const float th, const bool bMono) {
  const cv::Mat Rcw = CurrentFrame.mTcw.rowRange(0, 3).colRange(0, 3);
  const cv::Mat tcw = CurrentFrame.mTcw.rowRange(0, 3).col(3);
  const cv::Mat twc = -Rcw.t() * tcw;
  const cv::Mat Rlw = LastFrame.mTcw.rowRange(0, 3).colRange(0, 3);
  const cv::Mat tlw = LastFrame.mTcw.rowRange(0, 3).col(3);
  const cv::Mat tlc = Rlw * twc + tlw;
  const bool bForward = tlc.at<float>(2) > CurrentFrame.mb && !bMono;
  const bool bBackward = -tlc.at<float>(2) > CurrentFrame.mb && !bMono;
  const int mode = bForward ? 1 : (bBackward ? 2 : 0);
  const int nq = LastFrame.N;
  vector<b2s_proj_query> q((size_t)nq);
  for (int i = 0; i < nq; i++) {
    b2s_proj_query& p = q[i];
    memset(&p, 0, sizeof(p));
    p.octave = -1;  // skipped before the search
    MapPoint* pMP = LastFrame.mvpMapPoints[i];
    if (!pMP || LastFrame.mvbOutlier[i]) continue;
    cv::Mat x3Dw = pMP->GetWorldPos();
    cv::Mat x3Dc = Rcw * x3Dw + tcw;
    const float xc = x3Dc.at<float>(0);
    const float yc = x3Dc.at<float>(1);
    const float invzc = 1.0 / x3Dc.at<float>(2);
    p.u = Frame::fx * xc * invzc + Frame::cx;
    p.v = Frame::fy * yc * invzc + Frame::cy;
    p.invz = invzc;
    p.angle = LastFrame.mvKeysUn[i].angle;
    p.octave = LastFrame.mvKeys[i].octave;
    p.has_obs = pMP->Observations() > 0;
    put_desc(p.desc, pMP);
  }
  Flat c;
  flatten(CurrentFrame, c);
  if (c.n == 0 || nq == 0) return 0;
  vector<uint8_t> occupied((size_t)c.n, 0);
  for (int j = 0; j < c.n; j++) occupied[j] = CurrentFrame.mvpMapPoints[j] && CurrentFrame.mvpMapPoints[j]->Observations() > 0;
  b2s_matcher* h = handle_for(std::max(c.n, nq));
  if (!h) return 0;
  const b2s_frame_geom g = geom_of(CurrentFrame);
  vector<int32_t> match((size_t)c.n, -1);
  int n = 0;
  if (!ok(b2s_search_by_projection_last(h, q.data(), nq, c.x.data(), c.y.data(), c.octave.data(), c.angle.data(), c.uright.data(),
                                        occupied.data(), c.desc, c.n, &g, th, mode, TH_HIGH, mbCheckOrientation, match.data(), &n),
          "SearchByProjection(Current, Last)"))
    return 0;
  for (int j = 0; j < c.n; j++)
    if (match[j] >= 0) CurrentFrame.mvpMapPoints[j] = LastFrame.mvpMapPoints[match[j]];
  return n;
}

// ---- Tracking::Relocalization (:1731-1863)
int ORBmatcher::SearchByProjection(Frame& CurrentFrame, KeyFrame* pKF, const set<MapPoint*>& sAlreadyFound, const float th,
                                   const int ORBdist) {
  const cv::Mat Rcw = CurrentFrame.mTcw.rowRange(0, 3).colRange(0, 3);
  const cv::Mat tcw = CurrentFrame.mTcw.rowRange(0, 3).col(3);
  const cv::Mat Ow = -Rcw.t() * tcw;
  const vector<MapPoint*> vpMPs = pKF->GetMapPointMatches();
  const int nq = (int)vpMPs.size();
  vector<b2s_proj_query> q((size_t)nq);
  for (int i = 0; i < nq; i++) {
    b2s_proj_query& p = q[i];
    memset(&p, 0, sizeof(p));
    p.octave = -1;
    MapPoint* pMP = vpMPs[i];
    if (!pMP || pMP->isBad() || sAlreadyFound.count(pMP)) continue;
    cv::Mat x3Dw = pMP->GetWorldPos();
    cv::Mat x3Dc = Rcw * x3Dw + tcw;
    const float xc = x3Dc.at<float>(0);
    const float yc = x3Dc.at<float>(1);
    const float invzc = 1.0 / x3Dc.at<float>(2);
    const float u = Frame::fx * xc * invzc + Frame::cx;
    const float v = Frame::fy * yc * invzc + Frame::cy;
    cv::Mat PO = x3Dw - Ow;
    const float dist3D = cv::norm(PO);
    if (dist3D < pMP->GetMinDistanceInvariance() || dist3D > pMP->GetMaxDistanceInvariance()) continue;
    p.u = u;
    p.v = v;
    p.invz = 1.0f;  // this overload neither tests nor uses the depth
    p.angle = pKF->mvKeysUn[i].angle;
    p.octave = pMP->PredictScale(dist3D, &CurrentFrame);
    p.has_obs = 1;
    put_desc(p.desc, pMP);
  }
  Flat c;
  flatten(CurrentFrame, c);
  if (c.n == 0 || nq == 0) return 0;
  vector<uint8_t> occupied((size_t)c.n, 0);
  for (int j = 0; j < c.n; j++) occupied[j] = CurrentFrame.mvpMapPoints[j] != NULL;
  vector<float> noRight((size_t)c.n, -1.f);  // no stereo gate in this overload
  b2s_matcher* h = handle_for(std::max(c.n, nq));
  if (!h) return 0;
  const b2s_frame_geom g = geom_of(CurrentFrame);
  vector<int32_t> match((size_t)c.n, -1);
  int n = 0;
  if (!ok(b2s_search_by_projection_last(h, q.data(), nq, c.x.data(), c.y.data(), c.octave.data(), c.angle.data(), noRight.data(),
                                        occupied.data(), c.desc, c.n, &g, th, /*mode=*/0, ORBdist, mbCheckOrientation,
                                        match.data(), &n),
          "SearchByProjection(Current, KeyFrame)"))
    return 0;
  for (int j = 0; j < c.n; j++)
    if (match[j] >= 0) CurrentFrame.mvpMapPoints[j] = vpMPs[match[j]];
  return n;
}

}  // namespace ORB_SLAM2
