#include "ORBmatcher.h"

#include <cstring>
#include <vector>

#include "b2s_host.h"

namespace ORB_SLAM2 {

using b2s_host::fail;

// ORBmatcher objects are stack temporaries in the reference (one per call site, several per tracked frame); the device
// handle — a stream and ~30 device buffers — is therefore owned by the calling THREAD, not by the object: created on
// first use, grown on demand, kept until the thread exits.  Handles that were outgrown stay alive as well, because a
// FrameGrid built on one of them must remain usable.
namespace {
struct ThreadHandles {
  std::vector<b2s_matcher*> all;
  b2s_matcher* cur = nullptr;
  int cap = 0;
  ~ThreadHandles() {
    for (b2s_matcher* h : all) b2s_matcher_destroy(h);
  }
};
ThreadHandles& thread_handles() {
  static thread_local ThreadHandles t;
  return t;
}
}  // namespace

ORBmatcher::ORBmatcher(float nnratio, bool checkOri) : mfNNratio(nnratio), mbCheckOrientation(checkOri) {}
ORBmatcher::~ORBmatcher() {}  // the handle belongs to the thread

void ORBmatcher::Ensure(int n) {
  ThreadHandles& t = thread_handles();
  if (!t.cur || n > t.cap) {
    const int cap = n < 4096 ? 4096 : n;
    b2s_matcher* h = nullptr;
    int rc = b2s_matcher_create(cap, 1, b2s_host::device(), &h);
    if (rc != B2S_OK) fail("ORBmatcher", rc);
    t.all.push_back(h);
    t.cur = h;
    t.cap = cap;
  }
  mpHandle = t.cur;
  mCap = t.cap;
}

int ORBmatcher::DescriptorDistance(const uint8_t* a, const uint8_t* b) {
  int d = 0;
  for (int i = 0; i < 4; i++) {
    uint64_t x, y;
    memcpy(&x, a + 8 * i, 8);
    memcpy(&y, b + 8 * i, 8);
    d += __builtin_popcountll(x ^ y);
  }
  return d;
}

int ORBmatcher::SearchByBoW(const BowSide& kf, const BowSide& f, std::vector<int32_t>& matchF) {
  Ensure(kf.n > f.n ? kf.n : f.n);
  matchF.assign(f.n, -1);
  int nm = 0;
  int rc = b2s_search_by_bow(mpHandle, kf.descriptors, kf.node, kf.valid, kf.angle, kf.n, f.descriptors, f.node, nullptr,
                             f.angle, f.n, TH_LOW, mfNNratio, 0, mbCheckOrientation, matchF.data(), &nm);
  if (rc != B2S_OK) fail("ORBmatcher::SearchByBoW", rc);
  return nm;
}

int ORBmatcher::SearchByBoWKF(const BowSide& k1, const BowSide& k2, std::vector<int32_t>& match2) {
  Ensure(k1.n > k2.n ? k1.n : k2.n);
  match2.assign(k2.n, -1);
  int nm = 0;
  int rc = b2s_search_by_bow(mpHandle, k1.descriptors, k1.node, k1.valid, k1.angle, k1.n, k2.descriptors, k2.node, k2.valid,
                             k2.angle, k2.n, TH_LOW, mfNNratio, 1, mbCheckOrientation, match2.data(), &nm);
  if (rc != B2S_OK) fail("ORBmatcher::SearchByBoW(KF,KF)", rc);
  return nm;
}

int ORBmatcher::SearchByProjection(const std::vector<b2s_proj_query>& q, const float* kpx, const float* kpy,
                                   const int32_t* octave, const float* angle, const float* uright, const uint8_t* occupied,
                                   const uint8_t* descriptors, int nF, const b2s_frame_geom& geom, float th, int mode,
                                   std::vector<int32_t>& matchCur) {
  Ensure((int)q.size() > nF ? (int)q.size() : nF);
  matchCur.assign(nF, -1);
  int nm = 0;
  int rc = b2s_search_by_projection_last(mpHandle, q.data(), (int)q.size(), kpx, kpy, octave, angle, uright, occupied,
                                         descriptors, nF, &geom, th, mode, TH_HIGH, mbCheckOrientation, matchCur.data(), &nm);
  if (rc != B2S_OK) fail("ORBmatcher::SearchByProjection", rc);
  return nm;
}

FrameGrid::FrameGrid(ORBmatcher& matcher, const float* kpx, const float* kpy, const int32_t* octave, const float* angle,
                     const float* uright, const uint8_t* descriptors, int nFeatures, const b2s_frame_geom& geom,
                     const float* invLevelSigma2)
    : mN(nFeatures) {
  int rc = b2s_frame_grid_create(matcher.handle(nFeatures), kpx, kpy, octave, angle, uright, descriptors, nFeatures, &geom,
                                 invLevelSigma2, &mpGrid);
  if (rc != B2S_OK) fail("FrameGrid", rc);
}
FrameGrid::~FrameGrid() { b2s_frame_grid_destroy(mpGrid); }

std::vector<size_t> FrameGrid::GetFeaturesInArea(const float& x, const float& y, const float& r, const int minLevel,
                                                 const int maxLevel) const {
  std::vector<int32_t> idx((size_t)(mN > 0 ? mN : 1));
  int n = 0;
  int rc = b2s_frame_grid_features_in_area(mpGrid, x, y, r, minLevel, maxLevel, idx.data(), (int)idx.size(), &n);
  if (rc != B2S_OK) fail("FrameGrid::GetFeaturesInArea", rc);
  return std::vector<size_t>(idx.begin(), idx.begin() + n);
}

int ORBmatcher::SearchByProjection(const FrameGrid& grid, const std::vector<b2s_proj_query>& q, const uint8_t* occupied,
                                   float th, int mode, std::vector<int32_t>& matchCur) {
  Ensure((int)q.size() > grid.N() ? (int)q.size() : grid.N());
  matchCur.assign(grid.N(), -1);
  int nm = 0;
  int rc = b2s_search_by_projection_last_grid(mpHandle, grid.handle(), q.data(), (int)q.size(), occupied, th, mode, TH_HIGH,
                                              mbCheckOrientation, matchCur.data(), &nm);
  if (rc != B2S_OK) fail("ORBmatcher::SearchByProjection(grid)", rc);
  return nm;
}

int ORBmatcher::SearchByProjection(const FrameGrid& grid, const std::vector<b2s_map_query>& mp, const uint8_t* occupied,
                                   float th, std::vector<int32_t>& matchF) {
  Ensure((int)mp.size() > grid.N() ? (int)mp.size() : grid.N());
  matchF.assign(grid.N(), -1);
  int nm = 0;
  int rc = b2s_search_by_projection_map_grid(mpHandle, grid.handle(), mp.data(), (int)mp.size(), occupied, th, TH_HIGH,
                                             mfNNratio, matchF.data(), &nm);
  if (rc != B2S_OK) fail("ORBmatcher::SearchByProjection(grid, map points)", rc);
  return nm;
}

int ORBmatcher::SearchWindows(const FrameGrid& grid, const std::vector<b2s_win_query>& mp, const uint8_t* occupied, int flags,
                              std::vector<int32_t>& bestIdx) {
  Ensure((int)mp.size() > grid.N() ? (int)mp.size() : grid.N());
  bestIdx.assign(mp.size(), -1);
  int na = 0;
  int rc = b2s_search_windows_grid(mpHandle, grid.handle(), mp.data(), (int)mp.size(), occupied, flags, TH_LOW, bestIdx.data(),
                                   nullptr, &na);
  if (rc != B2S_OK) fail("ORBmatcher::SearchWindows(grid)", rc);
  return na;
}

int ORBmatcher::SearchForInitialization(const float* kpx1, const float* kpy1, const int32_t* octave1, const float* angle1,
                                        const uint8_t* d1, int n1, const float* kpx2, const float* kpy2,
                                        const int32_t* octave2, const float* angle2, const uint8_t* d2, int n2,
                                        const b2s_frame_geom& geom, std::vector<float>& vbPrevMatched,
                                        std::vector<int>& vnMatches12, int windowSize) {
  (void)kpx1;
  (void)kpy1;  // F1's own coordinates only seed vbPrevMatched (done by the caller, src/Tracking.cc:905-907)
  Ensure(n1 > n2 ? n1 : n2);
  vnMatches12.assign(n1, -1);
  if ((int)vbPrevMatched.size() < 2 * n1) fail("ORBmatcher::SearchForInitialization: vbPrevMatched too short", B2S_ERR_BAD_ARG);
  std::vector<float> px(n1), py(n1);
  for (int i = 0; i < n1; i++) {
    px[i] = vbPrevMatched[2 * i];
    py[i] = vbPrevMatched[2 * i + 1];
  }
  int nm = 0;
  static_assert(sizeof(int) == sizeof(int32_t), "vnMatches12 is vector<int> in the reference");
  int rc = b2s_search_for_initialization(mpHandle, px.data(), py.data(), octave1, angle1, d1, n1, kpx2, kpy2, octave2, angle2, d2,
                                         n2, &geom, windowSize, TH_LOW, mfNNratio, mbCheckOrientation,
                                         reinterpret_cast<int32_t*>(vnMatches12.data()), &nm);
  if (rc != B2S_OK) fail("ORBmatcher::SearchForInitialization", rc);
  for (int i = 0; i < n1; i++)
    if (vnMatches12[i] >= 0) {  // :636-638
      vbPrevMatched[2 * i] = kpx2[vnMatches12[i]];
      vbPrevMatched[2 * i + 1] = kpy2[vnMatches12[i]];
    }
  return nm;
}

int ORBmatcher::SearchByProjectionReloc(std::vector<b2s_proj_query> q, const float* kpx, const float* kpy,
                                        const int32_t* octave, const float* angle, const uint8_t* occupied,
                                        const uint8_t* descriptors, int nF, const b2s_frame_geom& geom, float th, int ORBdist,
                                        std::vector<int32_t>& matchCur) {
  Ensure((int)q.size() > nF ? (int)q.size() : nF);
  matchCur.assign(nF, -1);
  for (size_t i = 0; i < q.size(); i++) {
    q[i].invz = 1.0f;   // src/ORBmatcher.cc:1766-1772 neither tests the sign of the depth nor uses it
    q[i].has_obs = 1;   // :1817 skips any feature that holds a map point, so every assignment occupies its feature
  }
  const std::vector<float> noStereo((size_t)nF, -1.0f);  // no |ur - uR| gate in this overload
  int nm = 0;
  int rc = b2s_search_by_projection_last(mpHandle, q.data(), (int)q.size(), kpx, kpy, octave, angle, noStereo.data(), occupied,
                                         descriptors, nF, &geom, th, /*mode: levels [l-1, l+1]*/ 0, ORBdist, mbCheckOrientation,
                                         matchCur.data(), &nm);
  if (rc != B2S_OK) fail("ORBmatcher::SearchByProjection(relocalisation)", rc);
  return nm;
}

int ORBmatcher::SearchByProjection(const std::vector<b2s_map_query>& mp, const float* kpx, const float* kpy,
                                   const int32_t* octave, const float* uright, const uint8_t* occupied,
                                   const uint8_t* descriptors, int nF, const b2s_frame_geom& geom, float th,
                                   std::vector<int32_t>& matchF) {
  Ensure((int)mp.size() > nF ? (int)mp.size() : nF);
  matchF.assign(nF, -1);
  int nm = 0;
  int rc = b2s_search_by_projection_map(mpHandle, mp.data(), (int)mp.size(), kpx, kpy, octave, uright, occupied,
                                        descriptors, nF, &geom, th, TH_HIGH, mfNNratio, matchF.data(), &nm);
  if (rc != B2S_OK) fail("ORBmatcher::SearchByProjection(map points)", rc);
  return nm;
}

int ORBmatcher::SearchWindows(const std::vector<b2s_win_query>& mp, const float* kpx, const float* kpy, const int32_t* octave,
                              const float* uright, const float* invLevelSigma2, const uint8_t* occupied,
                              const uint8_t* descriptors, int nF, const b2s_frame_geom& geom, int flags,
                              std::vector<int32_t>& bestIdx) {
  Ensure((int)mp.size() > nF ? (int)mp.size() : nF);
  bestIdx.assign(mp.size(), -1);
  int n = 0;
  int rc = b2s_search_windows(mpHandle, mp.data(), (int)mp.size(), kpx, kpy, octave, uright, invLevelSigma2, occupied,
                              descriptors, nF, &geom, flags, TH_LOW, bestIdx.data(), nullptr, &n);
  if (rc != B2S_OK) fail("ORBmatcher::SearchWindows", rc);
  return n;
}

int ORBmatcher::SearchForTriangulation(const b2s_kf_features& kf1, const b2s_kf_features& kf2, const float F12[9], float ex,
                                       float ey, const float* scaleFactors2, const float* levelSigma2_2, int nLevels,
                                       bool bOnlyStereo, std::vector<std::pair<size_t, size_t> >& vMatchedPairs) {
  Ensure(kf1.n > kf2.n ? kf1.n : kf2.n);
  std::vector<int32_t> m12(kf1.n > 0 ? kf1.n : 1, -1);
  int nm = 0;
  int rc = b2s_search_for_triangulation(mpHandle, &kf1, &kf2, F12, ex, ey, scaleFactors2, levelSigma2_2, nLevels,
                                        bOnlyStereo, mbCheckOrientation, m12.data(), &nm);
  if (rc != B2S_OK) fail("ORBmatcher::SearchForTriangulation", rc);
  vMatchedPairs.clear();
  vMatchedPairs.reserve(nm);
  for (int i = 0; i < kf1.n; i++)
    if (m12[i] >= 0) vMatchedPairs.push_back(std::make_pair((size_t)i, (size_t)m12[i]));  // :999-1005
  return nm;
}

}  // namespace ORB_SLAM2
