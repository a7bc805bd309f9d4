// Drop-in replacement for the reference's src/Initializer.cc, against its unchanged include/Initializer.h: the
// constructor keeps what the reference keeps; Initialize compacts the matches and draws mvSets with DUtils::Random
// exactly as src/Initializer.cc:82-168 does (so the process consumes the same rand() stream), then makes one
// b2s_initialize call with batch 1 and writes R21, t21, vP3D and vbTriangulated as the reference does: only on success,
// except that a failed ReconstructF leaves R21 and t21 empty.  On a library error it prints to stderr and returns false.
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <vector>

#include "Initializer.h"
#include "Thirdparty/DBoW2/DUtils/Random.h"

#include "b200slam.h"

namespace ORB_SLAM2 {
namespace {

// One handle for the process (Tracking calls Initialize from one thread), grown on demand.
struct InitSlot {
  b2s_init_solver* h = nullptr;
  int keys = 0, iterations = 0;
  std::mutex m;
  b2s_init_solver* get(int nKeys, int nIt) {
    if (h && nKeys <= keys && nIt <= iterations) return h;
    b2s_init_destroy(h);
    h = nullptr;
    keys = nKeys > 4096 ? nKeys : 4096;
    iterations = nIt > 200 ? nIt : 200;
    const char* e = getenv("B2S_DEVICE");
    if (b2s_init_create(keys, iterations, 1, e ? atoi(e) : 0, &h) != B2S_OK) {
      fprintf(stderr, "Initializer (b200): %s\n", b2s_last_error());
      h = nullptr;
      keys = iterations = 0;
    }
    return h;
  }
} g_init;

}  // namespace

Initializer::Initializer(const Frame& ReferenceFrame, float sigma, int iterations) {
  mK = ReferenceFrame.mK.clone();
  mvKeys1 = ReferenceFrame.mvKeysUn;
  mSigma = sigma;
  mSigma2 = sigma * sigma;
  mMaxIterations = iterations;
}

bool Initializer::Initialize(const Frame& CurrentFrame, const vector<int>& vMatches12, cv::Mat& R21, cv::Mat& t21,
                             vector<cv::Point3f>& vP3D, vector<bool>& vbTriangulated) {
  // :82-124
  mvKeys2 = CurrentFrame.mvKeysUn;
  mvMatches12.clear();
  mvMatches12.reserve(mvKeys2.size());
  mvbMatched1.resize(mvKeys1.size());
  for (size_t i = 0, iend = vMatches12.size(); i < iend; i++) {
    if (vMatches12[i] >= 0) {
      mvMatches12.push_back(make_pair(i, vMatches12[i]));
      mvbMatched1[i] = true;
    } else
      mvbMatched1[i] = false;
  }
  const int N = mvMatches12.size();
  vector<size_t> vAllIndices;
  vAllIndices.reserve(N);
  vector<size_t> vAvailableIndices;
  for (int i = 0; i < N; i++) vAllIndices.push_back(i);

  // :132-168: the same draws, in the same order
  mvSets = vector<vector<size_t> >(mMaxIterations, vector<size_t>(8, 0));
  DUtils::Random::SeedRandOnce(0);
  for (int it = 0; it < mMaxIterations; it++) {
    vAvailableIndices = vAllIndices;
    for (size_t j = 0; j < 8; j++) {
      int randi = DUtils::Random::RandomInt(0, vAvailableIndices.size() - 1);
      int idx = vAvailableIndices[randi];
      mvSets[it][j] = idx;
      vAvailableIndices[randi] = vAvailableIndices.back();
      vAvailableIndices.pop_back();
    }
  }

  // one batch-1 call
  const int n1 = (int)mvKeys1.size(), n2 = (int)mvKeys2.size();
  std::vector<float> kp1((size_t)n1 * 2), kp2((size_t)n2 * 2);
  for (int i = 0; i < n1; i++) {
    kp1[2 * i] = mvKeys1[i].pt.x;
    kp1[2 * i + 1] = mvKeys1[i].pt.y;
  }
  for (int i = 0; i < n2; i++) {
    kp2[2 * i] = mvKeys2[i].pt.x;
    kp2[2 * i + 1] = mvKeys2[i].pt.y;
  }
  std::vector<int32_t> m12((size_t)n1, -1), sets((size_t)mMaxIterations * 8);
  for (size_t i = 0; i < vMatches12.size() && i < (size_t)n1; i++) m12[i] = vMatches12[i];
  for (int it = 0; it < mMaxIterations; it++)
    for (int j = 0; j < 8; j++) sets[8 * (size_t)it + j] = (int32_t)mvSets[it][j];
  b2s_init_problem q;
  q.n1 = n1;
  q.n2 = n2;
  q.kp1 = kp1.data();
  q.kp2 = kp2.data();
  q.matches12 = m12.data();
  for (int i = 0; i < 9; i++) q.K[i] = mK.at<float>(i / 3, i % 3);
  q.sigma = mSigma;
  q.iterations = mMaxIterations;
  q.sets = sets.data();
  std::vector<float> p3d((size_t)n1 * 3);
  std::vector<uint8_t> tri((size_t)n1);
  b2s_init_result r;
  r.p3d = p3d.data();
  r.triangulated = tri.data();
  r.inliers_h = r.inliers_f = nullptr;
  int rc;
  {
    std::lock_guard<std::mutex> lock(g_init.m);
    b2s_init_solver* h = g_init.get(n1 > n2 ? n1 : n2, mMaxIterations);
    rc = h ? b2s_initialize(h, 1, &q, &r) : B2S_ERR_CUDA;
  }
  if (rc != B2S_OK) {
    fprintf(stderr, "Initializer::Initialize: libb200slam error %d: %s\n", rc, b2s_last_error());
    return false;
  }
  if (r.rt_state == -1) {  // ReconstructF clears its outputs before deciding (:1032-1033)
    R21 = cv::Mat();
    t21 = cv::Mat();
  }
  if (!r.ret) return false;
  cv::Mat(3, 3, CV_32F, r.R21).copyTo(R21);
  cv::Mat(3, 1, CV_32F, r.t21).copyTo(t21);
  vP3D.assign((size_t)n1, cv::Point3f());
  vbTriangulated.assign((size_t)n1, false);
  for (int i = 0; i < n1; i++) {
    vP3D[i] = cv::Point3f(p3d[3 * i], p3d[3 * i + 1], p3d[3 * i + 2]);
    vbTriangulated[i] = tri[i] != 0;
  }
  return true;
}

}  // namespace ORB_SLAM2
