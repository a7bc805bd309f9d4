// Drop-in replacement for the reference's src/Sim3Solver.cc, against its unchanged include/Sim3Solver.h.  The
// constructor and SetRansacParameters are the reference's; iterate draws the sets it may use with DUtils::Random in the
// reference's pattern (:228-249), makes one b2s_sim3solver_iterate call with batch 1 and writes the members and outputs
// as the reference does.  On a library error it prints to stderr and returns an empty matrix.
//
// The one difference: iterate(k) draws min(k, mRansacMaxIts - mnIterations) sets before the call, where the reference
// draws 3 indices per iteration as it goes.  After an early return at iteration j < k the process's rand() stream is
// 3*(k-j) draws further on than the reference's; no output of the call changes, later draws in the process shift.
//
// mvSigmaSquare1 / mvSigmaSquare2, which the reference declares and never uses, hold the bit patterns of each
// correspondence's float sigma2, so that iterate passes the device what the constructor read.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

#include "Sim3Solver.h"
#include "Thirdparty/DBoW2/DUtils/Random.h"

#include "b200slam.h"

namespace ORB_SLAM2 {
namespace {

// One handle for the process (LoopClosing runs the solvers from one thread), grown on demand.
struct Sim3SolverSlot {
  b2s_sim3solver* h = nullptr;
  int matches = 0, sets = 0;
  std::mutex m;
  b2s_sim3solver* get(int n, int k) {
    if (h && n <= matches && k <= sets) return h;
    b2s_sim3solver_destroy(h);
    h = nullptr;
    matches = n > 1024 ? n : 1024;
    sets = k > 300 ? k : 300;
    const char* e = getenv("B2S_DEVICE");
    if (b2s_sim3solver_create(matches, sets, 1, e ? atoi(e) : 0, &h) != B2S_OK) {
      fprintf(stderr, "Sim3Solver (b200): %s\n", b2s_last_error());
      h = nullptr;
      matches = sets = 0;
    }
    return h;
  }
} g_sim3solver;

size_t float_bits(float f) {
  uint32_t u;
  memcpy(&u, &f, sizeof(u));
  return u;
}

float bits_float(size_t s) {
  const uint32_t u = (uint32_t)s;
  float f;
  memcpy(&f, &u, sizeof(f));
  return f;
}

}  // namespace

// :48-140
Sim3Solver::Sim3Solver(KeyFrame* pKF1, KeyFrame* pKF2, const std::vector<MapPoint*>& vpMatched12,
                       const bool bFixScale)
    : mnIterations(0), mnBestInliers(0), mbFixScale(bFixScale) {
  mpKF1 = pKF1;
  mpKF2 = pKF2;
  std::vector<MapPoint*> vpKeyFrameMP1 = pKF1->GetMapPointMatches();
  mN1 = vpMatched12.size();
  mvpMapPoints1.reserve(mN1);
  mvpMapPoints2.reserve(mN1);
  mvpMatches12 = vpMatched12;
  mvnIndices1.reserve(mN1);
  mvX3Dc1.reserve(mN1);
  mvX3Dc2.reserve(mN1);
  cv::Mat Rcw1 = pKF1->GetRotation();
  cv::Mat tcw1 = pKF1->GetTranslation();
  cv::Mat Rcw2 = pKF2->GetRotation();
  cv::Mat tcw2 = pKF2->GetTranslation();
  mvAllIndices.reserve(mN1);
  size_t idx = 0;
  for (int i1 = 0; i1 < mN1; i1++) {
    if (!vpMatched12[i1]) continue;
    MapPoint* pMP1 = vpKeyFrameMP1[i1];
    MapPoint* pMP2 = vpMatched12[i1];
    if (!pMP1) continue;
    if (pMP1->isBad() || pMP2->isBad()) continue;
    const int indexKF1 = pMP1->GetIndexInKeyFrame(pKF1);
    const int indexKF2 = pMP2->GetIndexInKeyFrame(pKF2);
    if (indexKF1 < 0 || indexKF2 < 0) continue;
    const float sigmaSquare1 = pKF1->mvLevelSigma2[pKF1->mvKeysUn[indexKF1].octave];
    const float sigmaSquare2 = pKF2->mvLevelSigma2[pKF2->mvKeysUn[indexKF2].octave];
    mvnMaxError1.push_back(9.210 * sigmaSquare1);
    mvnMaxError2.push_back(9.210 * sigmaSquare2);
    mvSigmaSquare1.push_back(float_bits(sigmaSquare1));
    mvSigmaSquare2.push_back(float_bits(sigmaSquare2));
    mvpMapPoints1.push_back(pMP1);
    mvpMapPoints2.push_back(pMP2);
    mvnIndices1.push_back(i1);
    cv::Mat X3D1w = pMP1->GetWorldPos();
    mvX3Dc1.push_back(Rcw1 * X3D1w + tcw1);
    cv::Mat X3D2w = pMP2->GetWorldPos();
    mvX3Dc2.push_back(Rcw2 * X3D2w + tcw2);
    mvAllIndices.push_back(idx);
    idx++;
  }
  mK1 = pKF1->mK;
  mK2 = pKF2->mK;
  SetRansacParameters();
}

// :143-196
void Sim3Solver::SetRansacParameters(double probability, int minInliers, int maxIterations) {
  mRansacProb = probability;
  mRansacMinInliers = minInliers;
  mRansacMaxIts = maxIterations;
  N = mvpMapPoints1.size();
  mvbInliersi.resize(N);
  float epsilon = (float)mRansacMinInliers / N;
  int nIterations;
  if (mRansacMinInliers == N)
    nIterations = 1;
  else
    nIterations = ceil(log(1 - mRansacProb) / log(1 - pow(epsilon, 3)));
  mRansacMaxIts = max(1, min(nIterations, mRansacMaxIts));
  mnIterations = 0;
}

cv::Mat Sim3Solver::iterate(int nIterations, bool& bNoMore, std::vector<bool>& vbInliers, int& nInliers) {
  bNoMore = false;
  vbInliers = std::vector<bool>(mN1, false);
  nInliers = 0;
  if (N < mRansacMinInliers) {
    bNoMore = true;
    return cv::Mat();
  }
  // the draws of the iterations this call may run, in the reference's order
  int k = mRansacMaxIts - mnIterations;
  if (nIterations < k) k = nIterations;
  if (k < 0) k = 0;
  std::vector<int32_t> sets((size_t)k * 3);
  std::vector<size_t> vAvailableIndices;
  for (int it = 0; it < k; it++) {
    vAvailableIndices = mvAllIndices;
    for (short i = 0; i < 3; ++i) {
      int randi = DUtils::Random::RandomInt(0, vAvailableIndices.size() - 1);
      sets[(size_t)it * 3 + i] = (int32_t)vAvailableIndices[randi];
      vAvailableIndices[randi] = vAvailableIndices.back();
      vAvailableIndices.pop_back();
    }
  }

  std::vector<float> X1((size_t)N * 3), X2((size_t)N * 3), s1((size_t)N), s2((size_t)N);
  for (int i = 0; i < N; i++) {
    for (int r = 0; r < 3; r++) {
      X1[(size_t)i * 3 + r] = mvX3Dc1[i].at<float>(r);
      X2[(size_t)i * 3 + r] = mvX3Dc2[i].at<float>(r);
    }
    s1[(size_t)i] = bits_float(mvSigmaSquare1[i]);
    s2[(size_t)i] = bits_float(mvSigmaSquare2[i]);
  }
  b2s_sim3solver_problem q;
  q.n = N;
  q.X1c = X1.data();
  q.X2c = X2.data();
  q.sigma2_1 = s1.data();
  q.sigma2_2 = s2.data();
  q.K1[0] = mK1.at<float>(0, 0);
  q.K1[1] = mK1.at<float>(1, 1);
  q.K1[2] = mK1.at<float>(0, 2);
  q.K1[3] = mK1.at<float>(1, 2);
  q.K2[0] = mK2.at<float>(0, 0);
  q.K2[1] = mK2.at<float>(1, 1);
  q.K2[2] = mK2.at<float>(0, 2);
  q.K2[3] = mK2.at<float>(1, 2);
  q.fix_scale = mbFixScale ? 1 : 0;
  q.min_inliers = mRansacMinInliers;
  q.max_its = mRansacMaxIts;
  q.iterations_done = mnIterations;
  q.best_inliers = mnBestInliers;
  q.k = k;
  q.sets = sets.data();
  std::vector<uint8_t> inl((size_t)(N > 0 ? N : 1));
  b2s_sim3solver_result r;
  r.inliers = inl.data();
  int rc;
  {
    std::lock_guard<std::mutex> lock(g_sim3solver.m);
    b2s_sim3solver* h = g_sim3solver.get(N, k);
    rc = h ? b2s_sim3solver_iterate(h, 1, &q, &r) : B2S_ERR_CUDA;
  }
  if (rc != B2S_OK) {
    fprintf(stderr, "Sim3Solver::iterate: libb200slam error %d: %s\n", rc, b2s_last_error());
    return cv::Mat();
  }
  mnIterations = r.iterations_done;
  mnBestInliers = r.best_inliers;
  if (r.best_changed) {
    mBestRotation = cv::Mat(3, 3, CV_32F, r.R).clone();
    mBestTranslation = cv::Mat(3, 1, CV_32F, r.t).clone();
    mBestScale = r.s;
  }
  if (r.returned) {
    for (int i = 0; i < N; i++) mvbInliersi[i] = inl[(size_t)i] != 0;
    mvbBestInliers = mvbInliersi;
    mBestT12 = cv::Mat(4, 4, CV_32F, r.T12).clone();
    nInliers = r.n_inliers;
    for (int i = 0; i < N; i++)
      if (inl[(size_t)i]) vbInliers[mvnIndices1[i]] = true;
    return mBestT12;
  }
  bNoMore = r.no_more != 0;
  return cv::Mat();
}

cv::Mat Sim3Solver::find(std::vector<bool>& vbInliers12, int& nInliers) {
  bool bFlag;
  return iterate(mRansacMaxIts, bFlag, vbInliers12, nInliers);
}

cv::Mat Sim3Solver::GetEstimatedRotation() { return mBestRotation.clone(); }

cv::Mat Sim3Solver::GetEstimatedTranslation() { return mBestTranslation.clone(); }

float Sim3Solver::GetEstimatedScale() { return mBestScale; }

}  // namespace ORB_SLAM2
