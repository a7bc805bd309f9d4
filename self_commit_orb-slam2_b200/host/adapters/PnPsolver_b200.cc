// Drop-in replacement for the reference's src/PnPsolver.cc, against its unchanged include/PnPsolver.h.  The constructor
// and SetRansacParameters are the reference's; iterate draws the sets it may use with DUtils::Random in the reference's
// pattern (:274-290), makes one b2s_pnpsolver_iterate call with batch 1 and writes the members and outputs as the
// reference does.  On a library error it prints to stderr and returns an empty matrix.
//
// The one difference: iterate(k) draws max(k, mRansacMaxIts - mnIterations) sets before the call (the iterations its ||
// loop condition runs without an early return), where the reference draws 4 indices per iteration as it goes.  After an
// early return at iteration j of those k the process's rand() stream is 4*(k-j) draws further on than the reference's;
// no output of the call changes, later draws in the process shift.
//
// mRansacTh, which the reference declares and never uses, keeps SetRansacParameters' th2, so that iterate passes the
// device the threshold scale the reference folds into mvMaxError.  The EPnP working arrays (pws, us, alphas, pcs) stay
// unallocated: the device holds them.
#include <cmath>
#include <cstring>
#include <mutex>
#include <vector>

#include "PnPsolver.h"
#include "Thirdparty/DBoW2/DUtils/Random.h"

#include "b200slam.h"
#include "../b2s_host.h"

namespace ORB_SLAM2 {
namespace {

// One handle for the process (Tracking runs the solvers from one thread), grown on demand.
b2s_host::Slot<b2s_pnpsolver, 2, b2s_pnpsolver_destroy> g_pnpsolver;

}  // namespace

// :120-168
PnPsolver::PnPsolver(const Frame& F, const vector<MapPoint*>& vpMapPointMatches)
    : pws(0), us(0), alphas(0), pcs(0), maximum_number_of_correspondences(0), number_of_correspondences(0),
      mnInliersi(0), mnIterations(0), mnBestInliers(0), N(0) {
  mvpMapPointMatches = vpMapPointMatches;
  mvP2D.reserve(F.mvpMapPoints.size());
  mvSigma2.reserve(F.mvpMapPoints.size());
  mvP3Dw.reserve(F.mvpMapPoints.size());
  mvKeyPointIndices.reserve(F.mvpMapPoints.size());
  mvAllIndices.reserve(F.mvpMapPoints.size());
  int idx = 0;
  for (size_t i = 0, iend = vpMapPointMatches.size(); i < iend; i++) {
    MapPoint* pMP = vpMapPointMatches[i];
    if (pMP && !pMP->isBad()) {
      const cv::KeyPoint& kp = F.mvKeysUn[i];
      mvP2D.push_back(kp.pt);
      mvSigma2.push_back(F.mvLevelSigma2[kp.octave]);
      cv::Mat Pos = pMP->GetWorldPos();
      mvP3Dw.push_back(cv::Point3f(Pos.at<float>(0), Pos.at<float>(1), Pos.at<float>(2)));
      mvKeyPointIndices.push_back(i);
      mvAllIndices.push_back(idx);
      idx++;
    }
  }
  fu = F.fx;
  fv = F.fy;
  uc = F.cx;
  vc = F.cy;
  SetRansacParameters();
}

PnPsolver::~PnPsolver() {
  delete[] pws;
  delete[] us;
  delete[] alphas;
  delete[] pcs;
}

// :181-230
void PnPsolver::SetRansacParameters(double probability, int minInliers, int maxIterations, int minSet, float epsilon,
                                    float th2) {
  mRansacProb = probability;
  mRansacMinInliers = minInliers;
  mRansacMaxIts = maxIterations;
  mRansacEpsilon = epsilon;
  mRansacMinSet = minSet;
  mRansacTh = th2;
  N = mvP2D.size();
  mvbInliersi.resize(N);
  int nMinInliers = N * mRansacEpsilon;
  if (nMinInliers < mRansacMinInliers) nMinInliers = mRansacMinInliers;
  if (nMinInliers < minSet) nMinInliers = minSet;
  mRansacMinInliers = nMinInliers;
  if (mRansacEpsilon < (float)mRansacMinInliers / N) mRansacEpsilon = (float)mRansacMinInliers / N;
  int nIterations;
  if (mRansacMinInliers == N)
    nIterations = 1;
  else
    nIterations = ceil(log(1 - mRansacProb) / log(1 - pow(mRansacEpsilon, 3)));
  mRansacMaxIts = max(1, min(nIterations, mRansacMaxIts));
  mvMaxError.resize(mvSigma2.size());
  for (size_t i = 0; i < mvSigma2.size(); i++) mvMaxError[i] = mvSigma2[i] * th2;
}

cv::Mat PnPsolver::find(vector<bool>& vbInliers, int& nInliers) {
  bool bFlag;
  return iterate(mRansacMaxIts, bFlag, vbInliers, nInliers);
}

cv::Mat PnPsolver::iterate(int nIterations, bool& bNoMore, vector<bool>& vbInliers, int& nInliers) {
  bNoMore = false;
  vbInliers.clear();
  nInliers = 0;
  if (N < mRansacMinInliers) {
    bNoMore = true;
    return cv::Mat();
  }
  // the draws of the iterations this call runs unless it returns early, in the reference's order
  int k = mRansacMaxIts - mnIterations;
  if (nIterations > k) k = nIterations;
  if (k < 0) k = 0;
  const int minSet = mRansacMinSet > 0 ? mRansacMinSet : 0;
  std::vector<int32_t> sets((size_t)k * minSet);
  std::vector<size_t> vAvailableIndices;
  for (int it = 0; it < k; it++) {
    vAvailableIndices = mvAllIndices;
    for (short i = 0; i < mRansacMinSet; ++i) {
      int randi = DUtils::Random::RandomInt(0, vAvailableIndices.size() - 1);
      sets[(size_t)it * minSet + i] = (int32_t)vAvailableIndices[randi];
      vAvailableIndices[randi] = vAvailableIndices.back();
      vAvailableIndices.pop_back();
    }
  }

  std::vector<float> P3((size_t)N * 3), P2((size_t)N * 2), bestTcw(16, 0.f);
  std::vector<uint8_t> bestIn((size_t)(N > 0 ? N : 1), 0), inl((size_t)(N > 0 ? N : 1)), bestOut(inl.size());
  for (int i = 0; i < N; i++) {
    P3[(size_t)i * 3] = mvP3Dw[i].x;
    P3[(size_t)i * 3 + 1] = mvP3Dw[i].y;
    P3[(size_t)i * 3 + 2] = mvP3Dw[i].z;
    P2[(size_t)i * 2] = mvP2D[i].x;
    P2[(size_t)i * 2 + 1] = mvP2D[i].y;
    bestIn[(size_t)i] = i < (int)mvbBestInliers.size() && mvbBestInliers[i];
  }
  if (mBestTcw.empty()) {
    for (int i = 0; i < 4; i++) bestTcw[(size_t)i * 5] = 1.f;
  } else {
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++) bestTcw[(size_t)r * 4 + c] = mBestTcw.at<float>(r, c);
  }
  b2s_pnpsolver_problem q;
  q.n = N;
  q.P3Dw = P3.data();
  q.P2D = P2.data();
  q.sigma2 = mvSigma2.data();
  q.fu = (float)fu;
  q.fv = (float)fv;
  q.uc = (float)uc;
  q.vc = (float)vc;
  q.th2 = mRansacTh;
  q.min_inliers = mRansacMinInliers;
  q.max_its = mRansacMaxIts;
  q.min_set = mRansacMinSet;
  q.iterations_done = mnIterations;
  q.best_inliers = mnBestInliers;
  q.best_Tcw = bestTcw.data();
  q.best_mask = bestIn.data();
  q.k = k;
  q.sets = sets.data();
  b2s_pnpsolver_result r;
  r.inliers = inl.data();
  r.best_mask = bestOut.data();
  int rc;
  {
    std::lock_guard<std::mutex> lock(g_pnpsolver.mutex);
    rc = g_pnpsolver.get({N, k}, {1024, 300}, [](const int* c, b2s_pnpsolver** h) {
      return b2s_pnpsolver_create(c[0], c[1], 1, b2s_host::device(), h);
    });
    if (rc == B2S_OK) rc = b2s_pnpsolver_iterate(g_pnpsolver.h, 1, &q, &r);
  }
  if (rc != B2S_OK) {
    b2s_host::report("PnPsolver::iterate", rc);
    return cv::Mat();
  }
  mnIterations = r.iterations_done;
  mnBestInliers = r.best_inliers;
  if (r.best_changed) {
    mvbBestInliers.assign((size_t)N, false);
    for (int i = 0; i < N; i++) mvbBestInliers[i] = bestOut[(size_t)i] != 0;
    mBestTcw = cv::Mat(4, 4, CV_32F, r.best_Tcw).clone();
  }
  if (!r.returned) {
    bNoMore = r.no_more != 0;
    return cv::Mat();
  }
  nInliers = r.n_inliers;
  vbInliers = vector<bool>(mvpMapPointMatches.size(), false);
  for (int i = 0; i < N; i++)
    if (inl[(size_t)i]) vbInliers[mvKeyPointIndices[i]] = true;
  if (r.no_more) {  // the loop ended: mBestTcw
    bNoMore = true;
    return mBestTcw.clone();
  }
  mnRefinedInliers = r.n_inliers;
  mvbRefinedInliers.assign((size_t)N, false);
  for (int i = 0; i < N; i++) mvbRefinedInliers[i] = inl[(size_t)i] != 0;
  mRefinedTcw = cv::Mat(4, 4, CV_32F, r.Tcw).clone();
  return mRefinedTcw.clone();
}

}  // namespace ORB_SLAM2
