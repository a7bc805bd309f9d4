// Optimizer_b200.cc — drop-in bodies of
//     void Optimizer::LocalBundleAdjustment(KeyFrame* pKF, bool* pbStopFlag, Map* pMap)   include/Optimizer.h:112
//     int  Optimizer::PoseOptimization(Frame* pFrame)                                      include/Optimizer.h:100
//     void Optimizer::GlobalBundleAdjustemnt(Map*, int, bool*, unsigned long, bool)       src/Optimizer.cc:55
//     void Optimizer::BundleAdjustment(const vector<KeyFrame*>&, const vector<MapPoint*>&, int, bool*, unsigned long,
//                                      bool)                                              src/Optimizer.cc:86
//     void Optimizer::OptimizeEssentialGraph(Map*, KeyFrame*, KeyFrame*, const KeyFrameAndPose&,
//                                            const KeyFrameAndPose&, const map<KeyFrame*, set<KeyFrame*>>&,
//                                            const bool&)                                src/Optimizer.cc:1017
//     int  Optimizer::OptimizeSim3(KeyFrame*, KeyFrame*, vector<MapPoint*>&, g2o::Sim3&, const float, const bool)
//                                                                                         src/Optimizer.cc:1364
// with the reference's exact signatures, for the LocalMapping / Tracking / LoopClosing threads to call unchanged
// (src/LocalMapping.cc:123, src/Tracking.cc:1081, 1219, 1398, 1834, 2078, 2152, src/LoopClosing.cc:460, 782, 880-895 ...).
// Compile this file INSIDE the reference tree (it includes the reference's own include/Optimizer.h) in place of those
// function bodies of src/Optimizer.cc (:55-341, :363-605, :629-997, :1017-1339, :1364-1590), that is every body of that
// file, and link libb200slam.so.
//
// What stays on the host is what touches the object graph: the window selection (local keyframes = pKF + covisibles,
// local map points = their matches, fixed cameras = other observers; the mnBALocalForKF / mnBAFixedForKF marks other
// threads rely on), and the write-back under Map::mMutexMapUpdate (erase the outlier observations, SetPose,
// SetWorldPos, UpdateNormalAndDepth).  Everything numeric — the graph, 5 + 10 Levenberg iterations, the outlier
// re-classification — is b2s_local_ba / b2s_pose_optimization on the GPU.  No exceptions, no return codes beyond the
// reference's: a library error is reported on stderr and the map is left untouched.
//
// tests: oracle/ref_optimizer_glue.cpp builds the same stub object graph for this file (oracle/_ref/libadapter_optimizer.so)
// and for the reference's own Optimizer.cc (libref_optimizer.so); tests/test_adapters_gpu.py requires identical erase
// lists and poses / landmarks within the parity bar.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <list>
#include <map>
#include <mutex>
#include <set>
#include <utility>
#include <vector>

#include "Optimizer.h"

#include "b200slam.h"
#include "../b2s_host.h"

namespace ORB_SLAM2 {
namespace {

using b2s_host::report;

int create_ba(const int* cap, b2s_ba_solver** h) {
  return b2s_ba_create(cap[0], cap[1], cap[2], 1, b2s_host::device(), h);
}

// One solver handle per calling thread role, grown on demand: LocalBA (LocalMapping), PoseOptimization (Tracking), the
// global bundle adjustment (LoopClosing's GBA thread, or Tracking's monocular initialisation), the essential graph
// (LoopClosing::CorrectLoop) and OptimizeSim3 (LoopClosing::ComputeSim3, one problem per call).
b2s_host::Slot<b2s_ba_solver, 3, b2s_ba_destroy> g_localBA, g_pose;
b2s_host::Slot<b2s_gba_solver, 3, b2s_gba_destroy> g_gba;
b2s_host::Slot<b2s_eg_solver, 3, b2s_eg_destroy> g_eg;
b2s_host::Slot<b2s_sim3opt_solver, 1, b2s_sim3opt_destroy> g_sim3;

b2s_sim3 to_b2s(const g2o::Sim3& S) {
  b2s_sim3 o;
  for (int i = 0; i < 4; i++) o.q[i] = S[i];
  for (int i = 0; i < 3; i++) o.t[i] = S[4 + i];
  o.s = S[7];
  return o;
}

void pose_to_floats(const cv::Mat& T, float* out) {
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) out[4 * i + j] = T.at<float>(i, j);
}

}  // namespace

void Optimizer::LocalBundleAdjustment(KeyFrame* pKF, bool* pbStopFlag, Map* pMap) {
  // ---- window selection (what src/Optimizer.cc:633-694 leaves behind: three lists and the marks on the objects)
  std::vector<KeyFrame*> localKFs(1, pKF);
  pKF->mnBALocalForKF = pKF->mnId;
  {
    const std::vector<KeyFrame*> neigh = pKF->GetVectorCovisibleKeyFrames();
    for (size_t i = 0; i < neigh.size(); i++) {
      neigh[i]->mnBALocalForKF = pKF->mnId;
      if (!neigh[i]->isBad()) localKFs.push_back(neigh[i]);
    }
  }
  std::vector<MapPoint*> localMPs;
  for (size_t k = 0; k < localKFs.size(); k++) {
    const std::vector<MapPoint*> matches = localKFs[k]->GetMapPointMatches();
    for (size_t i = 0; i < matches.size(); i++) {
      MapPoint* p = matches[i];
      if (!p || p->isBad() || p->mnBALocalForKF == pKF->mnId) continue;
      p->mnBALocalForKF = pKF->mnId;
      localMPs.push_back(p);
    }
  }
  std::vector<KeyFrame*> fixedKFs;
  std::vector<std::map<KeyFrame*, size_t> > observations(localMPs.size());
  for (size_t m = 0; m < localMPs.size(); m++) {
    observations[m] = localMPs[m]->GetObservations();
    for (std::map<KeyFrame*, size_t>::const_iterator it = observations[m].begin(); it != observations[m].end(); ++it) {
      KeyFrame* k = it->first;
      if (k->mnBALocalForKF == pKF->mnId || k->mnBAFixedForKF == pKF->mnId) continue;
      k->mnBAFixedForKF = pKF->mnId;
      if (!k->isBad()) fixedKFs.push_back(k);
    }
  }
  if (pbStopFlag && *pbStopFlag) return;  // :858-860 (nothing has been changed yet)

  // ---- flatten: local keyframes first, then the fixed cameras; one edge per observation of a non-bad keyframe
  std::map<KeyFrame*, int> kfIndex;
  std::vector<KeyFrame*> allKFs(localKFs);
  allKFs.insert(allKFs.end(), fixedKFs.begin(), fixedKFs.end());
  const int nKF = (int)allKFs.size(), nLocal = (int)localKFs.size(), nMP = (int)localMPs.size();
  std::vector<float> Tcw((size_t)nKF * 16), pts((size_t)nMP * 3);
  std::vector<uint8_t> fixed((size_t)nKF, 0);
  for (int k = 0; k < nKF; k++) {
    kfIndex[allKFs[k]] = k;
    pose_to_floats(allKFs[k]->GetPose(), &Tcw[(size_t)16 * k]);
    fixed[k] = (k >= nLocal) || (allKFs[k]->mnId == 0);  // :722, :736
  }
  std::vector<b2s_ba_edge> edges;
  std::vector<std::pair<KeyFrame*, MapPoint*> > edgeOwner;
  for (int m = 0; m < nMP; m++) {
    const cv::Mat X = localMPs[m]->GetWorldPos();
    for (int c = 0; c < 3; c++) pts[(size_t)3 * m + c] = X.at<float>(c);
    for (std::map<KeyFrame*, size_t>::const_iterator it = observations[m].begin(); it != observations[m].end(); ++it) {
      KeyFrame* k = it->first;
      if (k->isBad()) continue;
      std::map<KeyFrame*, int>::const_iterator ki = kfIndex.find(k);
      if (ki == kfIndex.end()) continue;  // (cannot happen: every non-bad observer is local or fixed)
      const cv::KeyPoint& kp = k->mvKeysUn[it->second];
      b2s_ba_edge e;
      e.kf = ki->second;
      e.mp = m;
      e.obs[0] = kp.pt.x;
      e.obs[1] = kp.pt.y;
      e.obs[2] = k->mvuRight[it->second];  // < 0: monocular observation (:794)
      e.inv_sigma2 = k->mvInvLevelSigma2[kp.octave];
      edges.push_back(e);
      edgeOwner.push_back(std::make_pair(k, localMPs[m]));
    }
  }
  const int nE = (int)edges.size();
  std::vector<float> TcwOut((size_t)nLocal * 16), ptsOut((size_t)nMP * 3);
  std::vector<uint8_t> outlier((size_t)(nE > 0 ? nE : 1), 0);
  b2s_ba_problem prob;
  prob.n_kf = nKF;
  prob.n_local = nLocal;
  prob.Tcw = Tcw.data();
  prob.fixed = fixed.data();
  prob.n_mp = nMP;
  prob.points = pts.data();
  prob.n_edges = nE;
  prob.edges = edges.data();
  prob.fx = pKF->fx;
  prob.fy = pKF->fy;
  prob.cx = pKF->cx;
  prob.cy = pKF->cy;
  prob.bf = pKF->mbf;
  prob.its1 = 5;   // optimizer.optimize(5)  (:864)
  prob.its2 = 10;  // optimizer.optimize(10) (:917)
  b2s_ba_result res;
  res.Tcw_out = TcwOut.data();
  res.points_out = ptsOut.data();
  res.edge_outlier = outlier.data();
  res.trace = nullptr;
  res.chi2_final = 0;
  res.n_trials = 0;
  {
    std::lock_guard<std::mutex> lock(g_localBA.mutex);
    int rc = g_localBA.get({nKF, nMP, nE}, {64, 8192, 65536}, create_ba);
    static_assert(sizeof(bool) == 1, "the stop flag is polled as one byte");
    if (rc == B2S_OK)
      rc = b2s_local_ba(g_localBA.h, &prob, reinterpret_cast<const volatile uint8_t*>(pbStopFlag), &res);
    if (rc == B2S_ERR_ABORTED) return;
    if (rc != B2S_OK) {
      report("Optimizer::LocalBundleAdjustment", rc);
      return;
    }
  }

  // ---- write-back (:921-996): monocular outliers first, then the stereo ones, each in edge order
  std::unique_lock<std::mutex> lock(pMap->mMutexMapUpdate);
  for (int pass = 0; pass < 2; pass++)
    for (int e = 0; e < nE; e++) {
      const bool stereo = edges[e].obs[2] >= 0;
      if (!outlier[e] || stereo != (pass == 1)) continue;
      edgeOwner[e].first->EraseMapPointMatch(edgeOwner[e].second);
      edgeOwner[e].second->EraseObservation(edgeOwner[e].first);
    }
  for (int k = 0; k < nLocal; k++) {
    cv::Mat T(4, 4, CV_32F);
    for (int i = 0; i < 4; i++)
      for (int j = 0; j < 4; j++) T.at<float>(i, j) = TcwOut[(size_t)16 * k + 4 * i + j];
    localKFs[k]->SetPose(T);
  }
  for (int m = 0; m < nMP; m++) {
    cv::Mat X(3, 1, CV_32F);
    for (int c = 0; c < 3; c++) X.at<float>(c) = ptsOut[(size_t)3 * m + c];
    localMPs[m]->SetWorldPos(X);
    localMPs[m]->UpdateNormalAndDepth();
  }
}

int Optimizer::PoseOptimization(Frame* pFrame) {
  const int N = pFrame->N;
  std::vector<uint8_t> hasMP((size_t)(N > 0 ? N : 1), 0), outl((size_t)(N > 0 ? N : 1), 0);
  std::vector<float> Xw((size_t)3 * (N > 0 ? N : 1), 0.f), kpx((size_t)(N > 0 ? N : 1)), kpy(kpx.size()), ur(kpx.size()),
      w(kpx.size());
  float Tcw[16], TcwOut[16];
  pose_to_floats(pFrame->mTcw, Tcw);
  int nCorr = 0;
  {
    std::unique_lock<std::mutex> lock(MapPoint::mGlobalMutex);  // :410
    for (int i = 0; i < N; i++) {
      MapPoint* p = pFrame->mvpMapPoints[i];
      const cv::KeyPoint& kp = pFrame->mvKeysUn[i];
      kpx[i] = kp.pt.x;
      kpy[i] = kp.pt.y;
      ur[i] = pFrame->mvuRight[i];
      w[i] = pFrame->mvInvLevelSigma2[kp.octave];
      if (!p) continue;
      hasMP[i] = 1;
      nCorr++;
      pFrame->mvbOutlier[i] = false;  // :421, :458
      const cv::Mat X = p->GetWorldPos();
      for (int c = 0; c < 3; c++) Xw[(size_t)3 * i + c] = X.at<float>(c);
    }
  }
  if (nCorr < 3) return 0;  // :492-493 (pose untouched)
  b2s_pose_problem prob;
  prob.Tcw = Tcw;
  prob.n = N;
  prob.has_mp = hasMP.data();
  prob.Xw = Xw.data();
  prob.kpx = kpx.data();
  prob.kpy = kpy.data();
  prob.uright = ur.data();
  prob.inv_sigma2 = w.data();
  prob.fx = pFrame->fx;
  prob.fy = pFrame->fy;
  prob.cx = pFrame->cx;
  prob.cy = pFrame->cy;
  prob.bf = pFrame->mbf;
  b2s_pose_result res;
  res.Tcw_out = TcwOut;
  res.outlier = outl.data();
  res.trace = nullptr;
  res.n_inliers = 0;
  res.n_trials = 0;
  {
    std::lock_guard<std::mutex> lock(g_pose.mutex);
    int rc = g_pose.get({0, 0, 0}, {4, 16, 64}, create_ba);
    if (rc == B2S_OK) rc = b2s_pose_optimization(g_pose.h, &prob, &res);
    if (rc != B2S_OK) {
      report("Optimizer::PoseOptimization", rc);
      return 0;
    }
  }
  for (int i = 0; i < N; i++)
    if (hasMP[i]) pFrame->mvbOutlier[i] = outl[i] != 0;
  cv::Mat T(4, 4, CV_32F);
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) T.at<float>(i, j) = TcwOut[4 * i + j];
  pFrame->SetPose(T);
  return res.n_inliers;
}

void Optimizer::GlobalBundleAdjustemnt(Map* pMap, int nIterations, bool* pbStopFlag, const unsigned long nLoopKF,
                                       const bool bRobust) {
  std::vector<KeyFrame*> vpKFs = pMap->GetAllKeyFrames();
  std::vector<MapPoint*> vpMP = pMap->GetAllMapPoints();
  BundleAdjustment(vpKFs, vpMP, nIterations, pbStopFlag, nLoopKF, bRobust);
}

void Optimizer::BundleAdjustment(const std::vector<KeyFrame*>& vpKFs, const std::vector<MapPoint*>& vpMP, int nIterations,
                                 bool* pbStopFlag, const unsigned long nLoopKF, const bool bRobust) {
  // ---- gather (src/Optimizer.cc:117-275): non-bad keyframes by ascending mnId (g2o orders vertices by id), mnId == 0
  // fixed; non-bad points by ascending mnId, one edge per observation of a non-bad keyframe with mnId <= maxKFid
  std::vector<KeyFrame*> kfs;
  unsigned long maxKFid = 0;
  for (size_t i = 0; i < vpKFs.size(); i++) {
    if (vpKFs[i]->isBad()) continue;
    kfs.push_back(vpKFs[i]);
    if (vpKFs[i]->mnId > maxKFid) maxKFid = vpKFs[i]->mnId;
  }
  std::sort(kfs.begin(), kfs.end(), [](KeyFrame* a, KeyFrame* b) { return a->mnId < b->mnId; });
  std::vector<MapPoint*> mps;
  for (size_t i = 0; i < vpMP.size(); i++)
    if (!vpMP[i]->isBad()) mps.push_back(vpMP[i]);
  std::sort(mps.begin(), mps.end(), [](MapPoint* a, MapPoint* b) { return a->mnId < b->mnId; });
  const int nKF = (int)kfs.size(), nMP = (int)mps.size();
  std::map<KeyFrame*, int> kfIndex;
  std::vector<float> Tcw((size_t)nKF * 16), pts((size_t)nMP * 3);
  std::vector<uint8_t> fixed((size_t)nKF, 0);
  float fx = 0, fy = 0, cx = 0, cy = 0, bf = 0;
  for (int k = 0; k < nKF; k++) {
    kfIndex[kfs[k]] = k;
    pose_to_floats(kfs[k]->GetPose(), &Tcw[(size_t)16 * k]);
    fixed[k] = kfs[k]->mnId == 0;  // :132
  }
  std::vector<b2s_ba_edge> edges;
  for (int m = 0; m < nMP; m++) {
    const cv::Mat X = mps[m]->GetWorldPos();
    for (int c = 0; c < 3; c++) pts[(size_t)3 * m + c] = X.at<float>(c);
    const std::map<KeyFrame*, size_t> observations = mps[m]->GetObservations();
    for (std::map<KeyFrame*, size_t>::const_iterator it = observations.begin(); it != observations.end(); ++it) {
      KeyFrame* k = it->first;
      if (k->isBad() || k->mnId > maxKFid) continue;  // :178-179
      std::map<KeyFrame*, int>::const_iterator ki = kfIndex.find(k);
      if (ki == kfIndex.end()) continue;  // (an observer outside the keyframe list: not a vertex of the graph)
      const cv::KeyPoint& kp = k->mvKeysUn[it->second];
      b2s_ba_edge e;
      e.kf = ki->second;
      e.mp = m;
      e.obs[0] = kp.pt.x;
      e.obs[1] = kp.pt.y;
      e.obs[2] = k->mvuRight[it->second];  // < 0: monocular observation (:186)
      e.inv_sigma2 = k->mvInvLevelSigma2[kp.octave];
      edges.push_back(e);
      if (edges.size() == 1) {
        fx = k->fx; fy = k->fy; cx = k->cx; cy = k->cy; bf = k->mbf;
      } else if (k->fx != fx || k->fy != fy || k->cx != cx || k->cy != cy || k->mbf != bf) {
        fprintf(stderr, "Optimizer::BundleAdjustment (b200): keyframes with different intrinsics are not supported\n");
        return;
      }
    }
  }
  const int nE = (int)edges.size();
  std::vector<float> TcwOut((size_t)(nKF > 0 ? nKF : 1) * 16), ptsOut((size_t)(nMP > 0 ? nMP : 1) * 3);
  std::vector<uint8_t> included((size_t)(nMP > 0 ? nMP : 1), 0);
  b2s_gba_problem prob;
  prob.n_kf = nKF;
  prob.Tcw = Tcw.data();
  prob.fixed = fixed.data();
  prob.n_mp = nMP;
  prob.points = pts.data();
  prob.n_edges = nE;
  prob.edges = edges.data();
  prob.fx = fx; prob.fy = fy; prob.cx = cx; prob.cy = cy; prob.bf = bf;
  prob.iterations = nIterations;
  prob.robust = bRobust ? 1 : 0;
  b2s_gba_result res;
  res.Tcw_out = TcwOut.data();
  res.points_out = ptsOut.data();
  res.point_included = included.data();
  res.trace = nullptr;
  res.chi2_final = 0;
  res.n_trials = 0;
  {
    std::lock_guard<std::mutex> lock(g_gba.mutex);
    int rc = g_gba.get({nKF, nMP, nE}, {256, 32768, 262144}, [](const int* c, b2s_gba_solver** h) {
      return b2s_gba_create(c[0], c[1], c[2], b2s_host::device(), h);
    });
    static_assert(sizeof(bool) == 1, "the stop flag is polled as one byte");
    if (rc == B2S_OK) rc = b2s_global_ba(g_gba.h, &prob, reinterpret_cast<const volatile uint8_t*>(pbStopFlag), &res);
    if (rc != B2S_OK) {
      report("Optimizer::BundleAdjustment", rc);
      return;
    }
  }

  // ---- scatter (:287-340): direct writes for the initial map (nLoopKF == 0), else the GBA copies for LoopClosing
  for (int k = 0; k < nKF; k++) {
    cv::Mat T(4, 4, CV_32F);
    for (int i = 0; i < 4; i++)
      for (int j = 0; j < 4; j++) T.at<float>(i, j) = TcwOut[(size_t)16 * k + 4 * i + j];
    if (nLoopKF == 0) {
      kfs[k]->SetPose(T);
    } else {
      kfs[k]->mTcwGBA.create(4, 4, CV_32F);
      T.copyTo(kfs[k]->mTcwGBA);
      kfs[k]->mnBAGlobalForKF = nLoopKF;
    }
  }
  for (int m = 0; m < nMP; m++) {
    if (!included[m]) continue;  // vbNotIncludedMP
    cv::Mat X(3, 1, CV_32F);
    for (int c = 0; c < 3; c++) X.at<float>(c) = ptsOut[(size_t)3 * m + c];
    if (nLoopKF == 0) {
      mps[m]->SetWorldPos(X);
      mps[m]->UpdateNormalAndDepth();
    } else {
      mps[m]->mPosGBA.create(3, 1, CV_32F);
      X.copyTo(mps[m]->mPosGBA);
      mps[m]->mnBAGlobalForKF = nLoopKF;
    }
  }
}

void Optimizer::OptimizeEssentialGraph(Map* pMap, KeyFrame* pLoopKF, KeyFrame* pCurKF,
                                       const LoopClosing::KeyFrameAndPose& NonCorrectedSim3,
                                       const LoopClosing::KeyFrameAndPose& CorrectedSim3,
                                       const map<KeyFrame*, set<KeyFrame*> >& LoopConnections, const bool& bFixScale) {
  const std::vector<KeyFrame*> vpKFs = pMap->GetAllKeyFrames();
  const std::vector<MapPoint*> vpMPs = pMap->GetAllMapPoints();
  const int minFeat = 100;

  // ---- gather, step 2 (:1059-1098): one vertex per non-bad keyframe, ascending mnId; vScw = CorrectedSim3 if present,
  // else Sim3(Rcw, tcw, 1)
  std::vector<KeyFrame*> kfs;
  for (size_t i = 0; i < vpKFs.size(); i++)
    if (!vpKFs[i]->isBad()) kfs.push_back(vpKFs[i]);
  std::sort(kfs.begin(), kfs.end(), [](KeyFrame* a, KeyFrame* b) { return a->mnId < b->mnId; });
  const int nKF = (int)kfs.size();
  std::map<unsigned long, int> index;  // mnId -> vertex
  std::vector<g2o::Sim3, Eigen::aligned_allocator<g2o::Sim3> > vScw((size_t)nKF);
  std::vector<b2s_sim3> Siw((size_t)nKF);
  for (int k = 0; k < nKF; k++) {
    KeyFrame* pKF = kfs[(size_t)k];
    index[pKF->mnId] = k;
    LoopClosing::KeyFrameAndPose::const_iterator it = CorrectedSim3.find(pKF);
    if (it != CorrectedSim3.end()) {
      vScw[(size_t)k] = it->second;
    } else {
      const cv::Mat R = pKF->GetRotation(), t = pKF->GetTranslation();
      Eigen::Matrix<double, 3, 3> Rcw;
      Eigen::Matrix<double, 3, 1> tcw;
      for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++) Rcw(i, j) = R.at<float>(i, j);
        tcw(i) = t.at<float>(i);
      }
      vScw[(size_t)k] = g2o::Sim3(Rcw, tcw, 1.0);
    }
    Siw[(size_t)k] = to_b2s(vScw[(size_t)k]);
  }
  std::map<unsigned long, int>::const_iterator li = index.find(pLoopKF->mnId);
  if (li == index.end()) {
    fprintf(stderr, "Optimizer::OptimizeEssentialGraph (b200): the loop keyframe is not in the map\n");
    return;
  }
  auto vertex = [&](KeyFrame* pKF) {
    std::map<unsigned long, int>::const_iterator it = index.find(pKF->mnId);
    return it == index.end() ? -1 : it->second;
  };
  // the pose an edge's measurement starts from: NonCorrectedSim3 if present, else vScw
  auto nonCorrected = [&](KeyFrame* pKF, int v) -> g2o::Sim3 {
    LoopClosing::KeyFrameAndPose::const_iterator it = NonCorrectedSim3.find(pKF);
    return it != NonCorrectedSim3.end() ? it->second : vScw[(size_t)v];
  };
  // an edge whose endpoint has no vertex would dereference a null vertex in the reference; it is left out here
  std::vector<b2s_sim3_edge> edges;
  auto add = [&](int i, int j, const g2o::Sim3& Sji) {
    if (i < 0 || j < 0) return;
    b2s_sim3_edge e;
    e.i = i;
    e.j = j;
    e.meas = to_b2s(Sji);
    edges.push_back(e);
  };
  std::set<std::pair<unsigned long, unsigned long> > sInsertedEdges;

  // ---- step 3 (:1108-1143): loop connections, measured from vScw
  for (map<KeyFrame*, set<KeyFrame*> >::const_iterator mit = LoopConnections.begin(); mit != LoopConnections.end(); mit++) {
    KeyFrame* pKF = mit->first;
    const unsigned long nIDi = pKF->mnId;
    const int vi = vertex(pKF);
    if (vi < 0) continue;
    const g2o::Sim3 Swi = vScw[(size_t)vi].inverse();
    for (set<KeyFrame*>::const_iterator sit = mit->second.begin(); sit != mit->second.end(); sit++) {
      const unsigned long nIDj = (*sit)->mnId;
      if ((nIDi != pCurKF->mnId || nIDj != pLoopKF->mnId) && pKF->GetWeight(*sit) < minFeat) continue;
      const int vj = vertex(*sit);
      if (vj < 0) continue;
      add(vi, vj, vScw[(size_t)vj] * Swi);
      sInsertedEdges.insert(std::make_pair(std::min(nIDi, nIDj), std::max(nIDi, nIDj)));
    }
  }
  // ---- step 4 (:1147-1262): spanning tree, loop edges and strong covisibility, measured from NonCorrectedSim3
  for (size_t i = 0; i < vpKFs.size(); i++) {
    KeyFrame* pKF = vpKFs[i];
    const int vi = vertex(pKF);
    if (vi < 0) continue;
    const g2o::Sim3 Swi = nonCorrected(pKF, vi).inverse();
    KeyFrame* pParentKF = pKF->GetParent();
    if (pParentKF) {
      const int vj = vertex(pParentKF);
      if (vj >= 0) add(vi, vj, nonCorrected(pParentKF, vj) * Swi);
    }
    const set<KeyFrame*> sLoopEdges = pKF->GetLoopEdges();
    for (set<KeyFrame*>::const_iterator sit = sLoopEdges.begin(); sit != sLoopEdges.end(); sit++) {
      KeyFrame* pLKF = *sit;
      if (pLKF->mnId < pKF->mnId) {
        const int vl = vertex(pLKF);
        if (vl >= 0) add(vi, vl, nonCorrected(pLKF, vl) * Swi);
      }
    }
    const std::vector<KeyFrame*> vpConnectedKFs = pKF->GetCovisiblesByWeight(minFeat);
    for (std::vector<KeyFrame*>::const_iterator vit = vpConnectedKFs.begin(); vit != vpConnectedKFs.end(); vit++) {
      KeyFrame* pKFn = *vit;
      if (pKFn && pKFn != pParentKF && !pKF->hasChild(pKFn) && !sLoopEdges.count(pKFn)) {
        if (!pKFn->isBad() && pKFn->mnId < pKF->mnId) {
          if (sInsertedEdges.count(std::make_pair(std::min(pKF->mnId, pKFn->mnId), std::max(pKF->mnId, pKFn->mnId))))
            continue;
          const int vn = vertex(pKFn);
          if (vn >= 0) add(vi, vn, nonCorrected(pKFn, vn) * Swi);
        }
      }
    }
  }
  // ---- points (:1304-1322): the non-bad ones, each with the vertex of its nIDr (-1: none, the point stays)
  std::vector<MapPoint*> mps;
  for (size_t i = 0; i < vpMPs.size(); i++)
    if (!vpMPs[i]->isBad()) mps.push_back(vpMPs[i]);
  const int nMP = (int)mps.size(), nE = (int)edges.size();
  std::vector<float> pts((size_t)(nMP > 0 ? nMP : 1) * 3), ptsOut((size_t)(nMP > 0 ? nMP : 1) * 3),
      TcwOut((size_t)(nKF > 0 ? nKF : 1) * 16);
  std::vector<int32_t> refKF((size_t)(nMP > 0 ? nMP : 1));
  for (int m = 0; m < nMP; m++) {
    MapPoint* pMP = mps[(size_t)m];
    const unsigned long nIDr =
        pMP->mnCorrectedByKF == pCurKF->mnId ? pMP->mnCorrectedReference : pMP->GetReferenceKeyFrame()->mnId;
    std::map<unsigned long, int>::const_iterator it = index.find(nIDr);
    refKF[(size_t)m] = it == index.end() ? -1 : it->second;
    const cv::Mat X = pMP->GetWorldPos();
    for (int c = 0; c < 3; c++) pts[(size_t)3 * m + c] = X.at<float>(c);
  }
  b2s_eg_problem prob;
  prob.n_kf = nKF;
  prob.Siw = Siw.data();
  prob.fixed_kf = li->second;
  prob.fix_scale = bFixScale ? 1 : 0;
  prob.n_edges = nE;
  prob.edges = edges.data();
  prob.n_mp = nMP;
  prob.points = pts.data();
  prob.ref_kf = refKF.data();
  b2s_eg_result res;
  res.Tcw_out = TcwOut.data();
  res.points_out = ptsOut.data();
  res.trace = nullptr;
  res.chi2_initial = res.chi2_final = 0;
  res.n_trials = 0;
  {
    std::lock_guard<std::mutex> lock(g_eg.mutex);
    int rc = g_eg.get({nKF, nE, nMP}, {1024, 16384, 65536}, [](const int* c, b2s_eg_solver** h) {
      return b2s_eg_create(c[0], c[1], c[2], b2s_host::device(), h);
    });
    if (rc == B2S_OK) rc = b2s_optimize_essential_graph(g_eg.h, &prob, &res);
    if (rc != B2S_OK) {
      report("Optimizer::OptimizeEssentialGraph", rc);
      return;
    }
  }

  // ---- scatter (:1274-1338) under the map-update lock: SetPose of every keyframe, SetWorldPos and
  // UpdateNormalAndDepth of every non-bad point
  std::unique_lock<std::mutex> lock(pMap->mMutexMapUpdate);
  for (int k = 0; k < nKF; k++) {
    cv::Mat T(4, 4, CV_32F);
    for (int i = 0; i < 4; i++)
      for (int j = 0; j < 4; j++) T.at<float>(i, j) = TcwOut[(size_t)16 * k + 4 * i + j];
    kfs[(size_t)k]->SetPose(T);
  }
  for (int m = 0; m < nMP; m++) {
    cv::Mat X(3, 1, CV_32F);
    for (int c = 0; c < 3; c++) X.at<float>(c) = ptsOut[(size_t)3 * m + c];
    mps[(size_t)m]->SetWorldPos(X);
    mps[(size_t)m]->UpdateNormalAndDepth();
  }
}

int Optimizer::OptimizeSim3(KeyFrame* pKF1, KeyFrame* pKF2, vector<MapPoint*>& vpMatches1, g2o::Sim3& g2oS12,
                            const float th2, const bool bFixScale) {
  const cv::Mat& K1 = pKF1->mK;
  const cv::Mat& K2 = pKF2->mK;
  const cv::Mat R1w = pKF1->GetRotation();
  const cv::Mat t1w = pKF1->GetTranslation();
  const cv::Mat R2w = pKF2->GetRotation();
  const cv::Mat t2w = pKF2->GetTranslation();

  // ---- gather (:1429-1520): the reference's skip rules in its order; the camera-frame points by its cv::Mat expression
  const int N = (int)vpMatches1.size();
  const std::vector<MapPoint*> vpMapPoints1 = pKF1->GetMapPointMatches();
  std::vector<size_t> vnIndexEdge;
  std::vector<float> X1c, X2c, obs1, obs2, is1, is2;
  for (int i = 0; i < N; i++) {
    if (!vpMatches1[i]) continue;
    MapPoint* pMP1 = vpMapPoints1[i];
    MapPoint* pMP2 = vpMatches1[i];
    const int i2 = pMP2->GetIndexInKeyFrame(pKF2);
    if (!pMP1 || !pMP2 || pMP1->isBad() || pMP2->isBad() || i2 < 0) continue;
    const cv::Mat P3D1c = R1w * pMP1->GetWorldPos() + t1w;
    const cv::Mat P3D2c = R2w * pMP2->GetWorldPos() + t2w;
    for (int c = 0; c < 3; c++) {
      X1c.push_back(P3D1c.at<float>(c));
      X2c.push_back(P3D2c.at<float>(c));
    }
    const cv::KeyPoint& kpUn1 = pKF1->mvKeysUn[i];
    const cv::KeyPoint& kpUn2 = pKF2->mvKeysUn[i2];
    obs1.push_back(kpUn1.pt.x);
    obs1.push_back(kpUn1.pt.y);
    obs2.push_back(kpUn2.pt.x);
    obs2.push_back(kpUn2.pt.y);
    is1.push_back(pKF1->mvInvLevelSigma2[kpUn1.octave]);
    is2.push_back(pKF2->mvInvLevelSigma2[kpUn2.octave]);
    vnIndexEdge.push_back((size_t)i);
  }
  const int n = (int)vnIndexEdge.size();
  b2s_sim3_problem prob;
  prob.n = n;
  prob.X1c = X1c.data();
  prob.X2c = X2c.data();
  prob.obs1 = obs1.data();
  prob.obs2 = obs2.data();
  prob.inv_sigma2_1 = is1.data();
  prob.inv_sigma2_2 = is2.data();
  prob.fx1 = K1.at<float>(0, 0);
  prob.fy1 = K1.at<float>(1, 1);
  prob.cx1 = K1.at<float>(0, 2);
  prob.cy1 = K1.at<float>(1, 2);
  prob.fx2 = K2.at<float>(0, 0);
  prob.fy2 = K2.at<float>(1, 1);
  prob.cx2 = K2.at<float>(0, 2);
  prob.cy2 = K2.at<float>(1, 2);
  prob.S12 = to_b2s(g2oS12);
  prob.th2 = th2;
  prob.fix_scale = bFixScale ? 1 : 0;
  std::vector<uint8_t> keep((size_t)(n > 0 ? n : 1));
  b2s_sim3_result res;
  res.keep = keep.data();
  res.trace = nullptr;
  res.n_inliers = res.n_trials = 0;
  {
    std::lock_guard<std::mutex> lock(g_sim3.mutex);
    int rc = g_sim3.get({n}, {4096}, [](const int* c, b2s_sim3opt_solver** h) {
      return b2s_sim3opt_create(c[0], 1, b2s_host::device(), h);
    });
    if (rc == B2S_OK) rc = b2s_optimize_sim3(g_sim3.h, 1, &prob, &res);
    if (rc != B2S_OK) {
      report("Optimizer::OptimizeSim3", rc);
      return 0;
    }
  }

  // ---- scatter: null the rejected matches; g2oS12 (S12_out is the input itself after the early return, :1549-1551)
  for (int k = 0; k < n; k++)
    if (!keep[(size_t)k]) vpMatches1[vnIndexEdge[(size_t)k]] = static_cast<MapPoint*>(NULL);
  for (int i = 0; i < 8; i++) g2oS12[i] = (&res.S12_out.q[0])[i];
  return res.n_inliers;
}

}  // namespace ORB_SLAM2
