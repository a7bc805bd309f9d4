// Optimizer.h — mirror of Optimizer::LocalBundleAdjustment (/root/reference/include/Optimizer.h:112) on a flattened
// window.  The adapter that walks KeyFrame/MapPoint (src/Optimizer.cc:633-854) and writes the results back under
// Map::mMutexMapUpdate (:961-996) is listed in INTEGRATION.md.
#pragma once
#include <cstdint>
#include <vector>

#include "../../include/b200slam.h"

namespace ORB_SLAM2 {

struct LocalBAWindow {
  int nLocal = 0;                    // lLocalKeyFrames.size(); local keyframes come first in Tcw/fixed
  std::vector<float> Tcw;            // nKF x 16 (KeyFrame::GetPose(), row-major)
  std::vector<uint8_t> fixed;        // nKF: mnId==0 or lFixedCameras
  std::vector<float> points;         // nMP x 3
  std::vector<b2s_ba_edge> edges;    // insertion order of :770-853
  float fx = 0, fy = 0, cx = 0, cy = 0, bf = 0;
};

struct LocalBAResult {
  std::vector<float> Tcw;            // nLocal x 16 -> KeyFrame::SetPose
  std::vector<float> points;         // nMP x 3    -> MapPoint::SetWorldPos
  std::vector<uint8_t> outlier;      // per edge   -> vToErase
  bool aborted = false;              // stop flag was set before round 1: nothing to write back (:858-860)
};

struct PoseProblem {                 // Optimizer::PoseOptimization(Frame*) on the flattened frame
  float Tcw[16];                     // pFrame->mTcw
  std::vector<uint8_t> hasMapPoint;  // N: mvpMapPoints[i] != NULL
  std::vector<float> Xw;             // N x 3: pMP->GetWorldPos() (ignored where hasMapPoint == 0)
  std::vector<float> kpx, kpy;       // N: mvKeysUn[i].pt
  std::vector<float> uRight;         // N: mvuRight[i] (< 0: monocular observation)
  std::vector<float> invSigma2;      // N: mvInvLevelSigma2[mvKeysUn[i].octave]
  float fx = 0, fy = 0, cx = 0, cy = 0, bf = 0;
};

struct GlobalBAMap {                 // Optimizer::BundleAdjustment on the flattened map (src/Optimizer.cc:86-275)
  std::vector<float> Tcw;            // nKF x 16: the non-bad keyframes by ascending mnId (KeyFrame::GetPose())
  std::vector<uint8_t> fixed;        // nKF: mnId == 0
  std::vector<float> points;         // nMP x 3: the non-bad map points by ascending mnId
  std::vector<b2s_ba_edge> edges;    // grouped by point, observations of non-bad keyframes with mnId <= maxKFid
  float fx = 0, fy = 0, cx = 0, cy = 0, bf = 0;
};

struct GlobalBAResult {
  std::vector<float> Tcw;            // nKF x 16 -> SetPose (nLoopKF == 0) or mTcwGBA
  std::vector<float> points;         // nMP x 3  -> SetWorldPos + UpdateNormalAndDepth, or mPosGBA (included points only)
  std::vector<uint8_t> included;     // nMP: 0 = no edge (vbNotIncludedMP): not written back
};

struct EssentialGraph {              // Optimizer::OptimizeEssentialGraph on the gathered graph (src/Optimizer.cc:1059-1322)
  std::vector<b2s_sim3> Siw;         // nKF: vScw of the non-bad keyframes by ascending mnId
  int fixedKF = 0;                   // vertex of pLoopKF
  bool fixScale = false;             // bFixScale
  std::vector<b2s_sim3_edge> edges;  // insertion order of :1108-1262, measurements computed as the reference does
  std::vector<float> points;         // nMP x 3: the non-bad map points
  std::vector<int32_t> refKF;        // nMP: vertex of the point's nIDr, -1 for none
};

struct EssentialGraphResult {
  std::vector<float> Tcw;            // nKF x 16 -> SetPose
  std::vector<float> points;         // nMP x 3  -> SetWorldPos + UpdateNormalAndDepth
};

struct Sim3Problem {                 // Optimizer::OptimizeSim3 on the gathered correspondences (src/Optimizer.cc:1429-1520)
  std::vector<float> X1c, X2c;       // n x 3: R1w*P3D1w + t1w, R2w*P3D2w + t2w as the cv::Mat expression gives them
  std::vector<float> obs1, obs2;     // n x 2: mvKeysUn[i] of pKF1, mvKeysUn[i2] of pKF2
  std::vector<float> invSigma2_1, invSigma2_2;  // n: mvInvLevelSigma2 at the keypoints' octaves
  float K1[4], K2[4];                // fx fy cx cy
  b2s_sim3 S12;                      // g2oS12
  float th2 = 10.f;
  bool fixScale = false;
};

struct Sim3Result {
  b2s_sim3 S12;                      // -> g2oS12 (the input itself after the early return)
  std::vector<uint8_t> keep;         // n: 0 -> vpMatches1[vnIndexEdge[k]] = NULL
  int nInliers = 0;                  // the return value
};

class Optimizer {
 public:
  // int static PoseOptimization(Frame* pFrame) (include/Optimizer.h:100, src/Optimizer.cc:363-605): fills TcwOut (the
  // pose for pFrame->SetPose) and outlier (pFrame->mvbOutlier), returns nInitialCorrespondences - nBad
  static int PoseOptimization(const PoseProblem& f, float TcwOut[16], std::vector<uint8_t>& outlier);
  // void static LocalBundleAdjustment(KeyFrame* pKF, bool* pbStopFlag, Map* pMap) on the flattened window
  static void LocalBundleAdjustment(const LocalBAWindow& w, bool* pbStopFlag, LocalBAResult& out);
  // void static BundleAdjustment(vpKF, vpMP, nIterations, pbStopFlag, nLoopKF, bRobust) on the flattened map
  static void BundleAdjustment(const GlobalBAMap& m, int nIterations, bool* pbStopFlag, bool bRobust, GlobalBAResult& out);
  // void static OptimizeEssentialGraph(pMap, pLoopKF, pCurKF, NonCorrectedSim3, CorrectedSim3, LoopConnections,
  // bFixScale) on the gathered graph
  static void OptimizeEssentialGraph(const EssentialGraph& g, EssentialGraphResult& out);
  // int static OptimizeSim3(pKF1, pKF2, vpMatches1, g2oS12, th2, bFixScale) on the gathered correspondences
  static int OptimizeSim3(const Sim3Problem& p, Sim3Result& out);
};

}  // namespace ORB_SLAM2
