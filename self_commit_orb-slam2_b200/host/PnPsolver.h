#pragma once
#include <cstdint>
#include <vector>

#include "../../include/b200slam.h"

namespace ORB_SLAM2 {

// PnPsolver::iterate (src/PnPsolver.cc:240-363) on a flattened relocalisation candidate, with the minimal sets drawn by
// the caller.  The state the reference keeps across calls (iterations, bestInliers, bestTcw, bestMask) is the caller's.
struct PnPRansacProblem {
  std::vector<float> P3Dw;              // N x 3: mvP3Dw
  std::vector<float> P2D;               // N x 2: mvP2D
  std::vector<float> sigma2;            // N: mvLevelSigma2[octave] of each correspondence's keypoint
  float K[4];                           // fx, fy, cx, cy
  float th2 = 5.991f;                   // SetRansacParameters' th2
  int minInliers = 8, maxIts = 300;     // mRansacMinInliers, mRansacMaxIts after SetRansacParameters
  int iterations = 0, bestInliers = 0;  // mnIterations, mnBestInliers on entry
  float bestTcw[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};  // mBestTcw on entry
  std::vector<uint8_t> bestMask;        // N: mvbBestInliers on entry (empty: none)
  std::vector<int32_t> sets;            // k x 4, in draw order (k = max(nIterations, maxIts - iterations))
};

struct PnPRansacResult {
  bool returned = false;                // the call returned a pose (noMore: mBestTcw, else mRefinedTcw)
  float Tcw[16];                        // when returned
  std::vector<uint8_t> inliers;         // N, compacted order (0 unless returned)
  int nInliers = 0;
  bool noMore = false;
  int iterationsUsed = 0, iterations = 0, bestInliers = 0;  // the state after the call
  bool bestChanged = false;
  float bestTcw[16];                    // mBestTcw after the call
  std::vector<uint8_t> bestMask;        // N: mvbBestInliers after the call
};

class PnPRansac {
 public:
  // Returns the library's status (B2S_OK, or the error of b2s_pnpsolver_iterate; b2s_last_error() has the text)
  static int Iterate(const PnPRansacProblem& p, PnPRansacResult& out);
};

}  // namespace ORB_SLAM2
