#pragma once
#include <cstdint>
#include <vector>

#include "../../include/b200slam.h"

namespace ORB_SLAM2 {

// Sim3Solver::iterate (src/Sim3Solver.cc:199-285) on a flattened loop candidate, with the minimal sets drawn by the
// caller.  The state the reference keeps across calls (iterations, bestInliers, the best model) is the caller's.
struct Sim3RansacProblem {
  std::vector<float> X1c, X2c;          // N x 3: mvX3Dc1 / mvX3Dc2
  std::vector<float> sigma2_1, sigma2_2; // N: mvLevelSigma2[octave] of each correspondence's keypoint
  float K1[4], K2[4];                   // fx, fy, cx, cy
  bool fixScale = true;
  int minInliers = 6, maxIts = 300;     // mRansacMinInliers, mRansacMaxIts after SetRansacParameters
  int iterations = 0, bestInliers = 0;  // mnIterations, mnBestInliers on entry
  std::vector<int32_t> sets;            // k x 3, in draw order (k <= maxIts - iterations)
};

struct Sim3RansacResult {
  bool returned = false;                // the call returned mBestT12
  float T12[16];                        // when returned
  bool bestChanged = false;             // R, t, s hold the new best model
  float R[9], t[3], s = 1.f;
  std::vector<uint8_t> inliers;         // N, compacted order (0 unless returned)
  int nInliers = 0;
  bool noMore = false;
  int iterationsUsed = 0, iterations = 0, bestInliers = 0;  // the state after the call
};

class Sim3Ransac {
 public:
  // Returns the library's status (B2S_OK, or the error of b2s_sim3solver_iterate; b2s_last_error() has the text)
  static int Iterate(const Sim3RansacProblem& p, Sim3RansacResult& out);
};

}  // namespace ORB_SLAM2
