#pragma once
#include <cstdint>
#include <vector>

#include "../../include/b200slam.h"

namespace ORB_SLAM2 {

// Initializer::Initialize (src/Initializer.cc:68-231) on flattened frames, with the minimal sets drawn by the caller
struct InitProblem {
  std::vector<float> kp1, kp2;       // n1 x 2 / n2 x 2: mvKeysUn[i].pt of the reference / current frame
  std::vector<int32_t> matches12;    // n1: vMatches12 (< 0: unmatched)
  float K[9];                        // mK, row-major
  float sigma = 1.0f;
  std::vector<int32_t> sets;         // iterations x 8: mvSets
};

struct InitResult {
  bool ret = false;
  int model = 0;                     // 1: homography, 2: fundamental matrix
  int rtState = 0;                   // R21 / t21: 1 written, -1 emptied, 0 untouched
  float R21[9], t21[3];
  std::vector<float> p3d;            // n1 x 3: vP3D (when ret)
  std::vector<uint8_t> triangulated; // n1: vbTriangulated (when ret)
};

class MonoInitializer {
 public:
  // Returns the library's status (B2S_OK, or the error of b2s_initialize; b2s_last_error() has the text)
  static int Initialize(const InitProblem& p, InitResult& out);
};

}  // namespace ORB_SLAM2
