// oracle/refshim/slam_stubs_init.h — TEST INFRASTRUCTURE ONLY.  Pre-included (`-include`) into the in-place build of
// src/Initializer.cc and its glue (oracle/init.mk): defines the include guards of Frame.h, Optimizer.h and ORBmatcher.h
// so that include/Initializer.h opens none of them, and stands in for Frame with the two members Initializer reads.
// `using namespace std` is what the real Frame.h brings in (through ORBVocabulary.h ->
// Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:36); with it the unqualified acos / sqrt / isfinite of Initializer.cc
// resolve to std's float overloads, as in the reference's own build.
#pragma once
#define FRAME_H
#define OPTIMIZER_H
#define ORBMATCHER_H
#include <cmath>
#include <utility>
#include <vector>

#include <opencv2/opencv.hpp>

using namespace std;

namespace ORB_SLAM2 {
class Frame {
 public:
  cv::Mat mK;
  std::vector<cv::KeyPoint> mvKeysUn;
};
}  // namespace ORB_SLAM2
