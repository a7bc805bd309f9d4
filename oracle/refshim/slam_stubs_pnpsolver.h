// oracle/refshim/slam_stubs_pnpsolver.h — TEST INFRASTRUCTURE ONLY.  Pre-included (`-include`) into the in-place build
// of src/PnPsolver.cc and its glue (oracle/pnpsolver.mk): defines the include guards of MapPoint.h and Frame.h so that
// include/PnPsolver.h opens neither, and stands in for Frame and MapPoint with the members the PnPsolver constructor
// reads.  `using namespace std` is what the real Frame.h brings in.
#pragma once
#define MAPPOINT_H
#define FRAME_H
#include <cmath>
#include <vector>

#include <opencv2/core/core.hpp>

using namespace std;

namespace ORB_SLAM2 {

class MapPoint {
 public:
  bool bad = false;
  cv::Mat pos;  // 3 x 1 CV_32F world position
  bool isBad() { return bad; }
  cv::Mat GetWorldPos() { return pos.clone(); }
};

class Frame {
 public:
  std::vector<MapPoint*> mvpMapPoints;
  std::vector<cv::KeyPoint> mvKeysUn;
  std::vector<float> mvLevelSigma2;
  float fx, fy, cx, cy;
};
}  // namespace ORB_SLAM2
