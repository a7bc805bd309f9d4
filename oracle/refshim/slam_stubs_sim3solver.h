// oracle/refshim/slam_stubs_sim3solver.h — TEST INFRASTRUCTURE ONLY.  Pre-included (`-include`) into the in-place build
// of src/Sim3Solver.cc and its glue (oracle/sim3solver.mk): defines the include guards of KeyFrame.h, MapPoint.h and
// ORBmatcher.h so that include/Sim3Solver.h opens none of them, and stands in for KeyFrame and MapPoint with the members
// the Sim3Solver constructor reads.  `using namespace std` is what the real KeyFrame.h brings in.
#pragma once
#define KEYFRAME_H
#define MAPPOINT_H
#define ORBMATCHER_H
#include <cmath>
#include <map>
#include <vector>

#include <opencv2/opencv.hpp>

using namespace std;

namespace ORB_SLAM2 {
class KeyFrame;

class MapPoint {
 public:
  bool bad = false;
  cv::Mat pos;                       // 3 x 1 world position
  std::map<KeyFrame*, int> index;    // observation index per keyframe
  bool isBad() { return bad; }
  int GetIndexInKeyFrame(KeyFrame* pKF) {
    const auto it = index.find(pKF);
    return it == index.end() ? -1 : it->second;
  }
  cv::Mat GetWorldPos() { return pos.clone(); }
};

class KeyFrame {
 public:
  cv::Mat Tcw, mK;
  std::vector<MapPoint*> mvpMapPoints;
  std::vector<cv::KeyPoint> mvKeysUn;
  std::vector<float> mvLevelSigma2;
  std::vector<MapPoint*> GetMapPointMatches() { return mvpMapPoints; }
  cv::Mat GetRotation() { return Tcw.rowRange(0, 3).colRange(0, 3).clone(); }
  cv::Mat GetTranslation() { return Tcw.rowRange(0, 3).col(3).clone(); }
};
}  // namespace ORB_SLAM2
