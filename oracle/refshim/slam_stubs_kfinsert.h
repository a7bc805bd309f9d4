// TEST INFRASTRUCTURE — for the keyframe-insertion checkers (oracle/kfinsert.mk), stand-ins so that the reference's src/LocalMapping.cc, src/KeyFrame.cc and src/MapPoint.cc compile
// IN PLACE, unmodified, with their own include/LocalMapping.h, include/KeyFrame.h, include/MapPoint.h and include/Frame.h
// (pre-included with `-include`; defines the include guards of LoopClosing.h, Tracking.h, Map.h, KeyFrameDatabase.h,
// ORBmatcher.h, Optimizer.h, Converter.h and ORBVocabulary.h so the real headers are skipped).  Only what those three
// files name, with empty bodies, except:
//   Map::EraseKeyFrame  records its argument: KeyFrame::SetBadFlag calls it last, only for a keyframe it really culls,
//                       so the record is the order of the culls.
//   Map::EraseMapPoint  records its argument likewise (MapPoint::SetBadFlag calls it last).
//   ORBmatcher::DescriptorDistance  the Hamming distance of two descriptor rows (8 floats holding 32 bytes each).
#ifndef B2S_REF_SLAM_STUBS_KFINSERT_H
#define B2S_REF_SLAM_STUBS_KFINSERT_H
#define LOOPCLOSING_H
#define TRACKING_H
#define MAP_H
#define KEYFRAMEDATABASE_H
#define ORBMATCHER_H
#define OPTIMIZER_H
#define CONVERTER_H
#define ORBVOCABULARY_H

#include <opencv2/core/core.hpp>

#include <cstring>
#include <mutex>
#include <set>
#include <thread>  // std::this_thread in LocalMapping.cc, which the real Tracking.h brings in
#include <utility>
#include <vector>

#include "Thirdparty/DBoW2/DBoW2/BowVector.h"
#include "Thirdparty/DBoW2/DBoW2/FeatureVector.h"

using namespace std;  // the reference headers rely on it

namespace ORB_SLAM2 {

class KeyFrame;
class MapPoint;

class Map {
 public:
  std::mutex mMutexMapUpdate, mMutexPointCreation;
  std::vector<KeyFrame*> erased;  // EraseKeyFrame's arguments, in call order
  std::vector<MapPoint*> erasedPoints;  // EraseMapPoint's arguments, in call order
  void EraseKeyFrame(KeyFrame* pKF) { erased.push_back(pKF); }
  void EraseMapPoint(MapPoint* pMP) { erasedPoints.push_back(pMP); }
  void AddKeyFrame(KeyFrame*) {}
  void AddMapPoint(MapPoint*) {}
  long unsigned int KeyFramesInMap() { return 0; }
};

class KeyFrameDatabase {
 public:
  void erase(KeyFrame*) {}
};

class LoopClosing {
 public:
  void InsertKeyFrame(KeyFrame*) {}
};

class Tracking {};

class ORBmatcher {
 public:
  ORBmatcher(float = 0.6, bool = true) {}
  static int DescriptorDistance(const cv::Mat& a, const cv::Mat& b) {
    int d = 0;
    for (int i = 0; i < 8; i++) {
      unsigned x, y;
      memcpy(&x, a.data + i, 4);
      memcpy(&y, b.data + i, 4);
      d += __builtin_popcount(x ^ y);
    }
    return d;
  }
  int SearchForTriangulation(KeyFrame*, KeyFrame*, cv::Mat, std::vector<std::pair<size_t, size_t> >&, const bool) {
    return 0;
  }
  int Fuse(KeyFrame*, const std::vector<MapPoint*>&, const float = 3.0) { return 0; }
};

class Optimizer {
 public:
  static void LocalBundleAdjustment(KeyFrame*, bool*, Map*) {}
};

class Converter {
 public:
  static std::vector<cv::Mat> toDescriptorVector(const cv::Mat&) { return std::vector<cv::Mat>(); }
};

class ORBVocabulary {
 public:
  void transform(const std::vector<cv::Mat>&, DBoW2::BowVector&, DBoW2::FeatureVector&, int) {}
};

}  // namespace ORB_SLAM2
#endif
