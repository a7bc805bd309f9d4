// TEST INFRASTRUCTURE — stand-ins so that the reference's src/KeyFrame.cc compiles IN PLACE, unmodified, with its own
// include/KeyFrame.h and include/Frame.h (pre-included with `-include`; defines the include guards of MapPoint.h, Map.h,
// KeyFrameDatabase.h, Converter.h and ORBVocabulary.h so the real headers are skipped).  Only what KeyFrame.cc touches:
//   MapPoint          GetObservations / isBad (UpdateConnections), EraseObservation / GetIndexInKeyFrame (SetBadFlag,
//                     EraseMapPointMatch), Observations (TrackedMapPoints), GetWorldPos (ComputeSceneMedianDepth)
//   Map               EraseKeyFrame (SetBadFlag)
//   KeyFrameDatabase  erase (SetBadFlag)
//   Converter / ORBVocabulary   toDescriptorVector / transform (ComputeBoW)
#ifndef B2S_REF_SLAM_STUBS_KEYFRAME_H
#define B2S_REF_SLAM_STUBS_KEYFRAME_H
#define MAPPOINT_H
#define MAP_H
#define KEYFRAMEDATABASE_H
#define CONVERTER_H
#define ORBVOCABULARY_H

#include <opencv2/core/core.hpp>

#include <map>
#include <mutex>
#include <set>
#include <vector>

#include "Thirdparty/DBoW2/DBoW2/BowVector.h"
#include "Thirdparty/DBoW2/DBoW2/FeatureVector.h"

using namespace std;  // the reference headers rely on it

namespace ORB_SLAM2 {

class KeyFrame;

class MapPoint {
 public:
  std::map<KeyFrame*, size_t> mObservations;
  bool mbBad = false;
  cv::Mat mWorldPos;
  std::map<KeyFrame*, size_t> GetObservations() { return mObservations; }
  bool isBad() { return mbBad; }
  int Observations() { return (int)mObservations.size(); }
  void EraseObservation(KeyFrame* pKF) { mObservations.erase(pKF); }
  int GetIndexInKeyFrame(KeyFrame* pKF) { return mObservations.count(pKF) ? (int)mObservations[pKF] : -1; }
  cv::Mat GetWorldPos() { return mWorldPos.clone(); }
};

class Map {
 public:
  void EraseKeyFrame(KeyFrame*) {}
};

class KeyFrameDatabase {
 public:
  void erase(KeyFrame*) {}
};

class Converter {
 public:
  static std::vector<cv::Mat> toDescriptorVector(const cv::Mat& Descriptors) {
    std::vector<cv::Mat> v;
    for (int j = 0; j < Descriptors.rows; j++) v.push_back(Descriptors.row(j));
    return v;
  }
};

class ORBVocabulary {
 public:
  void transform(const std::vector<cv::Mat>&, DBoW2::BowVector&, DBoW2::FeatureVector&, int) {}
};

}  // namespace ORB_SLAM2
#endif
