// ORBVocabulary.h — mirror of ORB_SLAM2::ORBVocabulary (= DBoW2::TemplatedVocabulary<FORB::TDescriptor, FORB>,
// /root/reference/include/ORBVocabulary.h:33) for the part on the hot path: loadFromTextFile and transform
// (Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1338-1425, :1127-1256).  The tree lives on the device (libb200slam.so);
// BowVector / FeatureVector are composed on the host from the per-feature (word, weight, node) arrays.
#pragma once
#include <cstdint>
#include <map>
#include <string>
#include <vector>

#include "../../include/b200slam.h"

namespace ORB_SLAM2 {

typedef std::map<unsigned int, double> BowVector;                       // DBoW2::BowVector (word id -> value)
typedef std::map<unsigned int, std::vector<unsigned int> > FeatureVector;  // DBoW2::FeatureVector (node id -> features)

class ORBVocabulary {
 public:
  ORBVocabulary() {}
  ~ORBVocabulary();
  ORBVocabulary(const ORBVocabulary&) = delete;
  ORBVocabulary& operator=(const ORBVocabulary&) = delete;

  // bool loadFromTextFile(const std::string& filename): "k L scoring weighting" then "parent isLeaf d0..d31 weight" lines
  bool loadFromTextFile(const std::string& filename);
  // same, from already parsed arrays (node 0 = root)
  bool load(int k, int L, const std::vector<int32_t>& parent, const std::vector<uint8_t>& leafFlag,
            const std::vector<uint8_t>& desc, const std::vector<double>& weight);
  bool empty() const { return mpHandle == nullptr; }
  unsigned int size() const { return mpHandle ? (unsigned int)b2s_vocabulary_words(mpHandle) : 0u; }

  // void transform(const std::vector<TDescriptor>& features, BowVector& v, FeatureVector& fv, int levelsup) const
  // for the ORB vocabulary's TF_IDF weighting and L1 scoring; descriptors: n x 32 bytes (cv::Mat rows)
  void transform(const uint8_t* descriptors, int n, BowVector& v, FeatureVector& fv, int levelsup) const;

  // double score(const BowVector& a, const BowVector& b) const (TemplatedVocabulary.h:1199-1203) for the ORB
  // vocabulary's L1 scoring (ScoringObject.cpp:23-68), on the host: LoopClosing::DetectLoop calls it per covisible
  // keyframe; the keyframe database scores on the device (b2s_kfdb_*).
  double score(const BowVector& a, const BowVector& b) const;

 protected:
  b2s_vocabulary* mpHandle = nullptr;
  int mScoring = 0, mWeighting = 0;
};

}  // namespace ORB_SLAM2
