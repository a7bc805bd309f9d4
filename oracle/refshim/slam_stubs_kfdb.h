// TEST INFRASTRUCTURE — stand-ins for KeyFrame / Frame so that the reference's src/KeyFrameDatabase.cc compiles IN PLACE,
// unmodified, with the reference's own include/KeyFrameDatabase.h and the vendored DBoW2 as ORBVocabulary (pre-included
// with `-include`; defines the KEYFRAME_H / FRAME_H include guards so the real headers are skipped).  Only what
// KeyFrameDatabase.cc touches is here: mnId, mBowVec, the six query fields of include/KeyFrame.h:328-338, an ordered
// covisibility list (GetBestCovisibilityKeyFrames) and the connected set (GetConnectedKeyFrames).
//
// mLoopScore / mRelocScore start at 0.0f (the reference leaves them uninitialised, src/KeyFrame.cc:49).  They are
// ScoreField: a float that remembers which query wrote it last, so the glue can count reads of a score that the current
// query did not write (the stale read of DetectRelocalizationCandidates, src/KeyFrameDatabase.cc:336-344).
#ifndef B2S_REF_SLAM_STUBS_KFDB_H
#define B2S_REF_SLAM_STUBS_KFDB_H
#define KEYFRAME_H
#define FRAME_H

#include <list>
#include <mutex>
#include <set>
#include <vector>

#include "Thirdparty/DBoW2/DBoW2/BowVector.h"

using namespace std;  // the reference headers rely on it (KeyFrameDatabase.h uses unqualified list)

namespace ORB_SLAM2 {

extern unsigned long long g_kfdb_query_serial;  // incremented by the glue before every query
extern long long g_kfdb_stale_loop_reads, g_kfdb_stale_reloc_reads;

template <int RELOC>
struct ScoreField {
  float v = 0.0f;
  unsigned long long written = 0;
  ScoreField& operator=(float x) {
    v = x;
    written = g_kfdb_query_serial;
    return *this;
  }
  operator float() const {
    if (written != g_kfdb_query_serial) ++(RELOC ? g_kfdb_stale_reloc_reads : g_kfdb_stale_loop_reads);
    return v;
  }
};

class KeyFrame {
 public:
  long unsigned int mnId = 0;
  DBoW2::BowVector mBowVec;
  long unsigned int mnLoopQuery = 0;
  int mnLoopWords = 0;
  ScoreField<0> mLoopScore;
  long unsigned int mnRelocQuery = 0;
  int mnRelocWords = 0;
  ScoreField<1> mRelocScore;

  std::vector<KeyFrame*> covis;      // GetBestCovisibilityKeyFrames order
  std::set<KeyFrame*> connected;
  std::set<KeyFrame*> GetConnectedKeyFrames() { return connected; }
  std::vector<KeyFrame*> GetBestCovisibilityKeyFrames(const int& N) {
    if ((int)covis.size() < N) return covis;
    return std::vector<KeyFrame*>(covis.begin(), covis.begin() + N);
  }
};

class Frame {
 public:
  long unsigned int mnId = 0;
  DBoW2::BowVector mBowVec;
};

}  // namespace ORB_SLAM2
#endif
