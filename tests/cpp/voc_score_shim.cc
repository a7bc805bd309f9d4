// C entry point around the product's ORBVocabulary::score (self_commit_orb-slam2_b200/host/ORBVocabulary.cc), for
// tests/test_kfdb_score.py: two BowVectors as (word, value) arrays in.
#include <cstdint>

#include "ORBVocabulary.h"

extern "C" double voc_score(const uint32_t* w1, const double* v1, int n1, const uint32_t* w2, const double* v2, int n2) {
  ORB_SLAM2::BowVector a, b;
  for (int i = 0; i < n1; i++) a[w1[i]] = v1[i];
  for (int i = 0; i < n2; i++) b[w2[i]] = v2[i];
  ORB_SLAM2::ORBVocabulary voc;  // score() needs no loaded tree
  return voc.score(a, b);
}
