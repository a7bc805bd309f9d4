#include "ORBVocabulary.h"

#include <cmath>
#include <cstdio>
#include <fstream>
#include <sstream>

#include "b2s_host.h"

namespace ORB_SLAM2 {

ORBVocabulary::~ORBVocabulary() { b2s_vocabulary_destroy(mpHandle); }

bool ORBVocabulary::load(int k, int L, const std::vector<int32_t>& parent, const std::vector<uint8_t>& leafFlag,
                         const std::vector<uint8_t>& desc, const std::vector<double>& weight) {
  b2s_vocabulary_destroy(mpHandle);
  mpHandle = nullptr;
  b2s_vocabulary_desc d;
  d.k = k; d.L = L; d.n_nodes = (int32_t)parent.size();
  d.parent = parent.data(); d.leaf_flag = leafFlag.data(); d.desc = desc.data(); d.weight = weight.data();
  const int rc = b2s_vocabulary_create(&d, b2s_host::device(), &mpHandle);
  if (rc != B2S_OK) {
    b2s_host::report("ORBVocabulary", rc);
    return false;
  }
  return true;
}

bool ORBVocabulary::loadFromTextFile(const std::string& filename) {
  std::ifstream f(filename.c_str());
  if (!f.is_open()) return false;
  std::string s;
  std::getline(f, s);
  std::stringstream ss(s);
  int k = 0, L = 0, n1 = 0, n2 = 0;
  ss >> k >> L >> n1 >> n2;
  if (k < 0 || k > 20 || L < 1 || L > 10 || n1 < 0 || n1 > 5 || n2 < 0 || n2 > 3) {  // :1359-1363
    fprintf(stderr, "Vocabulary loading failure: This is not a correct text file!\n");
    return false;
  }
  mScoring = n1;
  mWeighting = n2;
  std::vector<int32_t> parent(1, -1);
  std::vector<uint8_t> leaf(1, 0), desc(32, 0);
  std::vector<double> weight(1, 0.0);
  while (std::getline(f, s)) {  // :1378-1418
    if (s.empty()) continue;
    std::stringstream sn(s);
    int pid = 0, isLeaf = 0;
    sn >> pid >> isLeaf;
    parent.push_back(pid);
    leaf.push_back(isLeaf > 0 ? 1 : 0);
    for (int i = 0; i < 32; i++) {  // FORB::fromString: 32 decimal byte values
      int v = 0;
      sn >> v;
      desc.push_back((uint8_t)v);
    }
    double w = 0;
    sn >> w;
    weight.push_back(w);
  }
  return load(k, L, parent, leaf, desc, weight);
}

void ORBVocabulary::transform(const uint8_t* descriptors, int n, BowVector& v, FeatureVector& fv, int levelsup) const {
  v.clear();
  fv.clear();
  if (empty() || n <= 0) return;
  std::vector<int32_t> word(n), node(n);
  std::vector<double> w(n);
  const int rc = b2s_bow_transform(mpHandle, descriptors, n, levelsup, word.data(), w.data(), node.data());
  if (rc != B2S_OK) b2s_host::fail("ORBVocabulary::transform", rc);
  for (int i = 0; i < n; i++) {  // :1145-1160 (TF_IDF): addWeight / addFeature in feature order, stopped words skipped
    if (w[i] > 0) {
      v[(unsigned int)word[i]] += w[i];
      fv[(unsigned int)node[i]].push_back((unsigned int)i);
    }
  }
  double norm = 0.0;  // L1 scoring: mustNormalize -> BowVector::normalize(L1) (BowVector.cpp:62-84)
  for (BowVector::iterator it = v.begin(); it != v.end(); ++it) norm += std::fabs(it->second);
  if (norm > 0.0)
    for (BowVector::iterator it = v.begin(); it != v.end(); ++it) it->second /= norm;
}

double ORBVocabulary::score(const BowVector& a, const BowVector& b) const {
  // L1Scoring::score: over the common words in ascending order, one sequential sum (the lower_bound jumps of the
  // reference only skip words that are not common)
  double s = 0.0;
  BowVector::const_iterator i = a.begin(), j = b.begin();
  while (i != a.end() && j != b.end()) {
    if (i->first == j->first) {
      const double v = i->second, w = j->second;
      s += std::fabs(v - w) - std::fabs(v) - std::fabs(w);
      ++i;
      ++j;
    } else if (i->first < j->first) {
      i = a.lower_bound(j->first);
    } else {
      j = b.lower_bound(i->first);
    }
  }
  return -s / 2.0;  // ||v - w||_1 scaled to [0, 1] (Nister, 2006)
}

}  // namespace ORB_SLAM2
