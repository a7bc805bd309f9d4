// KeyFrameDatabase_b200.cc — drop-in implementation of the reference's KeyFrameDatabase class
// (include/KeyFrameDatabase.h, unchanged) on top of libb200slam.so: the constructor, add, erase, clear,
// DetectLoopCandidates (LoopClosing::DetectLoop, src/LoopClosing.cc:184) and DetectRelocalizationCandidates
// (Tracking::Relocalization, src/Tracking.cc:2039) keep their exact signatures.  Compile this file INSIDE the reference
// tree in place of src/KeyFrameDatabase.cc and link libb200slam.so (INTEGRATION.md §3d).
//
// The BowVectors and the per-keyframe query state (mnLoopQuery ... mRelocScore) live on the device; the KeyFrame fields of
// that name are no longer written (nothing else in the system reads them).  The header is unchanged, so the device handle
// and the id -> KeyFrame* map of each database live in a registry keyed by the object.  A query gathers what only the
// object graph knows — GetBestCovisibilityKeyFrames(10) of every keyframe in the database, and GetConnectedKeyFrames() of
// the query keyframe — makes one C-ABI call under mMutex and maps the returned ids back to KeyFrame*.
//
// tests: oracle/ref_kfdb_glue.cpp drives this file (oracle/_ref/libadapter_kfdb.so) and the reference's own
// src/KeyFrameDatabase.cc (libref_kfdb.so) on the same stand-in objects; tests/test_kfdb_gpu.py requires the same
// vector<KeyFrame*>.
#include <cstdint>
#include <cstdlib>
#include <map>
#include <mutex>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "KeyFrameDatabase.h"

#include "b200slam.h"

using namespace std;

namespace ORB_SLAM2 {

namespace {

struct DbState {
  b2s_kfdb* h = nullptr;
  std::unordered_map<uint64_t, KeyFrame*> live;  // keyframes in the database, by mnId
};

std::mutex g_registry_mutex;
std::map<const KeyFrameDatabase*, DbState> g_registry;

DbState& state_of(const KeyFrameDatabase* db) {
  std::lock_guard<std::mutex> lock(g_registry_mutex);
  return g_registry[db];
}

void check(int rc, const char* what) {
  if (rc != B2S_OK) throw std::runtime_error(std::string(what) + ": libb200slam error " + std::to_string(rc) + ": " +
                                             b2s_last_error());
}

void flatten(const DBoW2::BowVector& v, std::vector<uint32_t>& w, std::vector<double>& x) {
  w.clear();
  x.clear();
  for (DBoW2::BowVector::const_iterator it = v.begin(); it != v.end(); ++it) {
    w.push_back((uint32_t)it->first);
    x.push_back(it->second);
  }
}

// GetBestCovisibilityKeyFrames(10) of every keyframe in the database, by id; `known` maps every id seen back to its object
struct Covis {
  std::vector<uint64_t> ids;
  std::vector<int32_t> n;
  std::unordered_map<uint64_t, KeyFrame*> known;
  b2s_kfdb_covis table;
  explicit Covis(const DbState& s) : known(s.live) {
    uint64_t rows = 0;
    for (const auto& kv : s.live) rows = std::max<uint64_t>(rows, kv.first + 1);
    ids.assign(rows * 10, 0);
    n.assign(rows, 0);
    for (const auto& kv : s.live) {
      const std::vector<KeyFrame*> nb = kv.second->GetBestCovisibilityKeyFrames(10);
      int k = 0;
      for (KeyFrame* p : nb) {
        if (k == 10) break;
        ids[kv.first * 10 + k++] = p->mnId;
        known[p->mnId] = p;
      }
      n[kv.first] = k;
    }
    table.ids = ids.data();
    table.n = n.data();
    table.n_rows = (int32_t)rows;
  }
  std::vector<KeyFrame*> objects(const std::vector<uint64_t>& out, int cnt) const {
    std::vector<KeyFrame*> r;
    r.reserve(cnt);
    for (int i = 0; i < cnt; i++) r.push_back(known.at(out[i]));
    return r;
  }
};

}  // namespace

KeyFrameDatabase::KeyFrameDatabase(const ORBVocabulary& voc) : mpVoc(&voc) {
  // no inverted file on the host: mvInvertedFile stays empty
  const char* e = getenv("B2S_DEVICE");
  DbState& s = state_of(this);
  check(b2s_kfdb_create((int)voc.size(), e ? atoi(e) : 0, &s.h), "KeyFrameDatabase");
}

void KeyFrameDatabase::add(KeyFrame* pKF) {
  unique_lock<mutex> lock(mMutex);
  DbState& s = state_of(this);
  std::vector<uint32_t> w;
  std::vector<double> x;
  flatten(pKF->mBowVec, w, x);
  check(b2s_kfdb_add(s.h, pKF->mnId, w.data(), x.data(), (int)w.size()), "KeyFrameDatabase::add");
  s.live[pKF->mnId] = pKF;
}

void KeyFrameDatabase::erase(KeyFrame* pKF) {
  unique_lock<mutex> lock(mMutex);
  DbState& s = state_of(this);
  auto it = s.live.find(pKF->mnId);
  if (it == s.live.end() || it->second != pKF) return;
  check(b2s_kfdb_erase(s.h, pKF->mnId), "KeyFrameDatabase::erase");
  s.live.erase(it);
}

void KeyFrameDatabase::clear() {
  unique_lock<mutex> lock(mMutex);
  DbState& s = state_of(this);
  check(b2s_kfdb_clear(s.h), "KeyFrameDatabase::clear");
  s.live.clear();
}

vector<KeyFrame*> KeyFrameDatabase::DetectLoopCandidates(KeyFrame* pKF, float minScore) {
  const set<KeyFrame*> spConnectedKeyFrames = pKF->GetConnectedKeyFrames();
  std::vector<uint64_t> conn;
  for (KeyFrame* p : spConnectedKeyFrames) conn.push_back(p->mnId);
  std::vector<uint32_t> w;
  std::vector<double> x;
  flatten(pKF->mBowVec, w, x);
  unique_lock<mutex> lock(mMutex);
  DbState& s = state_of(this);
  const Covis c(s);
  std::vector<uint64_t> out(s.live.size() + 1);
  int cnt = 0;
  check(b2s_kfdb_detect_loop_candidates(s.h, pKF->mnId, w.data(), x.data(), (int)w.size(), conn.data(), (int)conn.size(),
                                        minScore, &c.table, out.data(), (int)out.size(), &cnt),
        "KeyFrameDatabase::DetectLoopCandidates");
  return c.objects(out, cnt);
}

vector<KeyFrame*> KeyFrameDatabase::DetectRelocalizationCandidates(Frame* F) {
  std::vector<uint32_t> w;
  std::vector<double> x;
  flatten(F->mBowVec, w, x);
  unique_lock<mutex> lock(mMutex);
  DbState& s = state_of(this);
  const Covis c(s);
  std::vector<uint64_t> out(s.live.size() + 1);
  int cnt = 0;
  check(b2s_kfdb_detect_relocalization_candidates(s.h, F->mnId, w.data(), x.data(), (int)w.size(), &c.table, out.data(),
                                                  (int)out.size(), &cnt),
        "KeyFrameDatabase::DetectRelocalizationCandidates");
  return c.objects(out, cnt);
}

}  // namespace ORB_SLAM2
