// TEST INFRASTRUCTURE — C entry points around the reference's KeyFrameDatabase (src/KeyFrameDatabase.cc compiled in place,
// unmodified, against the stand-in KeyFrame / Frame of refshim/slam_stubs_kfdb.h and the vendored DBoW2 as ORBVocabulary,
// so size() and score() are DBoW2's own).  Built into oracle/_ref/libref_kfdb.so (git-ignored).
//
// The glue owns the KeyFrame objects, one per id: add / erase hand the same object to the database, so a re-added
// keyframe keeps its query fields as in the reference; clear() deletes them all (Tracking::Reset deletes every keyframe
// and restarts KeyFrame::nNextId at 0, so ids are reused by fresh objects).  Before a query the covisibility table
// (GetBestCovisibilityKeyFrames(10) by id) is copied into the objects; neighbour ids without an object get a fresh one,
// which the database never saw.  The query keyframe / frame is a separate object with the query's id and BowVector:
// KeyFrameDatabase.cc only reads its mnId, mBowVec and GetConnectedKeyFrames().
//
// built with -DB2S_ADAPTER_BUILD into _ref/libadapter_kfdb.so, the entry points are adp_* and KeyFrameDatabase:: resolves
// to the product's drop-in (host/adapters/KeyFrameDatabase_b200.cc) instead of the reference's src/KeyFrameDatabase.cc.
#ifdef B2S_ADAPTER_BUILD
#define KFDB_FN(name) adp_kfdb_##name
#else
#define KFDB_FN(name) ref_kfdb_##name
#endif
#include <cstdint>
#include <cstring>
#include <map>
#include <set>
#include <vector>

#include "KeyFrameDatabase.h"

namespace ORB_SLAM2 {
unsigned long long g_kfdb_query_serial = 1;
long long g_kfdb_stale_loop_reads = 0, g_kfdb_stale_reloc_reads = 0;
}  // namespace ORB_SLAM2

using namespace ORB_SLAM2;

namespace {
// ORBVocabulary with n words: only size() and score() (L1, the ORB vocabulary's scoring) are used by the database
struct StandInVoc : public ORBVocabulary {
  explicit StandInVoc(int n_words) : ORBVocabulary(10, 6, DBoW2::TF_IDF, DBoW2::L1_NORM) { m_words.resize(n_words); }
};

struct Glue {
  StandInVoc voc;
  KeyFrameDatabase* db;
  std::map<uint64_t, KeyFrame*> objs;
  std::set<uint64_t> live;
  explicit Glue(int n_words) : voc(n_words), db(new KeyFrameDatabase(voc)) {}
  ~Glue() {
    delete db;
    for (auto& kv : objs) delete kv.second;
  }
  KeyFrame* obj(uint64_t id) {
    KeyFrame*& p = objs[id];
    if (!p) {
      p = new KeyFrame();
      p->mnId = id;
    }
    return p;
  }
  void set_covis(const uint64_t* ids, const int32_t* n, int n_rows) {
    for (uint64_t id : live) {
      KeyFrame* kf = obj(id);
      kf->covis.clear();
      if (id < (uint64_t)n_rows)
        for (int k = 0; k < n[id] && k < 10; k++) kf->covis.push_back(obj(ids[id * 10 + k]));
    }
  }
  int write(const std::vector<KeyFrame*>& v, uint64_t* out, int cap) {
    for (size_t i = 0; i < v.size() && (int)i < cap; i++) out[i] = v[i]->mnId;
    return (int)v.size();
  }
};

DBoW2::BowVector bow(const uint32_t* w, const double* v, int n) {
  DBoW2::BowVector b;
  for (int i = 0; i < n; i++) b[w[i]] = v[i];
  return b;
}

struct State {  // layout of b2s_kfdb_state
  uint64_t loop_query;
  int32_t loop_words;
  float loop_score;
  uint64_t reloc_query;
  int32_t reloc_words;
  float reloc_score;
};
}  // namespace

extern "C" {
void* KFDB_FN(create)(int n_words) { return new Glue(n_words); }
void KFDB_FN(destroy)(void* h) { delete static_cast<Glue*>(h); }

// -1: the id is already in the database
int KFDB_FN(add)(void* h, uint64_t id, const uint32_t* w, const double* v, int n) {
  Glue* g = static_cast<Glue*>(h);
  if (g->live.count(id)) return -1;
  KeyFrame* kf = g->obj(id);
  kf->mBowVec = bow(w, v, n);
  g->db->add(kf);
  g->live.insert(id);
  return 0;
}

void KFDB_FN(erase)(void* h, uint64_t id) {
  Glue* g = static_cast<Glue*>(h);
  if (!g->live.count(id)) return;
  g->db->erase(g->obj(id));
  g->live.erase(id);
}

void KFDB_FN(clear)(void* h) {
  Glue* g = static_cast<Glue*>(h);
  g->db->clear();
  for (auto& kv : g->objs) delete kv.second;
  g->objs.clear();
  g->live.clear();
}

int KFDB_FN(size)(void* h) { return (int)static_cast<Glue*>(h)->live.size(); }

// return the number of candidates (ids of the first min(cap, n) in out)
int KFDB_FN(detect_loop)(void* h, uint64_t qid, const uint32_t* w, const double* v, int n, const uint64_t* conn, int n_conn,
                         float min_score, const uint64_t* covis_ids, const int32_t* covis_n, int n_rows, uint64_t* out,
                         int cap) {
  Glue* g = static_cast<Glue*>(h);
  g->set_covis(covis_ids, covis_n, n_rows);
  KeyFrame q;
  q.mnId = qid;
  q.mBowVec = bow(w, v, n);
  for (int i = 0; i < n_conn; i++) q.connected.insert(g->obj(conn[i]));
  ++g_kfdb_query_serial;
  return g->write(g->db->DetectLoopCandidates(&q, min_score), out, cap);
}

int KFDB_FN(detect_reloc)(void* h, uint64_t qid, const uint32_t* w, const double* v, int n, const uint64_t* covis_ids,
                          const int32_t* covis_n, int n_rows, uint64_t* out, int cap) {
  Glue* g = static_cast<Glue*>(h);
  g->set_covis(covis_ids, covis_n, n_rows);
  Frame f;
  f.mnId = qid;
  f.mBowVec = bow(w, v, n);
  ++g_kfdb_query_serial;
  return g->write(g->db->DetectRelocalizationCandidates(&f), out, cap);
}

// the six query fields of keyframe `id` (zeros for an id without an object)
void KFDB_FN(state)(void* h, uint64_t id, void* out) {
  Glue* g = static_cast<Glue*>(h);
  State s;
  memset(&s, 0, sizeof(s));
  auto it = g->objs.find(id);
  if (it != g->objs.end()) {
    const KeyFrame* k = it->second;
    s.loop_query = k->mnLoopQuery;
    s.loop_words = k->mnLoopWords;
    s.loop_score = k->mLoopScore.v;
    s.reloc_query = k->mnRelocQuery;
    s.reloc_words = k->mnRelocWords;
    s.reloc_score = k->mRelocScore.v;
  }
  memcpy(out, &s, sizeof(s));
}

// ORBVocabulary::score (TemplatedVocabulary.h:1199-1203 -> L1Scoring::score)
double KFDB_FN(score)(const uint32_t* w1, const double* v1, int n1, const uint32_t* w2, const double* v2, int n2) {
  StandInVoc voc(1);
  return voc.score(bow(w1, v1, n1), bow(w2, v2, n2));
}

// reads of mLoopScore / mRelocScore that the running query had not written, since the library was loaded
void KFDB_FN(counters)(long long* stale_loop, long long* stale_reloc) {
  *stale_loop = g_kfdb_stale_loop_reads;
  *stale_reloc = g_kfdb_stale_reloc_reads;
}
}
