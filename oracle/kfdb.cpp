// TEST INFRASTRUCTURE — CPU restatement of KeyFrameDatabase (src/KeyFrameDatabase.cc:45-374) with DBoW2's L1 score
// (Thirdparty/DBoW2/DBoW2/ScoringObject.cpp:23-68), the checker for csrc/kfdb.cu.  It keeps the reference's inverted
// file (one list per word, add() order, erase() without reordering), so it checks the device's merge formulation by an
// independent route.  The per-keyframe query state (include/KeyFrame.h:328-338) is kept by id, starts at 0 / 0 / 0.0f,
// survives erase() and is dropped by clear(), as documented for b2s_kfdb_* in include/b200slam.h.
// It also counts two paths the tests want to see taken: covisibility neighbours whose score was read although this query
// did not write it (the stale mRelocScore of :336-344), and best keyframes dropped by the first-occurrence dedupe.
// Built into oracle/liborb_kfdb.so by oracle/kfdb.mk; bound by tests/kfdb_binding.py.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <list>
#include <set>
#include <unordered_map>
#include <vector>

namespace {

struct Kf {
  std::vector<uint32_t> w;
  std::vector<double> v;
  bool live = false;
  uint64_t loop_query = 0;
  int32_t loop_words = 0;
  float loop_score = 0.0f;
  uint64_t reloc_query = 0;
  int32_t reloc_words = 0;
  float reloc_score = 0.0f;
  uint64_t loop_written = 0, reloc_written = 0;  // query serial of the last score write
};

struct Db {
  int n_words = 0;
  std::unordered_map<uint64_t, Kf> kfs;
  std::unordered_map<uint32_t, std::list<uint64_t> > inv;
  uint64_t serial = 0;
  long long stale_reads = 0, dedupes = 0;
};

// L1Scoring::score: the common words in ascending order, one sequential double sum, then -s/2
double l1_score(const uint32_t* aw, const double* av, int na, const std::vector<uint32_t>& bw, const std::vector<double>& bv) {
  double s = 0.0;
  size_t i = 0, j = 0;
  while (i < (size_t)na && j < bw.size()) {
    if (aw[i] == bw[j]) {
      const double x = av[i], y = bv[j];
      s += std::fabs(x - y) - std::fabs(x) - std::fabs(y);
      i++;
      j++;
    } else if (aw[i] < bw[j]) {
      i++;
    } else {
      j++;
    }
  }
  return -s / 2.0;
}

const Kf* find(const Db* d, uint64_t id) {
  auto it = d->kfs.find(id);
  return it == d->kfs.end() ? nullptr : &it->second;
}

int detect(Db* d, bool loop, uint64_t qid, const uint32_t* w, const double* v, int n, const uint64_t* conn, int n_conn,
           float min_score, const uint64_t* covis_ids, const int32_t* covis_n, int n_rows, uint64_t* out, int cap) {
  d->serial++;
  const std::set<uint64_t> connected(conn, conn + n_conn);
  // step 1: keyframes sharing a word, in inverted-file order, and their word counts
  std::vector<uint64_t> listed;
  for (int i = 0; i < n; i++) {
    auto it = d->inv.find(w[i]);
    if (it == d->inv.end()) continue;
    for (uint64_t id : it->second) {
      Kf& k = d->kfs[id];
      if (loop) {
        if (k.loop_query != qid) {
          k.loop_words = 0;
          if (!connected.count(id)) {
            k.loop_query = qid;
            listed.push_back(id);
          }
        }
        k.loop_words++;
      } else {
        if (k.reloc_query != qid) {
          k.reloc_words = 0;
          k.reloc_query = qid;
          listed.push_back(id);
        }
        k.reloc_words++;
      }
    }
  }
  if (listed.empty()) return 0;
  // step 2: the common-word gate
  int max_common = 0;
  for (uint64_t id : listed) {
    const Kf& k = d->kfs[id];
    max_common = std::max(max_common, loop ? k.loop_words : k.reloc_words);
  }
  const int min_common = (int)((float)max_common * 0.8f);
  // step 3: scores
  std::vector<std::pair<float, uint64_t> > scored;
  for (uint64_t id : listed) {
    Kf& k = d->kfs[id];
    if ((loop ? k.loop_words : k.reloc_words) <= min_common) continue;
    const float si = (float)l1_score(w, v, n, k.w, k.v);
    if (loop) {
      k.loop_score = si;
      k.loop_written = d->serial;
      if (si >= min_score) scored.push_back(std::make_pair(si, id));
    } else {
      k.reloc_score = si;
      k.reloc_written = d->serial;
      scored.push_back(std::make_pair(si, id));
    }
  }
  if (scored.empty()) return 0;
  // step 4: covisibility groups
  std::vector<std::pair<float, uint64_t> > groups;
  float best_acc = loop ? min_score : 0.0f;
  for (const auto& e : scored) {
    float acc = e.first, best = e.first;
    uint64_t best_id = e.second;
    if (e.second < (uint64_t)n_rows) {
      for (int k = 0; k < covis_n[e.second] && k < 10; k++) {
        const uint64_t nb = covis_ids[e.second * 10 + k];
        const Kf* s = find(d, nb);
        const Kf zero;
        if (!s) s = &zero;
        float sc;
        if (loop) {
          if (s->loop_query != qid || s->loop_words <= min_common) continue;
          sc = s->loop_score;
          if (s->loop_written != d->serial) d->stale_reads++;
        } else {
          if (s->reloc_query != qid) continue;
          sc = s->reloc_score;
          if (s->reloc_written != d->serial) d->stale_reads++;
        }
        acc += sc;
        if (sc > best) {
          best = sc;
          best_id = nb;
        }
      }
    }
    groups.push_back(std::make_pair(acc, best_id));
    if (acc > best_acc) best_acc = acc;
  }
  // step 5: retain and dedupe
  const float min_retain = 0.75f * best_acc;
  std::set<uint64_t> added;
  int cnt = 0;
  for (const auto& gr : groups) {
    if (!(gr.first > min_retain)) continue;
    if (added.count(gr.second)) {
      d->dedupes++;
      continue;
    }
    added.insert(gr.second);
    if (cnt < cap) out[cnt] = gr.second;
    cnt++;
  }
  return cnt;
}

}  // namespace

extern "C" {
void* orc_kfdb_create(int n_words) {
  Db* d = new Db();
  d->n_words = n_words;
  return d;
}
void orc_kfdb_destroy(void* h) { delete static_cast<Db*>(h); }

// -1: the id is already in the database
int orc_kfdb_add(void* h, uint64_t id, const uint32_t* w, const double* v, int n) {
  Db* d = static_cast<Db*>(h);
  Kf& k = d->kfs[id];
  if (k.live) return -1;
  k.live = true;
  k.w.assign(w, w + n);
  k.v.assign(v, v + n);
  for (int i = 0; i < n; i++) d->inv[w[i]].push_back(id);
  return 0;
}

void orc_kfdb_erase(void* h, uint64_t id) {
  Db* d = static_cast<Db*>(h);
  auto it = d->kfs.find(id);
  if (it == d->kfs.end() || !it->second.live) return;
  it->second.live = false;
  for (uint32_t w : it->second.w) {
    std::list<uint64_t>& l = d->inv[w];
    for (auto li = l.begin(); li != l.end(); ++li)
      if (*li == id) {
        l.erase(li);
        break;
      }
  }
}

void orc_kfdb_clear(void* h) {
  Db* d = static_cast<Db*>(h);
  d->kfs.clear();
  d->inv.clear();
}

int orc_kfdb_size(void* h) {
  int n = 0;
  for (const auto& kv : static_cast<Db*>(h)->kfs) n += kv.second.live;
  return n;
}

int orc_kfdb_detect_loop(void* h, uint64_t qid, const uint32_t* w, const double* v, int n, const uint64_t* conn, int n_conn,
                         float min_score, const uint64_t* covis_ids, const int32_t* covis_n, int n_rows, uint64_t* out,
                         int cap) {
  return detect(static_cast<Db*>(h), true, qid, w, v, n, conn, n_conn, min_score, covis_ids, covis_n, n_rows, out, cap);
}

int orc_kfdb_detect_reloc(void* h, uint64_t qid, const uint32_t* w, const double* v, int n, const uint64_t* covis_ids,
                          const int32_t* covis_n, int n_rows, uint64_t* out, int cap) {
  return detect(static_cast<Db*>(h), false, qid, w, v, n, nullptr, 0, 0.0f, covis_ids, covis_n, n_rows, out, cap);
}

// b2s_kfdb_state layout: u64, i32, f32, u64, i32, f32
void orc_kfdb_state(void* h, uint64_t id, void* out) {
  const Kf* k = find(static_cast<Db*>(h), id);
  const Kf zero;
  if (!k) k = &zero;
  unsigned char* o = static_cast<unsigned char*>(out);
  memcpy(o + 0, &k->loop_query, 8);
  memcpy(o + 8, &k->loop_words, 4);
  memcpy(o + 12, &k->loop_score, 4);
  memcpy(o + 16, &k->reloc_query, 8);
  memcpy(o + 24, &k->reloc_words, 4);
  memcpy(o + 28, &k->reloc_score, 4);
}

void orc_kfdb_counters(void* h, long long* stale_reads, long long* dedupes) {
  *stale_reads = static_cast<Db*>(h)->stale_reads;
  *dedupes = static_cast<Db*>(h)->dedupes;
}

// ORBVocabulary::score for L1 (the product's host/ORBVocabulary.cc restates it; DBoW2's is in libref_kfdb.so)
double orc_l1_score(const uint32_t* aw, const double* av, int na, const uint32_t* bw, const double* bv, int nb) {
  return l1_score(aw, av, na, std::vector<uint32_t>(bw, bw + nb), std::vector<double>(bv, bv + nb));
}
}
