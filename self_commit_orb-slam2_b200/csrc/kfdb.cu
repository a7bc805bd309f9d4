// kfdb.cu — KeyFrameDatabase (src/KeyFrameDatabase.cc) on the device: DetectLoopCandidates (:104-239) and
// DetectRelocalizationCandidates (:252-374) with DBoW2's L1 score (Thirdparty/DBoW2/DBoW2/ScoringObject.cpp:23-68).
//
// No inverted file.  The reference's result is a function of three per-keyframe quantities: the number of query words the
// keyframe shares, the rank (in the query's ascending word order) of the first one, and the L1 score.  The inverted file
// is only the CPU's way of visiting the keyframes that share a word; a merge of the query against every live keyframe's
// sorted BowVector gives the same quantities exactly.  Step 1 of the reference appends a keyframe to lKFsSharingWords
// when it meets it for the first time: while walking the first query word it shares, at its position in that word's
// inverted list, which is add() order (erase() keeps the order of the rest).  So the list order is the order of the key
// (first shared rank, add sequence), and the live list below is kept in add order.
//
//   k_kfdb_match   one warp per live keyframe: shared-word count (ballot / popc), first shared rank, the L1 score as one
//                  left-to-right double chain over the common words in word order, and the per-keyframe state update of
//                  step 1 (mnLoopQuery / mnLoopWords, mnRelocQuery / mnRelocWords).
//   k_kfdb_finish  one CTA: max common words over the listed keyframes and the 0.8 gate, the score write-back, the list
//                  order (a stable counting sort by first rank over the add-ordered live list), the covisibility group
//                  sums, the 0.75 retain step and the first-occurrence dedupe.
//
// The score is computed for every keyframe that shares a word, gated or not: it costs one predicated load per common
// word, saves a launch, and only the gated ones are written back or read.
#include <algorithm>
#include <vector>

#include "common.cuh"

namespace b2s {
namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kMatchWarps = 8;
constexpr int kFinThreads = 1024;
constexpr int kFreePos = 0x7f7f7f7f;  // first_pos[] "unused" (cudaMemset byte 0x7f)
constexpr int64_t kPoolMin = 1 << 16;

struct LiveRec {  // one live keyframe, in add order
  int64_t off;    // into the BowVector pool
  int32_t n;
  int32_t id;
};
struct SlotRec {  // per live keyframe, per query
  int32_t words;  // mnLoopWords / mnRelocWords after step 1
  int32_t rank;   // first shared query rank (-1: none)
  float score;    // (float) L1 score
  int32_t listed; // appended to lKFsSharingWords by this query
};

__device__ __forceinline__ bool sorted_contains(const uint64_t* a, int n, uint64_t x) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo < n && a[lo] == x;
}

__global__ void __launch_bounds__(kMatchWarps * 32)
    k_kfdb_match(const uint32_t* __restrict__ pw, const double* __restrict__ pv, const LiveRec* __restrict__ live, int n_live,
                 const uint32_t* __restrict__ qw, const double* __restrict__ qv, int nq, const uint64_t* __restrict__ conn,
                 int n_conn, int loop, unsigned long long qid, b2s_kfdb_state* __restrict__ state, SlotRec* __restrict__ rec) {
  extern __shared__ __align__(16) unsigned char smem[];
  double* sv = reinterpret_cast<double*>(smem);
  uint32_t* sw = reinterpret_cast<uint32_t*>(sv + nq);
  for (int i = threadIdx.x; i < nq; i += blockDim.x) {
    sw[i] = qw[i];
    sv[i] = qv[i];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int slot = blockIdx.x * kMatchWarps + (threadIdx.x >> 5);
  if (slot >= n_live) return;
  const LiveRec kf = live[slot];
  const uint32_t qlo = sw[0], qhi = sw[nq - 1];
  int cnt = 0, first = -1;
  double s = 0.0;
  for (int base = 0; base < kf.n; base += 32) {
    const int j = base + lane;
    int r = -1;
    double t = 0.0;
    if (j < kf.n) {
      const uint32_t w = pw[kf.off + j];
      if (w >= qlo && w <= qhi) {
        int lo = 0, hi = nq - 1;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (sw[mid] < w) lo = mid + 1; else hi = mid;
        }
        if (sw[lo] == w) {
          r = lo;
          const double v = sv[lo], x = pv[kf.off + j];
          t = fabs(v - x) - fabs(v) - fabs(x);  // ScoringObject.cpp:40 (v1 = the query)
        }
      }
    }
    unsigned m = __ballot_sync(kFull, r >= 0);
    if (m) {
      // both vectors ascend, so the first common word in keyframe order has the smallest query rank
      if (first < 0) first = __shfl_sync(kFull, r, __ffs(m) - 1);
      cnt += __popc(m);
      while (m) {  // the reference's sequential sum, in ascending word order
        s += __shfl_sync(kFull, t, __ffs(m) - 1);
        m &= m - 1;
      }
    }
    if (pw[kf.off + min(base + 31, kf.n - 1)] > qhi) break;  // the rest of the keyframe's words are past the query's
  }
  if (lane != 0) return;
  SlotRec o;
  o.words = 0;
  o.rank = first;
  o.score = (float)(-s / 2.0);  // ScoringObject.cpp:66, then `float si = mpVoc->score(..)`
  o.listed = 0;
  if (cnt > 0) {
    b2s_kfdb_state st = state[kf.id];
    if (!loop) {  // :271-277
      if (st.reloc_query != qid) {
        st.reloc_words = 0;
        st.reloc_query = qid;
        o.listed = 1;
      }
      st.reloc_words += cnt;
      o.words = st.reloc_words;
    } else {  // :126-135: a connected keyframe is reset at every shared word and never flagged
      if (st.loop_query != qid) {
        if (sorted_contains(conn, n_conn, (uint64_t)kf.id)) {
          st.loop_words = 1;
        } else {
          st.loop_words = cnt;
          st.loop_query = qid;
          o.listed = 1;
        }
      } else {
        st.loop_words += cnt;
      }
      o.words = st.loop_words;
    }
    state[kf.id] = st;
  }
  rec[slot] = o;
}

__device__ int block_max_i(int v, int* red) {
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(kFull, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  v = red[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); w++) v = max(v, red[w]);
  return v;
}
__device__ float block_max_f(float v, float* red) {
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(kFull, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  v = red[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); w++) v = fmaxf(v, red[w]);
  return v;
}
// exclusive prefix sum over the block (kFinThreads = 32 warps); *total = the sum
__device__ int block_excl_scan(int v, int* red, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int inc = warp_incl_scan(v, lane);
  __syncthreads();
  if (lane == 31) red[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    const int t = red[lane];
    const int ti = warp_incl_scan(t, lane);
    red[lane] = ti - t;
    if (lane == 31) *total = ti;
  }
  __syncthreads();
  return red[wid] + inc - v;
}

__device__ __forceinline__ bool is_entry(const SlotRec& o, int min_common, int loop, float min_score) {
  return o.listed && o.words > min_common && (!loop || o.score >= min_score);  // :166-175 / :306-311
}

__global__ void __launch_bounds__(kFinThreads)
    k_kfdb_finish(const LiveRec* __restrict__ live, int n_live, const SlotRec* __restrict__ rec, int nq, int loop,
                  unsigned long long qid, float min_score, const uint64_t* __restrict__ covis_ids,
                  const int32_t* __restrict__ covis_n, int n_rows, b2s_kfdb_state* state, int state_cap,
                  int32_t* __restrict__ order, float* __restrict__ acc, int32_t* __restrict__ best,
                  int32_t* __restrict__ first_pos, int32_t* __restrict__ out) {
  __shared__ int hist[B2S_KFDB_MAX_WORDS];
  __shared__ int red_i[32];
  __shared__ float red_f[32];
  __shared__ int s_total;
  const int tid = threadIdx.x, lane = tid & 31;
  for (int r = tid; r < nq; r += kFinThreads) hist[r] = 0;
  // maxCommonWords over lKFsSharingWords (:148-155 / :286-293)
  int mx = 0, any = 0;
  for (int i = tid; i < n_live; i += kFinThreads) {
    const SlotRec o = rec[i];
    if (o.listed) {
      any = 1;
      mx = max(mx, o.words);
    }
  }
  mx = block_max_i(mx, red_i);
  any = block_max_i(any, red_i);
  if (!any) {  // lKFsSharingWords empty
    if (tid == 0) out[0] = 0;
    return;
  }
  const int min_common = (int)((float)mx * 0.8f);
  // score write-back for every scored keyframe, and the first-rank histogram of the entries of lScoreAndMatch
  for (int i = tid; i < n_live; i += kFinThreads) {
    const SlotRec o = rec[i];
    if (o.listed && o.words > min_common) {
      if (loop) state[live[i].id].loop_score = o.score;
      else state[live[i].id].reloc_score = o.score;
      if (!loop || o.score >= min_score) atomicAdd(&hist[o.rank], 1);
    }
  }
  __syncthreads();
  {  // exclusive scan of hist[0, nq): the first list position of each rank
    const int per = (nq + kFinThreads - 1) / kFinThreads, b0 = min(tid * per, nq), b1 = min(b0 + per, nq);
    int sum = 0;
    for (int r = b0; r < b1; r++) sum += hist[r];
    int run = block_excl_scan(sum, red_i, &s_total);
    for (int r = b0; r < b1; r++) {
      const int c = hist[r];
      hist[r] = run;
      run += c;
    }
  }
  __syncthreads();
  const int E = s_total;
  if (E == 0) {  // lScoreAndMatch empty
    if (tid == 0) out[0] = 0;
    return;
  }
  // list order: stable within a rank (the live list is in add order), one warp, 32 keyframes per step
  if (tid < 32) {
    for (int base = 0; base < n_live; base += 32) {
      const int i = base + lane;
      int e = 0, r = 0;
      if (i < n_live) {
        const SlotRec o = rec[i];
        if (is_entry(o, min_common, loop, min_score)) {
          e = 1;
          r = o.rank;
        }
      }
      const unsigned peers = __match_any_sync(kFull, e ? r : -1 - lane);
      const int leader = __ffs(peers) - 1;
      int s = 0;
      if (e && lane == leader) {
        s = hist[r];
        hist[r] = s + __popc(peers);
      }
      s = __shfl_sync(kFull, s, leader);
      if (e) order[s + __popc(peers & ((1u << lane) - 1u))] = i;
      __syncwarp();
    }
  }
  __syncthreads();
  // covisibility groups (:190-215 / :325-350); the neighbours' state is read after this query's write-back
  float amax = loop ? min_score : 0.0f;  // bestAccScore
  for (int p = tid; p < E; p += kFinThreads) {
    const int i = order[p];
    const int id = live[i].id;
    const float sc = rec[i].score;
    float a = sc, b = sc;
    int bid = id;
    if (id < n_rows) {
      const int nn = min(covis_n[id], 10);
      for (int k = 0; k < nn; k++) {
        const uint64_t nb = covis_ids[(size_t)id * 10 + k];
        b2s_kfdb_state st = {0, 0, 0.0f, 0, 0, 0.0f};  // a keyframe the database never saw
        if (nb < (uint64_t)state_cap) st = state[nb];
        // loop: flagged by this query id with enough words; reloc: flagged only, so a stale mRelocScore may be read
        if (loop ? (st.loop_query == qid && st.loop_words > min_common) : (st.reloc_query == qid)) {
          const float v = loop ? st.loop_score : st.reloc_score;
          a += v;
          if (v > b && nb < (uint64_t)state_cap) {  // (an unseen keyframe's 0.0f never beats a score >= 0)
            b = v;
            bid = (int)nb;
          }
        }
      }
    }
    acc[p] = a;
    best[p] = bid;
    if (a > amax) amax = a;
  }
  amax = block_max_f(amax, red_f);
  const float min_retain = 0.75f * amax;
  // first occurrence of each best keyframe among the retained groups, in list order (:220-236 / :355-371)
  for (int p = tid; p < E; p += kFinThreads)
    if (acc[p] > min_retain) atomicMin(&first_pos[best[p]], p);
  __syncthreads();
  int n_out = 0;
  for (int base = 0; base < E; base += kFinThreads) {
    const int p = base + tid;
    int f = 0, bid = 0;
    if (p < E && acc[p] > min_retain) {
      bid = best[p];
      f = first_pos[bid] == p;
    }
    const int pos = block_excl_scan(f, red_i, &s_total);
    if (f) out[1 + n_out + pos] = bid;
    n_out += s_total;
    __syncthreads();
  }
  for (int p = tid; p < E; p += kFinThreads)
    if (acc[p] > min_retain) first_pos[best[p]] = kFreePos;
  if (tid == 0) out[0] = n_out;
}

__global__ void k_kfdb_move(const uint32_t* __restrict__ ow, const double* __restrict__ ov, const LiveRec* __restrict__ from,
                            const LiveRec* __restrict__ to, uint32_t* __restrict__ nw, double* __restrict__ nv) {
  const LiveRec a = from[blockIdx.x], b = to[blockIdx.x];
  for (int j = threadIdx.x; j < a.n; j += blockDim.x) {
    nw[b.off + j] = ow[a.off + j];
    nv[b.off + j] = ov[a.off + j];
  }
}

}  // namespace
}  // namespace b2s

using namespace b2s;

struct b2s_kfdb : b2s::Stage {
  int n_words = 0;
  // BowVector pool (uint32_t words, double values): [0, pool_tail) holds the vectors of live and erased keyframes;
  // pool_live entries are live
  DevBuf d_pw, d_pv;
  int64_t pool_cap = 0, pool_tail = 0, pool_live = 0;
  std::vector<LiveRec> live;  // in add order (= the order of every inverted list)
  bool live_dirty = true;
  std::vector<int32_t> slot_of_id;  // -1: not in the database
  // per-id query state (b2s_kfdb_state) and dedupe scratch (int32_t), grown on demand
  DevBuf d_state, d_first_pos;
  int state_cap = 0;
  // per-live-keyframe scratch: LiveRec, SlotRec, int32_t order / best, float acc; int32_t count + ids out
  int live_cap = 0;
  DevBuf d_live, d_rec, d_order, d_best, d_acc, d_out;
  HostBuf h_out;
  // one upload per query: query words + values, connected ids, covisibility table
  Packed q;
};

namespace {

int ensure_live_cap(b2s_kfdb* db, int n) {
  if (n <= db->live_cap) return B2S_OK;
  const int cap = std::max(n, std::max(2 * db->live_cap, 256));
  db->live_cap = 0;  // until every buffer has grown
  db->live_dirty = true;
  int rc = grow(db->d_live, (size_t)cap * sizeof(LiveRec));
  if (rc == B2S_OK) rc = grow(db->d_rec, (size_t)cap * sizeof(SlotRec));
  if (rc == B2S_OK) rc = grow(db->d_order, (size_t)cap * 4);
  if (rc == B2S_OK) rc = grow(db->d_best, (size_t)cap * 4);
  if (rc == B2S_OK) rc = grow(db->d_acc, (size_t)cap * 4);
  if (rc == B2S_OK) rc = grow(db->d_out, (size_t)(cap + 1) * 4);
  if (rc == B2S_OK) rc = grow(db->h_out, (size_t)(cap + 1) * 4);
  if (rc != B2S_OK) return rc;
  db->live_cap = cap;
  return B2S_OK;
}

int ensure_state_cap(b2s_kfdb* db, int n) {
  if (n <= db->state_cap) return B2S_OK;
  const int cap = (int)std::min<int64_t>(INT32_MAX, std::max<int64_t>(n, std::max<int64_t>(2 * (int64_t)db->state_cap, 1024)));
  // new arrays, then swapped in: the old ones are freed on return, or kept if anything fails
  DevBuf s, f;
  cudaError_t e = cudaSuccess;
  if (grow(s, (size_t)cap * sizeof(b2s_kfdb_state)) != B2S_OK || grow(f, (size_t)cap * 4) != B2S_OK)
    e = cudaErrorMemoryAllocation;
  if (e == cudaSuccess) e = cudaMemsetAsync(s.p, 0, (size_t)cap * sizeof(b2s_kfdb_state), db->stream);
  if (e == cudaSuccess) e = cudaMemsetAsync(f.p, 0x7f, (size_t)cap * 4, db->stream);
  if (e == cudaSuccess && db->state_cap)
    e = cudaMemcpyAsync(s.p, db->d_state.p, (size_t)db->state_cap * sizeof(b2s_kfdb_state), cudaMemcpyDeviceToDevice, db->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(db->stream);
  if (e != cudaSuccess) {
    set_error("b2s_kfdb: state arrays for %d ids: %s", cap, cudaGetErrorString(e));
    return B2S_ERR_CUDA;
  }
  swap(db->d_state, s);
  swap(db->d_first_pos, f);
  db->state_cap = cap;
  return B2S_OK;
}

// Moves the live vectors to the front of a new pool with room for `extra` more entries.
int compact_pool(b2s_kfdb* db, int64_t extra) {
  const int64_t cap = std::max(kPoolMin, 2 * (db->pool_live + extra));
  // a new pool, then swapped in as in ensure_state_cap
  DevBuf nw, nv, from;
  cudaError_t e = cudaSuccess;
  if (grow(nw, (size_t)cap * 4) != B2S_OK || grow(nv, (size_t)cap * 8) != B2S_OK) e = cudaErrorMemoryAllocation;
  std::vector<LiveRec> moved(db->live);
  int64_t off = 0;
  for (LiveRec& r : moved) {
    r.off = off;
    off += r.n;
  }
  const int n = (int)moved.size();
  if (e == cudaSuccess && n && grow(from, (size_t)2 * n * sizeof(LiveRec)) != B2S_OK) e = cudaErrorMemoryAllocation;
  LiveRec* d_from = (LiveRec*)from.p;
  if (e == cudaSuccess && n) e = cudaMemcpyAsync(d_from, db->live.data(), (size_t)n * sizeof(LiveRec), cudaMemcpyHostToDevice, db->stream);
  if (e == cudaSuccess && n) e = cudaMemcpyAsync(d_from + n, moved.data(), (size_t)n * sizeof(LiveRec), cudaMemcpyHostToDevice, db->stream);
  if (e == cudaSuccess && n) {
    k_kfdb_move<<<n, 128, 0, db->stream>>>((const uint32_t*)db->d_pw.p, (const double*)db->d_pv.p, d_from, d_from + n,
                                           (uint32_t*)nw.p, (double*)nv.p);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(db->stream);
  if (e != cudaSuccess) {
    set_error("b2s_kfdb: pool compaction: %s", cudaGetErrorString(e));
    return B2S_ERR_CUDA;
  }
  swap(db->d_pw, nw);
  swap(db->d_pv, nv);
  db->pool_cap = cap;
  db->pool_tail = off;
  db->live.swap(moved);
  db->live_dirty = true;
  return B2S_OK;
}

int check_bow(const b2s_kfdb* db, const uint32_t* words, const double* values, int n, const char* fn) {
  if (n < 0 || (n > 0 && (!words || !values))) {
    set_error("%s: bad BowVector argument", fn);
    return B2S_ERR_BAD_ARG;
  }
  if (n > B2S_KFDB_MAX_WORDS) {
    set_error("%s: BowVector of %d entries (at most %d)", fn, n, B2S_KFDB_MAX_WORDS);
    return B2S_ERR_CAPACITY;
  }
  for (int i = 0; i < n; i++)
    if (words[i] >= (uint32_t)db->n_words || (i > 0 && words[i] <= words[i - 1])) {
      set_error("%s: word ids must ascend and be below %d (entry %d: %u)", fn, db->n_words, i, words[i]);
      return B2S_ERR_BAD_ARG;
    }
  return B2S_OK;
}

int query(b2s_kfdb* db, int loop, uint64_t qid, const uint32_t* words, const double* values, int n, const uint64_t* conn,
          int n_conn, float min_score, const b2s_kfdb_covis* covis, uint64_t* out_ids, int cap, int* n_out, const char* fn) {
  if (!db || !n_out || cap < 0 || (cap > 0 && !out_ids) || n_conn < 0 || (n_conn > 0 && !conn) ||
      (covis && (covis->n_rows < 0 || (covis->n_rows > 0 && (!covis->ids || !covis->n))))) {
    set_error("%s: bad argument", fn);
    return B2S_ERR_BAD_ARG;
  }
  *n_out = 0;
  int rc = check_bow(db, words, values, n, fn);
  if (rc != B2S_OK) return rc;
  db->lastMs = 0.0f;
  const int n_live = (int)db->live.size();
  if (n == 0 || n_live == 0) return B2S_OK;  // no keyframe shares a word: nothing is touched
  B2S_CUDA(cudaSetDevice(db->device));
  if ((rc = ensure_live_cap(db, n_live)) != B2S_OK) return rc;
  if (db->live_dirty) {
    B2S_CUDA(cudaMemcpyAsync(db->d_live.p, db->live.data(), (size_t)n_live * sizeof(LiveRec), cudaMemcpyHostToDevice,
                             db->stream));
    db->live_dirty = false;
  }
  const int n_rows = covis ? covis->n_rows : 0;
  Packed& q = db->q;
  q.clear();
  const Seg<double> qv = q.add<double>(n);
  const Seg<uint32_t> qw = q.add<uint32_t>(n);
  const Seg<uint64_t> qc = q.add<uint64_t>(n_conn), cid = q.add<uint64_t>((size_t)n_rows * 10);
  const Seg<int32_t> cn = q.add<int32_t>(n_rows);
  if ((rc = q.fit(fn)) != B2S_OK) return rc;
  q.stage(qv, values);
  q.stage(qw, words);
  q.stage(qc, conn);
  std::sort(q.host(qc), q.host(qc) + n_conn);
  q.stage(cid, n_rows ? covis->ids : nullptr);
  q.stage(cn, n_rows ? covis->n : nullptr);
  if ((rc = q.upload(db->stream)) != B2S_OK) return rc;
  const LiveRec* live = (const LiveRec*)db->d_live.p;
  SlotRec* rec = (SlotRec*)db->d_rec.p;
  b2s_kfdb_state* state = (b2s_kfdb_state*)db->d_state.p;
  if ((rc = db->begin()) != B2S_OK) return rc;
  k_kfdb_match<<<div_up(n_live, kMatchWarps), kMatchWarps * 32, (size_t)n * 12, db->stream>>>(
      (const uint32_t*)db->d_pw.p, (const double*)db->d_pv.p, live, n_live, q.dev(qw), q.dev(qv), n, q.dev(qc), n_conn,
      loop, (unsigned long long)qid, state, rec);
  B2S_CUDA(cudaGetLastError());
  k_kfdb_finish<<<1, kFinThreads, 0, db->stream>>>(live, n_live, rec, n, loop, (unsigned long long)qid, min_score,
                                                   q.dev(cid), q.dev(cn), n_rows, state, db->state_cap,
                                                   (int32_t*)db->d_order.p, (float*)db->d_acc.p, (int32_t*)db->d_best.p,
                                                   (int32_t*)db->d_first_pos.p, (int32_t*)db->d_out.p);
  B2S_CUDA(cudaGetLastError());
  B2S_CUDA(cudaEventRecord(db->ev[1], db->stream));  // the kernels only: the download is not timed
  const int n_dl = 1 + std::min(cap, n_live);
  B2S_CUDA(cudaMemcpyAsync(db->h_out.p, db->d_out.p, (size_t)n_dl * 4, cudaMemcpyDeviceToHost, db->stream));
  B2S_CUDA(cudaStreamSynchronize(db->stream));
  B2S_CUDA(cudaEventElapsedTime(&db->lastMs, db->ev[0], db->ev[1]));
  const int32_t* hout = (const int32_t*)db->h_out.p;
  const int cnt = hout[0];
  *n_out = cnt;
  if (cnt > cap) {
    set_error("%s: %d candidates, cap %d", fn, cnt, cap);
    return B2S_ERR_CAPACITY;
  }
  for (int i = 0; i < cnt; i++) out_ids[i] = (uint64_t)hout[1 + i];
  return B2S_OK;
}

}  // namespace

extern "C" void b2s_kfdb_destroy(b2s_kfdb* db) {
  if (!db) return;
  db->close();
  delete db;
}

extern "C" int b2s_kfdb_create(int n_words, int device, b2s_kfdb** out) {
  if (!out || n_words < 1) {
    set_error("b2s_kfdb_create: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  *out = nullptr;
  int rc = select_device(device);
  if (rc != B2S_OK) return rc;
  b2s_kfdb* db = new b2s_kfdb();
  db->n_words = n_words;
  db->open(device);
  cudaError_t e = db->error;
  if (e == cudaSuccess && (grow(db->d_pw, (size_t)kPoolMin * 4) != B2S_OK || grow(db->d_pv, (size_t)kPoolMin * 8) != B2S_OK))
    e = cudaErrorMemoryAllocation;
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(k_kfdb_match, cudaFuncAttributeMaxDynamicSharedMemorySize, B2S_KFDB_MAX_WORDS * 12);
  if (e != cudaSuccess) {
    set_error("b2s_kfdb_create: %s", cudaGetErrorString(e));
    b2s_kfdb_destroy(db);
    return B2S_ERR_CUDA;
  }
  db->pool_cap = kPoolMin;
  *out = db;
  return B2S_OK;
}

extern "C" int b2s_kfdb_add(b2s_kfdb* db, uint64_t kf_id, const uint32_t* words, const double* values, int n) {
  if (!db || kf_id >= (uint64_t)INT32_MAX) {
    set_error("b2s_kfdb_add: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  int rc = check_bow(db, words, values, n, "b2s_kfdb_add");
  if (rc != B2S_OK) return rc;
  const int id = (int)kf_id;
  if (id < (int)db->slot_of_id.size() && db->slot_of_id[id] >= 0) {
    set_error("b2s_kfdb_add: keyframe %d is already in the database", id);
    return B2S_ERR_BAD_ARG;
  }
  B2S_CUDA(cudaSetDevice(db->device));
  if ((rc = ensure_state_cap(db, id + 1)) != B2S_OK) return rc;
  if (db->pool_tail + n > db->pool_cap && (rc = compact_pool(db, n)) != B2S_OK) return rc;
  if (n) {
    B2S_CUDA(cudaMemcpyAsync((uint32_t*)db->d_pw.p + db->pool_tail, words, (size_t)n * 4, cudaMemcpyHostToDevice, db->stream));
    B2S_CUDA(cudaMemcpyAsync((double*)db->d_pv.p + db->pool_tail, values, (size_t)n * 8, cudaMemcpyHostToDevice, db->stream));
  }
  if (id >= (int)db->slot_of_id.size()) db->slot_of_id.resize((size_t)id + 1, -1);
  db->slot_of_id[id] = (int32_t)db->live.size();
  db->live.push_back(LiveRec{db->pool_tail, n, id});
  db->pool_tail += n;
  db->pool_live += n;
  db->live_dirty = true;
  return B2S_OK;
}

extern "C" int b2s_kfdb_erase(b2s_kfdb* db, uint64_t kf_id) {
  if (!db) {
    set_error("b2s_kfdb_erase: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  if (kf_id >= db->slot_of_id.size() || db->slot_of_id[kf_id] < 0) return B2S_OK;
  const int slot = db->slot_of_id[kf_id];
  db->pool_live -= db->live[slot].n;
  db->live.erase(db->live.begin() + slot);
  db->slot_of_id[kf_id] = -1;
  for (size_t i = slot; i < db->live.size(); i++) db->slot_of_id[db->live[i].id] = (int32_t)i;
  db->live_dirty = true;
  if (db->pool_tail - db->pool_live > std::max(db->pool_live, kPoolMin)) {  // more dead than live entries
    B2S_CUDA(cudaSetDevice(db->device));
    return compact_pool(db, 0);
  }
  return B2S_OK;
}

extern "C" int b2s_kfdb_clear(b2s_kfdb* db) {
  if (!db) {
    set_error("b2s_kfdb_clear: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  B2S_CUDA(cudaSetDevice(db->device));
  db->live.clear();
  db->slot_of_id.clear();
  db->pool_tail = db->pool_live = 0;
  db->live_dirty = true;
  if (db->state_cap) {
    B2S_CUDA(cudaMemsetAsync(db->d_state.p, 0, (size_t)db->state_cap * sizeof(b2s_kfdb_state), db->stream));
    B2S_CUDA(cudaStreamSynchronize(db->stream));
  }
  return B2S_OK;
}

extern "C" int b2s_kfdb_size(const b2s_kfdb* db, int* n) {
  if (!db || !n) {
    set_error("b2s_kfdb_size: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  *n = (int)db->live.size();
  return B2S_OK;
}

extern "C" int b2s_kfdb_detect_loop_candidates(b2s_kfdb* db, uint64_t query_kf_id, const uint32_t* words, const double* values,
                                               int n, const uint64_t* connected_ids, int n_connected, float min_score,
                                               const b2s_kfdb_covis* covis, uint64_t* out_ids, int cap, int* n_out) {
  return query(db, 1, query_kf_id, words, values, n, connected_ids, n_connected, min_score, covis, out_ids, cap, n_out,
               "b2s_kfdb_detect_loop_candidates");
}

extern "C" int b2s_kfdb_detect_relocalization_candidates(b2s_kfdb* db, uint64_t frame_id, const uint32_t* words,
                                                         const double* values, int n, const b2s_kfdb_covis* covis,
                                                         uint64_t* out_ids, int cap, int* n_out) {
  return query(db, 0, frame_id, words, values, n, nullptr, 0, 0.0f, covis, out_ids, cap, n_out,
               "b2s_kfdb_detect_relocalization_candidates");
}

extern "C" int b2s_kfdb_keyframe_state(b2s_kfdb* db, uint64_t kf_id, b2s_kfdb_state* state) {
  if (!db || !state) {
    set_error("b2s_kfdb_keyframe_state: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  memset(state, 0, sizeof(*state));
  if (kf_id >= (uint64_t)db->state_cap) return B2S_OK;
  B2S_CUDA(cudaSetDevice(db->device));
  B2S_CUDA(cudaMemcpyAsync(state, (const b2s_kfdb_state*)db->d_state.p + kf_id, sizeof(*state), cudaMemcpyDeviceToHost,
                           db->stream));
  B2S_CUDA(cudaStreamSynchronize(db->stream));
  return B2S_OK;
}

extern "C" float b2s_kfdb_last_query_ms(const b2s_kfdb* db) { return db ? db->lastMs : 0.0f; }
