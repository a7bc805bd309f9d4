// covis.cu — KeyFrame::UpdateConnections (src/KeyFrame.cc:386-507) for a batch of keyframes, with the AddConnection
// (:159-178) and UpdateBestCovisibles (:185-209) it calls on the partners.  Integer work only.
//
// Three launches, no host synchronisation between them:
//   k_covis_count   one CTA per call: the counter KFcounter (:405-427) as a histogram over table indices, emitted in
//                   index order (std::map<KeyFrame*,int> order, index order standing for address order), nmax / pKFmax
//                   (:445-454) and the strong pairs (:455-463) or the fallback pair (:467-474), ordered as the sort +
//                   push_front of :477-485 leaves them: (weight desc, index desc).
//   k_covis_group   one CTA: the calls' events grouped by target keyframe, a stable counting sort on batch position.  A
//                   call makes one member event (its own replacement, :488-505, and the reads around it) and one
//                   AddConnection event per partner it connects to.
//   k_covis_replay  one warp per keyframe: its events replayed in batch order.  The counters are independent of each
//                   other (counting reads only observations and bad flags, which the calls never write), so only this
//                   merge has to follow the call order.
#include <cub/cub.cuh>

#include <algorithm>

#include "common.cuh"

using namespace b2s;

namespace {

constexpr int kTh = 15;          // the strong-pair threshold th (:438)
constexpr int kCountThreads = 256;
constexpr int kGroupThreads = 1024;
constexpr int kReplayWarps = 8;

struct Args {
  int n, B, maxConn;
  // input (device copies of the problem)
  const int *mapOff, *mapKf, *mapW, *listOff, *listKf, *listW;
  const int* kfFlags;  // bit 0: mbFirstConnection, bit 1: mnId == 0
  const int *parentIn, *mpBad, *obsOff, *obsKf, *member, *slotOff, *slotMp;
  // scratch, rows of stride n per call
  int* hist;  // all zero between calls: k_covis_count clears what it read
  int *cntKf, *cntW, *cntN, *strKf, *strW, *strN;
  int *evCnt, *evStart, *cur, *bound, *evPos, *evK;
  // outputs: small arrays (downloaded first) and areas
  int *flag, *outOff, *memOff, *changed, *parent, *first, *mapN, *listN, *startN, *afterN, *pair;
  int *oMapKf, *oMapW, *oListKf, *oListW, *oStartKf, *oAfterKf, *oAfterW;
};

// Block-wide exclusive scan of a[0, n) in place, a[n] = total (n + 1 entries written).
template <int T>
__device__ void block_exclusive_scan(int* a, int n) {
  typedef cub::BlockScan<int, T> Scan;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += T) {
    const int i = base + threadIdx.x;
    const int v = i < n ? a[i] : 0;
    int x, tot;
    Scan(tmp).ExclusiveSum(v, x, tot);
    if (i < n) a[i] = carry + x;
    __syncthreads();
    if (threadIdx.x == 0) carry += tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) a[n] = carry;
  __syncthreads();
}

__global__ void __launch_bounds__(kCountThreads) k_covis_count(Args a) {
  const int b = blockIdx.x, n = a.n, m = a.member[b];
  int* hist = a.hist + (size_t)b * n;
  for (int s = a.slotOff[b] + threadIdx.x; s < a.slotOff[b + 1]; s += kCountThreads) {
    const int mp = a.slotMp[s];
    if (mp < 0 || a.mpBad[mp]) continue;  // :409-413
    for (int o = a.obsOff[mp]; o < a.obsOff[mp + 1]; o++) {
      const int kf = a.obsKf[o];
      if (kf != m) atomicAdd(&hist[kf], 1);  // :421-423
    }
  }
  __syncthreads();

  typedef cub::BlockScan<int, kCountThreads> Scan;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int carry, nStrong;
  __shared__ unsigned long long best;  // (weight << 32) | (INT_MAX - index): the first strict maximum in index order
  if (threadIdx.x == 0) {
    carry = 0;
    nStrong = 0;
    best = 0ull;
  }
  __syncthreads();
  int* cKf = a.cntKf + (size_t)b * n;
  int* cW = a.cntW + (size_t)b * n;
  for (int base = 0; base < n; base += kCountThreads) {
    const int i = base + threadIdx.x;
    int v = 0;
    if (i < n) {
      v = hist[i];
      if (v) hist[i] = 0;
    }
    int x, tot;
    Scan(tmp).ExclusiveSum(v > 0 ? 1 : 0, x, tot);
    if (v > 0) {
      cKf[carry + x] = i;
      cW[carry + x] = v;
      atomicMax(&best, ((unsigned long long)v << 32) | (unsigned)(0x7fffffff - i));
      if (v >= kTh) atomicAdd(&nStrong, 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) carry += tot;
    __syncthreads();
  }
  const int C = carry, S = nStrong;
  int* sKf = a.strKf + (size_t)b * n;
  int* sW = a.strW + (size_t)b * n;
  // rank of each strong pair in (weight desc, index desc) order
  for (int i = threadIdx.x; i < C; i += kCountThreads) {
    const int wi = cW[i], ki = cKf[i];
    if (wi < kTh) continue;
    int r = 0;
    for (int j = 0; j < C; j++) {
      const int wj = cW[j];
      r += wj >= kTh && (wj > wi || (wj == wi && cKf[j] > ki));
    }
    sKf[r] = ki;
    sW[r] = wi;
  }
  if (threadIdx.x == 0) {
    a.cntN[b] = C;
    if (C > 0 && S == 0) {  // no strong pair: (nmax, pKFmax)
      sKf[0] = 0x7fffffff - (int)(best & 0xffffffffu);
      sW[0] = (int)(best >> 32);
    }
    a.strN[b] = C == 0 ? 0 : (S > 0 ? S : 1);
  }
}

__global__ void __launch_bounds__(kGroupThreads) k_covis_group(Args a) {
  const int n = a.n, B = a.B, tid = threadIdx.x;
  for (int t = tid; t < n; t += kGroupThreads) {
    a.evCnt[t] = 0;
    a.cur[t] = 0;
  }
  __syncthreads();
  for (int b = tid; b < B; b += kGroupThreads) {
    atomicAdd(&a.evCnt[a.member[b]], 1);
    for (int k = 0; k < a.strN[b]; k++) atomicAdd(&a.evCnt[a.strKf[(size_t)b * n + k]], 1);
  }
  __syncthreads();
  for (int t = tid; t <= n; t += kGroupThreads) a.evStart[t] = t < n ? a.evCnt[t] : 0;
  __syncthreads();
  block_exclusive_scan<kGroupThreads>(a.evStart, n);
  // a call's targets are distinct (its member is never its own partner), so one pass per call needs no atomics
  for (int b = 0; b < B; b++) {
    if (tid == 0) {
      const int m = a.member[b], e = a.evStart[m] + a.cur[m]++;
      a.evPos[e] = b;
      a.evK[e] = -1;
    }
    for (int k = tid; k < a.strN[b]; k += kGroupThreads) {
      const int t = a.strKf[(size_t)b * n + k], e = a.evStart[t] + a.cur[t]++;
      a.evPos[e] = b;
      a.evK[e] = k;
    }
    __syncthreads();
  }
  // room for each touched keyframe's map and list: the largest it starts from plus one per AddConnection
  for (int t = tid; t < n; t += kGroupThreads) {
    int bound = 0;
    if (a.evCnt[t] > 0) {
      int mx = max(a.mapOff[t + 1] - a.mapOff[t], a.listOff[t + 1] - a.listOff[t]), adds = 0;
      for (int e = a.evStart[t]; e < a.evStart[t] + a.evCnt[t]; e++)
        if (a.evK[e] < 0)
          mx = max(mx, a.cntN[a.evPos[e]]);
        else
          adds++;
      bound = mx + adds;
    }
    a.bound[t] = bound;
    a.outOff[t] = bound;
  }
  __syncthreads();
  block_exclusive_scan<kGroupThreads>(a.outOff, n);
  for (int b = tid; b < B; b += kGroupThreads) a.memOff[b] = a.bound[a.member[b]];
  __syncthreads();
  block_exclusive_scan<kGroupThreads>(a.memOff, B);
  if (tid == 0) a.flag[0] = a.outOff[n] > a.maxConn || a.memOff[B] > a.maxConn;
}

// UpdateBestCovisibles (:185-209): the whole map in (weight desc, index desc) order
__device__ void sort_map(const int* mKf, const int* mW, int ms, int* lKf, int* lW, int lane) {
  for (int i = lane; i < ms; i += 32) {
    const int wi = mW[i], ki = mKf[i];
    int r = 0;
    for (int j = 0; j < ms; j++) {
      const int wj = mW[j];
      r += wj > wi || (wj == wi && mKf[j] > ki);
    }
    lKf[r] = ki;
    lW[r] = wi;
  }
  __syncwarp();
}

__device__ void copy_row(int* dst, const int* src, int len, int lane) {
  for (int i = lane; i < len; i += 32) dst[i] = src[i];
}

__global__ void __launch_bounds__(kReplayWarps * 32) k_covis_replay(Args a) {
  const int lane = threadIdx.x & 31, t = blockIdx.x * kReplayWarps + (threadIdx.x >> 5), n = a.n;
  if (t >= n) return;
  int parent = a.parentIn[t], first = a.kfFlags[t] & 1;
  const bool idZero = (a.kfFlags[t] & 2) != 0;
  const int c = a.evCnt[t];
  if (c == 0 || a.flag[0]) {
    if (lane == 0) {
      a.changed[t] = 0;
      a.parent[t] = parent;
      a.first[t] = first;
      a.mapN[t] = a.listN[t] = 0;
    }
    return;
  }
  const int o = a.outOff[t];
  int *mKf = a.oMapKf + o, *mW = a.oMapW + o, *lKf = a.oListKf + o, *lW = a.oListW + o;
  int ms = a.mapOff[t + 1] - a.mapOff[t], ls = a.listOff[t + 1] - a.listOff[t];
  copy_row(mKf, a.mapKf + a.mapOff[t], ms, lane);
  copy_row(mW, a.mapW + a.mapOff[t], ms, lane);
  copy_row(lKf, a.listKf + a.listOff[t], ls, lane);
  copy_row(lW, a.listW + a.listOff[t], ls, lane);
  __syncwarp();
  bool stale = false;  // the list is UpdateBestCovisibles of the current map, not yet materialised
  int changed = 0;
  for (int e = a.evStart[t]; e < a.evStart[t] + c; e++) {
    const int b = a.evPos[e], k = a.evK[e];
    if (k < 0) {  // this keyframe's own call
      if (stale) {
        sort_map(mKf, mW, ms, lKf, lW, lane);
        ls = ms;
        stale = false;
      }
      const int so = a.memOff[b];
      copy_row(a.oStartKf + so, lKf, ls, lane);  // GetVectorCovisibleKeyFrames() before the call
      const int startN = ls, C = a.cntN[b];
      int pp = -1;
      if (C > 0) {  // :488-505
        __syncwarp();
        copy_row(mKf, a.cntKf + (size_t)b * n, C, lane);
        copy_row(mW, a.cntW + (size_t)b * n, C, lane);
        ms = C;
        ls = a.strN[b];
        copy_row(lKf, a.strKf + (size_t)b * n, ls, lane);
        copy_row(lW, a.strW + (size_t)b * n, ls, lane);
        changed = 1;
        if (first && !idZero) {
          parent = pp = a.strKf[(size_t)b * n];
          first = 0;
        }
        __syncwarp();
      }
      copy_row(a.oAfterKf + so, mKf, ms, lane);  // the connection map right after the call
      copy_row(a.oAfterW + so, mW, ms, lane);
      if (lane == 0) {
        a.startN[b] = startN;
        a.afterN[b] = ms;
        a.pair[b] = pp;
      }
    } else {  // AddConnection(member, w) (:159-178)
      const int K = a.member[b], w = a.strW[(size_t)b * n + k];
      int pos = 0;
      for (int base = 0; base < ms; base += 32) {
        const int i = base + lane;
        pos += __popc(__ballot_sync(0xffffffffu, i < ms && mKf[i] < K));
      }
      const bool found = pos < ms && mKf[pos] == K;
      if (found && mW[pos] == w) continue;  // the same weight: no effect
      if (!found) {
        for (int hi = ms - 1; hi >= pos; hi -= 32) {
          const int i = hi - lane;
          int kv = 0, wv = 0;
          if (i >= pos) {
            kv = mKf[i];
            wv = mW[i];
          }
          __syncwarp();
          if (i >= pos) {
            mKf[i + 1] = kv;
            mW[i + 1] = wv;
          }
          __syncwarp();
        }
        ms++;
      }
      if (lane == 0) {
        mKf[pos] = K;
        mW[pos] = w;
      }
      __syncwarp();
      changed = 1;
      stale = true;
    }
  }
  if (stale) {
    sort_map(mKf, mW, ms, lKf, lW, lane);
    ls = ms;
  }
  if (lane == 0) {
    a.changed[t] = changed;
    a.parent[t] = parent;
    a.first[t] = first;
    a.mapN[t] = changed ? ms : 0;
    a.listN[t] = changed ? ls : 0;
  }
}

}  // namespace

struct b2s_covis : b2s::Stage {
  int maxKf, maxMp, maxObs, maxSlots, maxConn, maxBatch;
  Args a{};      // the scratch pointers; the rest are set per call
  Packed scr;    // scratch only the device touches
  Packed in;     // the problem
  Packed out;    // the small outputs, downloaded first, then the output areas of maxConn entries each
  Seg<int> mapOff, mapKf, mapW, listOff, listKf, listW, kfFlags, parentIn, mpBad, obsOff, obsKf, member, slotOff, slotMp;
  Seg<int> flag, outOff, memOff, changed, parent, first, mapN, listN, startN, afterN, pair, area[7];
  // n keyframes, B calls, M map and L list entries, nmp points with O observers, S slots
  void lay(size_t n, size_t B, size_t M, size_t L, size_t nmp, size_t O, size_t S) {
    in.clear();
    mapOff = in.add<int>(n + 1);
    mapKf = in.add<int>(M);
    mapW = in.add<int>(M);
    listOff = in.add<int>(n + 1);
    listKf = in.add<int>(L);
    listW = in.add<int>(L);
    kfFlags = in.add<int>(n);
    parentIn = in.add<int>(n);
    mpBad = in.add<int>(nmp);
    obsOff = in.add<int>(nmp + 1);
    obsKf = in.add<int>(O);
    member = in.add<int>(B);
    slotOff = in.add<int>(B + 1);
    slotMp = in.add<int>(S);
    out.clear();
    flag = out.add<int>(1);
    outOff = out.add<int>(n + 1);
    memOff = out.add<int>(B + 1);
    changed = out.add<int>(n);
    parent = out.add<int>(n);
    first = out.add<int>(n);
    mapN = out.add<int>(n);
    listN = out.add<int>(n);
    startN = out.add<int>(B);
    afterN = out.add<int>(B);
    pair = out.add<int>(B);
    for (Seg<int>& g : area) g = out.add<int>(maxConn);
  }
};

extern "C" int b2s_covis_create(int max_kf, int max_mp, int max_obs, int max_slots, int max_conn, int max_batch,
                                int device, b2s_covis** out) {
  if (!out || max_kf < 1 || max_mp < 0 || max_obs < 0 || max_slots < 0 || max_conn < 0 || max_batch < 1) {
    set_error("b2s_covis_create: bad argument (max_kf, max_batch >= 1; the others >= 0)");
    return B2S_ERR_BAD_ARG;
  }
  *out = nullptr;
  int rc = select_device(device);
  if (rc != B2S_OK) return rc;
  b2s_covis* h = new b2s_covis();
  h->maxKf = max_kf;
  h->maxMp = max_mp;
  h->maxObs = max_obs;
  h->maxSlots = max_slots;
  h->maxConn = max_conn;
  h->maxBatch = max_batch;
  const size_t K = max_kf, B = max_batch, C = max_conn, KB = K * B;
  Packed& scr = h->scr;
  const Seg<int> hist = scr.add<int>(KB), cntKf = scr.add<int>(KB), cntW = scr.add<int>(KB), strKf = scr.add<int>(KB),
                 strW = scr.add<int>(KB), evPos = scr.add<int>(KB), evK = scr.add<int>(KB), cntN = scr.add<int>(B),
                 strN = scr.add<int>(B), evCnt = scr.add<int>(K + 1), evStart = scr.add<int>(K + 1),
                 cur = scr.add<int>(K + 1), bound = scr.add<int>(K + 1);
  h->lay(K, B, C, C, max_mp, max_obs, max_slots);
  h->open(device);
  scr.reserve(h->error, false);
  h->in.reserve(h->error);
  h->out.reserve(h->error);
  cudaError_t e = h->error;
  if (e == cudaSuccess) e = cudaMemset(scr.dev(hist), 0, KB * 4);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    set_error("b2s_covis_create: %s", cudaGetErrorString(e));
    b2s_covis_destroy(h);
    return B2S_ERR_CUDA;
  }
  Args& a = h->a;
  a.hist = scr.dev(hist);
  a.cntKf = scr.dev(cntKf);
  a.cntW = scr.dev(cntW);
  a.strKf = scr.dev(strKf);
  a.strW = scr.dev(strW);
  a.evPos = scr.dev(evPos);
  a.evK = scr.dev(evK);
  a.cntN = scr.dev(cntN);
  a.strN = scr.dev(strN);
  a.evCnt = scr.dev(evCnt);
  a.evStart = scr.dev(evStart);
  a.cur = scr.dev(cur);
  a.bound = scr.dev(bound);
  a.maxConn = max_conn;
  *out = h;
  return B2S_OK;
}

extern "C" void b2s_covis_destroy(b2s_covis* h) {
  if (!h) return;
  h->close();
  delete h;
}

extern "C" float b2s_covis_last_ms(const b2s_covis* h) { return h ? h->lastMs : 0.f; }

extern "C" int b2s_update_connections(b2s_covis* h, const b2s_covis_problem* p, b2s_covis_result* r) {
  if (!h || !p || !r || p->batch < 1 || p->n_kf < 1 || p->n_mp < 0 || !p->kf_id || !p->map_off || !p->list_off ||
      !p->first_connection || !p->parent || !p->obs_off || !p->member || !p->slot_off ||
      (p->n_mp > 0 && !p->mp_bad) || !r->changed || !r->parent || !r->first_connection || !r->map_off ||
      !r->list_off || !r->child_pairs || !r->start_off || !r->after_off) {
    set_error("b2s_update_connections: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  const int n = p->n_kf, B = p->batch, nmp = p->n_mp;
  if (n > h->maxKf || nmp > h->maxMp || B > h->maxBatch) {
    set_error("b2s_update_connections: n_kf %d, n_mp %d or batch %d exceeds the handle's capacity", n, nmp, B);
    return B2S_ERR_CAPACITY;
  }
  const int64_t big = INT32_MAX;
  if (!csr_ok(p->map_off, n, big) || !csr_ok(p->list_off, n, big) || !csr_ok(p->obs_off, nmp, big) ||
      !csr_ok(p->slot_off, B, big)) {
    set_error("b2s_update_connections: an offset array is not a CSR");
    return B2S_ERR_BAD_ARG;
  }
  const int M = p->map_off[n], L = p->list_off[n], O = p->obs_off[nmp], S = p->slot_off[B];
  if (M > h->maxConn || L > h->maxConn || O > h->maxObs || S > h->maxSlots) {
    set_error("b2s_update_connections: %d map, %d list, %d observer or %d slot entries exceed the handle's capacity", M,
              L, O, S);
    return B2S_ERR_CAPACITY;
  }
  if ((M > 0 && (!p->map_kf || !p->map_w)) || (L > 0 && (!p->list_kf || !p->list_w)) || (O > 0 && !p->obs_kf) ||
      (S > 0 && !p->slot_mp)) {
    set_error("b2s_update_connections: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  for (int i = 1; i < n; i++)
    if (p->kf_id[i] <= p->kf_id[i - 1]) {
      set_error("b2s_update_connections: keyframe ids are not strictly ascending at %d", i);
      return B2S_ERR_BAD_ARG;
    }
  bool ok = entries_ok(p->map_off, p->map_kf, n, 0, n, true) && entries_ok(p->list_off, p->list_kf, n, 0, n, false) &&
            entries_ok(p->obs_off, p->obs_kf, nmp, 0, n, true) && entries_ok(p->slot_off, p->slot_mp, B, -1, nmp, false);
  for (int i = 0; ok && i < n; i++) ok = p->parent[i] >= -1 && p->parent[i] < n;
  for (int b = 0; ok && b < B; b++) ok = p->member[b] >= 0 && p->member[b] < n;
  if (!ok) {
    set_error("b2s_update_connections: an index is out of range, or a map or observer row is not strictly ascending");
    return B2S_ERR_BAD_ARG;
  }
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;

  // pack the problem: one upload
  h->lay(n, B, M, L, nmp, O, S);
  int rc = h->in.fit("b2s_update_connections");
  if (rc == B2S_OK) rc = h->out.fit("b2s_update_connections");
  if (rc != B2S_OK) return rc;
  Packed &in = h->in, &out = h->out;
  Args a = h->a;
  a.n = n;
  a.B = B;
  a.mapOff = in.stage(h->mapOff, p->map_off);
  a.mapKf = in.stage(h->mapKf, p->map_kf);
  a.mapW = in.stage(h->mapW, p->map_w);
  a.listOff = in.stage(h->listOff, p->list_off);
  a.listKf = in.stage(h->listKf, p->list_kf);
  a.listW = in.stage(h->listW, p->list_w);
  int* flags = in.host(h->kfFlags);
  for (int i = 0; i < n; i++) flags[i] = (p->first_connection[i] ? 1 : 0) | (p->kf_id[i] == 0 ? 2 : 0);
  a.kfFlags = in.dev(h->kfFlags);
  a.parentIn = in.stage(h->parentIn, p->parent);
  int* bad = in.host(h->mpBad);
  for (int i = 0; i < nmp; i++) bad[i] = p->mp_bad[i] ? 1 : 0;
  a.mpBad = in.dev(h->mpBad);
  a.obsOff = in.stage(h->obsOff, p->obs_off);
  a.obsKf = in.stage(h->obsKf, p->obs_kf);
  a.member = in.stage(h->member, p->member);
  a.slotOff = in.stage(h->slotOff, p->slot_off);
  a.slotMp = in.stage(h->slotMp, p->slot_mp);
  a.flag = out.dev(h->flag);
  a.outOff = out.dev(h->outOff);
  a.memOff = out.dev(h->memOff);
  a.changed = out.dev(h->changed);
  a.parent = out.dev(h->parent);
  a.first = out.dev(h->first);
  a.mapN = out.dev(h->mapN);
  a.listN = out.dev(h->listN);
  a.startN = out.dev(h->startN);
  a.afterN = out.dev(h->afterN);
  a.pair = out.dev(h->pair);
  int** areas[7] = {&a.oMapKf, &a.oMapW, &a.oListKf, &a.oListW, &a.oStartKf, &a.oAfterKf, &a.oAfterW};
  for (int i = 0; i < 7; i++) *areas[i] = out.dev(h->area[i]);

  if ((rc = h->begin()) != B2S_OK) return rc;
  if ((rc = in.upload(s)) != B2S_OK) return rc;
  k_covis_count<<<B, kCountThreads, 0, s>>>(a);
  k_covis_group<<<1, kGroupThreads, 0, s>>>(a);
  k_covis_replay<<<div_up(n, kReplayWarps), kReplayWarps * 32, 0, s>>>(a);
  B2S_CUDA(cudaGetLastError());
  // the small outputs first: they size the areas
  if ((rc = out.download(s, 0, h->pair.end())) != B2S_OK) return rc;
  B2S_CUDA(cudaStreamSynchronize(s));
  const int *outOff = out.host(h->outOff), *memOff = out.host(h->memOff);
  if (*out.host(h->flag)) {
    set_error("b2s_update_connections: the outputs need %d and %d entries, beyond the handle's max_conn %d",
              outOff[n], memOff[B], h->maxConn);
    return B2S_ERR_CAPACITY;
  }
  const int nOut = outOff[n], nMem = memOff[B];
  for (int i = 0; i < 7; i++) {
    const Seg<int>& g = h->area[i];
    if ((rc = out.download(s, g.off, g.off + (size_t)(i < 4 ? nOut : nMem) * 4)) != B2S_OK) return rc;
  }
  if ((rc = h->finish()) != B2S_OK) return rc;

  const int *changed = out.host(h->changed), *parent = out.host(h->parent), *first = out.host(h->first),
            *mapN = out.host(h->mapN), *listN = out.host(h->listN), *startN = out.host(h->startN),
            *afterN = out.host(h->afterN), *pair = out.host(h->pair);
  int64_t needMap = 0, needList = 0, needStart = 0, needAfter = 0;
  for (int t = 0; t < n; t++) {
    needMap += mapN[t];
    needList += listN[t];
  }
  for (int b = 0; b < B; b++) {
    needStart += startN[b];
    needAfter += afterN[b];
  }
  const bool fits =
      needMap <= r->map_cap && needList <= r->list_cap && needStart <= r->start_cap && needAfter <= r->after_cap;
  if (fits && ((needMap && (!r->map_kf || !r->map_w)) || (needList && (!r->list_kf || !r->list_w)) ||
               (needStart && !r->start_kf) || (needAfter && (!r->after_kf || !r->after_w)))) {
    set_error("b2s_update_connections: bad argument (a null output array)");
    return B2S_ERR_BAD_ARG;
  }
  r->map_need = (int)needMap;
  r->list_need = (int)needList;
  r->start_need = (int)needStart;
  r->after_need = (int)needAfter;
  if (!fits) {
    set_error("b2s_update_connections: the outputs need %lld / %lld / %lld / %lld entries (map / list / start / after)",
              (long long)needMap, (long long)needList, (long long)needStart, (long long)needAfter);
    return B2S_ERR_CAPACITY;
  }
  const int* A[7];
  for (int i = 0; i < 7; i++) A[i] = out.host(h->area[i]);
  int cm = 0, cl = 0;
  r->map_off[0] = r->list_off[0] = 0;
  for (int t = 0; t < n; t++) {
    r->changed[t] = (uint8_t)changed[t];
    r->parent[t] = parent[t];
    r->first_connection[t] = (uint8_t)first[t];
    if (mapN[t]) {
      memcpy(r->map_kf + cm, A[0] + outOff[t], (size_t)mapN[t] * 4);
      memcpy(r->map_w + cm, A[1] + outOff[t], (size_t)mapN[t] * 4);
    }
    if (listN[t]) {
      memcpy(r->list_kf + cl, A[2] + outOff[t], (size_t)listN[t] * 4);
      memcpy(r->list_w + cl, A[3] + outOff[t], (size_t)listN[t] * 4);
    }
    cm += mapN[t];
    cl += listN[t];
    r->map_off[t + 1] = cm;
    r->list_off[t + 1] = cl;
  }
  int cs = 0, ca = 0, np = 0;
  r->start_off[0] = r->after_off[0] = 0;
  for (int b = 0; b < B; b++) {
    if (startN[b]) memcpy(r->start_kf + cs, A[4] + memOff[b], (size_t)startN[b] * 4);
    if (afterN[b]) {
      memcpy(r->after_kf + ca, A[5] + memOff[b], (size_t)afterN[b] * 4);
      memcpy(r->after_w + ca, A[6] + memOff[b], (size_t)afterN[b] * 4);
    }
    cs += startN[b];
    ca += afterN[b];
    r->start_off[b + 1] = cs;
    r->after_off[b + 1] = ca;
    if (pair[b] >= 0) {
      r->child_pairs[2 * np] = pair[b];
      r->child_pairs[2 * np + 1] = p->member[b];
      np++;
    }
  }
  r->n_pairs = np;
  return B2S_OK;
}
