// culling.cu — LocalMapping::KeyFrameCulling (src/LocalMapping.cc:873-956) for a batch of independent local maps, with
// the point-side effects of the KeyFrame::SetBadFlag (src/KeyFrame.cc:599-722) it calls: MapPoint::EraseObservation
// (src/MapPoint.cc:170-200) on every non-NULL slot of the culled keyframe and, where nObs drops to 2 or less,
// MapPoint::SetBadFlag (:217-234) with its EraseMapPointMatch(idx) on the remaining observers.  Integer work plus one
// double multiply per keyframe.
//
// Two launches, no host synchronisation between them:
//   k_cull_count  one CTA per (problem, local keyframe): nMPs and nRedundantObservations (:884-949) from the entry
//                 state, the slots strided over the CTA and reduced with warp sums.
//   k_cull_walk   one CTA per problem: the verdicts in list order.  Until the first cull that changes the state, the
//                 precomputed counts are the counts the reference sees; after it, each later keyframe is recounted from
//                 the current state.  A cull's effects run in parallel over its slots.  Within one cull they do not
//                 depend on the order: each point's observation of the culled keyframe is claimed once (atomicExch on
//                 its alive flag, so a duplicate slot does nothing, as the reference's second EraseObservation does),
//                 only the claiming thread touches that point's nObs and observer row, and slot nulling only writes
//                 -1.  The culled keyframe's own slots are never nulled by its own cull: its observation is gone before
//                 any of its points turns bad.
#include <vector>

#include "common.cuh"

using namespace b2s;

namespace {

constexpr int kThreads = 128;
constexpr int kWarps = kThreads / 32;

struct Desc {  // one problem's extent and its bases in the packed arrays
  int nkf, nmp, nloc, kf, mp, obs, obsOff, loc, slotOff, slot, mono;
};

struct Args {
  const Desc* desc;
  const int* locProb;  // the problem of each local keyframe over the batch
  // input, packed over the batch; row offsets (obsOff, slotOff) are relative to their problem's base
  const int* kfFlags;  // bit 0: mnId == 0, bit 1: mbNotErase
  const float* thDepth;
  const int *mpBad, *mpNobs, *obsOff, *obsKf, *obsIdx, *obsOct, *obsStereo;
  const int *localKf, *slotOff, *slotMp, *slotOct;
  const float* slotDepth;
  // scratch
  int *cntM, *cntR, *localPos;
  // outputs (one area, downloaded in one copy); bad / nobs / alive / slot are the walk's working state
  int *verdict, *nM, *nR, *bad, *nobs, *alive, *slot, *nCulled;
};

__device__ int2 block_sum2(int x, int y) {
  __shared__ int sx[kWarps], sy[kWarps];
  x = warp_reduce_sum(x);
  y = warp_reduce_sum(y);
  if ((threadIdx.x & 31) == 0) {
    sx[threadIdx.x >> 5] = x;
    sy[threadIdx.x >> 5] = y;
  }
  __syncthreads();
  int2 r = make_int2(0, 0);
#pragma unroll
  for (int i = 0; i < kWarps; i++) {
    r.x += sx[i];
    r.y += sy[i];
  }
  __syncthreads();
  return r;
}

// (nMPs, nRedundantObservations) of local keyframe l of problem d (:884-949) on the state (slot, bad, nobs, alive);
// alive == nullptr: every observation is in place (the entry state).  The observer scan stops at 3, so its order does
// not matter.
__device__ int2 count_local(const Args& a, const Desc& d, int l, const int* slot, const int* bad, const int* nobs,
                            const int* alive) {
  const int k = a.localKf[d.loc + l];
  const float th = a.thDepth[d.kf + k];
  const int* off = a.obsOff + d.obsOff;
  const int s0 = a.slotOff[d.slotOff + l], s1 = a.slotOff[d.slotOff + l + 1];
  int nm = 0, nr = 0;
  for (int s = d.slot + s0 + threadIdx.x; s < d.slot + s1; s += kThreads) {
    const int mp = slot[s];
    if (mp < 0 || bad[d.mp + mp]) continue;
    if (!d.mono) {
      const float z = a.slotDepth[s];
      if (z > th || z < 0.f) continue;  // :911; a NaN depth passes
    }
    nm++;
    if (nobs[d.mp + mp] > 3) {  // :917
      const long long lvl = (long long)a.slotOct[s] + 1;
      int c = 0;
      for (int o = d.obs + off[mp]; o < d.obs + off[mp + 1]; o++) {
        if ((alive && !alive[o]) || a.obsKf[o] == k) continue;
        if (a.obsOct[o] <= lvl && ++c >= 3) break;  // :933-938
      }
      nr += c >= 3;
    }
  }
  return block_sum2(nm, nr);
}

__global__ void __launch_bounds__(kThreads) k_cull_count(Args a) {
  const int g = blockIdx.x;
  const Desc d = a.desc[a.locProb[g]];
  if (a.kfFlags[d.kf + a.localKf[g]] & 1) return;  // mnId 0: never counted
  const int2 c = count_local(a, d, g - d.loc, a.slotMp, a.mpBad, a.mpNobs, nullptr);
  if (threadIdx.x == 0) {
    a.cntM[g] = c.x;
    a.cntR[g] = c.y;
  }
}

__global__ void __launch_bounds__(kThreads) k_cull_walk(Args a) {
  const int b = blockIdx.x, tid = threadIdx.x;
  const Desc d = a.desc[b];
  const int* off = a.obsOff + d.obsOff;
  const int* sOff = a.slotOff + d.slotOff;
  const int nObs = off[d.nmp], nSlots = sOff[d.nloc];
  for (int i = tid; i < d.nmp; i += kThreads) {
    a.bad[d.mp + i] = a.mpBad[d.mp + i];
    a.nobs[d.mp + i] = a.mpNobs[d.mp + i];
  }
  for (int o = tid; o < nObs; o += kThreads) a.alive[d.obs + o] = 1;
  for (int s = tid; s < nSlots; s += kThreads) a.slot[d.slot + s] = a.slotMp[d.slot + s];
  for (int k = tid; k < d.nkf; k += kThreads) a.localPos[d.kf + k] = -1;
  __syncthreads();
  for (int l = tid; l < d.nloc; l += kThreads) a.localPos[d.kf + a.localKf[d.loc + l]] = l;
  __syncthreads();

  bool dirty = false;  // uniform over the CTA: a cull has changed the state the precomputed counts came from
  int culled = 0;
  for (int l = 0; l < d.nloc; l++) {
    const int g = d.loc + l, k = a.localKf[g], fl = a.kfFlags[d.kf + k];
    if (fl & 1) {  // :887
      if (tid == 0) {
        a.verdict[g] = B2S_CULL_SKIPPED;
        a.nM[g] = a.nR[g] = 0;
      }
      continue;
    }
    const int2 c = dirty ? count_local(a, d, l, a.slot, a.bad, a.nobs, a.alive) : make_int2(a.cntM[g], a.cntR[g]);
    const bool redundant = (double)c.y > __dmul_rn(0.9, (double)c.x);  // :952, an int against a double
    const int v = !redundant ? B2S_CULL_KEPT : (fl & 2) ? B2S_CULL_DEFERRED : B2S_CULL_CULLED;
    if (tid == 0) {
      a.verdict[g] = v;
      a.nM[g] = c.x;
      a.nR[g] = c.y;
    }
    if (v != B2S_CULL_CULLED) continue;
    culled++;
    // KeyFrame::SetBadFlag (:619-621): EraseObservation(this) on every non-NULL slot
    bool changed = false;
    for (int s = d.slot + sOff[l] + tid; s < d.slot + sOff[l + 1]; s += kThreads) {
      const int mp = a.slot[s];
      if (mp < 0) continue;
      int lo = d.obs + off[mp], hi = d.obs + off[mp + 1];  // the observer row is ascending: find k
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a.obsKf[mid] < k)
          lo = mid + 1;
        else
          hi = mid;
      }
      if (lo == d.obs + off[mp + 1] || a.obsKf[lo] != k) continue;  // not an observer: nothing happens
      if (atomicExch(&a.alive[lo], 0) == 0) continue;              // erased already (a duplicate slot)
      changed = true;
      const int n = a.nobs[d.mp + mp] - (a.obsStereo[lo] ? 2 : 1);
      a.nobs[d.mp + mp] = n;
      if (n <= 2) {  // MapPoint::SetBadFlag: the remaining observers lose slot idx, whatever point it holds
        a.bad[d.mp + mp] = 1;
        for (int o = d.obs + off[mp]; o < d.obs + off[mp + 1]; o++) {
          if (!a.alive[o]) continue;
          a.alive[o] = 0;
          const int p = a.localPos[d.kf + a.obsKf[o]];
          if (p >= 0) a.slot[d.slot + sOff[p] + a.obsIdx[o]] = -1;
        }
      }
    }
    dirty = __syncthreads_or(changed) || dirty;
  }
  if (tid == 0) a.nCulled[b] = culled;
}

}  // namespace

struct b2s_culling : b2s::Stage {
  int maxKf, maxMp, maxObs, maxLocal, maxSlots, maxBatch;
  Packed in, out;  // the packed problems; outputs, then scratch
};

extern "C" int b2s_culling_create(int max_kf, int max_mp, int max_obs, int max_local, int max_slots, int max_batch,
                                  int device, b2s_culling** out) {
  if (!out || max_kf < 1 || max_mp < 0 || max_obs < 0 || max_local < 0 || max_slots < 0 || max_batch < 1) {
    set_error("b2s_culling_create: bad argument (max_kf, max_batch >= 1; the others >= 0)");
    return B2S_ERR_BAD_ARG;
  }
  *out = nullptr;
  int rc = select_device(device);
  if (rc != B2S_OK) return rc;
  b2s_culling* h = new b2s_culling();
  h->maxKf = max_kf;
  h->maxMp = max_mp;
  h->maxObs = max_obs;
  h->maxLocal = max_local;
  h->maxSlots = max_slots;
  h->maxBatch = max_batch;
  h->open(device);
  if (h->error != cudaSuccess) {
    set_error("b2s_culling_create: %s", cudaGetErrorString(h->error));
    b2s_culling_destroy(h);
    return B2S_ERR_CUDA;
  }
  *out = h;
  return B2S_OK;
}

extern "C" void b2s_culling_destroy(b2s_culling* h) {
  if (!h) return;
  h->close();
  delete h;
}

extern "C" float b2s_culling_last_ms(const b2s_culling* h) { return h ? h->lastMs : 0.f; }

namespace {

// B2S_OK, or the error of the first invalid problem (the message set)
int check_problem(const b2s_culling* h, int b, const b2s_culling_problem& p, const b2s_culling_result& r) {
  if (p.n_kf < 0 || p.n_mp < 0 || p.n_local < 0 || !p.obs_off || !p.slot_off ||
      (p.n_kf > 0 && (!p.kf_id || !p.not_erase || !p.th_depth)) || (p.n_mp > 0 && (!p.mp_bad || !p.mp_nobs)) ||
      (p.n_local > 0 && !p.local_kf) || (p.n_local > 0 && (!r.verdict || !r.n_mps || !r.n_redundant)) ||
      (p.n_mp > 0 && (!r.mp_bad || !r.mp_nobs))) {
    set_error("b2s_keyframe_culling: problem %d: bad argument (a null array or a negative count)", b);
    return B2S_ERR_BAD_ARG;
  }
  if (p.n_kf > h->maxKf || p.n_mp > h->maxMp || p.n_local > h->maxLocal) {
    set_error("b2s_keyframe_culling: problem %d: n_kf %d, n_mp %d or n_local %d exceeds the handle's capacity", b,
              p.n_kf, p.n_mp, p.n_local);
    return B2S_ERR_CAPACITY;
  }
  if (!csr_ok(p.obs_off, p.n_mp, INT32_MAX) || !csr_ok(p.slot_off, p.n_local, INT32_MAX)) {
    set_error("b2s_keyframe_culling: problem %d: an offset array is not a CSR", b);
    return B2S_ERR_BAD_ARG;
  }
  const int O = p.obs_off[p.n_mp], S = p.slot_off[p.n_local];
  if (O > h->maxObs || S > h->maxSlots) {
    set_error("b2s_keyframe_culling: problem %d: %d observations or %d slots exceed the handle's capacity", b, O, S);
    return B2S_ERR_CAPACITY;
  }
  if ((O > 0 && (!p.obs_kf || !p.obs_idx || !p.obs_octave || !p.obs_stereo || !r.obs_alive)) ||
      (S > 0 && (!p.slot_mp || !p.slot_octave || !r.slot_mp)) || (S > 0 && !p.monocular && !p.slot_depth)) {
    set_error("b2s_keyframe_culling: problem %d: bad argument (a null array)", b);
    return B2S_ERR_BAD_ARG;
  }
  bool ok = entries_ok(p.obs_off, p.obs_kf, p.n_mp, 0, p.n_kf, true) &&
            entries_ok(p.slot_off, p.slot_mp, p.n_local, -1, p.n_mp, false);
  std::vector<int> pos((size_t)p.n_kf, -1);
  for (int l = 0; ok && l < p.n_local; l++) {
    const int k = p.local_kf[l];
    ok = k >= 0 && k < p.n_kf && pos[(size_t)k] < 0;
    if (ok) pos[(size_t)k] = l;
  }
  // EraseMapPointMatch(idx) on a local observer must land inside its slot row
  for (int o = 0; ok && o < O; o++) {
    const int l = pos[(size_t)p.obs_kf[o]];
    ok = p.obs_idx[o] >= 0 && (l < 0 || p.obs_idx[o] < p.slot_off[l + 1] - p.slot_off[l]);
  }
  if (!ok) {
    set_error("b2s_keyframe_culling: problem %d: an index is out of range, an observer row is not strictly ascending, "
              "a local keyframe is repeated, or an obs_idx lies outside its keyframe's slots", b);
    return B2S_ERR_BAD_ARG;
  }
  return B2S_OK;
}

}  // namespace

extern "C" int b2s_keyframe_culling(b2s_culling* h, int batch, const b2s_culling_problem* p, b2s_culling_result* r) {
  if (!h || !p || !r || batch < 1) {
    set_error("b2s_keyframe_culling: bad argument");
    return B2S_ERR_BAD_ARG;
  }
  if (batch > h->maxBatch) {
    set_error("b2s_keyframe_culling: batch %d exceeds the handle's max_batch %d", batch, h->maxBatch);
    return B2S_ERR_CAPACITY;
  }
  for (int b = 0; b < batch; b++) {
    const int rc = check_problem(h, b, p[b], r[b]);
    if (rc != B2S_OK) return rc;
  }
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;

  // extents and bases
  std::vector<Desc> desc((size_t)batch);
  size_t K = 0, M = 0, O = 0, L = 0, S = 0;
  for (int b = 0; b < batch; b++) {
    const b2s_culling_problem& q = p[b];
    Desc& d = desc[(size_t)b];
    d.nkf = q.n_kf;
    d.nmp = q.n_mp;
    d.nloc = q.n_local;
    d.kf = (int)K;
    d.mp = (int)M;
    d.obs = (int)O;
    d.obsOff = (int)(M + b);
    d.loc = (int)L;
    d.slotOff = (int)(L + b);
    d.slot = (int)S;
    d.mono = q.monocular != 0;
    K += q.n_kf;
    M += q.n_mp;
    O += q.obs_off[q.n_mp];
    L += q.n_local;
    S += q.slot_off[q.n_local];
  }
  if (K + M + O + L + S + 2 * (size_t)batch >= (size_t)INT32_MAX / 4) {
    set_error("b2s_keyframe_culling: the batch is too large for one call");
    return B2S_ERR_CAPACITY;
  }
  Packed &in = h->in, &out = h->out;
  in.clear();
  const Seg<Desc> gDesc = in.add<Desc>(batch);
  const Seg<int> gLocProb = in.add<int>(L), gFlags = in.add<int>(K);
  const Seg<float> gTh = in.add<float>(K);
  const Seg<int> gBad = in.add<int>(M), gNobs = in.add<int>(M), gObsOff = in.add<int>(M + batch),
                 gObsKf = in.add<int>(O), gObsIdx = in.add<int>(O), gObsOct = in.add<int>(O), gObsSt = in.add<int>(O),
                 gLocal = in.add<int>(L), gSlotOff = in.add<int>(L + batch), gSlotMp = in.add<int>(S),
                 gSlotOct = in.add<int>(S);
  const Seg<float> gDepth = in.add<float>(S);
  out.clear();
  const Seg<int> gVerdict = out.add<int>(L), gNM = out.add<int>(L), gNR = out.add<int>(L), gBadOut = out.add<int>(M),
                 gNobsOut = out.add<int>(M), gAlive = out.add<int>(O), gSlot = out.add<int>(S),
                 gCulled = out.add<int>(batch), gCntM = out.add<int>(L), gCntR = out.add<int>(L),
                 gLocalPos = out.add<int>(K);
  int rc = in.fit("b2s_keyframe_culling");
  if (rc == B2S_OK) rc = out.fit("b2s_keyframe_culling");
  if (rc != B2S_OK) return rc;

  // pack: one upload
  memcpy(in.host(gDesc), desc.data(), (size_t)batch * sizeof(Desc));
  for (int b = 0; b < batch; b++) {
    const b2s_culling_problem& pb = p[b];
    const Desc& d = desc[(size_t)b];
    const int nO = pb.obs_off[pb.n_mp], nS = pb.slot_off[pb.n_local];
    for (int l = 0; l < d.nloc; l++) in.host(gLocProb)[d.loc + l] = b;
    for (int k = 0; k < d.nkf; k++) in.host(gFlags)[d.kf + k] = (pb.kf_id[k] == 0 ? 1 : 0) | (pb.not_erase[k] ? 2 : 0);
    if (d.nkf) memcpy(in.host(gTh) + d.kf, pb.th_depth, (size_t)d.nkf * 4);
    for (int m = 0; m < d.nmp; m++) in.host(gBad)[d.mp + m] = pb.mp_bad[m] ? 1 : 0;
    if (d.nmp) memcpy(in.host(gNobs) + d.mp, pb.mp_nobs, (size_t)d.nmp * 4);
    memcpy(in.host(gObsOff) + d.obsOff, pb.obs_off, (size_t)(d.nmp + 1) * 4);
    if (nO) {
      memcpy(in.host(gObsKf) + d.obs, pb.obs_kf, (size_t)nO * 4);
      memcpy(in.host(gObsIdx) + d.obs, pb.obs_idx, (size_t)nO * 4);
      memcpy(in.host(gObsOct) + d.obs, pb.obs_octave, (size_t)nO * 4);
      for (int i = 0; i < nO; i++) in.host(gObsSt)[d.obs + i] = pb.obs_stereo[i] ? 1 : 0;
    }
    if (d.nloc) memcpy(in.host(gLocal) + d.loc, pb.local_kf, (size_t)d.nloc * 4);
    memcpy(in.host(gSlotOff) + d.slotOff, pb.slot_off, (size_t)(d.nloc + 1) * 4);
    if (nS) {
      memcpy(in.host(gSlotMp) + d.slot, pb.slot_mp, (size_t)nS * 4);
      memcpy(in.host(gSlotOct) + d.slot, pb.slot_octave, (size_t)nS * 4);
      if (pb.slot_depth)
        memcpy(in.host(gDepth) + d.slot, pb.slot_depth, (size_t)nS * 4);
      else
        memset(in.host(gDepth) + d.slot, 0, (size_t)nS * 4);
    }
  }
  const Args a = {in.dev(gDesc),    in.dev(gLocProb),  in.dev(gFlags),   in.dev(gTh),      in.dev(gBad),
                  in.dev(gNobs),    in.dev(gObsOff),   in.dev(gObsKf),   in.dev(gObsIdx),  in.dev(gObsOct),
                  in.dev(gObsSt),   in.dev(gLocal),    in.dev(gSlotOff), in.dev(gSlotMp),  in.dev(gSlotOct),
                  in.dev(gDepth),   out.dev(gCntM),    out.dev(gCntR),   out.dev(gLocalPos), out.dev(gVerdict),
                  out.dev(gNM),     out.dev(gNR),      out.dev(gBadOut), out.dev(gNobsOut), out.dev(gAlive),
                  out.dev(gSlot),   out.dev(gCulled)};

  if ((rc = h->begin()) != B2S_OK) return rc;
  if ((rc = in.upload(s)) != B2S_OK) return rc;
  if (L) k_cull_count<<<(unsigned)L, kThreads, 0, s>>>(a);
  k_cull_walk<<<batch, kThreads, 0, s>>>(a);
  B2S_CUDA(cudaGetLastError());
  if ((rc = out.download(s, 0, gCulled.end())) != B2S_OK) return rc;  // not the scratch
  if ((rc = h->finish()) != B2S_OK) return rc;

  const int *verdict = out.host(gVerdict), *nM = out.host(gNM), *nR = out.host(gNR), *bad = out.host(gBadOut),
            *nobs = out.host(gNobsOut), *alive = out.host(gAlive), *slot = out.host(gSlot),
            *nCulled = out.host(gCulled);
  for (int b = 0; b < batch; b++) {
    const Desc& d = desc[(size_t)b];
    b2s_culling_result& rb = r[b];
    const int nO = p[b].obs_off[d.nmp], nS = p[b].slot_off[d.nloc];
    for (int l = 0; l < d.nloc; l++) rb.verdict[l] = (uint8_t)verdict[d.loc + l];
    if (d.nloc) {
      memcpy(rb.n_mps, nM + d.loc, (size_t)d.nloc * 4);
      memcpy(rb.n_redundant, nR + d.loc, (size_t)d.nloc * 4);
    }
    for (int m = 0; m < d.nmp; m++) rb.mp_bad[m] = (uint8_t)bad[d.mp + m];
    if (d.nmp) memcpy(rb.mp_nobs, nobs + d.mp, (size_t)d.nmp * 4);
    for (int i = 0; i < nO; i++) rb.obs_alive[i] = (uint8_t)alive[d.obs + i];
    if (nS) memcpy(rb.slot_mp, slot + d.slot, (size_t)nS * 4);
    rb.n_culled = nCulled[b];
  }
  return B2S_OK;
}
