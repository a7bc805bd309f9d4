// mappoint.cu — the per-point map refreshes on the matcher handle:
//   b2s_update_normal_and_depth  MapPoint::UpdateNormalAndDepth (src/MapPoint.cc:477-521) for a batch of points
//   b2s_process_new_keyframe     the association loop of LocalMapping::ProcessNewKeyFrame (src/LocalMapping.cc:217-249)
//                                and LocalMapping::MapPointCulling (:261-308) for a batch of independent problems
//
// Two kernels, no host synchronisation between them:
//   k_kfi_list   one CTA per problem: the association and the culling as parallel passes.  The association's first-slot
//                rule is an atomicMin per point, its appends a stable block-scan compaction in slot order; the culling's
//                verdicts come from the state after the association (a SetBadFlag changes no input of another point's
//                verdict), a later entry of a point an earlier entry set bad becomes B2S_KFI_BAD (first occurrence by
//                atomicMin), and the SetBadFlag effects run after every verdict is taken.
//   k_mp_point   one warp per point: UpdateNormalAndDepth on one lane, serially in observer order, so the float result
//                does not depend on the launch shape; then ComputeDistinctiveDescriptors on the warp (distinctive.cuh).
//                The standalone entry runs it alone.
// The float arithmetic is written with explicit round-to-nearest intrinsics (and the file is built with --fmad=false):
// the OpenCV forms it restates are listed in include/b200slam.h and DESIGN.md §7.
#include <vector>

#include "common.cuh"
#include "distinctive.cuh"
#include "matcher.cuh"

using namespace b2s;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

struct Desc {  // one problem's extent and its bases in the packed arrays
  int nkf, nmp, nslot, nrec, kf, mp, obs, obsOff, slot, rec, list, sf, nlev, cur, curId, mono;
};

struct Args {
  const Desc* desc;
  const int* mpProb;  // the problem of each point over the batch
  // input, packed over the batch; obsOff rows are relative to their problem's base
  const float *kfC, *mpPos, *sf;
  const int *kfBad, *slotMp, *slotSt, *mpBad, *mpRef, *mpNobs, *mpFound, *mpVis, *mpFirst, *obsOff, *obsKf, *obsIdx,
      *obsOct, *recent;
  const uint8_t *obsDesc, *slotDesc;
  // outputs (one area, downloaded in one copy)
  int *nobs, *bad, *added, *alive, *updated, *descPos, *slot, *list, *verdict, *nList, *nCulled;
  float *normal, *minD, *maxD;
  // scratch
  int *firstSlot, *firstEntry, *gather, *gatherPos;
};

// exclusive block scan of one flag per thread; *total: the sum over the block
__device__ int block_excl_scan(int x, int* total) {
  __shared__ int sw[kWarps];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int incl = warp_incl_scan(x, lane);
  if (lane == 31) sw[w] = incl;
  __syncthreads();
  int before = 0, sum = 0;
#pragma unroll
  for (int i = 0; i < kWarps; i++) {
    before += i < w ? sw[i] : 0;
    sum += sw[i];
  }
  __syncthreads();
  *total = sum;
  return before + incl - x;
}

// the position of keyframe k in point m's observer row (absolute), or -1
__device__ int find_obs(const Args& a, const Desc& d, int m, int k) {
  const int* off = a.obsOff + d.obsOff;
  int lo = d.obs + off[m], hi = d.obs + off[m + 1];
  const int end = hi;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a.obsKf[mid] < k)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo < end && a.obsKf[lo] == k ? lo : -1;
}

// MapPointCulling's rules (:276-306) on the state after the association
__device__ int verdict_of(const Args& a, const Desc& d, int g) {
  if (a.bad[g]) return B2S_KFI_BAD;
  const float ratio = __fdiv_rn(__int2float_rn(a.mpFound[g]), __int2float_rn(a.mpVis[g]));  // GetFoundRatio
  if (ratio < 0.25f) return B2S_KFI_CULLED_RATIO;                                            // NaN / inf: no
  const int age = (int)((unsigned)d.curId - (unsigned)a.mpFirst[g]);                        // (int)a - (int)b, wrapping
  if (age >= 2 && a.nobs[g] <= (d.mono ? 2 : 3)) return B2S_KFI_CULLED_OBS;
  return age >= 3 ? B2S_KFI_RETIRED : B2S_KFI_KEPT;
}

__device__ __forceinline__ bool culls(int v) { return v == B2S_KFI_CULLED_RATIO || v == B2S_KFI_CULLED_OBS; }

__global__ void __launch_bounds__(kThreads) k_kfi_list(Args a) {
  const int tid = threadIdx.x;
  const Desc d = a.desc[blockIdx.x];
  const int* off = a.obsOff + d.obsOff;
  for (int m = tid; m < d.nmp; m += kThreads) {
    const int g = d.mp + m;
    a.bad[g] = a.mpBad[g];
    a.nobs[g] = a.mpNobs[g];
    a.added[g] = -1;
    a.firstSlot[g] = a.firstEntry[g] = INT_MAX;
  }
  for (int o = tid; o < off[d.nmp]; o += kThreads) a.alive[d.obs + o] = 1;
  for (int s = tid; s < d.nslot; s += kThreads) a.slot[d.slot + s] = a.slotMp[d.slot + s];
  __syncthreads();
  for (int s = tid; s < d.nslot; s += kThreads) {
    const int m = a.slotMp[d.slot + s];
    if (m >= 0 && !a.mpBad[d.mp + m]) atomicMin(&a.firstSlot[d.mp + m], s);
  }
  __syncthreads();
  // the association (:222-247): the first slot of a point that does not list cur adds the observation, every other
  // slot of a good point appends it to the recent list
  int appended = 0;
  for (int base = 0; base < d.nslot; base += kThreads) {
    const int s = base + tid;
    int app = 0, m = -1;
    if (s < d.nslot) {
      m = a.slotMp[d.slot + s];
      if (m >= 0 && !a.mpBad[d.mp + m]) {
        if (a.firstSlot[d.mp + m] == s && find_obs(a, d, m, d.cur) < 0) {
          a.added[d.mp + m] = s;
          a.nobs[d.mp + m] += a.slotSt[d.slot + s] ? 2 : 1;
        } else {
          app = 1;
        }
      }
    }
    int total;
    const int pos = block_excl_scan(app, &total);
    if (app) a.list[d.list + d.nrec + appended + pos] = m;
    appended += total;
  }
  for (int e = tid; e < d.nrec; e += kThreads) a.list[d.list + e] = a.recent[d.rec + e];
  const int nList = d.nrec + appended;
  __syncthreads();
  for (int e = tid; e < nList; e += kThreads) atomicMin(&a.firstEntry[d.mp + a.list[d.list + e]], e);
  __syncthreads();
  // the culling (:276-306): verdicts from the state after the association
  int nCulled = 0;
  for (int e = tid; e < nList; e += kThreads) {
    const int g = d.mp + a.list[d.list + e];
    int v = verdict_of(a, d, g);
    if (culls(v) && a.firstEntry[g] != e) v = B2S_KFI_BAD;  // an earlier entry set it bad
    a.verdict[d.list + e] = v;
    nCulled += culls(v);
  }
  __syncthreads();  // every verdict reads the state after the association before any SetBadFlag writes
  // MapPoint::SetBadFlag (:217-234): mbBad, the observations cleared, EraseMapPointMatch(idx) on each observer (here the
  // current keyframe's slot; each point is set bad once, and the slot writes are all -1)
  for (int e = tid; e < nList; e += kThreads) {
    if (!culls(a.verdict[d.list + e])) continue;
    const int m = a.list[d.list + e], g = d.mp + m;
    a.bad[g] = 1;
    for (int o = d.obs + off[m]; o < d.obs + off[m + 1]; o++) {
      a.alive[o] = 0;
      if (a.obsKf[o] == d.cur) a.slot[d.slot + a.obsIdx[o]] = -1;
    }
    if (a.added[g] >= 0) a.slot[d.slot + a.added[g]] = -1;
  }
  int sum;
  block_excl_scan(nCulled, &sum);
  if (tid == 0) {
    a.nList[blockIdx.x] = nList;
    a.nCulled[blockIdx.x] = sum;
  }
}

// cv::norm of a float 3 x 1 column: the squares summed in double in order, (x^2 + y^2) + z^2 (a 1 x 3 row takes two
// lanes instead; both pinned against cv2.norm)
__device__ __forceinline__ double norm3(float x, float y, float z) {
  const double X = x, Y = y, Z = z;
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(X, X), __dmul_rn(Y, Y)), __dmul_rn(Z, Z)));
}

// One warp per point.  kInsert: b2s_process_new_keyframe (the point is refreshed where the association added the
// current keyframe's observation, which takes the keyframe's table position in the row); otherwise
// b2s_update_normal_and_depth (every good, observed point; the one problem's bases are 0).
template <bool kInsert>
__global__ void __launch_bounds__(kThreads) k_mp_point(Args a, int nPoints) {
  __shared__ int hist[kWarps][264];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int g = blockIdx.x * kWarps + wid;
  if (g >= nPoints) return;
  const Desc d = a.desc[kInsert ? a.mpProb[g] : 0];
  const int m = g - d.mp;
  const int* off = a.obsOff + d.obsOff;
  const int o0 = d.obs + off[m], nIn = off[m + 1] - off[m];
  const int s = kInsert ? a.added[g] : -1;
  const bool refresh = kInsert ? s >= 0 : !a.mpBad[g] && nIn > 0;
  if (!refresh) {
    if (lane == 0) {
      a.updated[g] = 0;
      if (kInsert) a.descPos[g] = -1;
    }
    return;
  }
  // the merged row: the entry row with the current keyframe inserted at its table position
  int ins = nIn;
  if (kInsert)
    for (int j = 0; j < nIn; j++)
      if (a.obsKf[o0 + j] > d.cur) {
        ins = j;
        break;
      }
  const int n = kInsert ? nIn + 1 : nIn;
  auto kfAt = [&](int j) { return !kInsert ? a.obsKf[o0 + j] : j < ins ? a.obsKf[o0 + j] : j == ins ? d.cur : a.obsKf[o0 + j - 1]; };
  if (lane == 0) {
    const float px = a.mpPos[3 * g], py = a.mpPos[3 * g + 1], pz = a.mpPos[3 * g + 2];
    float nx = 0.f, ny = 0.f, nz = 0.f;
    for (int j = 0; j < n; j++) {
      const float* O = a.kfC + 3 * (d.kf + kfAt(j));
      const float dx = __fsub_rn(px, O[0]), dy = __fsub_rn(py, O[1]), dz = __fsub_rn(pz, O[2]);  // mWorldPos - Owi
      const float al = __double2float_rn(__ddiv_rn(1.0, norm3(dx, dy, dz)));  // scaleAdd's alpha, rounded to float
      nx = __fmaf_rn(dx, al, nx);  // normal + normali/norm: scaleAdd, fused
      ny = __fmaf_rn(dy, al, ny);
      nz = __fmaf_rn(dz, al, nz);
    }
    const int ref = a.mpRef[g];
    int refO = o0;
    while (a.obsKf[refO] != ref) refO++;  // validated: the reference keyframe observes the point
    const float* O = a.kfC + 3 * (d.kf + ref);
    const float dist =
        __double2float_rn(norm3(__fsub_rn(px, O[0]), __fsub_rn(py, O[1]), __fsub_rn(pz, O[2])));
    const float* sf = a.sf + d.sf;
    const float mx = __fmul_rn(dist, sf[a.obsOct[refO]]);
    a.maxD[g] = mx;
    a.minD[g] = __fdiv_rn(mx, sf[d.nlev - 1]);
    const float inv = __double2float_rn(__ddiv_rn(1.0, (double)n));  // normal/n: convertTo with (float)(1./n)
    a.normal[3 * g] = __fadd_rn(__fmul_rn(nx, inv), 0.f);
    a.normal[3 * g + 1] = __fadd_rn(__fmul_rn(ny, inv), 0.f);
    a.normal[3 * g + 2] = __fadd_rn(__fmul_rn(nz, inv), 0.f);
    a.updated[g] = 1;
  }
  if (!kInsert) return;
  // ComputeDistinctiveDescriptors: the good observers' descriptors in row order, gathered as sources (an observation
  // index, or ~slot for the current keyframe's) with their row positions
  int* src = a.gather + o0 + g;  // n <= nIn + 1 entries per point: O + M over the batch
  int* pos = a.gatherPos + o0 + g;
  int N = 0;
  for (int base = 0; base < n; base += 32) {
    const int j = base + lane;
    int sj = 0;
    bool good = false;
    if (j < n) {
      const int k = kfAt(j);
      good = !a.kfBad[d.kf + k];
      sj = j < ins ? o0 + j : j == ins ? ~(d.slot + s) : o0 + j - 1;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, good);
    if (good) {
      const int at = N + __popc(bal & ((1u << lane) - 1));
      src[at] = sj;
      pos[at] = j;
    }
    N += __popc(bal);
  }
  __syncwarp();
  int best = -1;
  if (N > 0) {
    const int b = distinctive_best(
        N,
        [&](int i) {
          const int v = src[i];
          return v >= 0 ? ld_u256(a.obsDesc + (size_t)v * 32) : ld_u256(a.slotDesc + (size_t)(~v) * 32);
        },
        hist[wid], lane);
    best = pos[b];
  }
  if (lane == 0) a.descPos[g] = best;
}

}  // namespace

namespace {

constexpr int kMaxProblem = INT32_MAX / 8;  // bound on each packed extent, so that every offset fits an int

// Host checks shared by both entries: the observer CSR, its rows, octaves and, for the points in `need`, that the
// reference keyframe is an observer.  false: the message is set.
bool rows_ok(const char* fn, int b, int nkf, int nmp, const int32_t* off, const int32_t* kf, const int32_t* oct,
             int nlev, const int32_t* ref, const std::vector<char>& need) {
  if (!csr_ok(off, nmp, kMaxProblem) || !entries_ok(off, kf, nmp, 0, nkf, true)) {
    set_error("%s: problem %d: the observer rows are not a CSR of strictly ascending keyframe indices in range", fn, b);
    return false;
  }
  for (int o = 0; o < off[nmp]; o++)
    if (oct[o] < 0 || oct[o] >= nlev) {
      set_error("%s: problem %d: observation %d has octave %d outside [0, %d)", fn, b, o, oct[o], nlev);
      return false;
    }
  for (int m = 0; m < nmp; m++) {
    if (!need[(size_t)m]) continue;
    bool found = false;
    for (int o = off[m]; o < off[m + 1] && !found; o++) found = kf[o] == ref[m];
    if (!found) {
      set_error("%s: problem %d: point %d's reference keyframe %d is not one of its observers", fn, b, m, ref[m]);
      return false;
    }
  }
  return true;
}

int check_kfinsert(int b, const b2s_kfinsert_problem& p, const b2s_kfinsert_result& r) {
  const char* fn = "b2s_process_new_keyframe";
  if (p.n_kf < 1 || p.n_mp < 0 || p.n_slots < 0 || p.n_recent < 0 || p.n_levels < 1 || p.n_kf > kMaxProblem ||
      p.n_mp > kMaxProblem || p.n_slots > kMaxProblem || p.n_recent > kMaxProblem || p.cur < 0 || p.cur >= p.n_kf ||
      !p.kf_center || !p.kf_bad || !p.obs_off || !p.scale_factors ||
      (p.n_slots && (!p.slot_mp || !p.slot_stereo || !p.slot_desc || !r.slot_mp)) ||
      (p.n_mp && (!p.mp_pos || !p.mp_bad || !p.mp_ref || !p.mp_nobs || !p.mp_found || !p.mp_visible ||
                  !p.mp_first_kf || !r.mp_nobs || !r.mp_bad || !r.mp_added || !r.mp_updated || !r.mp_normal ||
                  !r.mp_min_dist || !r.mp_max_dist || !r.mp_desc)) ||
      (p.n_recent && !p.recent) || ((p.n_recent || p.n_slots) && (!r.list_mp || !r.list_verdict))) {
    set_error("%s: problem %d: bad argument (a null array, a count out of range, or cur outside the table)", fn, b);
    return B2S_ERR_BAD_ARG;
  }
  if (!csr_ok(p.obs_off, p.n_mp, kMaxProblem)) {
    set_error("%s: problem %d: obs_off is not a CSR", fn, b);
    return B2S_ERR_BAD_ARG;
  }
  const int O = p.obs_off[p.n_mp];
  if (O && (!p.obs_kf || !p.obs_idx || !p.obs_octave || !p.obs_desc || !r.obs_alive)) {
    set_error("%s: problem %d: bad argument (a null observation array)", fn, b);
    return B2S_ERR_BAD_ARG;
  }
  for (int s = 0; s < p.n_slots; s++)
    if (p.slot_mp[s] < -1 || p.slot_mp[s] >= p.n_mp) {
      set_error("%s: problem %d: slot %d holds point %d outside [-1, %d)", fn, b, s, p.slot_mp[s], p.n_mp);
      return B2S_ERR_BAD_ARG;
    }
  for (int e = 0; e < p.n_recent; e++)
    if (p.recent[e] < 0 || p.recent[e] >= p.n_mp) {
      set_error("%s: problem %d: recent entry %d is point %d outside [0, %d)", fn, b, e, p.recent[e], p.n_mp);
      return B2S_ERR_BAD_ARG;
    }
  for (int o = 0; o < O; o++)
    if (p.obs_idx[o] < 0 || (p.obs_kf && p.obs_kf[o] == p.cur && p.obs_idx[o] >= p.n_slots)) {
      set_error("%s: problem %d: observation %d has idx %d outside its keyframe", fn, b, o, p.obs_idx[o]);
      return B2S_ERR_BAD_ARG;
    }
  // the points the association refreshes: the first slot of a good point that does not list cur
  std::vector<char> need((size_t)p.n_mp, 0), seen((size_t)p.n_mp, 0);
  for (int s = 0; s < p.n_slots; s++) {
    const int m = p.slot_mp[s];
    if (m < 0 || p.mp_bad[m] || seen[(size_t)m]) continue;
    seen[(size_t)m] = 1;
    bool lists = false;
    for (int o = p.obs_off[m]; o < p.obs_off[m + 1] && !lists; o++) lists = p.obs_kf[o] == p.cur;
    need[(size_t)m] = !lists;
  }
  if (!rows_ok(fn, b, p.n_kf, p.n_mp, p.obs_off, p.obs_kf, p.obs_octave, p.n_levels, p.mp_ref, need))
    return B2S_ERR_BAD_ARG;
  return B2S_OK;
}

// Extents of a batch: keyframes, points, observations, slots, recent entries, scale levels, problems
struct Sizes {
  size_t K = 0, M = 0, O = 0, S = 0, R = 0, F = 0, B = 0;
};

}  // namespace

extern "C" float b2s_matcher_last_ms(const b2s_matcher* h) { return h ? h->lastMs : 0.f; }

extern "C" int b2s_update_normal_and_depth(b2s_matcher* h, const b2s_normal_depth_problem* p,
                                           b2s_normal_depth_result* r) {
  const char* fn = "b2s_update_normal_and_depth";
  if (!h || !p || !r || p->n_kf < 0 || p->n_mp < 0 || p->n_levels < 1 || p->n_kf > kMaxProblem ||
      p->n_mp > kMaxProblem || !p->obs_off || !p->scale_factors || (p->n_kf && !p->kf_center) ||
      (p->n_mp && (!p->mp_pos || !p->mp_bad || !p->mp_ref || !r->normal || !r->min_dist || !r->max_dist ||
                   !r->updated))) {
    set_error("%s: bad argument (a null array or a count out of range)", fn);
    return B2S_ERR_BAD_ARG;
  }
  if (!csr_ok(p->obs_off, p->n_mp, kMaxProblem)) {
    set_error("%s: obs_off is not a CSR", fn);
    return B2S_ERR_BAD_ARG;
  }
  const int nM = p->n_mp, nK = p->n_kf, O = p->obs_off[nM];
  if (O && (!p->obs_kf || !p->obs_octave)) {
    set_error("%s: bad argument (a null observation array)", fn);
    return B2S_ERR_BAD_ARG;
  }
  std::vector<char> need((size_t)nM);
  for (int m = 0; m < nM; m++) need[(size_t)m] = !p->mp_bad[m] && p->obs_off[m + 1] > p->obs_off[m];
  if (!rows_ok(fn, 0, nK, nM, p->obs_off, p->obs_kf, p->obs_octave, p->n_levels, p->mp_ref, need))
    return B2S_ERR_BAD_ARG;
  if (nM == 0) return B2S_OK;
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->stream;

  Packed &in = h->mpIn, &out = h->mpOut;
  in.clear();
  const Seg<Desc> gDesc = in.add<Desc>(1);
  const Seg<float> gC = in.add<float>(3 * (size_t)nK), gP = in.add<float>(3 * (size_t)nM);
  const Seg<int> gBad = in.add<int>(nM), gRef = in.add<int>(nM), gOff = in.add<int>(nM + 1), gKf = in.add<int>(O),
                 gOct = in.add<int>(O);
  const Seg<float> gSf = in.add<float>(p->n_levels);
  out.clear();
  const Seg<float> gNormal = out.add<float>(3 * (size_t)nM), gMinD = out.add<float>(nM), gMaxD = out.add<float>(nM);
  const Seg<int> gUpdated = out.add<int>(nM);
  int rc = in.fit(fn);
  if (rc == B2S_OK) rc = out.fit(fn);
  if (rc != B2S_OK) return rc;
  Desc* d = in.host(gDesc);
  *d = Desc{};
  d->nkf = nK;
  d->nmp = nM;
  d->nlev = p->n_levels;
  d->cur = -1;
  Args a{};
  a.desc = in.dev(gDesc);
  a.kfC = in.stage(gC, p->kf_center);
  a.mpPos = in.stage(gP, p->mp_pos);
  int* bad = in.host(gBad);
  for (int m = 0; m < nM; m++) bad[m] = p->mp_bad[m] ? 1 : 0;
  a.mpBad = in.dev(gBad);
  a.mpRef = in.stage(gRef, p->mp_ref);
  a.obsOff = in.stage(gOff, p->obs_off);
  a.obsKf = in.stage(gKf, p->obs_kf);
  a.obsOct = in.stage(gOct, p->obs_octave);
  a.sf = in.stage(gSf, p->scale_factors);
  a.normal = out.dev(gNormal);
  a.minD = out.dev(gMinD);
  a.maxD = out.dev(gMaxD);
  a.updated = out.dev(gUpdated);

  if ((rc = h->begin()) != B2S_OK) return rc;
  if ((rc = in.upload(st)) != B2S_OK) return rc;
  k_mp_point<false><<<div_up(nM, kWarps), kThreads, 0, st>>>(a, nM);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  if ((rc = out.download(st)) != B2S_OK) return rc;
  if ((rc = h->finish()) != B2S_OK) return rc;

  const float *normal = out.host(gNormal), *minD = out.host(gMinD), *maxD = out.host(gMaxD);
  const int* updated = out.host(gUpdated);
  for (int m = 0; m < nM; m++) {
    r->updated[m] = (uint8_t)updated[m];
    if (!r->updated[m]) continue;
    memcpy(r->normal + 3 * (size_t)m, normal + 3 * (size_t)m, 12);
    r->min_dist[m] = minD[m];
    r->max_dist[m] = maxD[m];
  }
  return B2S_OK;
}

extern "C" int b2s_process_new_keyframe(b2s_matcher* h, int batch, const b2s_kfinsert_problem* p,
                                        b2s_kfinsert_result* r) {
  const char* fn = "b2s_process_new_keyframe";
  if (!h || !p || !r || batch < 1) {
    set_error("%s: bad argument", fn);
    return B2S_ERR_BAD_ARG;
  }
  for (int b = 0; b < batch; b++) {
    const int rc = check_kfinsert(b, p[b], r[b]);
    if (rc != B2S_OK) return rc;
  }
  std::vector<Desc> desc((size_t)batch);
  Sizes z;
  z.B = batch;
  for (int b = 0; b < batch; b++) {
    const b2s_kfinsert_problem& q = p[b];
    Desc& d = desc[(size_t)b];
    d.nkf = q.n_kf;
    d.nmp = q.n_mp;
    d.nslot = q.n_slots;
    d.nrec = q.n_recent;
    d.kf = (int)z.K;
    d.mp = (int)z.M;
    d.obs = (int)z.O;
    d.obsOff = (int)(z.M + b);
    d.slot = (int)z.S;
    d.rec = (int)z.R;
    d.list = (int)(z.R + z.S);
    d.sf = (int)z.F;
    d.nlev = q.n_levels;
    d.cur = q.cur;
    d.curId = (int)(uint32_t)q.cur_id;  // (int)nCurrentKFid
    d.mono = q.monocular != 0;
    z.K += q.n_kf;
    z.M += q.n_mp;
    z.O += q.obs_off[q.n_mp];
    z.S += q.n_slots;
    z.R += q.n_recent;
    z.F += q.n_levels;
    if (3 * z.K + 8 * z.M + 4 * z.O + 4 * z.S + 2 * z.R + z.F + 2 * z.B >= (size_t)kMaxProblem) {
      set_error("%s: the batch is too large for one call", fn);
      return B2S_ERR_CAPACITY;
    }
  }
  B2S_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->stream;
  const size_t B = z.B, K = z.K, M = z.M, O = z.O, S = z.S, R = z.R, L = R + S;
  Packed &in = h->mpIn, &out = h->mpOut;
  in.clear();
  const Seg<Desc> gDesc = in.add<Desc>(B);
  const Seg<int> gProb = in.add<int>(M);
  const Seg<float> gC = in.add<float>(3 * K);
  const Seg<int> gKb = in.add<int>(K), gSm = in.add<int>(S), gSs = in.add<int>(S);
  const Seg<float> gP = in.add<float>(3 * M);
  const Seg<int> gBad = in.add<int>(M), gRef = in.add<int>(M), gNobs = in.add<int>(M), gFound = in.add<int>(M),
                 gVis = in.add<int>(M), gFirst = in.add<int>(M), gOff = in.add<int>(M + B), gKf = in.add<int>(O),
                 gIdx = in.add<int>(O), gOct = in.add<int>(O), gRec = in.add<int>(R);
  const Seg<float> gSf = in.add<float>(z.F);
  const Seg<uint8_t> gObsDesc = in.add<uint8_t>(32 * O), gSlotDesc = in.add<uint8_t>(32 * S);
  out.clear();
  const Seg<int> gNobsOut = out.add<int>(M), gBadOut = out.add<int>(M), gAdded = out.add<int>(M),
                 gUpdated = out.add<int>(M), gDescPos = out.add<int>(M), gAlive = out.add<int>(O);
  const Seg<float> gNormal = out.add<float>(3 * M), gMinD = out.add<float>(M), gMaxD = out.add<float>(M);
  const Seg<int> gSlot = out.add<int>(S), gList = out.add<int>(L), gVerdict = out.add<int>(L), gNList = out.add<int>(B),
                 gCulled = out.add<int>(B), gFirstSlot = out.add<int>(M), gFirstEntry = out.add<int>(M),
                 gGather = out.add<int>(O + M), gGatherPos = out.add<int>(O + M);
  int rc = in.fit(fn);
  if (rc == B2S_OK) rc = out.fit(fn);
  if (rc != B2S_OK) return rc;

  // pack: one upload
  memcpy(in.host(gDesc), desc.data(), B * sizeof(Desc));
  for (int b = 0; b < batch; b++) {
    const b2s_kfinsert_problem& pb = p[b];
    const Desc& d = desc[(size_t)b];
    const int nO = pb.obs_off[pb.n_mp];
    for (int m = 0; m < d.nmp; m++) {
      in.host(gProb)[d.mp + m] = b;
      in.host(gBad)[d.mp + m] = pb.mp_bad[m] ? 1 : 0;
      in.host(gFirst)[d.mp + m] = (int)(uint32_t)(uint64_t)pb.mp_first_kf[m];  // (int)mnFirstKFid
    }
    memcpy(in.host(gC) + 3 * (size_t)d.kf, pb.kf_center, 12 * (size_t)d.nkf);
    for (int k = 0; k < d.nkf; k++) in.host(gKb)[d.kf + k] = pb.kf_bad[k] ? 1 : 0;
    if (d.nslot) {
      memcpy(in.host(gSm) + d.slot, pb.slot_mp, 4 * (size_t)d.nslot);
      for (int s = 0; s < d.nslot; s++) in.host(gSs)[d.slot + s] = pb.slot_stereo[s] ? 1 : 0;
      memcpy(in.host(gSlotDesc) + 32 * (size_t)d.slot, pb.slot_desc, 32 * (size_t)d.nslot);
    }
    if (d.nmp) {
      memcpy(in.host(gP) + 3 * (size_t)d.mp, pb.mp_pos, 12 * (size_t)d.nmp);
      memcpy(in.host(gRef) + d.mp, pb.mp_ref, 4 * (size_t)d.nmp);
      memcpy(in.host(gNobs) + d.mp, pb.mp_nobs, 4 * (size_t)d.nmp);
      memcpy(in.host(gFound) + d.mp, pb.mp_found, 4 * (size_t)d.nmp);
      memcpy(in.host(gVis) + d.mp, pb.mp_visible, 4 * (size_t)d.nmp);
    }
    memcpy(in.host(gOff) + d.obsOff, pb.obs_off, 4 * (size_t)(d.nmp + 1));
    if (nO) {
      memcpy(in.host(gKf) + d.obs, pb.obs_kf, 4 * (size_t)nO);
      memcpy(in.host(gIdx) + d.obs, pb.obs_idx, 4 * (size_t)nO);
      memcpy(in.host(gOct) + d.obs, pb.obs_octave, 4 * (size_t)nO);
      memcpy(in.host(gObsDesc) + 32 * (size_t)d.obs, pb.obs_desc, 32 * (size_t)nO);
    }
    if (d.nrec) memcpy(in.host(gRec) + d.rec, pb.recent, 4 * (size_t)d.nrec);
    memcpy(in.host(gSf) + d.sf, pb.scale_factors, 4 * (size_t)d.nlev);
  }
  const Args a = {in.dev(gDesc),       in.dev(gProb),        in.dev(gC),           in.dev(gP),
                  in.dev(gSf),         in.dev(gKb),          in.dev(gSm),          in.dev(gSs),
                  in.dev(gBad),        in.dev(gRef),         in.dev(gNobs),        in.dev(gFound),
                  in.dev(gVis),        in.dev(gFirst),       in.dev(gOff),         in.dev(gKf),
                  in.dev(gIdx),        in.dev(gOct),         in.dev(gRec),         in.dev(gObsDesc),
                  in.dev(gSlotDesc),   out.dev(gNobsOut),    out.dev(gBadOut),     out.dev(gAdded),
                  out.dev(gAlive),     out.dev(gUpdated),    out.dev(gDescPos),    out.dev(gSlot),
                  out.dev(gList),      out.dev(gVerdict),    out.dev(gNList),      out.dev(gCulled),
                  out.dev(gNormal),    out.dev(gMinD),       out.dev(gMaxD),       out.dev(gFirstSlot),
                  out.dev(gFirstEntry), out.dev(gGather),    out.dev(gGatherPos)};

  if ((rc = h->begin()) != B2S_OK) return rc;
  if ((rc = in.upload(st)) != B2S_OK) return rc;
  k_kfi_list<<<batch, kThreads, 0, st>>>(a);
  h->launches++;
  if (M) {
    k_mp_point<true><<<div_up((int)M, kWarps), kThreads, 0, st>>>(a, (int)M);
    h->launches++;
  }
  B2S_CUDA(cudaGetLastError());
  if ((rc = out.download(st, 0, gCulled.end())) != B2S_OK) return rc;  // not the scratch
  if ((rc = h->finish()) != B2S_OK) return rc;

  const int *nobs = out.host(gNobsOut), *bad = out.host(gBadOut), *added = out.host(gAdded),
            *updated = out.host(gUpdated), *descPos = out.host(gDescPos), *alive = out.host(gAlive),
            *slot = out.host(gSlot), *list = out.host(gList), *verdict = out.host(gVerdict), *nList = out.host(gNList),
            *nCulled = out.host(gCulled);
  const float *normal = out.host(gNormal), *minD = out.host(gMinD), *maxD = out.host(gMaxD);
  for (int b = 0; b < batch; b++) {
    const Desc& d = desc[(size_t)b];
    b2s_kfinsert_result& rb = r[b];
    const int nO = p[b].obs_off[d.nmp];
    for (int m = 0; m < d.nmp; m++) {
      const int g = d.mp + m;
      rb.mp_nobs[m] = nobs[g];
      rb.mp_bad[m] = (uint8_t)bad[g];
      rb.mp_added[m] = added[g];
      rb.mp_updated[m] = (uint8_t)updated[g];
      rb.mp_desc[m] = updated[g] ? descPos[g] : -1;
      if (!updated[g]) continue;
      memcpy(rb.mp_normal + 3 * (size_t)m, normal + 3 * (size_t)g, 12);
      rb.mp_min_dist[m] = minD[g];
      rb.mp_max_dist[m] = maxD[g];
    }
    for (int i = 0; i < nO; i++) rb.obs_alive[i] = (uint8_t)alive[d.obs + i];
    if (d.nslot) memcpy(rb.slot_mp, slot + d.slot, 4 * (size_t)d.nslot);
    rb.n_list = nList[b];
    for (int e = 0; e < nList[b]; e++) {
      rb.list_mp[e] = list[d.list + e];
      rb.list_verdict[e] = (uint8_t)verdict[d.list + e];
    }
    rb.n_culled = nCulled[b];
  }
  return B2S_OK;
}
