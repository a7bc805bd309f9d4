/*
 * include/b200slam.h — C ABI of libb200slam.so: the H100-native (sm_90a) replacement for the hot path of
 * DreamWaterFound/self_commit_ORB-SLAM2.
 *
 * The reference has no FFI layer: its boundary is three C++ classes (SURVEY.md §8b).  The entry points below
 * are what a C++ shim with the reference's own signatures binds to (the shim lives in
 * self_commit_orb-slam2_b200/host/, the reference-side patch in INTEGRATION.md):
 *
 *   ORBextractor::ORBextractor(...)            /root/reference/include/ORBextractor.h:92,  src/ORBextractor.cc:492
 *   ORBextractor::operator()(...)              include/ORBextractor.h:110, src/ORBextractor.cc:1544
 *   ORBextractor::Get*()                       include/ORBextractor.h:118-161
 *   ORBmatcher::DescriptorDistance             include/ORBmatcher.h,  src/ORBmatcher.cc:1913
 *   ORBmatcher::SearchByBoW (2 overloads)      src/ORBmatcher.cc:230, :656
 *   ORBmatcher::SearchByProjection(F,F,th,mono) src/ORBmatcher.cc:1569
 *   Optimizer::LocalBundleAdjustment           include/Optimizer.h:112, src/Optimizer.cc:629
 *
 * Conventions: plain pointers and sizes, no C++/torch types; every function returns an int status
 * (B2S_OK = 0) and never throws; buffers are caller-owned, device memory is owned by handles; handles are
 * independent (one CUDA stream each, no global mutable state) so left/right extractors may run on two
 * threads like src/Frame.cc:159-167.  There is NO CPU fallback: without a CUDA device every call fails
 * with B2S_ERR_NO_DEVICE.
 */
#ifndef B200SLAM_H
#define B200SLAM_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

enum {
  B2S_OK = 0,
  B2S_ERR_NO_DEVICE = 1,    /* no CUDA device / driver: the product does not fall back to the CPU */
  B2S_ERR_BAD_ARG = 2,
  B2S_ERR_CUDA = 3,         /* a CUDA call failed; b2s_last_error() has the text */
  B2S_ERR_CAPACITY = 4,     /* caller buffer (cap) too small */
  B2S_ERR_ABORTED = 5       /* LocalBA: stop flag was set before the first round (no write-back) */
};

const char* b2s_last_error(void);   /* thread-local text of the last failure */
int b2s_version(void);
int b2s_device_count(void);
/* Issue-rate micro-benchmarks of `device` (about 20 ms): out8[0] packed u16x2 min/max (ALU pipe) and [1] IMAD (FMA pipe) in
 * G warp-instructions/s, [2] FP64 DFMA TFLOP/s, [3] POPC G warp-instructions/s, [4] ALU + FMA interleaved, [5] IMMA.16832.U8.U8 (the integer
 * tensor pipe as mma.sync reaches it) in G warp-instructions/s; the rest 0.
 * bench.py reports the kernels' figures against these measured bounds. */
int b2s_measure_peaks(int device, double* out8);

/* Layout-identical to cv::KeyPoint (28 bytes): pt.x, pt.y, size, angle, response, octave, class_id */
typedef struct {
  float x, y, size, angle, response;
  int32_t octave, class_id;
} b2s_keypoint;

/* ------------------------------------------------------------------ extractor */
typedef struct b2s_extractor b2s_extractor;

/* ctor: src/ORBextractor.cc:492-609. max_width/max_height/max_batch size the device buffers.
 * Accepted parameters: nfeatures >= 1 (up to the quadtree's shared-memory limit, about 12,000 at 1.2 / 8 levels: above
 * it B2S_ERR_BAD_ARG), scaleFactor > 1, nlevels 1..12, 1 <= minThFAST <= iniThFAST <= 254, max_width / max_height
 * 64..8192, max_batch >= 1.
 * Accepted images: width <= max_width, height <= max_height, and every pyramid level w_l x h_l
 * (w_l = cvRound(width / scaleFactor^l)) at least 62 x 62 (one 30-px FAST cell inside the 16-px border; 221 x 221 for
 * 8 levels at 1.2) with width >= about half the height.  Other images fail with B2S_ERR_BAD_ARG ("pyramid level l
 * (w x h) is too small for the 30-px FAST cell grid"); the reference would still return the keypoints of the larger
 * levels there.  Within that domain extraction succeeds for any image content: the internal candidate buffers are sized
 * for the worst case; B2S_ERR_CAPACITY reports a record cap (`cap`) that is too small. */
int b2s_extractor_create(int nfeatures, float scaleFactor, int nlevels, int iniThFAST, int minThFAST, int max_width,
                         int max_height, int max_batch, int device, b2s_extractor** out);
void b2s_extractor_destroy(b2s_extractor* h);
/* GetScaleFactors / GetInverseScaleFactors / GetScaleSigmaSquares / GetInverseScaleSigmaSquares + per-level quotas;
 * any pointer may be NULL; arrays hold nlevels entries. */
int b2s_extractor_tables(const b2s_extractor* h, float* scale, float* inv_scale, float* sigma2, float* inv_sigma2,
                         int32_t* nfeatures_per_level);
int b2s_extractor_max_keypoints(const b2s_extractor* h); /* upper bound of N for one image (nfeatures + 2*nlevels..) */

/* operator(): one image, HOST buffers (H2D/D2H inside). kps: cap entries; desc: cap x 32 bytes.
 * pyr_out: optional array of nlevels host pointers that receive mvImagePyramid level images (tightly packed
 * w_l x h_l) — needed by Frame::ComputeStereoMatches (src/Frame.cc:1044); NULL to skip the D2H.
 * Empty image (w<=0||h<=0||img==NULL) -> *n_out = 0, B2S_OK (src/ORBextractor.cc:1553). */
int b2s_extract(b2s_extractor* h, const uint8_t* img, int width, int height, int stride, b2s_keypoint* kps, uint8_t* desc,
                int cap, int* n_out, uint8_t* const* pyr_out);

/* Batched: B same-sized images (e.g. L/R pairs of several frames), HOST buffers; imgs = B pointers;
 * kps: B*cap, desc: B*cap*32, n_out: B. */
int b2s_extract_batch(b2s_extractor* h, const uint8_t* const* imgs, int batch, int width, int height, int stride,
                      b2s_keypoint* kps, uint8_t* desc, int cap, int* n_out);

/* Batched, DEVICE-resident: d_imgs = batch images at d_imgs + b*img_pitch_bytes (row stride `stride`), results stay
 * in HBM as fixed-size records (the layout that is all-gathered over NVLink, SURVEY.md §8e):
 *   d_kps[b*cap + i], d_desc[(b*cap + i)*32], d_counts[b].   stream: a cudaStream_t (NULL = the handle's own stream);
 * the call is asynchronous on that stream. */
int b2s_extract_batch_device(b2s_extractor* h, const uint8_t* d_imgs, size_t img_pitch_bytes, int batch, int width,
                             int height, int stride, b2s_keypoint* d_kps, uint8_t* d_desc, int32_t* d_counts, int cap,
                             void* stream);
/* status of the last device batch (candidate-buffer overflow etc.); synchronises the handle's stream. */
int b2s_extractor_check(b2s_extractor* h);
/* number of kernel launches issued by this handle so far (bench.py's gpu_launches) */
long long b2s_extractor_launch_count(const b2s_extractor* h);

/* per-stage CUDA-event timing on the launching stream (bench.py roofline): enable, run, then read the accumulated
 * device milliseconds of {pyramid resize chain, FAST cells, quadtree, blur, orient+describe} and the call count. */
int b2s_extractor_set_timing(b2s_extractor* h, int enable);
int b2s_extractor_get_timing(b2s_extractor* h, double* stage_ms5, long long* calls);

/* test hooks: device -> host copies of intermediates of image `b` of the last call */
int b2s_extractor_debug_level(b2s_extractor* h, int b, int level, int blurred, uint8_t* out, int* w, int* hgt);
int b2s_extractor_debug_candidates(b2s_extractor* h, int b, int level, int32_t* xy /*2*cap*/, int32_t* resp, int cap,
                                   int* n);
/* test hook, host only (needs no device): the per-image buffer sizes of a handle created for max_width x max_height and
 * the pyramid / cell geometry of a width x height image in it.  out: 8 + 8 * nlevels entries (layout in extractor.cu);
 * returns the status extraction of such an image would get from its geometry (B2S_OK or B2S_ERR_BAD_ARG). */
int b2s_debug_extractor_plan(int nfeatures, float scaleFactor, int nlevels, int max_width, int max_height, int width,
                             int height, int64_t* out);

/* ------------------------------------------------------------------ stereo matching (SURVEY.md §8f rank 1) */
/* Frame::ComputeStereoMatches (src/Frame.cc:1026-1421) for the stereo pairs of the batch this handle extracted last; the
 * image pyramids (mvImagePyramid, the function's only other input) are still resident, so no image leaves the device.
 * Pair p = (image first_left+p, image first_right+p) of that batch, p in [0, n_pairs).
 * bf = Frame::mbf; mb = the baseline the reference sees when the function runs (this fork assigns mb AFTER the call,
 * src/Frame.cc:125,186,1108, so it sees 0 and the disparity bound maxD = mbf/mb is +inf; pass the real baseline to get
 * the upstream behaviour).  Outputs per left feature: mvuRight / mvDepth (-1 = no stereo match); n_matched[p] = matches
 * that survive the median cull (:1395-1415).
 *
 * _device: d_kps/d_desc/d_counts are the device record arrays of that batch (e.g. the buffers given to
 * b2s_extract_batch_device, `cap` records per image, cap <= 4096); d_uright/d_depth: device float [n_pairs][cap];
 * asynchronous on `stream`.  The host variant uses the records b2s_extract_batch left on the device and writes
 * [n_pairs][cap_out] host arrays (cap_out >= the cap of that call). */
int b2s_stereo_match_device(b2s_extractor* h, int first_left, int first_right, int n_pairs, const b2s_keypoint* d_kps,
                            const uint8_t* d_desc, const int32_t* d_counts, int cap, float bf, float mb, float* d_uright,
                            float* d_depth, int32_t* d_nmatched, void* stream);
int b2s_stereo_match(b2s_extractor* h, int first_left, int first_right, int n_pairs, float bf, float mb, float* uright,
                     float* depth, int cap_out, int32_t* n_matched);

/* ------------------------------------------------------------------ matcher */
typedef struct b2s_matcher b2s_matcher;
int b2s_matcher_create(int max_features, int max_batch, int device, b2s_matcher** out);
void b2s_matcher_destroy(b2s_matcher* h);
long long b2s_matcher_launch_count(const b2s_matcher* h);

/* DescriptorDistance (src/ORBmatcher.cc:1913): n pairs a[i] vs b[i], HOST buffers -> dist[n] */
int b2s_descriptor_distance(b2s_matcher* h, const uint8_t* a, const uint8_t* b, int n, int32_t* dist);

/* SearchByBoW on flattened arrays (HOST buffers).  A = keyframe side, B = frame side.
 * nodeA/nodeB: DBoW2 FeatureVector node id per feature (features with equal ids are candidates);
 * validA/validB: 1 = has a usable MapPoint (validB may be NULL: SearchByBoW(KF,F) does not need it);
 * strict_lt: 0 -> best<=th_low (KF,F variant :308), 1 -> best<th_low (KF,KF variant :741).
 * matchB[j] = index into A, or -1. */
int b2s_search_by_bow(b2s_matcher* h, const uint8_t* descA, const int32_t* nodeA, const uint8_t* validA, const float* angA,
                      int nA, const uint8_t* descB, const int32_t* nodeB, const uint8_t* validB, const float* angB, int nB,
                      int th_low, float nnratio, int strict_lt, int check_ori, int32_t* matchB, int* nmatches);

/* Batched HOST-buffer variant: `batch` independent (A,B) pairs laid out with strides capA/capB features;
 * nA/nB: host int arrays [batch]; matchB: batch*capB; nmatches: batch. One H2D per array, one D2H per result. */
int b2s_search_by_bow_batch(b2s_matcher* h, int batch, const uint8_t* descA, const int32_t* nodeA, const uint8_t* validA,
                            const float* angA, const int32_t* nA, int capA, const uint8_t* descB, const int32_t* nodeB,
                            const uint8_t* validB, const float* angB, const int32_t* nB, int capB, int th_low,
                            float nnratio, int strict_lt, int check_ori, int32_t* matchB, int32_t* nmatches);

/* Test hook (host only, no GPU needed): the distance from which a frame-side candidate cannot influence SearchByBoW for
 * (TH_LOW, ratio) — the K-list stage lists and counts only candidates below it (257 = no cut).  tests/test_bow_cut_logic.py
 * checks by enumeration that no decision of src/ORBmatcher.cc:284-310 can depend on a candidate at or beyond it. */
int b2s_debug_bow_distance_cut(int th_low, float nnratio);

/* Batched device-resident variant: `batch` independent (A,B) pairs with strides capA/capB features. All pointers are
 * DEVICE pointers; nA/nB are device int arrays [batch]. Asynchronous on `stream`. */
int b2s_search_by_bow_device(b2s_matcher* h, int batch, const uint8_t* d_descA, const int32_t* d_nodeA,
                             const uint8_t* d_validA, const float* d_angA, const int32_t* d_nA, int capA,
                             const uint8_t* d_descB, const int32_t* d_nodeB, const uint8_t* d_validB,
                             const float* d_angB, const int32_t* d_nB, int capB, int th_low, float nnratio, int strict_lt,
                             int check_ori, int32_t* d_matchB, int32_t* d_nmatches, void* stream);

/* SearchByProjection(CurrentFrame, LastFrame, th, bMono) (src/ORBmatcher.cc:1569) after projection. */
typedef struct {
  float u, v;      /* projection of the last frame's map point into the current frame (:1620-1621) */
  float invz;      /* 1/zc (:1614) */
  float angle;     /* LastFrame.mvKeysUn[i].angle */
  int32_t octave;  /* LastFrame.mvKeys[i].octave */
  int32_t has_obs; /* pMP->Observations()>0 */
  uint8_t desc[32];/* pMP->GetDescriptor() */
} b2s_proj_query;

typedef struct {
  float mnMinX, mnMinY, mnMaxX, mnMaxY; /* Frame::mnMinX.. (src/Frame.cc:193-214) */
  float bf;                             /* Frame::mbf */
  const float* scale_factors;           /* mvScaleFactors, nlevels entries (host pointer) */
  int nlevels;
} b2s_frame_geom;

/* mode: 0 levels [oct-1,oct+1]; 1 forward (>=oct); 2 backward ([0,oct]) (:1637-1642).
 * match_cur[j] = query index or -1; *nmatches as the reference counts them. HOST buffers. */
int b2s_search_by_projection_last(b2s_matcher* h, const b2s_proj_query* q, int nq, const float* kpx, const float* kpy,
                                  const int32_t* octave, const float* angle, const float* uright,
                                  const uint8_t* occupied, const uint8_t* desc, int nf, const b2s_frame_geom* g, float th,
                                  int mode, int th_high, int check_ori, int32_t* match_cur, int* nmatches);

/* Batched, device-resident form for a sequence (the stream mode of SURVEY.md 8d / 8e): pair b matches the queries
 * d_q[b*capQ .. +d_nq[b]) against the current frame b given as the extractor's device records (d_kps, d_desc: stride capF
 * entries per pair, d_nf[b] valid) and the stereo matcher's d_uright.  Same candidate order, thresholds, greedy resolution and
 * rotation culling as b2s_search_by_projection_last (occupied = none: the current frame holds no MapPoint yet,
 * src/Tracking.cc:881-883).  d_match_cur: [batch][capF], d_nmatches: [batch].  Asynchronous on `stream` (NULL = the
 * matcher's own stream); needs batch <= max_batch and capQ, capF <= max_features of b2s_matcher_create. */
int b2s_search_by_projection_last_device(b2s_matcher* h, int batch, const b2s_proj_query* d_q, const int32_t* d_nq, int capQ,
                                         const b2s_keypoint* d_kps, const float* d_uright, const uint8_t* d_desc,
                                         const int32_t* d_nf, int capF, const b2s_frame_geom* g, float th, int mode,
                                         int th_high, int check_ori, int32_t* d_match_cur, int32_t* d_nmatches, void* stream);
/* The same with HOST buffers (one upload, one download, synchronous): q [batch][capQ], kps / uright / desc [batch][capF]. */
int b2s_search_by_projection_last_batch(b2s_matcher* h, int batch, const b2s_proj_query* q, const int32_t* nq, int capQ,
                                        const b2s_keypoint* kps, const float* uright, const uint8_t* desc, const int32_t* nf,
                                        int capF, const b2s_frame_geom* g, float th, int mode, int th_high, int check_ori,
                                        int32_t* match_cur, int32_t* nmatches);
/* HOST-buffer form for a frame sequence: kps / desc / depth hold batch + 1 consecutive frames ([batch + 1][cap]), uright the
 * mvuRight of frames 1 .. batch; frame b + 1 is matched against frame b, the queries being formed on the device exactly as
 * b2s_track_queries_device forms them (Tcl: [batch][12]).  match_cur [batch][cap], nmatches [batch].  Synchronous. */
int b2s_search_by_projection_sequence(b2s_matcher* h, int batch, const b2s_keypoint* kps, const uint8_t* desc,
                                      const float* depth, const float* uright, const int32_t* n, int cap, const float* Tcl,
                                      float fx, float fy, float cx, float cy, int has_obs, const b2s_frame_geom* g, float th,
                                      int mode, int th_high, int check_ori, int32_t* match_cur, int32_t* nmatches);
/* The projection half of the same function (src/ORBmatcher.cc:1600-1626) for a stereo sequence, on the device: feature i of
 * last frame b with stereo depth d_depth_last > 0 stands for the map point Frame::UnprojectStereo (src/Frame.cc:679-696)
 * gives it, is moved into the current camera by d_Tcl[b] = [R | t] (3 x 4 row-major floats) and projected with fx, fy, cx, cy;
 * query i belongs to feature i (features without depth become skipped queries), d_nq[b] = d_n_last[b].  has_obs = what
 * pMP->Observations() > 0 is for these points (0 for the temporal points of Tracking::UpdateLastFrame). */
int b2s_track_queries_device(b2s_matcher* h, int batch, const b2s_keypoint* d_kps_last, const uint8_t* d_desc_last,
                             const float* d_depth_last, const int32_t* d_n_last, int cap, const float* d_Tcl, float fx,
                             float fy, float cx, float cy, int has_obs, b2s_proj_query* d_q, int32_t* d_nq, void* stream);

/* SearchByProjection(Frame& F, const vector<MapPoint*>& vpMapPoints, float th) (src/ORBmatcher.cc:70-175), the local-map
 * matcher of Tracking::SearchLocalPoints; queries are the map points after Frame::isInFrustum (src/Frame.cc:608-735). */
typedef struct {
  float u, v, ur;    /* mTrackProjX, mTrackProjY, mTrackProjXR */
  float view_cos;    /* mTrackViewCos (RadiusByViewingCos, :178-185) */
  int32_t level;     /* mnTrackScaleLevel */
  uint8_t in_view;   /* mbTrackInView && !isBad() (:83-87) */
  uint8_t has_obs;   /* pMP->Observations()>0 */
  uint8_t pad[2];
  uint8_t desc[32];  /* pMP->GetDescriptor() */
} b2s_map_query;

/* Levels [level-1, level], radius RadiusByViewingCos(view_cos) (x th when th != 1) x scale[level], stereo gate on `ur`,
 * best <= th_high (TH_HIGH), ratio test `best > nnratio*second` only when both candidates share the pyramid level.
 * occupied[j] = the feature already holds a MapPoint with Observations()>0 (:123-125; may be NULL).
 * match_cur[j] = query index or -1 (last writer wins); *nmatches as the reference counts them. HOST buffers. */
int b2s_search_by_projection_map(b2s_matcher* h, const b2s_map_query* q, int nq, const float* kpx, const float* kpy,
                                 const int32_t* octave, const float* uright, const uint8_t* occupied, const uint8_t* desc,
                                 int nf, const b2s_frame_geom* g, float th, int th_high, float nnratio, int32_t* match_cur,
                                 int* nmatches);

/* Windowed best-match search on a KeyFrame's feature grid: the search core shared by
 *   ORBmatcher::Fuse(KeyFrame*, const vector<MapPoint*>&, th)                        src/ORBmatcher.cc:1020-1174 (B2S_WIN_CHI2)
 *   ORBmatcher::Fuse(KeyFrame*, cv::Mat Scw, vpPoints, th, vpReplacePoint)          :1179-1310                  (no flag)
 *   ORBmatcher::SearchByProjection(KeyFrame*, cv::Mat Scw, vpPoints, vpMatched, th) :388-512                    (B2S_WIN_GREEDY)
 * The caller keeps the projection (Rcw/tcw or Sim3), the visibility / distance / normal tests and the map bookkeeping
 * (Replace / AddObservation) and passes one query per surviving map point, in the reference's iteration order. */
typedef struct {
  float u, v, ur;      /* projection into the keyframe (ur = u - bf*invz; only the chi-square gate reads it) */
  float radius;        /* th * pKF->mvScaleFactors[nPredictedLevel] */
  int32_t min_level;   /* nPredictedLevel-1 */
  int32_t max_level;   /* nPredictedLevel   */
  uint8_t valid;       /* 0: skipped by the reference before the search (bad / behind the camera / out of range ...) */
  uint8_t pad[3];
  uint8_t desc[32];    /* pMP->GetDescriptor() */
} b2s_win_query;
#define B2S_WIN_CHI2 1   /* reprojection gate e2*mvInvLevelSigma2[level] <= 7.8 (mvuRight >= 0) / 5.99 (:1097-1124) */
#define B2S_WIN_GREEDY 2 /* features with occupied[j] != 0 or chosen by an earlier query are skipped (:462-463,498-502) */

/* best_idx[i] = keyframe feature with the smallest descriptor distance (first minimum in GetFeaturesInArea order,
 * src/KeyFrame.cc:752-796) if that distance <= th_dist (TH_LOW), else -1; best_dist may be NULL; occupied is only
 * read with B2S_WIN_GREEDY (may be NULL); inv_level_sigma2 only with B2S_WIN_CHI2.  HOST buffers. */
int b2s_search_windows(b2s_matcher* h, const b2s_win_query* q, int nq, const float* kpx, const float* kpy,
                       const int32_t* octave, const float* uright, const float* inv_level_sigma2, const uint8_t* occupied,
                       const uint8_t* desc, int nf, const b2s_frame_geom* g, int flags, int th_dist, int32_t* best_idx,
                       int32_t* best_dist, int* n_accepted);

/* ORBmatcher::SearchForTriangulation(KeyFrame* pKF1, KeyFrame* pKF2, cv::Mat F12, vMatchedPairs, bOnlyStereo)
 * (src/ORBmatcher.cc:810-1009, CheckDistEpipolarLine :186-215) on flattened keyframes (LocalMapping::CreateNewMapPoints). */
typedef struct {
  const uint8_t* desc;    /* mDescriptors, n x 32 */
  const int32_t* node;    /* DBoW2 FeatureVector node id per feature (mFeatVec) */
  const uint8_t* has_mp;  /* GetMapPoint(idx) != NULL */
  const uint8_t* stereo;  /* mvuRight[idx] >= 0 */
  const float* x;         /* mvKeysUn[idx].pt.x */
  const float* y;
  const int32_t* octave;  /* mvKeysUn[idx].octave */
  const float* angle;     /* mvKeysUn[idx].angle */
  int32_t n;
} b2s_kf_features;

/* ---- persistent Frame feature grid (SURVEY §8f rank 4) -------------------------------------------------------------------
 * Frame::AssignFeaturesToGrid (src/Frame.cc:461-491) once per frame; the frame's keypoints, descriptors and the 64 x 48
 * cell index then stay on the device, so the consecutive matchers Tracking runs on one frame (SearchByProjection against
 * the last frame, SearchLocalPoints, relocalisation, Fuse / loop searches on a keyframe) upload only their queries.
 * The grid belongs to the matcher handle it was created with.  inv_level_sigma2 (mvInvLevelSigma2) may be NULL unless
 * B2S_WIN_CHI2 searches are made.  _create_device takes the extractor's device-resident records (b2s_extract_batch_device)
 * and an optional device array of mvuRight (b2s_stereo_match_device); NULL = monocular (-1). */
typedef struct b2s_frame_grid b2s_frame_grid;
int b2s_frame_grid_create(b2s_matcher* h, const float* kpx, const float* kpy, const int32_t* octave, const float* angle,
                          const float* uright, const uint8_t* desc, int nf, const b2s_frame_geom* g,
                          const float* inv_level_sigma2, b2s_frame_grid** out);
int b2s_frame_grid_create_device(b2s_matcher* h, const b2s_keypoint* d_kps, const uint8_t* d_desc, int nf,
                                 const float* d_uright, const b2s_frame_geom* g, const float* inv_level_sigma2, void* stream,
                                 b2s_frame_grid** out);
void b2s_frame_grid_destroy(b2s_frame_grid* grid);
int b2s_frame_grid_size(const b2s_frame_grid* grid);
/* Frame::GetFeaturesInArea (src/Frame.cc:741-852): indices in the reference's order; *n = count (B2S_ERR_CAPACITY if > cap) */
int b2s_frame_grid_features_in_area(b2s_frame_grid* grid, float x, float y, float r, int min_level, int max_level,
                                    int32_t* out, int cap, int* n);
/* b2s_search_by_projection_last / _map / b2s_search_windows on a resident grid (same semantics, same results) */
int b2s_search_by_projection_last_grid(b2s_matcher* h, b2s_frame_grid* grid, const b2s_proj_query* q, int nq,
                                       const uint8_t* occupied, float th, int mode, int th_high, int check_ori,
                                       int32_t* match_cur, int* nmatches);
int b2s_search_by_projection_map_grid(b2s_matcher* h, b2s_frame_grid* grid, const b2s_map_query* q, int nq,
                                      const uint8_t* occupied, float th, int th_high, float nnratio, int32_t* match_cur,
                                      int* nmatches);
int b2s_search_windows_grid(b2s_matcher* h, b2s_frame_grid* grid, const b2s_win_query* q, int nq, const uint8_t* occupied,
                            int flags, int th_dist, int32_t* best_idx, int32_t* best_dist, int* n_accepted);

/* ORBmatcher::SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize) — src/ORBmatcher.cc:515-643
 * (Tracking::MonocularInitialization, src/Tracking.cc:937-944).  prevx / prevy = vbPrevMatched; octave1 / angle1 / desc1 =
 * F1.mvKeysUn / F1.mDescriptors (only level-0 keypoints search, :537); the F2 side as for the other projection matchers;
 * window = windowSize; th_low = TH_LOW; nnratio / check_ori = the matcher's constructor arguments.
 * match12[i1] = F2 feature or -1 (vnMatches12); the caller then sets vbPrevMatched[i1] = F2.mvKeysUn[match12[i1]].pt
 * (:636-638). */
int b2s_search_for_initialization(b2s_matcher* h, const float* prevx, const float* prevy, const int32_t* octave1,
                                  const float* angle1, const uint8_t* desc1, int n1, const float* kpx2, const float* kpy2,
                                  const int32_t* octave2, const float* angle2, const uint8_t* desc2, int n2,
                                  const b2s_frame_geom* g, int window, int th_low, float nnratio, int check_ori,
                                  int32_t* match12, int* nmatches);

/* F12: 3x3 row-major float; (ex, ey): epipole of camera 1 in image 2 (:815-823); scale_factors / level_sigma2:
 * pKF2->mvScaleFactors / mvLevelSigma2.  match12[idx1] = idx2 or -1 (vMatchedPairs in ascending idx1). HOST buffers. */
int b2s_search_for_triangulation(b2s_matcher* h, const b2s_kf_features* kf1, const b2s_kf_features* kf2, const float* F12,
                                 float ex, float ey, const float* scale_factors, const float* level_sigma2, int nlevels,
                                 int only_stereo, int check_ori, int32_t* match12, int* nmatches);

/* MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:359-440; SURVEY.md §8f rank 4) for a batch of map points:
 * point p owns descriptors [offsets[p], offsets[p+1]) (its observations in map order, bad keyframes removed);
 * best_idx[p] = descriptor (relative index) with the least median distance to the others, -1 without descriptors. */
int b2s_distinctive_descriptors(b2s_matcher* h, const uint8_t* desc, const int32_t* offsets, int n_points,
                                int32_t* best_idx);

/* ------------------------------------------------------------------ DBoW2 vocabulary (SURVEY.md §8f rank 3) */
/* TemplatedVocabulary<FORB>::transform (Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1127-1256) as used by
 * Frame::ComputeBoW / KeyFrame::ComputeBoW (src/Frame.cc:880-896, src/KeyFrame.cc, levelsup = 4): it produces the word
 * ids / weights of mBowVec and the node ids of mFeatVec that SearchByBoW and SearchForTriangulation consume.
 * The vocabulary is passed flattened: node 0 = root, nodes 1..n-1 in the order of the text file (loadFromTextFile
 * :1338-1425: "parent isLeaf d0..d31 weight" per line); children keep the file order, word ids go to the flagged leaves in
 * file order. */
typedef struct {
  int32_t k, L, n_nodes;
  const int32_t* parent;    /* [n_nodes], parent[0] = -1; parents precede their children */
  const uint8_t* leaf_flag; /* [n_nodes] */
  const uint8_t* desc;      /* [n_nodes][32] */
  const double* weight;     /* [n_nodes] */
} b2s_vocabulary_desc;
typedef struct b2s_vocabulary b2s_vocabulary;
int b2s_vocabulary_create(const b2s_vocabulary_desc* d, int device, b2s_vocabulary** out);
void b2s_vocabulary_destroy(b2s_vocabulary* v);
int b2s_vocabulary_words(const b2s_vocabulary* v);
/* Per feature: word id, word weight (0 = stopped word, skipped by DBoW2; may be NULL), node id `levelsup` levels above the
 * leaves (0 = root when L - levelsup <= 0).  The host composes BowVector (sum of weights per word, L1-normalised) and
 * FeatureVector (features per node) from these arrays; the device variant feeds b2s_search_by_bow_device directly. */
int b2s_bow_transform(b2s_vocabulary* v, const uint8_t* features, int n, int levelsup, int32_t* word_id, double* weight,
                      int32_t* node_id);
int b2s_bow_transform_device(b2s_vocabulary* v, const uint8_t* d_features, int n, int levelsup, int32_t* d_word_id,
                             double* d_weight, int32_t* d_node_id, void* stream);

/* ------------------------------------------------------------------ keyframe database */
/* KeyFrameDatabase (src/KeyFrameDatabase.cc): place recognition over the BowVectors of the map's keyframes, with the
 * reference's candidate semantics (DetectLoopCandidates :104-239 for LoopClosing::DetectLoop, DetectRelocalizationCandidates
 * :252-374 for Tracking::Relocalization) and DBoW2's L1 score (Thirdparty/DBoW2/DBoW2/ScoringObject.cpp:23-68).
 * The BowVectors live in a device pool indexed by keyframe id; the per-keyframe query state of include/KeyFrame.h:328-338
 * (mnLoopQuery, mnLoopWords, mLoopScore, mnRelocQuery, mnRelocWords, mRelocScore) is owned by the database, starts at
 * 0 / 0 / 0.0f and persists across queries exactly as the reference's KeyFrame fields do (the results depend on it).
 * A BowVector is passed as `n` (word id, value) pairs in ascending word order (std::map order), n <= B2S_KFDB_MAX_WORDS
 * (longer: B2S_ERR_CAPACITY).  Keyframe ids are < 2^31.  Queries are serialised on the handle's stream; each does one
 * upload and one download.
 * covis: GetBestCovisibilityKeyFrames(10) of every keyframe at query time, by keyframe id: covis_ids[id*10 + k] for
 * k < covis_n[id], id < n_rows (rows at or beyond n_rows are empty).  Neighbours that are not in the database are allowed.
 * out_ids receives the candidates in the reference's order; *n_out = their number (B2S_ERR_CAPACITY if > cap). */
#define B2S_KFDB_MAX_WORDS 8192
typedef struct b2s_kfdb b2s_kfdb;
typedef struct {
  uint64_t loop_query;  /* mnLoopQuery */
  int32_t loop_words;   /* mnLoopWords */
  float loop_score;     /* mLoopScore */
  uint64_t reloc_query; /* mnRelocQuery */
  int32_t reloc_words;  /* mnRelocWords */
  float reloc_score;    /* mRelocScore */
} b2s_kfdb_state;
typedef struct {
  const uint64_t* ids;  /* [n_rows][10] */
  const int32_t* n;     /* [n_rows], each <= 10 */
  int32_t n_rows;
} b2s_kfdb_covis;
/* n_words = ORBVocabulary::size() (word ids must be below it) */
int b2s_kfdb_create(int n_words, int device, b2s_kfdb** out);
void b2s_kfdb_destroy(b2s_kfdb* db);
/* add(pKF) (:53-60).  A keyframe id that is already in the database: B2S_ERR_BAD_ARG (the system adds each keyframe once). */
int b2s_kfdb_add(b2s_kfdb* db, uint64_t kf_id, const uint32_t* words, const double* values, int n);
/* erase(pKF) (:63-84): no effect for an id that is not in the database; the keyframe's query state is kept. */
int b2s_kfdb_erase(b2s_kfdb* db, uint64_t kf_id);
/* clear() (:87-91); also resets every keyframe's query state (the system then reuses ids for new keyframes). */
int b2s_kfdb_clear(b2s_kfdb* db);
int b2s_kfdb_size(const b2s_kfdb* db, int* n);
/* DetectLoopCandidates(pKF, minScore): connected_ids = pKF->GetConnectedKeyFrames() (any order). */
int b2s_kfdb_detect_loop_candidates(b2s_kfdb* db, uint64_t query_kf_id, const uint32_t* words, const double* values, int n,
                                    const uint64_t* connected_ids, int n_connected, float min_score,
                                    const b2s_kfdb_covis* covis, uint64_t* out_ids, int cap, int* n_out);
/* DetectRelocalizationCandidates(F): frame_id = F->mnId. */
int b2s_kfdb_detect_relocalization_candidates(b2s_kfdb* db, uint64_t frame_id, const uint32_t* words, const double* values,
                                              int n, const b2s_kfdb_covis* covis, uint64_t* out_ids, int cap, int* n_out);
/* The query state of keyframe kf_id (the initial state for an id the database never saw). */
int b2s_kfdb_keyframe_state(b2s_kfdb* db, uint64_t kf_id, b2s_kfdb_state* state);
/* Device time (CUDA events on the handle's stream) of the kernels of the last query, in ms. */
float b2s_kfdb_last_query_ms(const b2s_kfdb* db);

/* ------------------------------------------------------------------ LocalBA */
typedef struct {
  int32_t kf;       /* index into Tcw[] */
  int32_t mp;       /* index into points[] */
  float obs[3];     /* kpUn.pt.x, kpUn.pt.y, mvuRight (<0: monocular edge, src/Optimizer.cc:794) */
  float inv_sigma2; /* mvInvLevelSigma2[octave] */
} b2s_ba_edge;

typedef struct {
  int n_kf;             /* local keyframes first [0,n_local), then fixed cameras */
  int n_local;
  const float* Tcw;     /* n_kf x 16, KeyFrame::GetPose() row-major 4x4 float */
  const uint8_t* fixed; /* n_kf: setFixed(true) (mnId==0 or lFixedCameras) */
  int n_mp;
  const float* points;  /* n_mp x 3, MapPoint::GetWorldPos() */
  int n_edges;
  const b2s_ba_edge* edges; /* insertion order of src/Optimizer.cc:770-853 */
  float fx, fy, cx, cy, bf;
  int its1, its2;       /* optimize(5), optimize(10) */
} b2s_ba_problem;

typedef struct {
  float* Tcw_out;        /* n_local x 16 (SetPose values) */
  float* points_out;     /* n_mp x 3 (SetWorldPos values) */
  uint8_t* edge_outlier; /* n_edges: 1 -> (KF,MP) goes to vToErase (:927-958) */
  int32_t* trace;        /* optional (>=256): accept(1)/reject(0) per LM trial, -1 terminated */
  double chi2_final;
  int n_trials;
} b2s_ba_result;

typedef struct b2s_ba_solver b2s_ba_solver;
int b2s_ba_create(int max_kf, int max_mp, int max_edges, int max_batch, int device, b2s_ba_solver** out);
void b2s_ba_destroy(b2s_ba_solver* h);
long long b2s_ba_launch_count(const b2s_ba_solver* h);
/* How many SMs (= thread blocks of the persistent LM kernel) one batched call may occupy; 0 = all of them (default).  A batch
 * of several windows deals this budget to the windows by estimated cost (the kernel ends with its slowest window).  All SMs
 * give the shortest LocalBA latency; a pipeline that runs other kernels next to LocalBA gets more total throughput from about
 * half of them, because a window's serial part (the reduced-system factorisation) idles fewer blocks.  One-window calls are
 * not affected (16 blocks). */
int b2s_ba_set_sm_budget(b2s_ba_solver* h, int sms);
/* Duration (CUDA events on the solver's stream) of the persistent LM kernel of the last b2s_local_ba(_batch) call and the
 * number of LM trials (accepted + rejected, all windows) it ran — measurement hook for bench.py's roofline. */
float b2s_ba_last_kernel_ms(const b2s_ba_solver* h, long long* lm_trials);
/* Optimizer::LocalBundleAdjustment from graph construction to write-back values. stop: pbStopFlag (may be NULL). */
int b2s_local_ba(b2s_ba_solver* h, const b2s_ba_problem* p, const volatile uint8_t* stop, b2s_ba_result* r);
/* `batch` independent windows solved concurrently (replicas; SURVEY.md §8e). */
int b2s_local_ba_batch(b2s_ba_solver* h, int batch, const b2s_ba_problem* p, b2s_ba_result* r);

/* ------------------------------------------------------------------ PoseOptimization (SURVEY.md §8f rank 2) */
/* Optimizer::PoseOptimization(Frame*) (src/Optimizer.cc:363-605) from graph construction to SetPose / mvbOutlier. */
typedef struct {
  const float* Tcw;        /* pFrame->mTcw, 16 floats row-major */
  int32_t n;               /* pFrame->N */
  const uint8_t* has_mp;   /* pFrame->mvpMapPoints[i] != NULL */
  const float* Xw;         /* pMP->GetWorldPos(), n x 3 (ignored where has_mp == 0) */
  const float* kpx;        /* mvKeysUn[i].pt.x */
  const float* kpy;
  const float* uright;     /* mvuRight[i]; < 0: monocular edge (:418) */
  const float* inv_sigma2; /* mvInvLevelSigma2[mvKeysUn[i].octave] */
  float fx, fy, cx, cy, bf;
} b2s_pose_problem;
typedef struct {
  float* Tcw_out;     /* 16 floats: the pose handed to pFrame->SetPose (:600-603) */
  uint8_t* outlier;   /* n: pFrame->mvbOutlier */
  int32_t* trace;     /* optional (>= 256): accept(1)/reject(0) per LM trial, -1 terminated */
  int32_t n_inliers;  /* return value: nInitialCorrespondences - nBad (:605) */
  int32_t n_trials;
} b2s_pose_result;
/* The handle is the LocalBA solver handle (b2s_ba_create); frames of a batch are independent (one CTA each). */
int b2s_pose_optimization(b2s_ba_solver* h, const b2s_pose_problem* p, b2s_pose_result* r);
int b2s_pose_optimization_batch(b2s_ba_solver* h, int batch, const b2s_pose_problem* p, b2s_pose_result* r);

/* ------------------------------------------------------------------ global bundle adjustment */
/* Optimizer::BundleAdjustment (src/Optimizer.cc:86-341), the body of GlobalBundleAdjustemnt: one Levenberg run of
 * `iterations` over every keyframe, map point and observation of the map (LoopClosing::RunGlobalBundleAdjustment, monocular
 * initialisation), from graph construction to the values handed to SetPose / SetWorldPos (or mTcwGBA / mPosGBA).
 * Keyframes without an edge and the fixed keyframes keep their estimate but are still written back through the Converter
 * quaternion round trip; points without an edge are excluded (vbNotIncludedMP) and their rows are not written.
 * With an empty graph, or the stop flag set before the first iteration, nothing is optimised and the write-back still
 * happens.  The LM loop runs on the host; every stage of a trial (linearisation, Schur complement, the tiled Cholesky of
 * the reduced camera system over its block envelope, the substitutions, the update) is FP64 kernels without
 * floating-point atomics, so two calls on the same input give bit-identical outputs. */
typedef struct {
  int n_kf;                 /* the non-bad keyframes, ascending mnId */
  const float* Tcw;         /* n_kf x 16, GetPose() */
  const uint8_t* fixed;     /* n_kf; the reference fixes exactly mnId == 0 (src/Optimizer.cc:132) */
  int n_mp;                 /* the non-bad map points, ascending mnId */
  const float* points;      /* n_mp x 3 */
  int n_edges;
  const b2s_ba_edge* edges; /* grouped by point (ascending), one per (keyframe, point) */
  float fx, fy, cx, cy, bf;
  int iterations;           /* nIterations */
  int robust;               /* bRobust: Huber sqrt(5.99) mono / sqrt(7.815) stereo, deltas passed as float (:141-142) */
} b2s_gba_problem;
typedef struct {
  float* Tcw_out;           /* n_kf x 16: every keyframe, via the Converter quaternion round trip (:294-308) */
  float* points_out;        /* n_mp x 3; rows of excluded points are not written */
  uint8_t* point_included;  /* n_mp: 0 = the point has no edge (vbNotIncludedMP, :266-274) */
  int32_t* trace;           /* optional (>= 256): accept(1)/reject(0) per LM trial, -1 terminated */
  double chi2_final;        /* robustified chi2 of the returned estimate */
  int n_trials;
} b2s_gba_result;
typedef struct b2s_gba_solver b2s_gba_solver;
/* Capacities of the problem arrays; the reduced-system storage is sized from each call's free keyframes and grows on
 * demand.  Supports at least max_kf = 2048, max_mp = 262144, max_edges = 2^21. */
int b2s_gba_create(int max_kf, int max_mp, int max_edges, int device, b2s_gba_solver** out);
void b2s_gba_destroy(b2s_gba_solver* h);
/* stop: pbStopFlag (may be NULL), polled before each iteration and in the trial loop.  Sizes above the handle's
 * capacities: B2S_ERR_CAPACITY; an index out of range, a duplicate (keyframe, point) pair or points not ascending:
 * B2S_ERR_BAD_ARG. */
int b2s_global_ba(b2s_gba_solver* h, const b2s_gba_problem* p, const volatile uint8_t* stop, b2s_gba_result* r);
/* Device time (CUDA events on the solver's stream) of the last b2s_global_ba call and the LM trials it ran. */
float b2s_gba_last_ms(const b2s_gba_solver* h, long long* lm_trials);

/* ------------------------------------------------------------------ essential graph */
/* Optimizer::OptimizeEssentialGraph (src/Optimizer.cc:1017-1339), the pose-graph step of LoopClosing::CorrectLoop: a Sim3
 * pose graph over every keyframe of the map, one fixed vertex (the loop keyframe), EdgeSim3 edges with identity
 * information, 20 Levenberg iterations from lambda 1e-16, g2o's numeric Jacobians (central differences, delta = 1e-9);
 * then every keyframe gets [R t/s; 0 1] of its optimised Sim3 and every point moves with its reference keyframe.
 * The caller builds the edge list and its measurements (the reference's loops :1108-1262, in their order); the device
 * never needs to know which pose an edge's measurement came from.  The LM loop runs on the host; every stage of a trial
 * is FP64 kernels without floating-point atomics, so two calls on the same input give bit-identical outputs.  With no
 * edge, nothing is optimised and everything is still written back. */
typedef struct {
  double q[4];  /* g2o::Sim3 operator[] order: qx qy qz qw, then t, then s */
  double t[3];
  double s;
} b2s_sim3;
typedef struct {
  int32_t i, j;   /* EdgeSim3: vertex 0 = keyframe i, vertex 1 = keyframe j */
  b2s_sim3 meas;  /* S_ji */
} b2s_sim3_edge;
typedef struct {
  int n_kf;                    /* the map's keyframes, ascending mnId */
  const b2s_sim3* Siw;         /* n_kf: initial estimates (vScw: CorrectedSim3 if present, else Sim3(Rcw, tcw, 1)) */
  int fixed_kf;                /* index of the loop keyframe, the only fixed vertex (:1086) */
  int fix_scale;               /* bFixScale: the scale component of every update is zeroed */
  int n_edges;
  const b2s_sim3_edge* edges;  /* in the reference's insertion order */
  int n_mp;                    /* the non-bad map points */
  const float* points;         /* n_mp x 3 */
  const int32_t* ref_kf;       /* n_mp: keyframe index of the point's nIDr (:1311-1322); -1: no such vertex, the point
                                  is written back unchanged */
} b2s_eg_problem;
typedef struct {
  float* Tcw_out;              /* n_kf x 16: SetPose([R t/s; 0 1]) of every keyframe (:1279-1299) */
  float* points_out;           /* n_mp x 3: correctedSwr.map(Srw.map(P)) (:1304-1338) */
  int32_t* trace;              /* optional (>= 256): accept(1)/reject(0) per LM trial, -1 terminated */
  double chi2_initial, chi2_final;
  int n_trials;
} b2s_eg_result;
typedef struct b2s_eg_solver b2s_eg_solver;
/* Capacities of the problem arrays; the tile storage of the factorisation is sized from each call's graph and grows on
 * demand.  Supports at least max_kf = 4096, max_edges = 2^17, max_mp = 2^22. */
int b2s_eg_create(int max_kf, int max_edges, int max_mp, int device, b2s_eg_solver** out);
void b2s_eg_destroy(b2s_eg_solver* h);
/* Sizes above the handle's capacities: B2S_ERR_CAPACITY.  An edge index out of range or i == j, fixed_kf out of range or a
 * ref_kf outside [-1, n_kf): B2S_ERR_BAD_ARG (the reference would dereference a missing vertex). */
int b2s_optimize_essential_graph(b2s_eg_solver* h, const b2s_eg_problem* p, b2s_eg_result* r);
/* Device time (CUDA events on the solver's stream) of the last call and the LM trials it ran. */
float b2s_eg_last_ms(const b2s_eg_solver* h, long long* lm_trials);

/* ------------------------------------------------------------------ Sim3 refinement (loop-closure verification) */
/* Optimizer::OptimizeSim3 (src/Optimizer.cc:1364-1590) after the graph is built: one free Sim3 S12 (fixed scale if
 * fix_scale), two Huber-robust projection edges per correspondence (S12 X2c into pKF1, S12^-1 X1c into pKF2), g2o's
 * numeric Jacobians (central differences, delta = 1e-9) and Levenberg steps; optimize(5), drop the pairs with an edge
 * chi2 above th2, return 0 if fewer than 10 remain, else optimize(10 if any was dropped, else 5) and count the inliers.
 * The caller applies the reference's skip rules (:1429-1520) and passes the surviving correspondences in its order.
 * One launch runs a whole batch, one CTA per problem; every sum is serial in edge order, so two calls on the same input
 * give bit-identical outputs and a batch equals its problems run one by one. */
typedef struct {
  int32_t n;                 /* correspondences that entered the graph, in the reference's order (vnIndexEdge) */
  const float* X1c;          /* n x 3: R1w*P3D1w + t1w as the caller's cv::Mat expression produced it */
  const float* X2c;          /* n x 3: R2w*P3D2w + t2w */
  const float* obs1;         /* n x 2: mvKeysUn[i] of pKF1 */
  const float* obs2;         /* n x 2: mvKeysUn[i2] of pKF2 */
  const float* inv_sigma2_1; /* n: pKF1->mvInvLevelSigma2[octave] */
  const float* inv_sigma2_2; /* n */
  float fx1, fy1, cx1, cy1, fx2, fy2, cx2, cy2;
  b2s_sim3 S12;              /* g2oS12 on entry */
  float th2;
  int32_t fix_scale;
} b2s_sim3_problem;
typedef struct {
  b2s_sim3 S12_out;          /* the optimised g2oS12; equals S12 on the early return */
  uint8_t* keep;             /* n: 0 -> vpMatches1[vnIndexEdge[k]] = NULL */
  int32_t* trace;            /* optional (>= 256): accept(1)/reject(0) per trial of both optimize() calls, -1 terminated */
  int32_t n_inliers;         /* the return value */
  int32_t n_trials;
} b2s_sim3_result;
typedef struct b2s_sim3opt_solver b2s_sim3opt_solver;
/* max_matches <= 65536 correspondences per problem, max_batch problems per call. */
int b2s_sim3opt_create(int max_matches, int max_batch, int device, b2s_sim3opt_solver** out);
void b2s_sim3opt_destroy(b2s_sim3opt_solver* h);
/* n > max_matches or batch > max_batch: B2S_ERR_CAPACITY.  batch < 1, n < 0, a null array with n > 0 or th2 <= 0:
 * B2S_ERR_BAD_ARG.  Nothing is written unless every problem is valid. */
int b2s_optimize_sim3(b2s_sim3opt_solver* h, int batch, const b2s_sim3_problem* p, b2s_sim3_result* r);
/* Device time (CUDA events on the solver's stream: upload, kernel, download) of the last call and its LM trials. */
float b2s_sim3opt_last_ms(const b2s_sim3opt_solver* h, long long* lm_trials);

/* ------------------------------------------------------------------ monocular initialisation */
/* Initializer::Initialize (src/Initializer.cc:68-231) with the minimal sets drawn by the caller (:132-168): normalise
 * both keypoint sets, score `iterations` homographies and fundamental matrices (ComputeH21 / ComputeF21 by Jacobi SVD,
 * CheckHomography / CheckFundamental), keep the first strict maximum of each, pick H when SH/(SH+SF) > 0.40 and
 * reconstruct the chosen model only (ReconstructH: 8 motion hypotheses, ReconstructF: 4) with minParallax = 1 and
 * minTriangulated = 50.  The cv::Mat arithmetic follows OpenCV's (float storage, double accumulators in gemm / dot /
 * norm, float scaling); DESIGN §7 lists it.  One call runs a batch of independent problems with no host synchronisation
 * between the stages; every score is a serial float sum in match order, so two calls give bit-identical outputs and a
 * batch equals its problems run one by one. */
typedef struct {
  int32_t n1, n2;             /* keypoints of the reference frame (1) and the current frame (2) */
  const float* kp1;           /* n1 x 2: mvKeysUn[i].pt of frame 1 */
  const float* kp2;           /* n2 x 2 */
  const int32_t* matches12;   /* n1: vMatches12, the frame-2 keypoint matched to frame-1 keypoint i, or < 0 */
  float K[9];                 /* mK, row-major */
  float sigma;
  int32_t iterations;         /* mMaxIterations */
  const int32_t* sets;        /* iterations x 8: mvSets, indices into the matches compacted in frame-1 order */
} b2s_init_problem;
typedef struct {
  int32_t ret;                /* Initialize's return value */
  int32_t model;              /* 1: homography (RH > 0.40), 2: fundamental matrix */
  int32_t rt_state;           /* R21 / t21: 1 written, -1 emptied (ReconstructF's failure after DecomposeE), 0 untouched */
  float R21[9], t21[3];
  float* p3d;                 /* n1 x 3: vP3D, written only when ret != 0 */
  uint8_t* triangulated;      /* n1: vbTriangulated, written only when ret != 0 */
  uint8_t* inliers_h;         /* optional, n_matches: the best homography's inlier flags */
  uint8_t* inliers_f;         /* optional, n_matches: the best fundamental matrix's inlier flags */
  int32_t n_matches;          /* matched frame-1 keypoints (the compacted match list's length) */
  int32_t best_h_iter, best_f_iter; /* -1 when no iteration scored above 0 */
  float SH, SF, RH;
  float H21[9], F21[9];       /* the best hypotheses (zero when none) */
  int32_t n_hyp;              /* motion hypotheses checked: 8 (H), 4 (F), 0 (ReconstructH's singular-value early-out) */
  int32_t n_good[8];          /* CheckRT's return value per hypothesis */
  float parallax[8];          /* CheckRT's parallax per hypothesis, degrees */
} b2s_init_result;
typedef struct b2s_init_solver b2s_init_solver;
/* max_keys keypoints per frame (<= 16384), max_iterations per problem, max_batch problems per call. */
int b2s_init_create(int max_keys, int max_iterations, int max_batch, int device, b2s_init_solver** out);
void b2s_init_destroy(b2s_init_solver* h);
/* n1, n2 > max_keys, iterations > max_iterations or batch > max_batch: B2S_ERR_CAPACITY.  batch < 1, sigma <= 0,
 * iterations < 1, n1 or n2 < 1, a null array, fewer than 8 matches, a match index outside [0, n2), a set index outside
 * [0, n_matches) or repeated within its set: B2S_ERR_BAD_ARG.  Nothing is written unless every problem is valid.  Where
 * neither model scored above 0 the reference would multiply an empty matrix; here the call returns 0 for that problem
 * with n_hyp = 0 and R21, t21, p3d and triangulated untouched. */
int b2s_initialize(b2s_init_solver* h, int batch, const b2s_init_problem* p, b2s_init_result* r);
/* Device time (CUDA events on the solver's stream: upload, kernels, download) of the last call. */
float b2s_init_last_ms(const b2s_init_solver* h);

/* ------------------------------------------------------------------ Sim3 RANSAC (loop-closure candidates) */
/* Sim3Solver::iterate (src/Sim3Solver.cc:199-285) with the minimal sets drawn by the caller: for each set, Horn's closed
 * form (ComputeSim3 :309-448: centroids, the 4 x 4 float Jacobi eigen, Rodrigues, scale, T12 and T21), CheckInliers in
 * both directions with the thresholds (size_t)(9.210 * sigma2), then the reference's scan: the best model replaced on
 * >=, an immediate return when an iteration has more than min_inliers inliers.  The solver state the reference keeps
 * across calls (mnIterations, mnBestInliers, the best model) goes in and comes out, so the ABI is stateless.  The
 * cv::Mat arithmetic follows OpenCV's; DESIGN §7 lists it.  One call runs a batch of independent solvers with no host
 * synchronisation between stages; inlier counts are integers, so a batch equals its problems run one by one. */
typedef struct {
  int32_t n;                  /* N: the correspondences the constructor kept (:78-127), in vpMatched12 order */
  const float* X1c;           /* n x 3: mvX3Dc1, Rcw1*Xw + tcw1 as the caller's cv::Mat expression produced it */
  const float* X2c;           /* n x 3: mvX3Dc2 */
  const float* sigma2_1;      /* n: pKF1->mvLevelSigma2[octave]; the threshold is (size_t)(9.210 * sigma2) */
  const float* sigma2_2;      /* n: pKF2->mvLevelSigma2[octave] */
  float K1[4], K2[4];         /* fx, fy, cx, cy of mK1 / mK2 */
  int32_t fix_scale;          /* mbFixScale */
  int32_t min_inliers;        /* mRansacMinInliers */
  int32_t max_its;            /* mRansacMaxIts after SetRansacParameters */
  int32_t iterations_done;    /* mnIterations on entry */
  int32_t best_inliers;       /* mnBestInliers on entry */
  int32_t k;                  /* minimal sets given: the iterations this call may run (<= max_its - iterations_done) */
  const int32_t* sets;        /* k x 3: indices into [0, n), in draw order; not read when n < min_inliers */
} b2s_sim3solver_problem;
typedef struct {
  int32_t returned;           /* 1: iterate returned mBestT12 (an iteration had more than min_inliers inliers) */
  float T12[16];              /* the returned T12, row-major 4 x 4, when returned */
  int32_t best_changed;       /* 1: an iteration of this call replaced the best model; R, t and s hold the new one */
  float R[9], t[3], s;        /* mBestRotation, mBestTranslation (3 x 1), mBestScale: written only when best_changed */
  uint8_t* inliers;           /* n: vbInliers in compacted order (entry i is vpMatched12[mvnIndices1[i]]); 0 unless
                                 returned */
  int32_t n_inliers;          /* nInliers: 0 unless returned */
  int32_t no_more;            /* bNoMore */
  int32_t iterations_used;    /* sets consumed by this call */
  int32_t iterations_done;    /* mnIterations after the call */
  int32_t best_inliers;       /* mnBestInliers after the call */
} b2s_sim3solver_result;
typedef struct b2s_sim3solver b2s_sim3solver;
/* max_matches correspondences (<= 65536) and max_sets sets per problem, max_batch problems per call. */
int b2s_sim3solver_create(int max_matches, int max_sets, int max_batch, int device, b2s_sim3solver** out);
void b2s_sim3solver_destroy(b2s_sim3solver* h);
/* n > max_matches, k > max_sets or batch > max_batch: B2S_ERR_CAPACITY.  batch < 1, a null array, n < 0, max_its < 1,
 * iterations_done < 0, best_inliers < 0, k < 0 or k > max_its - iterations_done, a sigma2 that is negative or not
 * finite, n < 3 where an iteration would run (n >= min_inliers and k > 0), a set index outside [0, n) or repeated within
 * its set: B2S_ERR_BAD_ARG.  Nothing is written unless every problem is valid.  Where n < min_inliers the call returns
 * no_more = 1 and consumes no set, as the reference does before it draws. */
int b2s_sim3solver_iterate(b2s_sim3solver* h, int batch, const b2s_sim3solver_problem* p, b2s_sim3solver_result* r);
/* Device time (CUDA events on the solver's stream: upload, kernels, download) of the last call. */
float b2s_sim3solver_last_ms(const b2s_sim3solver* h);

/* ---------------------------------------------------------------------------------------------------------------------
 * EPnP RANSAC for relocalisation candidates: PnPsolver::iterate (src/PnPsolver.cc:240-363) with the minimal sets drawn
 * by the caller.  Each iteration runs compute_pose (EPnP: control points, barycentric coordinates, the 12 x 12 SVD of
 * MtM, three beta approximations with 5 Gauss-Newton steps each) on its 4 correspondences and CheckInliers over all n;
 * then the reference's scan: the best model replaced on >, and on an iteration with at least min_inliers inliers a
 * Refine (compute_pose on the best mask's correspondences) that returns when it keeps more than min_inliers inliers.
 * The loop runs until iterations_done reaches max_its and at least the caller's nIterations times (its condition is
 * ||), so a call that does not return early runs exactly k iterations.  The solver state the reference keeps across
 * calls (mnIterations, mnBestInliers, mBestTcw, mvbBestInliers) goes in and comes out, so the ABI is stateless.  The
 * arithmetic is the reference's double precision with OpenCV's C API (cvMulTransposed, cvSVD, cvInvert, cvSolve) as
 * OpenCV computes it; DESIGN §7 lists it.  One call runs a batch of independent solvers with no host synchronisation
 * between stages; a batch equals its problems run one by one. */
typedef struct {
  int32_t n;                  /* N: the correspondences the constructor kept (:120-168), in vpMapPointMatches order */
  const float* P3Dw;          /* n x 3: mvP3Dw */
  const float* P2D;           /* n x 2: mvP2D (undistorted keypoints) */
  const float* sigma2;        /* n: mvSigma2, F.mvLevelSigma2[octave]; mvMaxError = sigma2 * th2 in float */
  float fu, fv, uc, vc;       /* F.fx, F.fy, F.cx, F.cy */
  float th2;                  /* SetRansacParameters' th2 */
  int32_t min_inliers;        /* mRansacMinInliers after SetRansacParameters */
  int32_t max_its;            /* mRansacMaxIts after SetRansacParameters */
  int32_t min_set;            /* mRansacMinSet: must be 4 */
  int32_t iterations_done;    /* mnIterations on entry */
  int32_t best_inliers;       /* mnBestInliers on entry */
  const float* best_Tcw;      /* 16: mBestTcw on entry, row-major (any values while best_inliers == 0) */
  const uint8_t* best_mask;   /* n: mvbBestInliers on entry (any values while best_inliers == 0) */
  int32_t k;                  /* minimal sets given: the iterations this call runs unless it returns early,
                                 max(nIterations, max_its - iterations_done); 0 when n < min_inliers */
  const int32_t* sets;        /* k x 4: indices into [0, n), in draw order; not read when n < min_inliers */
} b2s_pnpsolver_problem;
typedef struct {
  int32_t returned;           /* 1: iterate returned a pose (no_more = 0: a Refine succeeded, Tcw is mRefinedTcw;
                                 no_more = 1: the loop ended with best_inliers >= min_inliers, Tcw is mBestTcw) */
  float Tcw[16];              /* the returned pose, row-major 4 x 4, when returned */
  uint8_t* inliers;           /* n: vbInliers in compacted order (mvbRefinedInliers or mvbBestInliers); 0 unless
                                 returned */
  int32_t n_inliers;          /* nInliers: 0 unless returned */
  int32_t no_more;            /* bNoMore */
  int32_t iterations_used;    /* sets consumed by this call */
  int32_t iterations_done;    /* mnIterations after the call */
  int32_t best_inliers;       /* mnBestInliers after the call */
  int32_t best_changed;       /* 1: an iteration of this call replaced the best model */
  float best_Tcw[16];         /* mBestTcw after the call (the entry value when best_changed is 0) */
  uint8_t* best_mask;         /* n: mvbBestInliers after the call (the entry value when best_changed is 0) */
} b2s_pnpsolver_result;
typedef struct b2s_pnpsolver b2s_pnpsolver;
/* max_matches correspondences (<= 65536) and max_sets sets per problem, max_batch (<= 65535) problems per call. */
int b2s_pnpsolver_create(int max_matches, int max_sets, int max_batch, int device, b2s_pnpsolver** out);
void b2s_pnpsolver_destroy(b2s_pnpsolver* h);
/* n > max_matches, k > max_sets or batch > max_batch: B2S_ERR_CAPACITY.  batch < 1, a null array, n < 0, max_its < 1,
 * min_set != 4, iterations_done < 0, best_inliers < 0 or > n, k < 0, k < max_its - iterations_done where n >=
 * min_inliers (the loop cannot stop before max_its), a sigma2 that is negative or not finite, a set index outside
 * [0, n) or repeated within its set: B2S_ERR_BAD_ARG.  Nothing is written unless every problem is valid.  Where
 * n < min_inliers the call returns no_more = 1 and consumes no set, as the reference does before it draws. */
int b2s_pnpsolver_iterate(b2s_pnpsolver* h, int batch, const b2s_pnpsolver_problem* p, b2s_pnpsolver_result* r);
/* Device time (CUDA events on the solver's stream: upload, kernels, download) of the last call. */
float b2s_pnpsolver_last_ms(const b2s_pnpsolver* h);

#ifdef __cplusplus
}
#endif
#endif
