/*
 * oracle/orb_oracle.h — C API of the CPU oracle.
 *
 * TEST INFRASTRUCTURE ONLY.  This is a CPU restatement of the reference algorithm for the hot
 * path (ORBextractor::operator(), ORBmatcher::SearchBy*, Optimizer::LocalBundleAdjustment of
 * DreamWaterFound/self_commit_ORB-SLAM2).  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs may load it.  The product (libb200slam.so) never links,
 * loads or calls anything in this directory.
 *
 * PARITY PINNING: the reference ships no tests or golden vectors (SURVEY.md §4) and its build
 * needs OpenCV C++/Eigen3/Pangolin (all absent).  The oracle is pinned where it can be:
 *  - OpenCV-owned stages (resize, FAST, GaussianBlur, fastAtan2): bit-for-bit against Python cv2
 *    4.13 (the same OpenCV code the reference links), tests/test_oracle_cv2.py;
 *  - the whole extractor (cell loop, quadtree, IC_Angle, rBRIEF): bit-for-bit against the
 *    reference's OWN src/ORBextractor.cc compiled in place against oracle/refshim (oracle/_ref,
 *    tests/test_oracle_reference_extractor.py);
 *  - every matcher (SearchByBoW x2, SearchByProjection x3, SearchForTriangulation, Fuse x2,
 *    SearchBySim3): match-for-match against the reference's OWN src/ORBmatcher.cc compiled in
 *    place against oracle/refshim (cv stand-in + Frame/KeyFrame/MapPoint data holders),
 *    oracle/_ref/libref_matcher.so, tests/test_oracle_reference_matcher.py;
 *  - the DBoW2 transform: exact (doubles included) against the reference's vendored
 *    Thirdparty/DBoW2 compiled in place (oracle/_ref/libref_dbow2.so,
 *    tests/test_oracle_reference_dbow2.py);
 *  - ComputeStereoMatches, the Frame feature grid, the isInFrustum -> SearchByProjection chain:
 *    against the reference's OWN src/Frame.cc compiled in place with its extractor and matcher
 *    (oracle/_ref/libref_frame.so, tests/test_oracle_reference_frame.py), float for float;
 *  - ComputeDistinctiveDescriptors: against the reference's OWN src/MapPoint.cc compiled in place
 *    (oracle/_ref/libref_mappoint.so, tests/test_oracle_reference_mappoint.py);
 *  - LocalBA, PoseOptimization: no independent pin ("parity unpinned", see DESIGN.md) —
 *    src/Optimizer.cc needs g2o + Eigen, and Eigen is not in this image.
 */
#ifndef ORB_ORACLE_H
#define ORB_ORACLE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* Layout-compatible with cv::KeyPoint (28 bytes): pt.x, pt.y, size, angle, response, octave, class_id */
typedef struct {
  float x, y, size, angle, response;
  int32_t octave, class_id;
} orc_keypoint;

/* ---------------- extractor (src/ORBextractor.cc) ---------------- */
void* orc_extractor_create(int nfeatures, float scaleFactor, int nlevels, int iniThFAST, int minThFAST);
void orc_extractor_destroy(void* h);
/* ORBextractor::operator() (src/ORBextractor.cc:1544-1668). Returns N (<= cap) or -1 if cap too small. */
int orc_extract(void* h, const uint8_t* img, int w, int hgt, int stride, orc_keypoint* kps, uint8_t* desc, int cap);
/* getters (include/ORBextractor.h:118-161) */
void orc_extractor_tables(void* h, float* scale, float* inv_scale, float* sigma2, float* inv_sigma2, int* nfeat_per_level,
                          int* umax16);
/* introspection of the last orc_extract() call (test hooks) */
int orc_level_dims(void* h, int level, int* w, int* hgt);
const uint8_t* orc_level_image(void* h, int level);   /* contiguous w*h, pyramid level (no border) */
const uint8_t* orc_level_blurred(void* h, int level); /* contiguous w*h, or NULL if the level had no keypoints */
int orc_level_candidates(void* h, int level, orc_keypoint* out, int cap); /* pre-quadtree, border-relative coords */
int orc_level_keypoints(void* h, int level, orc_keypoint* out, int cap);  /* post-quadtree, level coords, with angle */

/* OpenCV-owned primitives, restated (SURVEY.md §8c); cross-checked against cv2 in tests */
void orc_resize_linear_u8(const uint8_t* src, int sw, int sh, int sstride, uint8_t* dst, int dw, int dh, int dstride);
void orc_gaussian_blur7_s2_u8(const uint8_t* src, int w, int h, int sstride, uint8_t* dst, int dstride);
/* cv::FAST(roi, kps, th, true): returns count; xy = (x,y) pairs in ROI coords, resp = score */
int orc_fast9_16_nms(const uint8_t* roi, int w, int h, int stride, int th, int* xy, int* resp, int cap);
/* full score map M (corner at th <=> M > th, response = M-1), 0 on the 3-px rim */
void orc_fast_score_map(const uint8_t* roi, int w, int h, int stride, uint8_t* score, int score_stride);
float orc_fast_atan2(float y, float x);
/* quadtree alone: DistributeOctTree (src/ORBextractor.cc:706-1049) */
int orc_distribute_octtree(const orc_keypoint* in, int n, int minX, int maxX, int minY, int maxY, int N, orc_keypoint* out,
                           int cap);

/* ---------------- matcher (src/ORBmatcher.cc) ---------------- */
int orc_descriptor_distance(const uint8_t* a, const uint8_t* b); /* :1913-1933 */

/* SearchByBoW(KeyFrame*,Frame&,...) :230-382 and (KeyFrame*,KeyFrame*,...) :656-799 on flattened arrays.
 * descA/nodeA/validA/angA: the keyframe side ("KF"); descB/nodeB/angB: the frame side ("F").
 * node ids: features sharing a node id are candidates of each other; iteration order = ascending node id,
 * ascending feature index inside a node (std::map + push_back order, SURVEY A4).
 * strict_lt=0: accept best<=th_low (M1); strict_lt=1: best<th_low (M2).
 * matchB[j] = index into A or -1.  Returns nmatches. */
int orc_search_by_bow(const uint8_t* descA, const int32_t* nodeA, const uint8_t* validA, const float* angA, int nA,
                      const uint8_t* descB, const int32_t* nodeB, const uint8_t* validB, const float* angB, int nB,
                      int th_low, float nnratio, int strict_lt, int check_ori, int32_t* matchB);

/* Frame feature grid (src/Frame.cc:461-491, 741-877) + SearchByProjection(Cur,Last,th,mono) (:1569-1728).
 * Queries are the last frame's map points already projected by the host shim with the current pose. */
typedef struct {
  float u, v;          /* projection in the current frame */
  float invz;          /* 1/zc (float, as computed at :1614) */
  float angle;         /* LastFrame.mvKeysUn[i].angle */
  int32_t octave;      /* LastFrame.mvKeys[i].octave */
  int32_t has_obs;     /* pMP->Observations()>0 */
  uint8_t desc[32];    /* pMP->GetDescriptor() */
} orc_proj_query;

typedef struct {
  float mnMinX, mnMinY, mnMaxX, mnMaxY;
  float bf;            /* CurrentFrame.mbf */
  const float* scale_factors; /* mvScaleFactors[nlevels] */
  int nlevels;
} orc_frame_geom;

/* ORBmatcher::SearchForInitialization (src/ORBmatcher.cc:515-643): prev = vbPrevMatched; octave1/angle1/desc1 = F1's
 * undistorted keypoints; F2 side like the other projection matchers; window = windowSize (Tracking uses 100).
 * match12[i1] = F2 feature or -1; returns nmatches.  The caller then sets vbPrevMatched[i1] = F2 keypoint (:636-638). */
int orc_search_for_initialization(const float* prevx, const float* prevy, const int32_t* octave1, const float* angle1,
                                  const uint8_t* desc1, int n1, const float* kpx2, const float* kpy2, const int32_t* octave2,
                                  const float* angle2, const uint8_t* desc2, int n2, const orc_frame_geom* g, int window,
                                  int th_low, float nnratio, int check_ori, int32_t* match12);

/* Frame::GetFeaturesInArea (src/Frame.cc:741-852): indices in the reference's order; returns the count, -1 if > cap */
int orc_features_in_area(const float* kpx, const float* kpy, const int32_t* octave, int nf, const orc_frame_geom* g, float x,
                         float y, float r, int min_level, int max_level, int32_t* out, int cap);

/* feats: current frame; kpx,kpy,octave,angle from mvKeysUn; uright = mvuRight; occupied = feature already holds a
 * MapPoint with Observations()>0 (src/ORBmatcher.cc:1658-1660).
 * mode: 0 = neither forward nor backward (levels [oct-1, oct+1]), 1 = forward (>= oct), 2 = backward ([0, oct]).
 * match_cur[j] = query index or -1. Returns nmatches (as the reference counts them). */
int orc_search_by_projection_last(const orc_proj_query* q, int nq, const float* kpx, const float* kpy,
                                  const int32_t* octave, const float* angle, const float* uright,
                                  const uint8_t* occupied, const uint8_t* desc, int nf, const orc_frame_geom* g,
                                  float th, int mode, int th_high, int check_ori, int32_t* match_cur);

/* SearchByProjection(Frame& F, const vector<MapPoint*>& vpMapPoints, float th) — src/ORBmatcher.cc:70-175: the local-map
 * matcher of Tracking::SearchLocalPoints.  Queries are the local map points after Frame::isInFrustum
 * (src/Frame.cc:608-735) filled mTrackProjX/Y/XR, mnTrackScaleLevel, mTrackViewCos. */
typedef struct {
  float u, v, ur;      /* mTrackProjX, mTrackProjY, mTrackProjXR */
  float view_cos;      /* mTrackViewCos -> RadiusByViewingCos (:178-185) */
  int32_t level;       /* mnTrackScaleLevel (predicted level) */
  uint8_t in_view;     /* mbTrackInView && !isBad()  (:83-87) */
  uint8_t has_obs;     /* pMP->Observations()>0: the feature it is assigned to becomes occupied (:123-125) */
  uint8_t pad[2];
  uint8_t desc[32];    /* pMP->GetDescriptor() */
} orc_map_query;

/* match_cur[j] = query index or -1 (last writer wins, :168). Returns nmatches as the reference counts them. */
int orc_search_by_projection_map(const orc_map_query* q, int nq, const float* kpx, const float* kpy,
                                 const int32_t* octave, const float* uright, const uint8_t* occupied,
                                 const uint8_t* desc, int nf, const orc_frame_geom* g, float th, int th_high,
                                 float nnratio, int32_t* match_cur);

/* Windowed best-match search on a KeyFrame's grid — the common core of
 *   ORBmatcher::Fuse(KeyFrame*, const vector<MapPoint*>&, th)                      src/ORBmatcher.cc:1020-1174  (flags = CHI2)
 *   ORBmatcher::Fuse(KeyFrame*, cv::Mat Scw, vpPoints, th, vpReplacePoint)        :1179-1310                   (flags = 0)
 *   ORBmatcher::SearchByProjection(KeyFrame*, cv::Mat Scw, vpPoints, vpMatched, th) :388-512                    (flags = GREEDY)
 * after the caller projected the map points (u, v, ur), predicted the level and computed radius = th*scale[level].
 * Candidates: KeyFrame::GetFeaturesInArea(u, v, radius) (src/KeyFrame.cc:752-796), level in [min_level, max_level];
 * CHI2: reprojection gate e2*invSigma2[level] <= 7.8 (stereo feature, mvuRight >= 0) / 5.99 (mono) (:1097-1124);
 * GREEDY: a feature with occupied[idx] != 0 or chosen by an earlier query is skipped (:462-463,498-502).
 * best_idx[i] = feature with the smallest distance (first minimum) if that distance <= th_dist, else -1. */
typedef struct {
  float u, v, ur, radius;
  int32_t min_level, max_level;
  uint8_t valid, pad[3];
  uint8_t desc[32];
} orc_win_query;
#define ORC_WIN_CHI2 1
#define ORC_WIN_GREEDY 2
int orc_search_windows(const orc_win_query* q, int nq, const float* kpx, const float* kpy, const int32_t* octave,
                       const float* uright, const float* inv_level_sigma2, const uint8_t* occupied, const uint8_t* desc,
                       int nf, const orc_frame_geom* g, int flags, int th_dist, int32_t* best_idx, int32_t* best_dist);

/* ORBmatcher::SearchForTriangulation(KeyFrame* pKF1, KeyFrame* pKF2, cv::Mat F12, vMatchedPairs, bOnlyStereo)
 * (src/ORBmatcher.cc:810-1009) + CheckDistEpipolarLine (:186-215) on flattened keyframes.
 * node: DBoW2 FeatureVector node id per feature (features of a node are visited in ascending feature index, nodes in
 * ascending id); has_mp: pKF->GetMapPoint(idx) != NULL; stereo: mvuRight[idx] >= 0; x, y, octave, angle: mvKeysUn.
 * F12: 3x3 row-major float (F12.at<float>(r,c)); ex, ey: epipole of camera 1 in image 2 (:821-823);
 * scale_factors / level_sigma2: pKF2->mvScaleFactors / mvLevelSigma2.
 * match12[idx1] = idx2 or -1 (the vMatchedPairs list in ascending idx1). Returns nmatches. */
typedef struct {
  const uint8_t* desc;
  const int32_t* node;
  const uint8_t* has_mp;
  const uint8_t* stereo;
  const float* x;
  const float* y;
  const int32_t* octave;
  const float* angle;
  int32_t n;
} orc_kf_features;
int orc_search_for_triangulation(const orc_kf_features* kf1, const orc_kf_features* kf2, const float* F12, float ex, float ey,
                                 const float* scale_factors, const float* level_sigma2, int only_stereo, int check_ori,
                                 int32_t* match12);

/* DBoW2 TemplatedVocabulary<FORB>::transform (Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1127-1256) as used by
 * Frame::ComputeBoW / KeyFrame::ComputeBoW (src/Frame.cc:880-896, levelsup = 4) on a flattened vocabulary:
 * node 0 is the root; nodes 1..n-1 in the order of the text file (loadFromTextFile :1338-1425): parent id, leaf flag,
 * 32-byte descriptor, weight; children are visited in file order, word ids are assigned to the leaves in file order. */
typedef struct {
  int32_t k, L, n_nodes;
  const int32_t* parent;    /* [n_nodes], parent[0] = -1 */
  const uint8_t* leaf_flag; /* [n_nodes] nIsLeaf > 0 */
  const uint8_t* desc;      /* [n_nodes][32] */
  const double* weight;     /* [n_nodes] */
} orc_vocabulary;
/* per feature: word id, word weight (0 = stopped word: DBoW2 skips it), id of the node `levelsup` levels above the leaves */
int orc_bow_transform(const orc_vocabulary* v, const uint8_t* features, int n, int levelsup, int32_t* word_id, double* weight,
                      int32_t* node_id);

/* MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:359-440) for a batch of map points: point p owns the
 * descriptors [offsets[p], offsets[p+1]) (its observations in std::map<KeyFrame*,size_t> order, bad keyframes removed).
 * best_idx[p] = index (relative to offsets[p]) of the descriptor with the least median distance to the others
 * (median = sorted row [0.5*(N-1)], first minimum wins), or -1 for a point without descriptors. */
void orc_distinctive_descriptors(const uint8_t* desc, const int32_t* offsets, int n_points, int32_t* best_idx);

/* Frame::ComputeStereoMatches (src/Frame.cc:1026-1421): row-band candidates, Hamming best (< (TH_HIGH+TH_LOW)/2),
 * 11x11 L1 block matching over +-5 px on the keypoint's pyramid level, parabola sub-pixel fit, median*2.1 cull.
 * kps: level-0 coordinates as produced by the extractor; pyr*: dense level images (stride = width), lvlW/lvlH their
 * sizes; scale / inv_scale = mvScaleFactors / mvInvScaleFactors; mb = the baseline the reference sees at that point
 * (0 in this fork: it is assigned after the call, so maxD = +inf).  Outputs mvuRight / mvDepth (-1 = no match).
 * Returns the number of stereo matches that survive the cull.
 * orc_compute_stereo_matches_reason computes the same and, where reason is not NULL, writes per left keypoint the
 * decision that settled it (ORC_ST_*). */
enum {
  ORC_ST_KEPT = 0,       /* matched and kept by the cull */
  ORC_ST_KEPT_ZERO = 1,  /* kept, with disparity <= 0 replaced by 0.01 (bestuR = uL - 0.01 in double) */
  ORC_ST_NO_ROW = 2,     /* the left row has no right keypoint in its band (or lies outside the image) */
  ORC_ST_MAXU = 3,       /* maxU = uL - minD < 0 */
  ORC_ST_NO_CAND = 4,    /* no right keypoint of the row passes the octave and u gates */
  ORC_ST_HAMMING = 5,    /* best Hamming distance >= thOrbDist (75) */
  ORC_ST_WINDOW = 6,     /* the 11x11 windows leave the pyramid level (the iniu / endu test, or a range OpenCV asserts on) */
  ORC_ST_EDGE = 7,       /* SAD minimum at bestincR == +-L */
  ORC_ST_DELTA = 8,      /* parabola offset outside [-1, 1] */
  ORC_ST_DISPARITY = 9,  /* disparity outside [minD, maxD) */
  ORC_ST_CULLED = 10     /* matched, then removed by the median cull (SAD >= 1.5f*1.4f*median) */
};
int orc_compute_stereo_matches(const orc_keypoint* kpsL, const uint8_t* descL, int nL, const orc_keypoint* kpsR,
                               const uint8_t* descR, int nR, const uint8_t* const* pyrL, const uint8_t* const* pyrR,
                               const int* lvlW, const int* lvlH, const float* scale, const float* inv_scale, int nlevels,
                               float mbf, float mb, float* uright, float* depth);
int orc_compute_stereo_matches_reason(const orc_keypoint* kpsL, const uint8_t* descL, int nL, const orc_keypoint* kpsR,
                                      const uint8_t* descR, int nR, const uint8_t* const* pyrL, const uint8_t* const* pyrR,
                                      const int* lvlW, const int* lvlH, const float* scale, const float* inv_scale,
                                      int nlevels, float mbf, float mb, float* uright, float* depth, int32_t* reason);

/* ---------------- PoseOptimization (src/Optimizer.cc:363-605 + vendored g2o; SURVEY §8f rank 2) ---------------- */
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
} orc_pose_problem;
typedef struct {
  float* Tcw_out;     /* 16 floats: pFrame->SetPose(...) (:600-603) */
  uint8_t* outlier;   /* n: pFrame->mvbOutlier */
  int32_t* trace;     /* optional: accept(1)/reject(0) of every LM trial, -1 terminated, >= 256 entries */
  int32_t n_trials;
} orc_pose_result;
/* returns nInitialCorrespondences - nBad (:605) */
int orc_pose_optimization(const orc_pose_problem* p, orc_pose_result* r);

/* ---------------- LocalBA (src/Optimizer.cc:629-997 + vendored g2o) ---------------- */
typedef struct {
  int32_t kf;        /* index into poses[] */
  int32_t mp;        /* index into points[] */
  float obs[3];      /* kpUn.pt.x, kpUn.pt.y, mvuRight (<0 => mono edge) */
  float inv_sigma2;  /* mvInvLevelSigma2[octave] */
} orc_ba_edge;

typedef struct {
  int n_kf;               /* local KFs first [0,n_local), then fixed cameras */
  int n_local;            /* number of local keyframes (lLocalKeyFrames) */
  const float* Tcw;       /* n_kf x 16 (row-major 4x4 float, KeyFrame::GetPose) */
  const uint8_t* fixed;   /* n_kf: 1 => setFixed(true) (id==0 or fixed camera) */
  int n_mp;
  const float* points;    /* n_mp x 3 float (MapPoint::GetWorldPos) */
  int n_edges;
  const orc_ba_edge* edges; /* insertion order */
  float fx, fy, cx, cy, bf;
  int its1, its2;         /* 5, 10 */
} orc_ba_problem;

typedef struct {
  float* Tcw_out;          /* n_local x 16 */
  float* points_out;       /* n_mp x 3 */
  uint8_t* edge_outlier;   /* n_edges: 1 => goes to vToErase (src/Optimizer.cc:927-958) */
  int32_t* trace;          /* optional, >= 256 ints: accept(1)/reject(0) sequence of LM trials, -1 terminated */
  double chi2_final;
  int n_trials;
} orc_ba_result;

/* stop: optional async abort flag (pbStopFlag). Returns 0 ok, 1 aborted before round 1 (no write-back). */
int orc_local_ba(const orc_ba_problem* p, const volatile uint8_t* stop, orc_ba_result* r);

/* test hooks (tests/test_oracle_ba_math.py): the linear system of the first LM iteration at the initial estimate
 * (Hpp n_free x 36, Hll n_mp x 9, Hpl n_edges x 18 = per-edge 6x3 block, b = [poses | points]), its damped Schur solve
 * x for (H + lambda I) x = b, and the pose retraction exp(upd) * T (upd = [omega, upsilon]).  Returns n_free. */
int orc_ba_debug_linear_system(const orc_ba_problem* p, int robust, double lambda, double* Hpp, double* Hll, double* Hpl,
                               double* b, double* err, double* chi2, int32_t* pose_index, double* x);
void orc_se3_oplus(const float* Tcw16, const double* upd6, double* R9, double* t3);
/* PoseOptimization: the 6x6 system of the first LM iteration at the initial pose, its damped solve, per-edge error / chi2 */
int orc_po_debug_linear_system(const orc_pose_problem* p, int robust, double lambda, double* H36, double* b6, double* x6,
                               double* err, double* chi2);

/* ---------------- helpers (orb_misc.cpp) ---------------- */
void orc_sincosf_batch(const float* in, long n, float* s, float* c, int threads); /* glibc sinf/cosf */
int orc_extract_many(int nfeatures, float scaleFactor, int nlevels, int iniTh, int minTh, const uint8_t* imgs, int count,
                     int w, int h, orc_keypoint* kps, uint8_t* desc, int cap, int* n_out, int threads);

/* CPU reference arm of bench.py: extract 2S images + ring SearchByBoW (one node) + LocalBA every ba_every frames on
 * `threads` host threads; returns wall seconds. imgs: L_0..L_{S-1}, R_0..R_{S-1}, each w*h tightly packed. */
double orc_stream_step(int nfeatures, float scaleFactor, int nlevels, int iniTh, int minTh, const uint8_t* imgs, int S,
                       int w, int h, const orc_ba_problem* ba, int ba_every, int threads, int* out_counts);

#ifdef __cplusplus
}
#endif
#endif
