// TEST INFRASTRUCTURE — C entry points around a Frame implementation that hold SEVERAL frames: stereo, RGB-D and
// monocular frames built one after another by the Frame constructors (so mnId, nNextId and the first-frame-only
// computations follow the construction order), copies made by the copy constructor, and every member the later stages
// read.  Compiled twice by oracle/frame.mk, with the same flags and stand-ins (MapPoint / KeyFrame / Converter /
// ORBVocabulary of slam_stubs.h in B2S_STUB_REAL_FRAME mode):
//   _ref/libref_frame_seq.so    the reference's own src/Frame.cc + src/ORBextractor.cc + src/ORBmatcher.cc, unmodified,
//                               with refshim/refshim_cv_undistort.h's cv::undistortPoints;
//   _ref/libadapter_frame.so    the product's host/adapters/Frame_b200.cc + host/ORBextractor.cc over libb200slam.so,
//                               with refshim_cv.h alone (its cv::undistortPoints aborts: the drop-in must not call it).
// tests/test_frame_adapter_gpu.py loads both and compares them member for member.
//
// The reference's extraction breaks DistributeOctTree's ties by heap address (see ref_glue.cpp): with
// rfs_reset(1) this library allocates from a bump arena until the next rfs_reset, so the reference follows the rule the
// device states ("later-created node first").  rfs_reset destroys every frame and extractor first.
#include <atomic>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <new>
#include <sys/mman.h>
#include <vector>

#include "Frame.h"

using namespace ORB_SLAM2;

// The stereo constructor extracts on two threads: the bump is atomic, so each thread's allocations still come at
// increasing addresses.  The arena is mapped by rfs_reset, before any frame is built.
static int g_monotonic = 0;
static char* g_arena = nullptr;
static std::atomic<size_t> g_off(0);
static const size_t kArena = (size_t)6 << 30;
static void* arena_alloc(size_t n) {
  const size_t a = g_off.fetch_add((n + 15) & ~(size_t)15);
  if (a + n > kArena) std::abort();
  return g_arena + a;
}
void* operator new(size_t n) {
  void* p = g_monotonic ? arena_alloc(n) : std::malloc(n ? n : 1);
  if (!p) throw std::bad_alloc();
  return p;
}
void* operator new[](size_t n) { return operator new(n); }
static inline bool in_arena(void* p) { return g_arena && (char*)p >= g_arena && (char*)p < g_arena + kArena; }
void operator delete(void* p) noexcept {
  if (p && !in_arena(p)) std::free(p);
}
void operator delete[](void* p) noexcept { operator delete(p); }
void operator delete(void* p, size_t) noexcept { operator delete(p); }
void operator delete[](void* p, size_t) noexcept { operator delete(p); }

namespace {
std::vector<std::unique_ptr<ORBextractor> >* g_ex = nullptr;
std::vector<std::unique_ptr<Frame> >* g_frames = nullptr;
ORBVocabulary g_voc;

cv::Mat mat_f(const float* p, int r, int c) {
  cv::Mat m(r, c, CV_32F);
  for (int i = 0; i < r; i++)
    for (int j = 0; j < c; j++) m.at<float>(i, j) = p[i * c + j];
  return m;
}
cv::Mat K_of(const float* K4) {
  const float k[9] = {K4[0], 0, K4[2], 0, K4[1], K4[3], 0, 0, 1};
  return mat_f(k, 3, 3);
}
void put_kps(const std::vector<cv::KeyPoint>& v, float* o) {
  for (size_t i = 0; i < v.size(); i++) {
    const cv::KeyPoint& k = v[i];
    float* p = o + 7 * i;
    p[0] = k.pt.x; p[1] = k.pt.y; p[2] = k.size; p[3] = k.angle; p[4] = k.response; p[5] = (float)k.octave;
    p[6] = (float)k.class_id;
  }
}
void put_desc(const cv::Mat& d, uint8_t* o) {
  for (int i = 0; i < d.rows; i++) std::memcpy(o + 32 * (size_t)i, d.ptr(i), 32);
}
int push(Frame* f) {
  g_frames->emplace_back(f);
  return (int)g_frames->size() - 1;
}
Frame& F(int i) { return *(*g_frames)[i]; }
}  // namespace

extern "C" {

/* Destroys every frame and extractor, resets Frame::nNextId to 0 and Frame::mbInitialComputations to true; then
 * allocates from the bump arena (monotonic = 1) or the system allocator (0). */
void rfs_reset(int monotonic) {
  if (g_frames) {
    g_frames->clear();
    g_ex->clear();
  }
  g_monotonic = 0;
  delete g_frames;
  delete g_ex;
  g_off = 0;  // nothing allocated from the arena is alive any more
  if (monotonic && !g_arena) {
    void* a = mmap(nullptr, kArena, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
    if (a == MAP_FAILED) std::abort();
    g_arena = (char*)a;
  }
  g_monotonic = monotonic;
  g_frames = new std::vector<std::unique_ptr<Frame> >();
  g_ex = new std::vector<std::unique_ptr<ORBextractor> >();
  g_frames->reserve(64);
  g_ex->reserve(16);
  Frame::nNextId = 0;
  Frame::mbInitialComputations = true;
}

/* ORBextractor(nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST); returns its index */
int rfs_extractor(int nfeatures, float scaleFactor, int nlevels, int iniTh, int minTh) {
  g_ex->emplace_back(new ORBextractor(nfeatures, scaleFactor, nlevels, iniTh, minTh));
  return (int)g_ex->size() - 1;
}

/* Frame(imLeft, imRight, 0.0, ex[exL], ex[exR], voc, K, D, bf, thDepth): the two images may differ in size and row
 * stride.  K4 = fx fy cx cy, dist: n_dist coefficients.  Returns the frame's index. */
int rfs_stereo(int exL, int exR, const uint8_t* L, int wL, int hL, int strideL, const uint8_t* R, int wR, int hR, int strideR,
               const float* K4, const float* dist, int n_dist, float bf, float thDepth) {
  cv::Mat imL(hL, wL, CV_8UC1, (void*)L, (size_t)strideL), imR(hR, wR, CV_8UC1, (void*)R, (size_t)strideR);
  cv::Mat K = K_of(K4), D = mat_f(dist, n_dist, 1);
  return push(new Frame(imL, imR, 0.0, (*g_ex)[exL].get(), (*g_ex)[exR].get(), &g_voc, K, D, bf, thDepth));
}

/* The RGB-D constructor when depth != NULL (h x w floats, row stride w), else the monocular one.  Returns the index. */
int rfs_mono_rgbd(int ex, const uint8_t* img, int w, int h, const float* depth, const float* K4, const float* dist, int n_dist,
                  float bf, float thDepth) {
  cv::Mat im(h, w, CV_8UC1, (void*)img, (size_t)w);
  cv::Mat K = K_of(K4), D = mat_f(dist, n_dist, 1);
  if (depth) {
    cv::Mat imD(h, w, CV_32F, (void*)depth, (size_t)w * 4);
    return push(new Frame(im, imD, 0.0, (*g_ex)[ex].get(), &g_voc, K, D, bf, thDepth));
  }
  return push(new Frame(im, 0.0, (*g_ex)[ex].get(), &g_voc, K, D, bf, thDepth));
}

/* Frame(const Frame&) of frame f; returns the copy's index */
int rfs_copy(int f) { return push(new Frame(F(f))); }

/* counts[13]: [0..7] N, mvKeys, mvKeysUn, mvKeysRight, mvuRight, mvDepth, mvpMapPoints sizes, mnId;
 * [8..12] descriptor rows, right descriptor rows, mnScaleLevels, the number of mvpMapPoints that are not NULL
 * plus the number of mvbOutlier entries that are true, mvbOutlier's size.
 * scalars[5]: mbf, mb, mThDepth, mfScaleFactor, mfLogScaleFactor */
void rfs_info(int f, int64_t* counts, float* scalars) {
  Frame& Fr = F(f);
  counts[0] = Fr.N;
  counts[1] = (int64_t)Fr.mvKeys.size();
  counts[2] = (int64_t)Fr.mvKeysUn.size();
  counts[3] = (int64_t)Fr.mvKeysRight.size();
  counts[4] = (int64_t)Fr.mvuRight.size();
  counts[5] = (int64_t)Fr.mvDepth.size();
  counts[6] = (int64_t)Fr.mvpMapPoints.size();
  counts[7] = (int64_t)Fr.mnId;
  counts[8] = Fr.mDescriptors.empty() ? 0 : Fr.mDescriptors.rows;
  counts[9] = Fr.mDescriptorsRight.empty() ? 0 : Fr.mDescriptorsRight.rows;
  counts[10] = Fr.mnScaleLevels;
  int64_t set = 0;
  for (MapPoint* p : Fr.mvpMapPoints) set += p != NULL;
  for (bool b : Fr.mvbOutlier) set += b;
  counts[11] = set;
  counts[12] = (int64_t)Fr.mvbOutlier.size();
  scalars[0] = Fr.mbf;
  scalars[1] = Fr.mb;
  scalars[2] = Fr.mThDepth;
  scalars[3] = Fr.mfScaleFactor;
  scalars[4] = Fr.mfLogScaleFactor;
}

/* Arrays sized by rfs_info: keypoints n x 7 floats (x y size angle response octave class_id), descriptors n x 32,
 * mvuRight / mvDepth, and the four scale tables (mnScaleLevels floats each: factors, inverses, sigma2, inverse sigma2).
 * Any pointer may be NULL. */
void rfs_get(int f, float* kps, float* kpsUn, float* kpsR, uint8_t* desc, uint8_t* descR, float* uright, float* depth,
             float* tables) {
  Frame& Fr = F(f);
  if (kps) put_kps(Fr.mvKeys, kps);
  if (kpsUn) put_kps(Fr.mvKeysUn, kpsUn);
  if (kpsR) put_kps(Fr.mvKeysRight, kpsR);
  if (desc && !Fr.mDescriptors.empty()) put_desc(Fr.mDescriptors, desc);
  if (descR && !Fr.mDescriptorsRight.empty()) put_desc(Fr.mDescriptorsRight, descR);
  if (uright) std::memcpy(uright, Fr.mvuRight.data(), Fr.mvuRight.size() * 4);
  if (depth) std::memcpy(depth, Fr.mvDepth.data(), Fr.mvDepth.size() * 4);
  if (tables) {
    const int L = Fr.mnScaleLevels;
    const std::vector<float>* t[4] = {&Fr.mvScaleFactors, &Fr.mvInvScaleFactors, &Fr.mvLevelSigma2, &Fr.mvInvLevelSigma2};
    for (int k = 0; k < 4; k++)
      for (int l = 0; l < L; l++) tables[k * L + l] = (int)t[k]->size() > l ? (*t[k])[l] : -1.0f;
  }
}

/* out12: fx fy cx cy invfx invfy mnMinX mnMaxX mnMinY mnMaxY mfGridElementWidthInv mfGridElementHeightInv;
 * out2: nNextId, mbInitialComputations */
void rfs_statics(float* out12, int64_t* out2) {
  const float v[12] = {Frame::fx, Frame::fy, Frame::cx, Frame::cy, Frame::invfx, Frame::invfy, Frame::mnMinX, Frame::mnMaxX,
                       Frame::mnMinY, Frame::mnMaxY, Frame::mfGridElementWidthInv, Frame::mfGridElementHeightInv};
  std::memcpy(out12, v, sizeof v);
  out2[0] = (int64_t)Frame::nNextId;
  out2[1] = Frame::mbInitialComputations ? 1 : 0;
}

/* mGrid of frame f: counts[col * FRAME_GRID_ROWS + row] and the indices, cell after cell in that order.  Returns the
 * total, or -1 when it exceeds cap. */
int rfs_grid(int f, int32_t* counts, int32_t* idx, int cap) {
  Frame& Fr = F(f);
  int t = 0;
  for (int i = 0; i < FRAME_GRID_COLS; i++)
    for (int j = 0; j < FRAME_GRID_ROWS; j++) {
      const std::vector<size_t>& c = Fr.mGrid[i][j];
      counts[i * FRAME_GRID_ROWS + j] = (int32_t)c.size();
      for (size_t k = 0; k < c.size(); k++) {
        if (t >= cap) return -1;
        idx[t++] = (int32_t)c[k];
      }
    }
  return t;
}

/* Frame::GetFeaturesInArea on frame f; -1 when the result exceeds cap */
int rfs_features_in_area(int f, float x, float y, float r, int minLevel, int maxLevel, int32_t* out, int cap) {
  std::vector<size_t> v = F(f).GetFeaturesInArea(x, y, r, minLevel, maxLevel);
  if ((int)v.size() > cap) return -1;
  for (size_t i = 0; i < v.size(); i++) out[i] = (int32_t)v[i];
  return (int)v.size();
}

/* Frame::SetPose(Tcw) then Frame::isInFrustum(pMP, cosLimit) for n map points.  out: n x 4 (mTrackProjX, mTrackProjY,
 * mTrackProjXR, mTrackViewCos); level: mnTrackScaleLevel; in_view: the return value. */
void rfs_is_in_frustum(int f, const float* Tcw16, const float* pos, const float* normal, const float* minDist,
                       const float* maxDist, int n, float cosLimit, float* out, int32_t* level, uint8_t* in_view) {
  Frame& Fr = F(f);
  Fr.SetPose(mat_f(Tcw16, 4, 4));
  for (int i = 0; i < n; i++) {
    MapPoint p;
    p.mWorldPos = mat_f(pos + 3 * i, 3, 1);
    p.mNormal = mat_f(normal + 3 * i, 3, 1);
    p.mfMinDistance = minDist[i];
    p.mfMaxDistance = maxDist[i];
    in_view[i] = Fr.isInFrustum(&p, cosLimit) ? 1 : 0;
    out[4 * i + 0] = p.mTrackProjX;
    out[4 * i + 1] = p.mTrackProjY;
    out[4 * i + 2] = p.mTrackProjXR;
    out[4 * i + 3] = p.mTrackViewCos;
    level[i] = p.mnTrackScaleLevel;
  }
}

/* Frame::UnprojectStereo(i) with the pose of the last rfs_is_in_frustum call: 1 and xyz, or 0 for an empty matrix */
int rfs_unproject_stereo(int f, int i, float* xyz) {
  cv::Mat m = F(f).UnprojectStereo(i);
  if (m.empty()) return 0;
  for (int k = 0; k < 3; k++) xyz[k] = m.at<float>(k);
  return 1;
}

/* the size of ORBextractor::mvImagePyramid and of its level `level` (0 x 0 when it was never written) */
int rfs_pyramid_level(int ex, int level, int* w, int* h) {
  const std::vector<cv::Mat>& p = (*g_ex)[ex]->mvImagePyramid;
  *w = *h = 0;
  if (level < (int)p.size() && !p[level].empty()) {
    *w = p[level].cols;
    *h = p[level].rows;
  }
  return (int)p.size();
}
}
