// TEST INFRASTRUCTURE — C entry points around the reference's own Frame (src/Frame.cc compiled in place, unmodified, with
// src/ORBextractor.cc and src/ORBmatcher.cc, against oracle/refshim with refshim/refshim_cv_undistort.h pre-included;
// MapPoint / KeyFrame / Converter / ORBVocabulary are the stand-ins of slam_stubs.h in B2S_STUB_REAL_FRAME mode).  The
// monocular (src/Frame.cc:351-458) and RGB-D (:238-348) constructors are built with a given calibration, distortion and
// depth image; UndistortKeyPoints / ComputeImageBounds run on the oracle's cv2-pinned cv::undistortPoints.  The glue
// exposes what they computed.  Built into oracle/_ref/libref_frame_undistort.so (oracle/undistort.mk, git-ignored);
// used only by tests.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <new>
#include <sys/mman.h>

#include "Frame.h"

using namespace ORB_SLAM2;

// The reference's DistributeOctTree breaks ties between equally large nodes by heap address (see ref_glue.cpp).  With
// ref_frame_set_monotonic_allocator(1) this library allocates from a bump arena, reset at each ref_frame_mono_rgbd, so
// the reference's extraction follows the rule the oracle and the device restate ("later-created node first"); by
// default it runs on the system malloc.
static int g_monotonic = 0;
static char* g_arena = nullptr;
static size_t g_off = 0;
static const size_t kArena = (size_t)3 << 30;
static void* arena_alloc(size_t n) {
  if (!g_arena) g_arena = (char*)mmap(nullptr, kArena, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
  const size_t a = (g_off + 15) & ~(size_t)15;
  if (a + n > kArena) std::abort();
  g_off = a + n;
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
std::unique_ptr<ORBextractor> g_ex;
std::unique_ptr<Frame> g_frame;
ORBVocabulary g_voc;

cv::Mat mat_f(const float* p, int r, int c) {
  cv::Mat m(r, c, CV_32F);
  for (int i = 0; i < r; i++)
    for (int j = 0; j < c; j++) m.at<float>(i, j) = p[i * c + j];
  return m;
}
void put_kp(const cv::KeyPoint& k, float* o) {
  o[0] = k.pt.x; o[1] = k.pt.y; o[2] = k.size; o[3] = k.angle; o[4] = k.response; o[5] = (float)k.octave; o[6] = (float)k.class_id;
}
}  // namespace

extern "C" {

void ref_frame_set_monotonic_allocator(int on) { g_monotonic = on; }

/* Frame(imGray, [imDepth,] ...) — the monocular constructor when depth is NULL, else the RGB-D one; depth: h x w floats
 * (row stride w).  K4 = fx fy cx cy, dist: n_dist coefficients.  Returns N. */
int ref_frame_mono_rgbd(const uint8_t* img, const float* depth, int w, int h, int nfeatures, float scaleFactor, int nlevels,
                        int iniTh, int minTh, const float* K4, const float* dist, int n_dist, float bf, float thDepth) {
  g_frame.reset();
  g_ex.reset();
  if (g_monotonic) g_off = 0;  // nothing this library allocated is alive any more
  g_ex.reset(new ORBextractor(nfeatures, scaleFactor, nlevels, iniTh, minTh));
  Frame::mbInitialComputations = true;  // recompute the image bounds / grid constants for this calibration (:321-340)
  cv::Mat im(h, w, CV_8UC1, (void*)img, (size_t)w);
  const float k[9] = {K4[0], 0, K4[2], 0, K4[1], K4[3], 0, 0, 1};
  cv::Mat K = mat_f(k, 3, 3), D = mat_f(dist, n_dist, 1);
  if (depth) {
    cv::Mat imD(h, w, CV_32F, (void*)depth, (size_t)w * 4);
    g_frame.reset(new Frame(im, imD, 0.0, g_ex.get(), &g_voc, K, D, bf, thDepth));
  } else {
    g_frame.reset(new Frame(im, 0.0, g_ex.get(), &g_voc, K, D, bf, thDepth));
  }
  return g_frame->N;
}

/* mvKeys and mvKeysUn (n x 7 floats each: x y size angle response octave class_id), mvuRight, mvDepth and
 * Frame::mnMinX, mnMaxX, mnMinY, mnMaxY of the frame built last */
void ref_frame_get_un(float* kps, float* kpsUn, float* uright, float* depth, float* bounds4) {
  Frame& F = *g_frame;
  for (int i = 0; i < F.N; i++) {
    put_kp(F.mvKeys[i], kps + 7 * (size_t)i);
    put_kp(F.mvKeysUn[i], kpsUn + 7 * (size_t)i);
    uright[i] = F.mvuRight[i];
    depth[i] = F.mvDepth[i];
  }
  bounds4[0] = Frame::mnMinX;
  bounds4[1] = Frame::mnMaxX;
  bounds4[2] = Frame::mnMinY;
  bounds4[3] = Frame::mnMaxY;
}

/* Frame::GetFeaturesInArea (src/Frame.cc:741-852) on the frame built last */
int ref_frame_features_in_area(float x, float y, float r, int minLevel, int maxLevel, int32_t* out, int cap) {
  std::vector<size_t> v = g_frame->GetFeaturesInArea(x, y, r, minLevel, maxLevel);
  if ((int)v.size() > cap) return -1;
  for (size_t i = 0; i < v.size(); i++) out[i] = (int32_t)v[i];
  return (int)v.size();
}
}
