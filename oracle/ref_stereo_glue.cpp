// TEST INFRASTRUCTURE — Frame::ComputeStereoMatches of the reference's own Frame (src/Frame.cc compiled in place,
// unmodified, with src/ORBextractor.cc and src/ORBmatcher.cc, against oracle/refshim; MapPoint / KeyFrame / Converter /
// ORBVocabulary are the stand-ins of slam_stubs.h in B2S_STUB_REAL_FRAME mode) on keypoints and descriptors the caller
// chooses.  Built into oracle/_ref/libref_stereo.so (git-ignored); used only by tests/test_stereo_edges.py.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <memory>
#include <vector>

#include "Frame.h"
#include "ORBmatcher.h"

using namespace ORB_SLAM2;

namespace {
std::unique_ptr<ORBextractor> g_exL, g_exR;
std::unique_ptr<Frame> g_frame;
ORBVocabulary g_voc;

cv::Mat mat_f(const float* p, int r, int c) {
  cv::Mat m(r, c, CV_32F);
  for (int i = 0; i < r; i++)
    for (int j = 0; j < c; j++) m.at<float>(i, j) = p[i * c + j];
  return m;
}

/* Frame(imLeft, imRight, ...) (src/Frame.cc:343-458) on the pair: the extractors keep the pair's pyramids */
void build_frame(const uint8_t* L, const uint8_t* R, int w, int h, int nfeatures, float scaleFactor, int nlevels, int iniTh,
                 int minTh, float bf) {
  g_frame.reset();
  g_exL.reset(new ORBextractor(nfeatures, scaleFactor, nlevels, iniTh, minTh));
  g_exR.reset(new ORBextractor(nfeatures, scaleFactor, nlevels, iniTh, minTh));
  Frame::mbInitialComputations = true;  // recompute the image bounds / grid constants for this image size (:424-446)
  cv::Mat imL(h, w, CV_8UC1, (void*)L, (size_t)w), imR(h, w, CV_8UC1, (void*)R, (size_t)w);
  const float k[9] = {500.f, 0, w * 0.5f, 0, 500.f, h * 0.5f, 0, 0, 1};
  const float d[4] = {0, 0, 0, 0};
  cv::Mat K = mat_f(k, 3, 3), D = mat_f(d, 4, 1);
  g_frame.reset(new Frame(imL, imR, 0.0, g_exL.get(), g_exR.get(), &g_voc, K, D, bf, 35.f));
}
}  // namespace

extern "C" {

/* Frame::ComputeStereoMatches (src/Frame.cc:1026-1421) on the caller's keypoints.  The Frame is built on the pair by
 * ref_frame_stereo, so the reference's extractors hold that pair's pyramids and the frame its scale tables; then N, mvKeys
 * (and mvKeysUn), mvKeysRight, both descriptor matrices, mbf and mb are overwritten through the public members and
 * ComputeStereoMatches runs once more.  kpsL / kpsR: n x 7 floats as ref_frame_get writes them.
 *
 * Input on which the reference is undefined is refused and nothing is computed (real OpenCV asserts in rowRange /
 * colRange, while the stand-in Mat reads past the level; vRowIndices is indexed unchecked):
 *   -1  N == 0 (the median reads vDistIdx[0] of an empty list)
 *   -2  an octave outside [0, nlevels)
 *   -3  a right keypoint whose band [floor(y-r), ceil(y+r)] leaves [0, rows), or a left row outside [0, rows)
 *   -4  a left keypoint with a candidate it could pick (row band, octave and u gates, Hamming < thOrbDist) whose 11x11
 *       window leaves its pyramid level, or whose right windows over +-5 px around that candidate would be read (the
 *       iniu / endu test passes) and leave the level. */
int ref_frame_stereo_inject(const uint8_t* L, const uint8_t* R, int w, int h, int nfeatures, float scaleFactor, int nlevels,
                            int iniTh, int minTh, const float* kpsL, const uint8_t* descL, int N, const float* kpsR,
                            const uint8_t* descR, int NR, float bf, float mb, float* uright, float* depth) {
  if (N <= 0) return -1;
  build_frame(L, R, w, h, nfeatures, scaleFactor, nlevels, iniTh, minTh, bf);
  Frame& F = *g_frame;
  const int nRows = g_exL->mvImagePyramid[0].rows;
  std::vector<cv::KeyPoint> kl(N), kr(NR);
  for (int i = 0; i < N + NR; i++) {
    const float* k = i < N ? kpsL + 7 * (size_t)i : kpsR + 7 * (size_t)(i - N);
    cv::KeyPoint kp(k[0], k[1], k[2], k[3], k[4], (int)k[5], (int)k[6]);
    if (kp.octave < 0 || kp.octave >= nlevels) return -2;
    (i < N ? kl[i] : kr[i - N]) = kp;
  }
  for (int iR = 0; iR < NR; iR++) {
    const float r = 2.0f * F.mvScaleFactors[kr[iR].octave];
    if ((int)std::floor(kr[iR].pt.y - r) < 0 || (int)std::ceil(kr[iR].pt.y + r) >= nRows) return -3;
  }
  const float maxD = bf / mb;
  for (int iL = 0; iL < N; iL++) {
    const cv::KeyPoint& kp = kl[iL];
    if (!(kp.pt.y >= 0.f) || (int)kp.pt.y >= nRows) return -3;
    const int lw = g_exL->mvImagePyramid[kp.octave].cols, lh = g_exL->mvImagePyramid[kp.octave].rows;
    const float inv = F.mvInvScaleFactors[kp.octave];
    const int cy = (int)std::round(kp.pt.y * inv), cxL = (int)std::round(kp.pt.x * inv);
    const bool leftIn = cy - 5 >= 0 && cy + 5 < lh && cxL - 5 >= 0 && cxL + 5 < lw;
    const int row = (int)kp.pt.y;
    for (int iR = 0; iR < NR; iR++) {
      const cv::KeyPoint& q = kr[iR];
      const float r = 2.0f * F.mvScaleFactors[q.octave];
      if (row < (int)std::floor(q.pt.y - r) || row > (int)std::ceil(q.pt.y + r)) continue;
      if (q.octave < kp.octave - 1 || q.octave > kp.octave + 1) continue;
      if (!(q.pt.x >= kp.pt.x - maxD && q.pt.x <= kp.pt.x - 0.f)) continue;
      if (ORBmatcher::DescriptorDistance(cv::Mat(1, 32, CV_8U, (void*)(descL + 32 * (size_t)iL), 32),
                                         cv::Mat(1, 32, CV_8U, (void*)(descR + 32 * (size_t)iR), 32)) >= (100 + 50) / 2)
        continue;
      if (!leftIn) return -4;
      const float su = std::round(q.pt.x * inv);
      const bool read = !(su < 0 || su + 11 >= lw);  // iniu = su, endu = su + 11 (:1269-1273)
      if (read && (int)su - 10 < 0) return -4;
    }
  }
  F.N = N;
  F.mvKeys = kl;
  F.mvKeysUn = kl;
  F.mvKeysRight = kr;
  F.mDescriptors = cv::Mat(N, 32, CV_8U);
  std::memcpy(F.mDescriptors.data, descL, 32 * (size_t)N);
  F.mDescriptorsRight = cv::Mat(std::max(NR, 1), 32, CV_8U);
  if (NR) std::memcpy(F.mDescriptorsRight.data, descR, 32 * (size_t)NR);
  F.mbf = bf;
  F.mb = mb;
  F.ComputeStereoMatches();
  for (int i = 0; i < N; i++) {
    uright[i] = F.mvuRight[i];
    depth[i] = F.mvDepth[i];
  }
  return 0;
}
}
