// ORBextractor.cc — host shim: reference signatures on top of the C ABI. No image processing happens here.
#include "ORBextractor.h"

#include <algorithm>
#include <cmath>
#include <cstring>

#include "b2s_host.h"

namespace ORB_SLAM2 {

static int g_device = -1;
void ORBextractor::SetDevice(int device) { g_device = device; }

ORBextractor::ORBextractor(int _nfeatures, float _scaleFactor, int _nlevels, int _iniThFAST, int _minThFAST)
    : nfeatures(_nfeatures), scaleFactor(_scaleFactor), nlevels(_nlevels), iniThFAST(_iniThFAST), minThFAST(_minThFAST) {
  mvImagePyramid.resize(nlevels);
  // The scale tables come from the library (same arithmetic as src/ORBextractor.cc:500-554); a 64x64 handle is enough
  // to read them, the real one is sized on the first image.
  EnsureHandle(64, 64);
}

ORBextractor::~ORBextractor() { b2s_extractor_destroy(mpHandle); }

int ORBextractor::EnsureHandle(int width, int height, int batch) {
  if (mpHandle && width <= mMaxW && height <= mMaxH && batch <= mMaxBatch) return B2S_OK;
  if (mpHandle) b2s_extractor_destroy(mpHandle);
  mpHandle = nullptr;
  mMaxW = std::max(width, mMaxW);
  mMaxH = std::max(height, mMaxH);
  mMaxBatch = std::max(batch, mMaxBatch);
  int rc = b2s_extractor_create(nfeatures, (float)scaleFactor, nlevels, iniThFAST, minThFAST, std::max(64, mMaxW),
                                std::max(64, mMaxH), mMaxBatch, g_device >= 0 ? g_device : b2s_host::device(), &mpHandle);
  if (rc != B2S_OK) {
    // The reference has neither exceptions nor return codes here (SURVEY.md §8b): report on stderr and leave the handle
    // empty; operator() then returns no keypoints, like the reference does for an empty image.  There is no CPU fallback.
    b2s_host::report("ORBextractor", rc);
    mpHandle = nullptr;
    return rc;
  }
  mvScaleFactor.resize(nlevels);
  mvInvScaleFactor.resize(nlevels);
  mvLevelSigma2.resize(nlevels);
  mvInvLevelSigma2.resize(nlevels);
  mnFeaturesPerLevel.resize(nlevels);
  b2s_extractor_tables(mpHandle, mvScaleFactor.data(), mvInvScaleFactor.data(), mvLevelSigma2.data(),
                       mvInvLevelSigma2.data(), mnFeaturesPerLevel.data());
  mvTmpKeys.resize(b2s_extractor_max_keypoints(mpHandle));
  return B2S_OK;
}

void ORBextractor::operator()(b2s_cv::InputArray _image, b2s_cv::InputArray /*_mask*/,
                              std::vector<b2s_cv::KeyPoint>& _keypoints, b2s_cv::OutputArray _descriptors) {
#ifdef B2S_HAVE_OPENCV
  if (_image.empty()) return;  // src/ORBextractor.cc:1553
  cv::Mat image = _image.getMat();
  assert(image.type() == CV_8UC1);
#else
  const b2s_cv::Mat& image = _image;
  if (image.empty()) return;
#endif
  EnsureHandle(image.cols, image.rows);
  if (!mpHandle) {  // no device / allocation failure (reported above): no keypoints
    _keypoints.clear();
    _descriptors.release();
    return;
  }
  std::vector<uint8_t*> pyr(nlevels, nullptr);
  if (mbDownloadPyramid) {
    for (int l = 0; l < nlevels; l++) {
      const int w = (int)lrintf((float)image.cols * mvInvScaleFactor[l]), h = (int)lrintf((float)image.rows * mvInvScaleFactor[l]);
#ifdef B2S_HAVE_OPENCV
      mvImagePyramid[l].create(h, w, CV_8UC1);
      pyr[l] = mvImagePyramid[l].data;
#else
      mvImagePyramid[l].create(h, w);
      pyr[l] = mvImagePyramid[l].data;
#endif
    }
  }
  const int cap = (int)mvTmpKeys.size();
  std::vector<uint8_t> desc((size_t)cap * 32);
  int n = 0;
  int rc = b2s_extract(mpHandle, image.data, image.cols, image.rows, (int)image.step, mvTmpKeys.data(), desc.data(), cap, &n,
                       mbDownloadPyramid ? pyr.data() : nullptr);
  if (rc != B2S_OK) {
    b2s_host::report("ORBextractor::operator()", rc);
    _keypoints.clear();
    _descriptors.release();
    return;
  }
  _keypoints.clear();
  _keypoints.resize(n);
  static_assert(sizeof(b2s_cv::KeyPoint) == sizeof(b2s_keypoint), "KeyPoint layout");
  if (n) memcpy((void*)_keypoints.data(), mvTmpKeys.data(), (size_t)n * sizeof(b2s_keypoint));
  if (n == 0) {
    _descriptors.release();  // :1590
    return;
  }
#ifdef B2S_HAVE_OPENCV
  _descriptors.create(n, 32, CV_8U);
  cv::Mat d = _descriptors.getMat();
  for (int i = 0; i < n; i++) memcpy(d.ptr(i), &desc[(size_t)i * 32], 32);
#else
  _descriptors.create(n, 32);
  memcpy(_descriptors.data, desc.data(), (size_t)n * 32);
#endif
}

// n records of `kps` -> keypoints, n descriptors of `desc` -> descriptors
static void take(const b2s_keypoint* kps, const uint8_t* desc, int n, std::vector<b2s_cv::KeyPoint>& keypoints,
                 std::vector<uint8_t>& descriptors) {
  keypoints.resize(n);
  if (n) memcpy((void*)keypoints.data(), kps, (size_t)n * sizeof(b2s_keypoint));
  descriptors.assign(desc, desc + (size_t)n * 32);
}

int ORBextractor::Extract(const uint8_t* image, int width, int height, size_t stride,
                          std::vector<b2s_cv::KeyPoint>& keypoints, std::vector<uint8_t>& descriptors) {
  keypoints.clear();
  descriptors.clear();
  if (!image || width <= 0 || height <= 0) return B2S_OK;  // an empty image has no keypoints (src/ORBextractor.cc:1553)
  int rc = EnsureHandle(width, height);
  if (!mpHandle) return rc != B2S_OK ? rc : B2S_ERR_NO_DEVICE;  // reported when the handle was made
  const int cap = (int)mvTmpKeys.size();
  std::vector<uint8_t> desc((size_t)cap * 32);
  int n = 0;
  rc = b2s_extract(mpHandle, image, width, height, (int)stride, mvTmpKeys.data(), desc.data(), cap, &n, nullptr);
  if (rc != B2S_OK) {
    b2s_host::report("ORBextractor::Extract", rc);
    return rc;
  }
  take(mvTmpKeys.data(), desc.data(), n, keypoints, descriptors);
  return B2S_OK;
}

int ORBextractor::ExtractStereo(const uint8_t* left, size_t strideLeft, const uint8_t* right, size_t strideRight, int width,
                                int height, float bf, float mb, std::vector<b2s_cv::KeyPoint>& keypointsLeft,
                                std::vector<uint8_t>& descriptorsLeft, std::vector<b2s_cv::KeyPoint>& keypointsRight,
                                std::vector<uint8_t>& descriptorsRight, std::vector<float>& uRight,
                                std::vector<float>& depth) {
  keypointsLeft.clear();
  keypointsRight.clear();
  descriptorsLeft.clear();
  descriptorsRight.clear();
  uRight.clear();
  depth.clear();
  if (!left || !right || width <= 0 || height <= 0) return B2S_OK;
  int rc = EnsureHandle(width, height, 2);
  if (!mpHandle) return rc != B2S_OK ? rc : B2S_ERR_NO_DEVICE;
  // one stride for both images: the right one is copied to the left one's when they differ
  if (strideRight != strideLeft) {
    mvPacked.resize(strideLeft * (size_t)(height - 1) + (size_t)width);
    for (int r = 0; r < height; r++) memcpy(&mvPacked[strideLeft * (size_t)r], right + strideRight * (size_t)r, (size_t)width);
    right = mvPacked.data();
  }
  const uint8_t* imgs[2] = {left, right};
  const int cap = (int)mvTmpKeys.size();
  std::vector<b2s_keypoint> kps((size_t)2 * cap);
  std::vector<uint8_t> desc((size_t)2 * cap * 32);
  int n[2] = {0, 0};
  rc = b2s_extract_batch(mpHandle, imgs, 2, width, height, (int)strideLeft, kps.data(), desc.data(), cap, n);
  if (rc != B2S_OK) {
    b2s_host::report("ORBextractor::ExtractStereo", rc);
    return rc;
  }
  rc = StereoMatch(bf, mb, n[0], uRight, depth);
  if (rc != B2S_OK) return rc;
  take(kps.data(), desc.data(), n[0], keypointsLeft, descriptorsLeft);
  take(kps.data() + cap, desc.data() + (size_t)cap * 32, n[1], keypointsRight, descriptorsRight);
  return B2S_OK;
}

int ORBextractor::StereoMatch(float bf, float mb, int n, std::vector<float>& uRight, std::vector<float>& depth) {
  uRight.clear();
  depth.clear();
  if (!mpHandle) return B2S_ERR_NO_DEVICE;  // reported when the handle was made
  const int cap = (int)mvTmpKeys.size();
  uRight.resize(cap);
  depth.resize(cap);
  int32_t matched = 0;
  const int rc = b2s_stereo_match(mpHandle, 0, 1, 1, bf, mb, uRight.data(), depth.data(), cap, &matched);
  if (rc != B2S_OK) {
    b2s_host::report("ORBextractor::StereoMatch", rc);
    uRight.clear();
    depth.clear();
    return rc;
  }
  uRight.resize(std::min(n, cap));
  depth.resize(std::min(n, cap));
  return B2S_OK;
}

int ORBextractor::UndistortPoints(const float* xy, int n, const float* K4, const float* dist, int n_dist, float* xy_out) {
  if (!mpHandle) return B2S_ERR_NO_DEVICE;
  const int rc = b2s_undistort_points(mpHandle, xy, n, K4, dist, n_dist, xy_out);
  if (rc != B2S_OK) b2s_host::report("ORBextractor::UndistortPoints", rc);
  return rc;
}

}  // namespace ORB_SLAM2
