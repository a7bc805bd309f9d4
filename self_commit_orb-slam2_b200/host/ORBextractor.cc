// ORBextractor.cc — host shim: reference signatures on top of the C ABI. No image processing happens here.
#include "ORBextractor.h"

#include <cmath>

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

void ORBextractor::EnsureHandle(int width, int height) {
  if (mpHandle && width <= mMaxW && height <= mMaxH) return;
  if (mpHandle) b2s_extractor_destroy(mpHandle);
  mpHandle = nullptr;
  mMaxW = std::max(width, mMaxW);
  mMaxH = std::max(height, mMaxH);
  int rc = b2s_extractor_create(nfeatures, (float)scaleFactor, nlevels, iniThFAST, minThFAST, std::max(64, mMaxW),
                                std::max(64, mMaxH), 1, g_device >= 0 ? g_device : b2s_host::device(), &mpHandle);
  if (rc != B2S_OK) {
    // The reference has neither exceptions nor return codes here (SURVEY.md §8b): report on stderr and leave the handle
    // empty; operator() then returns no keypoints, like the reference does for an empty image.  There is no CPU fallback.
    b2s_host::report("ORBextractor", rc);
    mpHandle = nullptr;
    return;
  }
  mvScaleFactor.resize(nlevels);
  mvInvScaleFactor.resize(nlevels);
  mvLevelSigma2.resize(nlevels);
  mvInvLevelSigma2.resize(nlevels);
  mnFeaturesPerLevel.resize(nlevels);
  b2s_extractor_tables(mpHandle, mvScaleFactor.data(), mvInvScaleFactor.data(), mvLevelSigma2.data(),
                       mvInvLevelSigma2.data(), mnFeaturesPerLevel.data());
  mvTmpKeys.resize(b2s_extractor_max_keypoints(mpHandle));
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

}  // namespace ORB_SLAM2
