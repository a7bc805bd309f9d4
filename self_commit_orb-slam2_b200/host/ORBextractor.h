// ORBextractor.h — header-compatible mirror of /root/reference/include/ORBextractor.h (class ORB_SLAM2::ORBextractor):
// same constructor, operator(), getters and public mvImagePyramid, so src/Frame.cc:494-515 and src/Tracking.cc:179-192
// compile against it unchanged.  The body runs on the GPU through libb200slam.so (include/b200slam.h).
#pragma once
#include <vector>

#include "../../include/b200slam.h"
#include "cv_compat.h"

namespace ORB_SLAM2 {

class ORBextractor {
 public:
  enum { HARRIS_SCORE = 0, FAST_SCORE = 1 };
  // include/ORBextractor.h:92
  ORBextractor(int nfeatures, float scaleFactor, int nlevels, int iniThFAST, int minThFAST);
  ~ORBextractor();
  ORBextractor(const ORBextractor&) = delete;
  ORBextractor& operator=(const ORBextractor&) = delete;

  // include/ORBextractor.h:110 — mask is ignored, exactly like the reference (src/ORBextractor.cc:1544-1668)
  void operator()(b2s_cv::InputArray image, b2s_cv::InputArray mask, std::vector<b2s_cv::KeyPoint>& keypoints,
                  b2s_cv::OutputArray descriptors);

  int inline GetLevels() { return nlevels; }
  float inline GetScaleFactor() { return (float)scaleFactor; }
  std::vector<float> inline GetScaleFactors() { return mvScaleFactor; }
  std::vector<float> inline GetInverseScaleFactors() { return mvInvScaleFactor; }
  std::vector<float> inline GetScaleSigmaSquares() { return mvLevelSigma2; }
  std::vector<float> inline GetInverseScaleSigmaSquares() { return mvInvLevelSigma2; }

  std::vector<b2s_cv::Mat> mvImagePyramid;  // filled after every operator() (Frame::ComputeStereoMatches reads it)

  // Device selection happens before the first image; B2S_DEVICE env var or SetDevice() (default 0).
  static void SetDevice(int device);
  // Skip the pyramid download when the caller does not need mvImagePyramid on the host (monocular / RGB-D frames).
  void SetDownloadPyramid(bool on) { mbDownloadPyramid = on; }

  // The calls the drop-in Frame (host/adapters/Frame_b200.cc) is built on.  None of them writes mvImagePyramid, whatever
  // SetDownloadPyramid says.  Each returns the library status (B2S_OK, or the code already reported on stderr with the
  // outputs cleared); descriptors are n x 32 bytes, row after row.
  //
  // One image (row stride `stride` bytes), as operator() without the pyramid download.
  int Extract(const uint8_t* image, int width, int height, size_t stride, std::vector<b2s_cv::KeyPoint>& keypoints,
              std::vector<uint8_t>& descriptors);
  // A same-sized stereo pair as one batch of two on this object's handle (image 0 = left, image 1 = right; the handle
  // grows to batch 2 once), then StereoMatch on it.  Images with different strides are packed to one stride first.
  int ExtractStereo(const uint8_t* left, size_t strideLeft, const uint8_t* right, size_t strideRight, int width, int height,
                    float bf, float mb, std::vector<b2s_cv::KeyPoint>& keypointsLeft, std::vector<uint8_t>& descriptorsLeft,
                    std::vector<b2s_cv::KeyPoint>& keypointsRight, std::vector<uint8_t>& descriptorsRight,
                    std::vector<float>& uRight, std::vector<float>& depth);
  // Frame::ComputeStereoMatches on the pair ExtractStereo extracted last, whose records and pyramids are still on the
  // device (b2s_stereo_match): n left features get mvuRight / mvDepth.
  int StereoMatch(float bf, float mb, int n, std::vector<float>& uRight, std::vector<float>& depth);
  // cv::undistortPoints(pts, K, dist, noArray(), K) on n points on this handle's device (b2s_undistort_points).
  int UndistortPoints(const float* xy, int n, const float* K4, const float* dist, int n_dist, float* xy_out);
  // Same constructor arguments: the two extractors give the same keypoints for the same image.
  bool SameParameters(const ORBextractor& other) const {
    return nfeatures == other.nfeatures && scaleFactor == other.scaleFactor && nlevels == other.nlevels &&
           iniThFAST == other.iniThFAST && minThFAST == other.minThFAST;
  }

 protected:
  int EnsureHandle(int width, int height, int batch = 1);  // B2S_OK with a handle for batch images of that size
  int nfeatures;
  double scaleFactor;
  int nlevels, iniThFAST, minThFAST;
  std::vector<int> mnFeaturesPerLevel;
  std::vector<float> mvScaleFactor, mvInvScaleFactor, mvLevelSigma2, mvInvLevelSigma2;
  b2s_extractor* mpHandle = nullptr;
  int mMaxW = 0, mMaxH = 0, mMaxBatch = 1;
  bool mbDownloadPyramid = true;
  std::vector<b2s_keypoint> mvTmpKeys;
  std::vector<uint8_t> mvPacked;  // ExtractStereo: the right image at the left image's stride
};

}  // namespace ORB_SLAM2
