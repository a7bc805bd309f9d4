// Frame_b200.cc — drop-in implementation of the reference's Frame class (include/Frame.h, unchanged) on top of
// libb200slam.so.  Compile this file INSIDE the reference tree in place of src/Frame.cc, next to the drop-in
// host/ORBextractor.{h,cc}, and link libb200slam.so.  Every member Frame.h declares is defined here with the same
// signature, and the same static members, so Tracking, KeyFrame, LocalMapping and LoopClosing compile and read them
// unchanged.
//
// Per frame, the work that touches pixels runs on the device:
//   * stereo:     ONE batch-2 extraction on the left extractor's handle (image 0 = left, image 1 = right), then
//                 b2s_stereo_match on the pyramids still resident there.  No pyramid is downloaded: the reference only
//                 downloads it for its CPU ComputeStereoMatches (src/Frame.cc:1026-1421, the one reader of
//                 mvImagePyramid).
//   * RGB-D:      ONE b2s_extract without the pyramid download, b2s_undistort_points on the keypoints when k1 != 0, and
//                 the depth lookup on the host (N floats of the caller's depth image: cheaper than uploading it).
//   * monocular:  ONE b2s_extract without the pyramid download and the same undistortion.
// ComputeImageBounds (first frame only) undistorts the four corners with b2s_undistort_points.  No OpenCV function runs
// on these paths; cv::Mat is only the container the header prescribes.
//
// The rest — the feature grid, GetFeaturesInArea, isInFrustum, the pose matrices, UnprojectStereo, ComputeBoW, the copy
// constructor — are host restatements in the reference's own expression order (file:line citations below), because
// KeyFrame copies mGrid and the later stages read these members: they must agree member for member.
//
// Errors: the reference has no error channel here.  A failed library call prints the one b2s_host::report line and the
// frame gets N = 0 (the reference's constructors return early for a frame without keypoints, as here).  The stereo
// constructor also refuses, with one stderr line, a pair the batch-2 call cannot take: left and right extractors built
// with different parameters, or images of different sizes (Tracking makes both extractors alike,
// src/Tracking.cc:179-189).
//
// tests: oracle/ref_frame_seq_glue.cpp drives this file (oracle/_ref/libadapter_frame.so) and the reference's own
// src/Frame.cc (oracle/_ref/libref_frame_seq.so) on the same inputs; tests/test_frame_adapter_gpu.py requires the same
// members, floats compared as bits.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "Converter.h"
#include "Frame.h"

#include "../b2s_host.h"

namespace ORB_SLAM2 {

// src/Frame.cc:42-52
long unsigned int Frame::nNextId = 0;
bool Frame::mbInitialComputations = true;
float Frame::cx, Frame::cy, Frame::fx, Frame::fy, Frame::invfx, Frame::invfy;
float Frame::mnMinX, Frame::mnMinY, Frame::mnMaxX, Frame::mnMaxY;
float Frame::mfGridElementWidthInv, Frame::mfGridElementHeightInv;

namespace {

// n rows of 32 descriptor bytes -> an n x 32 CV_8U matrix; no keypoints -> an empty matrix, as the extractor leaves it
void to_mat(const std::vector<uint8_t>& d, size_t n, cv::Mat& m) {
  if (n == 0) {
    m.release();
    return;
  }
  m.create((int)n, 32, CV_8U);
  for (size_t i = 0; i < n; i++) memcpy(m.ptr((int)i), &d[32 * i], 32);
}

// mK as the library's K4 = fx, fy, cx, cy
void k4_of(const cv::Mat& K, float* K4) {
  K4[0] = K.at<float>(0, 0);
  K4[1] = K.at<float>(1, 1);
  K4[2] = K.at<float>(0, 2);
  K4[3] = K.at<float>(1, 2);
}

// mDistCoef's entries: 4 or 5, whichever Tracking built (src/Tracking.cc:115-127)
std::vector<float> dist_of(const cv::Mat& D) {
  std::vector<float> d((size_t)D.rows * D.cols);
  for (size_t i = 0; i < d.size(); i++) d[i] = D.at<float>((int)i);
  return d;
}

// a frame without features: what the reference's constructors leave when the extraction found nothing
void drop_features(Frame& F) {
  F.N = 0;
  F.mvKeys.clear();
  F.mvKeysUn.clear();
  F.mvKeysRight.clear();
  F.mDescriptors.release();
  F.mDescriptorsRight.release();
  F.mvuRight.clear();
  F.mvDepth.clear();
  F.mvpMapPoints.clear();
  F.mvbOutlier.clear();
}

// UndistortKeyPoints (src/Frame.cc:899-964) with its status
int undistort_keys(Frame& F) {
  if (F.mDistCoef.at<float>(0) == 0.0) {  // :905-910: k1 == 0 means no distortion, whatever the other coefficients
    F.mvKeysUn = F.mvKeys;
    return B2S_OK;
  }
  std::vector<float> xy((size_t)2 * F.N);
  for (int i = 0; i < F.N; i++) {
    xy[2 * i] = F.mvKeys[i].pt.x;
    xy[2 * i + 1] = F.mvKeys[i].pt.y;
  }
  float K4[4];
  k4_of(F.mK, K4);
  const std::vector<float> dist = dist_of(F.mDistCoef);
  if (F.N > 0) {
    const int rc = F.mpORBextractorLeft->UndistortPoints(xy.data(), F.N, K4, dist.data(), (int)dist.size(), xy.data());
    if (rc != B2S_OK) return rc;
  }
  // :950-962: the distorted keypoint with the undistorted position
  F.mvKeysUn.resize(F.N);
  for (int i = 0; i < F.N; i++) {
    cv::KeyPoint kp = F.mvKeys[i];
    kp.pt.x = xy[2 * i];
    kp.pt.y = xy[2 * i + 1];
    F.mvKeysUn[i] = kp;
  }
  return B2S_OK;
}

// ComputeImageBounds (src/Frame.cc:967-1014) with its status: the undistorted corners (0,0), (cols,0), (0,rows),
// (cols,rows) when k1 != 0, else the image rectangle
int image_bounds(Frame& F, int cols, int rows) {
  if (F.mDistCoef.at<float>(0) != 0.0) {
    float c[8] = {0.0f, 0.0f, (float)cols, 0.0f, 0.0f, (float)rows, (float)cols, (float)rows};
    float K4[4];
    k4_of(F.mK, K4);
    const std::vector<float> dist = dist_of(F.mDistCoef);
    const int rc = F.mpORBextractorLeft->UndistortPoints(c, 4, K4, dist.data(), (int)dist.size(), c);
    if (rc != B2S_OK) return rc;
    Frame::mnMinX = min(c[0], c[4]);  // :999-1002
    Frame::mnMaxX = max(c[2], c[6]);
    Frame::mnMinY = min(c[1], c[3]);
    Frame::mnMaxY = max(c[5], c[7]);
  } else {
    Frame::mnMinX = 0.0f;  // :1007-1010
    Frame::mnMaxX = cols;
    Frame::mnMinY = 0.0f;
    Frame::mnMaxY = rows;
  }
  return B2S_OK;
}

// The first frame's computations (src/Frame.cc:207-226, 319-338, 429-450): image bounds, grid cell size, calibration.
int initial_computations(Frame& F, const cv::Mat& im, const cv::Mat& K) {
  const int rc = image_bounds(F, im.cols, im.rows);
  if (rc != B2S_OK) return rc;
  Frame::mfGridElementWidthInv = static_cast<float>(FRAME_GRID_COLS) / static_cast<float>(Frame::mnMaxX - Frame::mnMinX);
  Frame::mfGridElementHeightInv = static_cast<float>(FRAME_GRID_ROWS) / static_cast<float>(Frame::mnMaxY - Frame::mnMinY);
  Frame::fx = K.at<float>(0, 0);
  Frame::fy = K.at<float>(1, 1);
  Frame::cx = K.at<float>(0, 2);
  Frame::cy = K.at<float>(1, 2);
  Frame::invfx = 1.0f / Frame::fx;
  Frame::invfy = 1.0f / Frame::fy;
  Frame::mbInitialComputations = false;
  return B2S_OK;
}

}  // namespace

// src/Frame.cc:56-57
Frame::Frame() {}

// src/Frame.cc:61-104: deep copies of the matrices, the grid cell by cell, the pose matrices recomputed when set
Frame::Frame(const Frame& frame)
    : mpORBvocabulary(frame.mpORBvocabulary),
      mpORBextractorLeft(frame.mpORBextractorLeft),
      mpORBextractorRight(frame.mpORBextractorRight),
      mTimeStamp(frame.mTimeStamp),
      mK(frame.mK.clone()),
      mDistCoef(frame.mDistCoef.clone()),
      mbf(frame.mbf),
      mb(frame.mb),
      mThDepth(frame.mThDepth),
      N(frame.N),
      mvKeys(frame.mvKeys),
      mvKeysRight(frame.mvKeysRight),
      mvKeysUn(frame.mvKeysUn),
      mvuRight(frame.mvuRight),
      mvDepth(frame.mvDepth),
      mBowVec(frame.mBowVec),
      mFeatVec(frame.mFeatVec),
      mDescriptors(frame.mDescriptors.clone()),
      mDescriptorsRight(frame.mDescriptorsRight.clone()),
      mvpMapPoints(frame.mvpMapPoints),
      mvbOutlier(frame.mvbOutlier),
      mnId(frame.mnId),
      mpReferenceKF(frame.mpReferenceKF),
      mnScaleLevels(frame.mnScaleLevels),
      mfScaleFactor(frame.mfScaleFactor),
      mfLogScaleFactor(frame.mfLogScaleFactor),
      mvScaleFactors(frame.mvScaleFactors),
      mvInvScaleFactors(frame.mvInvScaleFactors),
      mvLevelSigma2(frame.mvLevelSigma2),
      mvInvLevelSigma2(frame.mvInvLevelSigma2) {
  for (int i = 0; i < FRAME_GRID_COLS; i++)
    for (int j = 0; j < FRAME_GRID_ROWS; j++) mGrid[i][j] = frame.mGrid[i][j];
  if (!frame.mTcw.empty()) SetPose(frame.mTcw);
}

// Stereo (src/Frame.cc:108-235).  This fork sets mb(0) and assigns mb = mbf/fx only after ComputeStereoMatches
// (:125, :231), so the matcher sees mb = 0 and its disparity bound mbf/mb is +inf: b2s_stereo_match gets mb = 0 too.
Frame::Frame(const cv::Mat& imLeft, const cv::Mat& imRight, const double& timeStamp, ORBextractor* extractorLeft,
             ORBextractor* extractorRight, ORBVocabulary* voc, cv::Mat& K, cv::Mat& distCoef, const float& bf,
             const float& thDepth)
    : mpORBvocabulary(voc),
      mpORBextractorLeft(extractorLeft),
      mpORBextractorRight(extractorRight),
      mTimeStamp(timeStamp),
      mK(K.clone()),
      mDistCoef(distCoef.clone()),
      mbf(bf),
      mb(0),
      mThDepth(thDepth),
      mpReferenceKF(static_cast<KeyFrame*>(NULL)) {
  mnId = nNextId++;  // :133

  // :141-153: the scale tables of the left extractor
  mnScaleLevels = mpORBextractorLeft->GetLevels();
  mfScaleFactor = mpORBextractorLeft->GetScaleFactor();
  mfLogScaleFactor = log(mfScaleFactor);
  mvScaleFactors = mpORBextractorLeft->GetScaleFactors();
  mvInvScaleFactors = mpORBextractorLeft->GetInverseScaleFactors();
  mvLevelSigma2 = mpORBextractorLeft->GetScaleSigmaSquares();
  mvInvLevelSigma2 = mpORBextractorLeft->GetInverseScaleSigmaSquares();

  // :159-167 and :186: both extractions and ComputeStereoMatches, as one batch-2 call on the left extractor's handle
  // (the right extractor is only checked to be alike: it would give the same keypoints)
  const bool sameSize = imLeft.cols == imRight.cols && imLeft.rows == imRight.rows;
  const bool sameParams = mpORBextractorLeft->SameParameters(*mpORBextractorRight);
  if (!sameSize || !sameParams) {
    fprintf(stderr, "Frame: stereo pair refused: %s; the frame has no features\n",
            !sameParams ? "the right extractor's parameters differ from the left one's"
                        : "the left and right images differ in size");
    drop_features(*this);
    return;
  }
  std::vector<uint8_t> descLeft, descRight;
  const int rc = mpORBextractorLeft->ExtractStereo(imLeft.data, (size_t)imLeft.step, imRight.data, (size_t)imRight.step,
                                                   imLeft.cols, imLeft.rows, mbf, mb, mvKeys, descLeft, mvKeysRight,
                                                   descRight, mvuRight, mvDepth);
  if (rc != B2S_OK) {  // reported by the extractor
    drop_features(*this);
    return;
  }
  to_mat(descLeft, mvKeys.size(), mDescriptors);
  to_mat(descRight, mvKeysRight.size(), mDescriptorsRight);

  N = mvKeys.size();  // :170-176
  if (mvKeys.empty()) return;

  if (undistort_keys(*this) != B2S_OK) {  // :181 (the stereo search read mvKeys, which this leaves as they are)
    drop_features(*this);
    return;
  }

  mvpMapPoints = vector<MapPoint*>(N, static_cast<MapPoint*>(NULL));  // :193-195
  mvbOutlier = vector<bool>(N, false);

  if (mbInitialComputations && initial_computations(*this, imLeft, K) != B2S_OK) {  // :207-226
    drop_features(*this);
    return;
  }

  mb = mbf / fx;  // :231

  AssignFeaturesToGrid();  // :234
}

// RGB-D (src/Frame.cc:238-348)
Frame::Frame(const cv::Mat& imGray, const cv::Mat& imDepth, const double& timeStamp, ORBextractor* extractor,
             ORBVocabulary* voc, cv::Mat& K, cv::Mat& distCoef, const float& bf, const float& thDepth)
    : mpORBvocabulary(voc),
      mpORBextractorLeft(extractor),
      mpORBextractorRight(static_cast<ORBextractor*>(NULL)),
      mTimeStamp(timeStamp),
      mK(K.clone()),
      mDistCoef(distCoef.clone()),
      mbf(bf),
      mThDepth(thDepth) {
  mnId = nNextId++;  // :259

  mnScaleLevels = mpORBextractorLeft->GetLevels();  // :265-277
  mfScaleFactor = mpORBextractorLeft->GetScaleFactor();
  mfLogScaleFactor = log(mfScaleFactor);
  mvScaleFactors = mpORBextractorLeft->GetScaleFactors();
  mvInvScaleFactors = mpORBextractorLeft->GetInverseScaleFactors();
  mvLevelSigma2 = mpORBextractorLeft->GetScaleSigmaSquares();
  mvInvLevelSigma2 = mpORBextractorLeft->GetInverseScaleSigmaSquares();

  ExtractORB(0, imGray);  // :283 (a failed extraction is reported and leaves no keypoints)

  N = mvKeys.size();  // :286-292
  if (mvKeys.empty()) return;

  if (undistort_keys(*this) != B2S_OK) {  // :299
    drop_features(*this);
    return;
  }

  ComputeStereoFromRGBD(imDepth);  // :302

  mvpMapPoints = vector<MapPoint*>(N, static_cast<MapPoint*>(NULL));  // :307-309
  mvbOutlier = vector<bool>(N, false);

  if (mbInitialComputations && initial_computations(*this, imGray, K) != B2S_OK) {  // :319-338
    drop_features(*this);
    return;
  }

  mb = mbf / fx;  // :344

  AssignFeaturesToGrid();  // :347
}

// Monocular (src/Frame.cc:351-458)
Frame::Frame(const cv::Mat& imGray, const double& timeStamp, ORBextractor* extractor, ORBVocabulary* voc, cv::Mat& K,
             cv::Mat& distCoef, const float& bf, const float& thDepth)
    : mpORBvocabulary(voc),
      mpORBextractorLeft(extractor),
      mpORBextractorRight(static_cast<ORBextractor*>(NULL)),
      mTimeStamp(timeStamp),
      mK(K.clone()),
      mDistCoef(distCoef.clone()),
      mbf(bf),
      mThDepth(thDepth) {
  mnId = nNextId++;  // :372

  mnScaleLevels = mpORBextractorLeft->GetLevels();  // :378-390
  mfScaleFactor = mpORBextractorLeft->GetScaleFactor();
  mfLogScaleFactor = log(mfScaleFactor);
  mvScaleFactors = mpORBextractorLeft->GetScaleFactors();
  mvInvScaleFactors = mpORBextractorLeft->GetInverseScaleFactors();
  mvLevelSigma2 = mpORBextractorLeft->GetScaleSigmaSquares();
  mvInvLevelSigma2 = mpORBextractorLeft->GetInverseScaleSigmaSquares();

  ExtractORB(0, imGray);  // :394

  N = mvKeys.size();  // :397-403
  if (mvKeys.empty()) return;

  if (undistort_keys(*this) != B2S_OK) {  // :407
    drop_features(*this);
    return;
  }

  mvuRight = vector<float>(N, -1);  // :411-412: no depth
  mvDepth = vector<float>(N, -1);

  mvpMapPoints = vector<MapPoint*>(N, static_cast<MapPoint*>(NULL));  // :417-419
  mvbOutlier = vector<bool>(N, false);

  if (mbInitialComputations && initial_computations(*this, imGray, K) != B2S_OK) {  // :429-450
    drop_features(*this);
    return;
  }

  mb = mbf / fx;  // :454

  AssignFeaturesToGrid();  // :457
}

// src/Frame.cc:461-491: every undistorted keypoint into the cell PosInGrid gives it, in index order
void Frame::AssignFeaturesToGrid() {
  int nReserve = 0.5f * N / (FRAME_GRID_COLS * FRAME_GRID_ROWS);
  for (unsigned int i = 0; i < FRAME_GRID_COLS; i++)
    for (unsigned int j = 0; j < FRAME_GRID_ROWS; j++) mGrid[i][j].reserve(nReserve);

  for (int i = 0; i < N; i++) {
    const cv::KeyPoint& kp = mvKeysUn[i];
    int nGridPosX, nGridPosY;
    if (PosInGrid(kp, nGridPosX, nGridPosY)) mGrid[nGridPosX][nGridPosY].push_back(i);
  }
}

// src/Frame.cc:494-515: flag 0 = left image -> mvKeys / mDescriptors, else right -> mvKeysRight / mDescriptorsRight.
// The extractor runs without its pyramid download.
void Frame::ExtractORB(int flag, const cv::Mat& im) {
  std::vector<uint8_t> desc;
  if (flag == 0) {
    mpORBextractorLeft->Extract(im.data, im.cols, im.rows, (size_t)im.step, mvKeys, desc);
    to_mat(desc, mvKeys.size(), mDescriptors);
  } else {
    mpORBextractorRight->Extract(im.data, im.cols, im.rows, (size_t)im.step, mvKeysRight, desc);
    to_mat(desc, mvKeysRight.size(), mDescriptorsRight);
  }
}

// src/Frame.cc:518-524
void Frame::SetPose(cv::Mat Tcw) {
  mTcw = Tcw.clone();
  UpdatePoseMatrices();
}

// src/Frame.cc:527-605
void Frame::UpdatePoseMatrices() {
  mRcw = mTcw.rowRange(0, 3).colRange(0, 3);
  mRwc = mRcw.t();
  mtcw = mTcw.rowRange(0, 3).col(3);
  mOw = -mRcw.t() * mtcw;  // the camera centre in world coordinates
}

// src/Frame.cc:608-738: projection, bounds, distance and viewing-angle gates, then the tracking fields of the point
bool Frame::isInFrustum(MapPoint* pMP, float viewingCosLimit) {
  pMP->mbTrackInView = false;

  cv::Mat P = pMP->GetWorldPos();
  const cv::Mat Pc = mRcw * P + mtcw;
  const float& PcX = Pc.at<float>(0);
  const float& PcY = Pc.at<float>(1);
  const float& PcZ = Pc.at<float>(2);
  if (PcZ < 0.0f) return false;  // :635

  const float invz = 1.0f / PcZ;  // :648-656
  const float u = fx * PcX * invz + cx;
  const float v = fy * PcY * invz + cy;
  if (u < mnMinX || u > mnMaxX) return false;
  if (v < mnMinY || v > mnMaxY) return false;

  const float maxDistance = pMP->GetMaxDistanceInvariance();  // :668-681
  const float minDistance = pMP->GetMinDistanceInvariance();
  const cv::Mat PO = P - mOw;
  const float dist = cv::norm(PO);
  if (dist < minDistance || dist > maxDistance) return false;

  cv::Mat Pn = pMP->GetNormal();  // :691-702
  const float viewCos = PO.dot(Pn) / dist;
  if (viewCos < viewingCosLimit) return false;

  const int nPredictedLevel = pMP->PredictScale(dist, this);  // :713

  pMP->mbTrackInView = true;  // :718-732
  pMP->mTrackProjX = u;
  pMP->mTrackProjXR = u - mbf * invz;
  pMP->mTrackProjY = v;
  pMP->mnTrackScaleLevel = nPredictedLevel;
  pMP->mTrackViewCos = viewCos;
  return true;
}

// src/Frame.cc:741-850: the cells the square [x-r, x+r] x [y-r, y+r] touches, column by column, and in them the
// undistorted keypoints strictly inside it (and within the level range when one is given)
vector<size_t> Frame::GetFeaturesInArea(const float& x, const float& y, const float& r, const int minLevel,
                                        const int maxLevel) const {
  vector<size_t> vIndices;
  vIndices.reserve(N);

  const int nMinCellX = max(0, (int)floor((x - mnMinX - r) * mfGridElementWidthInv));
  if (nMinCellX >= FRAME_GRID_COLS) return vIndices;
  const int nMaxCellX = min((int)FRAME_GRID_COLS - 1, (int)ceil((x - mnMinX + r) * mfGridElementWidthInv));
  if (nMaxCellX < 0) return vIndices;
  const int nMinCellY = max(0, (int)floor((y - mnMinY - r) * mfGridElementHeightInv));
  if (nMinCellY >= FRAME_GRID_ROWS) return vIndices;
  const int nMaxCellY = min((int)FRAME_GRID_ROWS - 1, (int)ceil((y - mnMinY + r) * mfGridElementHeightInv));
  if (nMaxCellY < 0) return vIndices;

  const bool bCheckLevels = (minLevel > 0) || (maxLevel >= 0);  // :792

  for (int ix = nMinCellX; ix <= nMaxCellX; ix++) {
    for (int iy = nMinCellY; iy <= nMaxCellY; iy++) {
      const vector<size_t>& vCell = mGrid[ix][iy];  // (the reference copies the cell; reading it in place is the same)
      for (size_t j = 0, jend = vCell.size(); j < jend; j++) {
        const cv::KeyPoint& kpUn = mvKeysUn[vCell[j]];
        if (bCheckLevels) {
          if (kpUn.octave < minLevel) continue;
          if (maxLevel >= 0)
            if (kpUn.octave > maxLevel) continue;
        }
        const float distx = kpUn.pt.x - x;
        const float disty = kpUn.pt.y - y;
        if (fabs(distx) < r && fabs(disty) < r) vIndices.push_back(vCell[j]);
      }
    }
  }
  return vIndices;
}

// src/Frame.cc:854-877
bool Frame::PosInGrid(const cv::KeyPoint& kp, int& posX, int& posY) {
  posX = round((kp.pt.x - mnMinX) * mfGridElementWidthInv);
  posY = round((kp.pt.y - mnMinY) * mfGridElementHeightInv);
  if (posX < 0 || posX >= FRAME_GRID_COLS || posY < 0 || posY >= FRAME_GRID_ROWS) return false;
  return true;
}

// src/Frame.cc:880-896 (the drop-in ORBVocabulary runs the descent on the device)
void Frame::ComputeBoW() {
  if (mBowVec.empty()) {
    vector<cv::Mat> vCurrentDesc = Converter::toDescriptorVector(mDescriptors);
    mpORBvocabulary->transform(vCurrentDesc, mBowVec, mFeatVec, 4);
  }
}

// src/Frame.cc:899-964 on the device (b2s_undistort_points).  A failure is reported and leaves mvKeysUn = mvKeys; the
// constructors, which call undistort_keys directly, give the frame N = 0 instead.
void Frame::UndistortKeyPoints() {
  if (undistort_keys(*this) != B2S_OK) mvKeysUn = mvKeys;
}

// src/Frame.cc:967-1014 on the device (b2s_undistort_points on the four corners).  A failure is reported and leaves the
// bounds as they were.
void Frame::ComputeImageBounds(const cv::Mat& imLeft) { image_bounds(*this, imLeft.cols, imLeft.rows); }

// src/Frame.cc:1026-1421 on the device: the pair the stereo constructor extracted is still resident on the left
// extractor's handle (records and pyramids), so this matches it again with the current mbf / mb.  A failure is reported
// and leaves every feature without a stereo match (-1).
void Frame::ComputeStereoMatches() {
  if (mpORBextractorLeft->StereoMatch(mbf, mb, N, mvuRight, mvDepth) != B2S_OK) {
    mvuRight = vector<float>(N, -1.0f);
    mvDepth = vector<float>(N, -1.0f);
  }
}

// src/Frame.cc:1423-1461 on the host: the depth at row (int)y, column (int)x of the distorted keypoint; a positive depth
// (not 0, negative or NaN) gives mvDepth and mvuRight = x_undistorted - mbf / d.  A keypoint whose truncated position is
// outside the image gets -1, as on the device (b2s_stereo_from_depth_device); the reference would read outside it.
void Frame::ComputeStereoFromRGBD(const cv::Mat& imDepth) {
  mvuRight = vector<float>(N, -1);
  mvDepth = vector<float>(N, -1);
  for (int i = 0; i < N; i++) {
    const cv::KeyPoint& kp = mvKeys[i];
    const cv::KeyPoint& kpU = mvKeysUn[i];
    const int v = (int)kp.pt.y;
    const int u = (int)kp.pt.x;
    if (v < 0 || v >= imDepth.rows || u < 0 || u >= imDepth.cols) continue;
    const float d = imDepth.at<float>(v, u);
    if (d > 0) {
      mvDepth[i] = d;
      mvuRight[i] = kpU.pt.x - mbf / d;
    }
  }
}

// src/Frame.cc:1464-1500: the keypoint's depth back-projected and moved to world coordinates; an empty matrix without
// depth
cv::Mat Frame::UnprojectStereo(const int& i) {
  const float z = mvDepth[i];
  if (z > 0) {
    const float u = mvKeysUn[i].pt.x;
    const float v = mvKeysUn[i].pt.y;
    const float x = (u - cx) * z * invfx;
    const float y = (v - cy) * z * invfy;
    cv::Mat x3Dc = (cv::Mat_<float>(3, 1) << x, y, z);
    return mRwc * x3Dc + mOw;
  } else
    return cv::Mat();
}

}  // namespace ORB_SLAM2
