// oracle/orb_stereo.cpp — CPU restatement of Frame::ComputeStereoMatches (src/Frame.cc:1026-1421).
// TEST INFRASTRUCTURE ONLY (see orb_oracle.h).  Arithmetic follows the reference statement by statement: float
// keypoint coordinates, C round() (half away from zero), integer-valued float SAD, float parabola fit.
#include <algorithm>
#include <climits>
#include <cmath>
#include <utility>
#include <vector>

#include "orb_oracle.h"

namespace {
const int TH_HIGH = 100, TH_LOW = 50;  // include/ORBmatcher.h:199-200
}

extern "C" int orc_compute_stereo_matches_reason(const orc_keypoint* kpsL, const uint8_t* descL, int N,
                                                 const orc_keypoint* kpsR, const uint8_t* descR, int Nr,
                                                 const uint8_t* const* pyrL, const uint8_t* const* pyrR, const int* lvlW,
                                                 const int* lvlH, const float* scale, const float* inv_scale, int nlevels,
                                                 float mbf, float mb, float* mvuRight, float* mvDepth, int32_t* reason) {
  (void)nlevels;
  int32_t noReason = 0;  // where reason is NULL every write goes here
  auto why = [&](int i) -> int32_t& { return reason ? reason[i] : noReason; };
  for (int i = 0; i < N; i++) {  // :1029-1030
    mvuRight[i] = -1.0f;
    mvDepth[i] = -1.0f;
  }
  const int thOrbDist = (TH_HIGH + TH_LOW) / 2;  // :1041
  const int nRows = lvlH[0];                     // mvImagePyramid[0].rows (:1044)
  // row-band table of the right keypoints (:1060-1097).  The reference indexes vRowIndices[yi] unchecked; keypoints
  // are >= 19 level-pixels away from the border so the band never leaves the image; the clamp only guards bad input.
  std::vector<std::vector<size_t> > vRowIndices(nRows);
  for (int iR = 0; iR < Nr; iR++) {
    const float kpY = kpsR[iR].y;
    const float r = 2.0f * scale[kpsR[iR].octave];
    const int maxr = (int)std::ceil(kpY + r);
    const int minr = (int)std::floor(kpY - r);
    for (int yi = std::max(minr, 0); yi <= std::min(maxr, nRows - 1); yi++) vRowIndices[yi].push_back(iR);
  }
  const float minZ = mb;  // :1108 (the reference runs this before mb is assigned; the caller passes what it would see)
  const float minD = 0;
  const float maxD = mbf / minZ;
  std::vector<std::pair<int, int> > vDistIdx;
  vDistIdx.reserve(N);
  for (int iL = 0; iL < N; iL++) {
    const orc_keypoint& kpL = kpsL[iL];
    const int levelL = kpL.octave;
    const float vL = kpL.y, uL = kpL.x;
    const int row = (int)vL;  // vRowIndices[vL]: float -> index conversion truncates
    why(iL) = ORC_ST_NO_ROW;
    if (row < 0 || row >= nRows) continue;
    const std::vector<size_t>& vCandidates = vRowIndices[row];
    if (vCandidates.empty()) continue;
    const float minU = uL - maxD, maxU = uL - minD;
    why(iL) = ORC_ST_MAXU;
    if (maxU < 0) continue;
    int bestDist = TH_HIGH;
    size_t bestIdxR = 0;
    why(iL) = ORC_ST_NO_CAND;
    for (size_t iC = 0; iC < vCandidates.size(); iC++) {  // :1169-1219
      const size_t iR = vCandidates[iC];
      const orc_keypoint& kpR = kpsR[iR];
      if (kpR.octave < levelL - 1 || kpR.octave > levelL + 1) continue;
      const float uR = kpR.x;
      if (uR >= minU && uR <= maxU) {
        why(iL) = ORC_ST_HAMMING;
        const int dist = orc_descriptor_distance(descL + (size_t)iL * 32, descR + iR * 32);
        if (dist < bestDist) {
          bestDist = dist;
          bestIdxR = iR;
        }
      }
    }
    if (bestDist < thOrbDist) {  // sub-pixel refinement by 11x11 L1 block matching on the keypoint's pyramid level
      const float uR0 = kpsR[bestIdxR].x;
      const float scaleFactor = inv_scale[kpL.octave];
      const float scaleduL = std::round(kpL.x * scaleFactor);
      const float scaledvL = std::round(kpL.y * scaleFactor);
      const float scaleduR0 = std::round(uR0 * scaleFactor);
      const int w = 5;
      const int lw = lvlW[kpL.octave], lh = lvlH[kpL.octave];
      const uint8_t* IL = pyrL[kpL.octave];
      const uint8_t* IR = pyrR[kpL.octave];
      const int cy = (int)scaledvL, cxL = (int)scaleduL, cxR0 = (int)scaleduR0;
      int bestDistS = INT_MAX;
      int bestincR = 0;
      const int L = 5;
      float vDists[2 * 5 + 1];
      const float iniu = scaleduR0 + L - w;
      const float endu = scaleduR0 + L + w + 1;
      why(iL) = ORC_ST_WINDOW;
      if (iniu < 0 || endu >= lw) continue;  // :1290
      // cv::Mat::rowRange/colRange would assert outside the image; guard the same accesses (never hit for real keypoints)
      if (cy - w < 0 || cy + w >= lh || cxL - w < 0 || cxL + w >= lw || cxR0 - L - w < 0) continue;
      const float cL = (float)IL[(size_t)cy * lw + cxL];
      for (int incR = -L; incR <= +L; incR++) {
        const int cxR = cxR0 + incR;
        const float cR = (float)IR[(size_t)cy * lw + cxR];
        float dist = 0;  // cv::norm(IL, IR, NORM_L1) of the centre-subtracted float patches (integer valued, exact)
        for (int dy = -w; dy <= w; dy++)
          for (int dx = -w; dx <= w; dx++) {
            const float a = (float)IL[(size_t)(cy + dy) * lw + cxL + dx] - cL;
            const float b = (float)IR[(size_t)(cy + dy) * lw + cxR + dx] - cR;
            dist += std::fabs(a - b);
          }
        if (dist < bestDistS) {  // float < int comparison as in the reference (:1308)
          bestDistS = (int)dist;
          bestincR = incR;
        }
        vDists[L + incR] = dist;
      }
      why(iL) = ORC_ST_EDGE;
      if (bestincR == -L || bestincR == L) continue;
      const float dist1 = vDists[L + bestincR - 1];
      const float dist2 = vDists[L + bestincR];
      const float dist3 = vDists[L + bestincR + 1];
      const float deltaR = (dist1 - dist3) / (2.0f * (dist1 + dist3 - 2.0f * dist2));
      why(iL) = ORC_ST_DELTA;
      if (deltaR < -1 || deltaR > 1) continue;
      float bestuR = scale[kpL.octave] * ((float)scaleduR0 + (float)bestincR + deltaR);
      float disparity = (uL - bestuR);
      why(iL) = ORC_ST_DISPARITY;
      if (disparity >= minD && disparity < maxD) {
        why(iL) = ORC_ST_KEPT;
        if (disparity <= 0) {
          disparity = 0.01;
          bestuR = uL - 0.01;
          why(iL) = ORC_ST_KEPT_ZERO;
        }
        mvDepth[iL] = mbf / disparity;
        mvuRight[iL] = bestuR;
        vDistIdx.push_back(std::pair<int, int>(bestDistS, iL));
      }
    }
  }
  if (vDistIdx.empty()) return 0;  // (the reference would index an empty vector here)
  std::sort(vDistIdx.begin(), vDistIdx.end());
  const float median = vDistIdx[vDistIdx.size() / 2].first;
  const float thDist = 1.5f * 1.4f * median;
  int kept = (int)vDistIdx.size();
  for (int i = (int)vDistIdx.size() - 1; i >= 0; i--) {
    if (vDistIdx[i].first < thDist) break;
    mvuRight[vDistIdx[i].second] = -1;
    mvDepth[vDistIdx[i].second] = -1;
    why(vDistIdx[i].second) = ORC_ST_CULLED;
    kept--;
  }
  return kept;
}

extern "C" int orc_compute_stereo_matches(const orc_keypoint* kpsL, const uint8_t* descL, int N, const orc_keypoint* kpsR,
                                          const uint8_t* descR, int Nr, const uint8_t* const* pyrL,
                                          const uint8_t* const* pyrR, const int* lvlW, const int* lvlH, const float* scale,
                                          const float* inv_scale, int nlevels, float mbf, float mb, float* mvuRight,
                                          float* mvDepth) {
  return orc_compute_stereo_matches_reason(kpsL, descL, N, kpsR, descR, Nr, pyrL, pyrR, lvlW, lvlH, scale, inv_scale,
                                           nlevels, mbf, mb, mvuRight, mvDepth, nullptr);
}
