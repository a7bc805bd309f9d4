// TEST INFRASTRUCTURE — drives the reference's OWN src/Initializer.cc (compiled in place, unmodified, against
// refshim/refshim_cv_init.h, with Thirdparty/DBoW2/DUtils/Random.cpp) on two stand-in Frames carrying mvKeysUn and mK.
// Built by `make -f init.mk init-ref` into _ref/libref_init.so; with -DB2S_ADAPTER_BUILD and the product's
// host/adapters/Initializer_b200.cc instead of the reference's Initializer.cc it is _ref/libadapter_init.so
// (adp_initialize only).
//
// Every entry point calls srand(0) first: DUtils::Random::SeedRandOnce seeds only once per process, so this is what
// lets two calls (and the two libraries) consume the same rand() stream.  Outputs the reference leaves alone keep the
// marker values they are given: R21 / t21 start as 3 x 3 / 3 x 1 matrices of -12345, vP3D as n1 points of -12345,
// vbTriangulated as n1 x true.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

#define private public  // the glue calls FindHomography / FindFundamental / ReconstructH / ReconstructF directly
#include "Initializer.h"
#undef private

#ifdef B2S_ADAPTER_BUILD
#define ref_initialize adp_initialize
#endif

using namespace ORB_SLAM2;

namespace {

const float MARK = -12345.f;

Frame frame(const float* kp, int n, const float* K) {
  Frame F;
  F.mK = cv::Mat(3, 3, CV_32F);
  for (int i = 0; i < 9; i++) F.mK.at<float>(i / 3, i % 3) = K[i];
  F.mvKeysUn.resize((size_t)n);
  for (int i = 0; i < n; i++) {
    F.mvKeysUn[(size_t)i].pt.x = kp[2 * i];
    F.mvKeysUn[(size_t)i].pt.y = kp[2 * i + 1];
  }
  return F;
}

struct Outputs {
  cv::Mat R21, t21;
  std::vector<cv::Point3f> vP3D;
  std::vector<bool> vbTriangulated;
  explicit Outputs(int n1)
      : R21(3, 3, CV_32F, cv::Scalar(MARK)), t21(3, 1, CV_32F, cv::Scalar(MARK)),
        vP3D((size_t)n1, cv::Point3f(MARK, MARK, MARK)), vbTriangulated((size_t)n1, true) {}
  // rt_state: 1 written, -1 emptied, 0 untouched
  void write(float* R, float* t, int32_t* rt_state, float* p3d, uint8_t* tri) const {
    if (R21.empty() || t21.empty()) {
      *rt_state = -1;
    } else {
      bool marked = true;
      for (int i = 0; i < 9; i++) marked = marked && R21.at<float>(i / 3, i % 3) == MARK;
      *rt_state = marked ? 0 : 1;
      for (int i = 0; i < 9; i++) R[i] = R21.at<float>(i / 3, i % 3);
      for (int i = 0; i < 3; i++) t[i] = t21.at<float>(i);
    }
    for (size_t i = 0; i < vP3D.size(); i++) {
      p3d[3 * i] = vP3D[i].x;
      p3d[3 * i + 1] = vP3D[i].y;
      p3d[3 * i + 2] = vP3D[i].z;
    }
    for (size_t i = 0; i < vbTriangulated.size(); i++) tri[i] = vbTriangulated[i] ? 1 : 0;
  }
};

}  // namespace

extern "C" {

// Initializer(F1, sigma, iterations).Initialize(F2, vMatches12, ...) after srand(0); mvSets -> sets_out (iterations x 8)
int ref_initialize(const b2s_init_problem* p, float* R21, float* t21, int32_t* rt_state, float* p3d, uint8_t* tri,
                   int32_t* sets_out) {
  const Frame F1 = frame(p->kp1, p->n1, p->K), F2 = frame(p->kp2, p->n2, p->K);
  const std::vector<int> m(p->matches12, p->matches12 + p->n1);
  Initializer I(F1, p->sigma, p->iterations);
  Outputs o(p->n1);
  srand(0);
  const bool ret = I.Initialize(F2, m, o.R21, o.t21, o.vP3D, o.vbTriangulated);
  o.write(R21, t21, rt_state, p3d, tri);
  for (int it = 0; it < p->iterations; it++)
    for (int j = 0; j < 8; j++) sets_out[8 * it + j] = (int32_t)I.mvSets[(size_t)it][(size_t)j];
  return ret ? 1 : 0;
}

#ifndef B2S_ADAPTER_BUILD
// The state Initialize builds before its two threads start (:82-168), with mvSets = p->sets
static void prepare(Initializer& I, const Frame& F2, const b2s_init_problem* p) {
  I.mvKeys2 = F2.mvKeysUn;
  I.mvMatches12.clear();
  I.mvbMatched1.assign((size_t)p->n1, false);
  for (int i = 0; i < p->n1; i++)
    if (p->matches12[i] >= 0) {
      I.mvMatches12.push_back(std::make_pair(i, p->matches12[i]));
      I.mvbMatched1[(size_t)i] = true;
    }
  I.mvSets.assign((size_t)p->iterations, std::vector<size_t>(8, 0));
  for (int it = 0; it < p->iterations; it++)
    for (int j = 0; j < 8; j++) I.mvSets[(size_t)it][(size_t)j] = (size_t)p->sets[8 * it + j];
}

// FindHomography / FindFundamental: score, the best matrix (zeros when none scored above 0), inlier flags
void ref_find(const b2s_init_problem* p, int homography, float* score, float* X, uint8_t* inl) {
  const Frame F1 = frame(p->kp1, p->n1, p->K), F2 = frame(p->kp2, p->n2, p->K);
  Initializer I(F1, p->sigma, p->iterations);
  prepare(I, F2, p);
  std::vector<bool> v;
  cv::Mat M;
  if (homography)
    I.FindHomography(v, *score, M);
  else
    I.FindFundamental(v, *score, M);
  for (int i = 0; i < 9; i++) X[i] = M.empty() ? 0.f : M.at<float>(i / 3, i % 3);
  for (size_t i = 0; i < v.size(); i++) inl[i] = v[i] ? 1 : 0;
}

// ReconstructH / ReconstructF(inliers, X, mK, R21, t21, vP3D, vbTriangulated, 1.0, 50) as Initialize calls them
int ref_reconstruct(const b2s_init_problem* p, int homography, const uint8_t* inl, const float* X, float* R21,
                    float* t21, int32_t* rt_state, float* p3d, uint8_t* tri) {
  const Frame F1 = frame(p->kp1, p->n1, p->K), F2 = frame(p->kp2, p->n2, p->K);
  Initializer I(F1, p->sigma, p->iterations);
  prepare(I, F2, p);
  std::vector<bool> v(I.mvMatches12.size());
  for (size_t i = 0; i < v.size(); i++) v[i] = inl[i] != 0;
  cv::Mat M(3, 3, CV_32F);
  for (int i = 0; i < 9; i++) M.at<float>(i / 3, i % 3) = X[i];
  Outputs o(p->n1);
  srand(0);
  const bool ret = homography ? I.ReconstructH(v, M, I.mK, o.R21, o.t21, o.vP3D, o.vbTriangulated, 1.0, 50)
                              : I.ReconstructF(v, M, I.mK, o.R21, o.t21, o.vP3D, o.vbTriangulated, 1.0, 50);
  o.write(R21, t21, rt_state, p3d, tri);
  return ret ? 1 : 0;
}
#endif

}  // extern "C"
