// TEST INFRASTRUCTURE — drives the reference's OWN src/Sim3Solver.cc (compiled in place, unmodified, against
// refshim/refshim_cv_sim3solver.h, with Thirdparty/DBoW2/DUtils/Random.cpp) on two stand-in KeyFrames built from a
// flattened scene.  Built by `make -f sim3solver.mk sim3solver-ref` into _ref/libref_sim3solver.so; with
// -DB2S_ADAPTER_BUILD and the product's host/adapters/Sim3Solver_b200.cc instead of the reference's Sim3Solver.cc it is
// _ref/libadapter_sim3solver.so, behind the same entry points.
//
// The solver draws from the process-global rand(): s3s_srand seeds it, and s3s_random_int is DUtils::Random::RandomInt,
// so a test can replay the draws a call made.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

#define protected public
#define private public
#include "Sim3Solver.h"
#undef private
#undef protected
#include "Thirdparty/DBoW2/DUtils/Random.h"

using namespace ORB_SLAM2;

extern "C" {

// A loop candidate flattened: KF1 has m keypoint slots (vpMatched12.size()), KF2 nk2 keypoints.
typedef struct {
  int32_t m, nk2, fix_scale;
  const float *Tcw1, *Tcw2;     // 4 x 4, row-major
  const float *K1, *K2;         // 3 x 3, row-major
  int32_t n_levels;
  const float *level_sigma2_1, *level_sigma2_2;  // mvLevelSigma2 of each keyframe
  const int32_t *octave1;       // m: mvKeysUn[i].octave of KF1
  const int32_t *octave2;       // nk2
  const int32_t *matched;       // m: vpMatched12[i] != NULL
  const int32_t *has_mp1;       // m: KF1's GetMapPointMatches()[i] != NULL
  const int32_t *bad1, *bad2;   // m: isBad() of the two map points
  const int32_t *idx1, *idx2;   // m: GetIndexInKeyFrame(pKF1) / (pKF2) (-1: not observed)
  const float *Xw1, *Xw2;       // m x 3: GetWorldPos()
} s3s_scene;

}  // extern "C"

namespace {

cv::Mat mat(int r, int c, const float* v) {
  cv::Mat M(r, c, CV_32F);
  for (int i = 0; i < r * c; i++) M.at<float>(i / c, i % c) = v[i];
  return M;
}

struct Holder {
  KeyFrame kf1, kf2;
  std::vector<MapPoint> mp1, mp2;
  std::vector<MapPoint*> matches12;
  Sim3Solver* solver = nullptr;
  ~Holder() { delete solver; }
};

void write_mat(const cv::Mat& M, float* out, int n) {
  for (int i = 0; i < n; i++) out[i] = M.empty() ? 0.f : M.at<float>(i / M.cols, i % M.cols);
}

}  // namespace

extern "C" {

void* s3s_create(const s3s_scene* s) {
  Holder* h = new Holder();
  h->kf1.Tcw = mat(4, 4, s->Tcw1);
  h->kf2.Tcw = mat(4, 4, s->Tcw2);
  h->kf1.mK = mat(3, 3, s->K1);
  h->kf2.mK = mat(3, 3, s->K2);
  h->kf1.mvLevelSigma2.assign(s->level_sigma2_1, s->level_sigma2_1 + s->n_levels);
  h->kf2.mvLevelSigma2.assign(s->level_sigma2_2, s->level_sigma2_2 + s->n_levels);
  h->kf1.mvKeysUn.resize((size_t)s->m);
  for (int i = 0; i < s->m; i++) h->kf1.mvKeysUn[(size_t)i].octave = s->octave1[i];
  h->kf2.mvKeysUn.resize((size_t)s->nk2);
  for (int i = 0; i < s->nk2; i++) h->kf2.mvKeysUn[(size_t)i].octave = s->octave2[i];
  h->mp1.resize((size_t)s->m);
  h->mp2.resize((size_t)s->m);
  h->kf1.mvpMapPoints.assign((size_t)s->m, nullptr);
  h->matches12.assign((size_t)s->m, nullptr);
  for (int i = 0; i < s->m; i++) {
    MapPoint &a = h->mp1[(size_t)i], &b = h->mp2[(size_t)i];
    a.bad = s->bad1[i] != 0;
    b.bad = s->bad2[i] != 0;
    a.pos = mat(3, 1, s->Xw1 + 3 * i);
    b.pos = mat(3, 1, s->Xw2 + 3 * i);
    if (s->idx1[i] >= 0) a.index[&h->kf1] = s->idx1[i];
    if (s->idx2[i] >= 0) b.index[&h->kf2] = s->idx2[i];
    if (s->has_mp1[i]) h->kf1.mvpMapPoints[(size_t)i] = &a;
    if (s->matched[i]) h->matches12[(size_t)i] = &b;
  }
  h->solver = new Sim3Solver(&h->kf1, &h->kf2, h->matches12, s->fix_scale != 0);
  return h;
}

void s3s_destroy(void* p) { delete (Holder*)p; }

void s3s_set_ransac_parameters(void* p, double probability, int min_inliers, int max_iterations) {
  ((Holder*)p)->solver->SetRansacParameters(probability, min_inliers, max_iterations);
}

// iterate(n_iterations, ...) (find() when n_iterations < 0): returns 1 when the returned matrix is not empty (then
// T12 holds it), no_more, inliers (mN1 entries), n_inliers
int s3s_iterate(void* p, int n_iterations, int32_t* no_more, uint8_t* inliers, int32_t* n_inliers, float* T12) {
  Sim3Solver* S = ((Holder*)p)->solver;
  std::vector<bool> v;
  int n = -7;
  bool nm = false;
  const cv::Mat T = n_iterations < 0 ? S->find(v, n) : S->iterate(n_iterations, nm, v, n);
  *no_more = n_iterations < 0 ? -1 : (nm ? 1 : 0);
  *n_inliers = n;
  for (size_t i = 0; i < v.size(); i++) inliers[i] = v[i] ? 1 : 0;
  write_mat(T, T12, 16);
  return T.empty() ? 0 : 1;
}

// The object's counters: N, mN1, mnIterations, mnBestInliers, mRansacMaxIts, mRansacMinInliers; the getters (R, t and
// s; has_best = 0 while GetEstimatedRotation() is empty)
void s3s_state(void* p, int32_t* counters, float* R, float* t, float* s, int32_t* has_best) {
  Sim3Solver* S = ((Holder*)p)->solver;
  counters[0] = S->N;
  counters[1] = S->mN1;
  counters[2] = S->mnIterations;
  counters[3] = S->mnBestInliers;
  counters[4] = S->mRansacMaxIts;
  counters[5] = S->mRansacMinInliers;
  const cv::Mat Rb = S->GetEstimatedRotation(), tb = S->GetEstimatedTranslation();
  *has_best = Rb.empty() ? 0 : 1;
  write_mat(Rb, R, 9);
  write_mat(tb, t, 3);
  *s = *has_best ? S->GetEstimatedScale() : 0.f;
}

// What the constructor kept: mvnIndices1 (N), mvX3Dc1 / mvX3Dc2 (N x 3), mvnMaxError1 / 2 (N)
void s3s_members(void* p, int32_t* indices1, float* X1c, float* X2c, uint64_t* max_err1, uint64_t* max_err2) {
  Sim3Solver* S = ((Holder*)p)->solver;
  for (int i = 0; i < S->N; i++) {
    indices1[i] = (int32_t)S->mvnIndices1[(size_t)i];
    for (int r = 0; r < 3; r++) {
      X1c[3 * i + r] = S->mvX3Dc1[(size_t)i].at<float>(r);
      X2c[3 * i + r] = S->mvX3Dc2[(size_t)i].at<float>(r);
    }
    max_err1[i] = S->mvnMaxError1[(size_t)i];
    max_err2[i] = S->mvnMaxError2[(size_t)i];
  }
}

void s3s_srand(unsigned seed) { srand(seed); }
int s3s_random_int(int lo, int hi) { return DUtils::Random::RandomInt(lo, hi); }

}  // extern "C"
