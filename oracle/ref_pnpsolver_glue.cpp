// TEST INFRASTRUCTURE — a C interface to the reference's own PnPsolver (src/PnPsolver.cc compiled in place against
// refshim/refshim_cv_pnpsolver.h, oracle/pnpsolver.mk), or to the product's drop-in behind the same header.  The scene
// is given flattened: correspondence i is keypoint i of a Frame stand-in with octave i, so its sigma2 is
// mvLevelSigma2[i].  Private members are opened to call compute_pose directly and to read the solver state.  Built
// with -DB2S_ADAPTER_BUILD and the product's host/adapters/PnPsolver_b200.cc into _ref/libadapter_pnpsolver.so, the
// same entry points drive the drop-in.
#define private public
#include "PnPsolver.h"
#undef private

#include <cstdint>
#include <cstdlib>
#include <cstring>

#include "Thirdparty/DBoW2/DUtils/Random.h"

using namespace ORB_SLAM2;

namespace {
struct Holder {
  Frame F;
  std::vector<MapPoint> mps;
  std::vector<MapPoint*> matches;
  PnPsolver* solver = nullptr;
  ~Holder() { delete solver; }
};

void write_Tcw(const cv::Mat& T, float* out) {
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++) out[4 * r + c] = (float)T.get(r, c);
}
}  // namespace

extern "C" {

void* pnp_create(int n, const float* P3Dw, const float* P2D, const float* sigma2, const float* cam) {
  Holder* h = new Holder();
  h->mps.resize((size_t)n);
  h->F.mvKeysUn.resize((size_t)n);
  h->F.mvLevelSigma2.assign(sigma2, sigma2 + n);
  for (int i = 0; i < n; i++) {
    h->mps[i].pos = cv::Mat(3, 1, CV_32F);
    for (int c = 0; c < 3; c++) h->mps[i].pos.at<float>(c) = P3Dw[3 * i + c];
    h->F.mvKeysUn[i].pt = cv::Point2f(P2D[2 * i], P2D[2 * i + 1]);
    h->F.mvKeysUn[i].octave = i;
    h->matches.push_back(&h->mps[i]);
  }
  h->F.mvpMapPoints = h->matches;
  h->F.fx = cam[0];
  h->F.fy = cam[1];
  h->F.cx = cam[2];
  h->F.cy = cam[3];
  h->solver = new PnPsolver(h->F, h->matches);
  return h;
}

void pnp_destroy(void* p) { delete (Holder*)p; }

void pnp_set_ransac_parameters(void* p, double probability, int min_inliers, int max_iterations, int min_set,
                               float epsilon, float th2) {
  ((Holder*)p)->solver->SetRansacParameters(probability, min_inliers, max_iterations, min_set, epsilon, th2);
}

// iterate(n_iterations) (or find() for n_iterations < 0): 1 and Tcw when the returned matrix is not empty
int pnp_iterate(void* p, int n_iterations, int32_t* no_more, uint8_t* inliers, int32_t* n_inliers, float* Tcw) {
  Holder* h = (Holder*)p;
  std::vector<bool> vb;
  int ni = 0;
  bool nm = false;
  const cv::Mat T = n_iterations < 0 ? h->solver->find(vb, ni) : h->solver->iterate(n_iterations, nm, vb, ni);
  *no_more = nm;
  *n_inliers = ni;
  for (size_t i = 0; i < h->matches.size(); i++) inliers[i] = i < vb.size() && vb[i];
  if (T.empty()) return 0;
  write_Tcw(T, Tcw);
  return 1;
}

// counters: mnIterations, mnBestInliers, mRansacMinInliers, mRansacMaxIts; best_mask n; returns 1 when mBestTcw is set
int pnp_state(void* p, int32_t* counters, float* best_Tcw, uint8_t* best_mask) {
  PnPsolver* s = ((Holder*)p)->solver;
  counters[0] = s->mnIterations;
  counters[1] = s->mnBestInliers;
  counters[2] = s->mRansacMinInliers;
  counters[3] = s->mRansacMaxIts;
  for (int i = 0; i < s->N; i++) best_mask[i] = i < (int)s->mvbBestInliers.size() && s->mvbBestInliers[i];
  if (s->mBestTcw.empty()) return 0;
  write_Tcw(s->mBestTcw, best_Tcw);
  return 1;
}

#ifndef B2S_ADAPTER_BUILD  // the drop-in runs EPnP on the device and has no compute_pose
// compute_pose on the m correspondences idx (as iterate's loop or Refine feeds it): R (9), t (3); returns the error
double pnp_compute_pose(void* p, const int* idx, int m, double* R, double* t) {
  PnPsolver* s = ((Holder*)p)->solver;
  s->set_maximum_number_of_correspondences(m);
  s->reset_correspondences();
  for (int i = 0; i < m; i++) {
    const int j = idx[i];
    s->add_correspondence(s->mvP3Dw[j].x, s->mvP3Dw[j].y, s->mvP3Dw[j].z, s->mvP2D[j].x, s->mvP2D[j].y);
  }
  const double e = s->compute_pose(s->mRi, s->mti);
  std::memcpy(R, s->mRi, sizeof(s->mRi));
  std::memcpy(t, s->mti, sizeof(s->mti));
  return e;
}
#endif

void pnp_srand(unsigned seed) { srand(seed); }
int pnp_random_int(int lo, int hi) { return DUtils::Random::RandomInt(lo, hi); }

}  // extern "C"
