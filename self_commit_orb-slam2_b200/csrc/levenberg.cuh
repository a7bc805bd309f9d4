// levenberg.cuh — g2o's Levenberg-Marquardt step control, shared by every optimiser of the library: LocalBA and
// PoseOptimization (localba.cu, on the device), the global bundle adjustment (gba.cu) and the essential graph
// (essential.cu, both on the host).
//
// Restates OptimizationAlgorithmLevenberg::solve of the reference's g2o (Thirdparty/g2o/g2o/core/
// optimization_algorithm_levenberg.cpp:47-51 constants, :61-163 solve) including ORB-SLAM's stop rule (:154-161, three
// iterations in a row that lower chi2 by less than 1e-3 of its initial value end the optimisation).  One iteration:
//   begin(chi2)                                   computeActiveErrors + activeRobustChi2 of the current state (:76-85)
//   init_lambda(l)                                on the first iteration only: computeLambdaInit (:93-97, :166-180)
//   do { solve; update; good = trial(...) }       one trial per lambda (:104-148); a rejected trial's state is restored
//   while (retry(stop))                           by the caller (pop)
//   if (end_iteration()) the optimisation stops   (:151-162)
// The caller computes chi2, the scale x^T (lambda x + b) (computeScale, :182-189) and the lambda to start from, and owns
// the state restore and the stop flag.  Everything here is plain arithmetic in the order of the reference lines, so the
// host and the device copies decide identically.
#pragma once
#include <float.h>
#include <math.h>

#include <cmath>

namespace b2s {

struct Levenberg {
  double lambda, ni;         // _currentLambda, _ni
  double currentChi, iniChi;  // chi2 of the current state, and at the iteration's start
  double rho;                // gain ratio of the last trial
  int qmax;                  // trials of this iteration (_levenbergIterations)
  int nBad;                  // consecutive iterations with a small gain
  int nTrials;               // trials of the whole optimisation (trace index)

  __host__ __device__ __forceinline__ void init_lambda(double lambda0) {
    lambda = lambda0;
    ni = 2;
    nBad = 0;
  }

  __host__ __device__ __forceinline__ void begin(double chi) {
    currentChi = chi;
    iniChi = chi;
    rho = 0;
    qmax = 0;
  }

  // One trial: `solved` is the linear solve's status, tempChi the chi2 after the update, scale computeScale().  Returns
  // whether the step is accepted (the caller keeps it, or restores the state saved before the trial).  trace[nTrials]
  // gets 1 / 0 while nTrials < 255.
  __host__ __device__ __forceinline__ bool trial(bool solved, double tempChi, double scale, int* trace) {
    if (!solved) {
      tempChi = DBL_MAX;
      scale = 0;
    }
    scale += 1e-3;
    double r = (currentChi - tempChi) / scale;
    if (!solved) r = -1;
    const bool good = r > 0 && isfinite(tempChi);
    if (nTrials < 255) trace[nTrials] = good ? 1 : 0;
    nTrials++;
    if (good) {
      double alpha = 1. - pow((2 * r - 1), 3);
      alpha = fmin(alpha, 2. / 3.);
      lambda *= fmax(1. / 3., alpha);
      ni = 2;
      currentChi = tempChi;
    } else {
      lambda *= ni;
      ni *= 2;
    }
    rho = r;
    qmax++;
    return good;
  }

  // Another trial with the larger lambda?  (`stop`: SparseOptimizer::terminate())
  __host__ __device__ __forceinline__ bool retry(bool stop) const { return rho < 0 && qmax < 10 && !stop; }

  // After the last trial of an iteration: does the optimisation stop here?
  __host__ __device__ __forceinline__ bool end_iteration() {
    if (qmax == 10 || rho == 0) return true;
    if ((iniChi - currentChi) * 1e3 < iniChi)
      nBad++;
    else
      nBad = 0;
    return nBad >= 3;
  }
};

}  // namespace b2s
