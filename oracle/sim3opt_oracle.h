/*
 * oracle/sim3opt_oracle.h — Optimizer::OptimizeSim3 for the CPU checkers (TEST INFRASTRUCTURE, see orb_oracle.h).
 *
 * orc_sim3_problem / orc_sim3_result are layout-identical to b2s_sim3_problem / b2s_sim3_result of include/b200slam.h.
 * orc_sim3_graph is the object graph ref_optimize_sim3 builds for the reference's own Optimizer::OptimizeSim3: two
 * keyframes and a pool of map points (map point m has mnId m).
 */
#pragma once
#include <stdint.h>

#include "essential_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  int32_t n;
  const float *X1c, *X2c, *obs1, *obs2, *inv_sigma2_1, *inv_sigma2_2;
  float fx1, fy1, cx1, cy1, fx2, fy2, cx2, cy2;
  orc_sim3 S12;
  float th2;
  int32_t fix_scale;
} orc_sim3_problem;
typedef struct {
  orc_sim3 S12_out;
  uint8_t* keep;
  int32_t* trace;
  int32_t n_inliers;
  int32_t n_trials;
} orc_sim3_result;
/* oracle/sim3opt.cpp: Optimizer::OptimizeSim3 after the graph is built.  chi2_out (optional, 2n): e12 / e21 chi2 of the
 * final classification (round 1's on the early return; pairs dropped in round 1 keep their round-1 values).
 * Returns 0. */
int orc_optimize_sim3(const orc_sim3_problem* p, orc_sim3_result* r, double* chi2_out);

typedef struct {
  const float* Tcw1;              /* 16 */
  const float* Tcw2;              /* 16 */
  const float* K1;                /* fx fy cx cy */
  const float* K2;
  int n1;                         /* keypoints of pKF1 = vpMatches1.size() */
  const float* kp1;               /* n1 x 2: mvKeysUn */
  const int32_t* oct1;            /* n1 */
  int n2;
  const float* kp2;               /* n2 x 2 */
  const int32_t* oct2;            /* n2 */
  int n_levels;
  const float* inv_sigma2_1;      /* n_levels: mvInvLevelSigma2 */
  const float* inv_sigma2_2;
  int n_mp;
  const float* points;            /* n_mp x 3 */
  const uint8_t* mp_bad;          /* n_mp */
  const int32_t* mp_idx2;         /* n_mp: index in pKF2 (its observation), -1: not observed in pKF2 */
  const int32_t* mp1;             /* n1: pKF1->GetMapPointMatches()[i] as a point index, -1: null */
  const int32_t* matches1;        /* n1: vpMatches1[i] as a point index, -1: null */
  orc_sim3 S12;
  float th2;
  int fix_scale;
} orc_sim3_graph;
typedef struct {
  uint8_t* match_kept;            /* n1: vpMatches1[i] is non-null after the call */
  orc_sim3 S12_out;               /* g2oS12 after the call */
  int32_t* trace;                 /* optional (>= 256), -1 terminated */
  int n_trials;
  int ret;                        /* the return value */
} orc_sim3_graph_result;
/* oracle/ref_sim3opt_glue.cpp: the reference's Optimizer::OptimizeSim3 (_ref/libref_sim3opt.so) on the object graph.
 * Returns 0, < 0 if the graph cannot be expressed. */
int ref_optimize_sim3(const orc_sim3_graph* g, orc_sim3_graph_result* r);
/* the same glue around the product's drop-in body (_ref/libadapter_sim3opt.so) */
int adp_optimize_sim3(const orc_sim3_graph* g, orc_sim3_graph_result* r);

#ifdef __cplusplus
}
#endif
