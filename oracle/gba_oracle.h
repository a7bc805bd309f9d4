/*
 * oracle/gba_oracle.h — flattened global bundle adjustment for the CPU checkers (TEST INFRASTRUCTURE, see orb_oracle.h).
 *
 * orc_gba_problem / orc_gba_result are layout-identical to b2s_gba_problem / b2s_gba_result of include/b200slam.h.
 * orc_gba_map is the object graph ref_global_ba builds for the reference's own Optimizer::GlobalBundleAdjustemnt: keyframe
 * k gets mnId = k, map point m gets mnId = m, bad objects stay in the map (the reference skips them itself).
 */
#pragma once
#include "orb_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  int n_kf;                  /* the non-bad keyframes, ascending mnId */
  const float* Tcw;          /* n_kf x 16 */
  const uint8_t* fixed;      /* n_kf: mnId == 0 */
  int n_mp;                  /* the non-bad map points, ascending mnId */
  const float* points;       /* n_mp x 3 */
  int n_edges;
  const orc_ba_edge* edges;  /* grouped by point (ascending), one per (keyframe, point) */
  float fx, fy, cx, cy, bf;
  int iterations;
  int robust;
} orc_gba_problem;

typedef struct {
  float* Tcw_out;            /* n_kf x 16 */
  float* points_out;         /* n_mp x 3 (rows of excluded points untouched) */
  uint8_t* point_included;   /* n_mp */
  int32_t* trace;            /* optional (>= 256), -1 terminated */
  double chi2_final;
  int n_trials;
} orc_gba_result;

/* Optimizer::BundleAdjustment on the flattened problem.  Returns 0. */
int orc_global_ba(const orc_gba_problem* p, const volatile uint8_t* stop, orc_gba_result* r);

typedef struct {
  int n_kf;                  /* keyframe k has mnId k */
  const float* Tcw;          /* n_kf x 16 */
  const uint8_t* kf_bad;     /* n_kf */
  int n_mp;                  /* map point m has mnId m */
  const float* points;       /* n_mp x 3 */
  const uint8_t* mp_bad;     /* n_mp */
  int n_obs;
  const orc_ba_edge* obs;    /* every observation (those of bad keyframes too), grouped by point, one per pair */
  float fx, fy, cx, cy, bf;
  int iterations;
  int robust;
  uint64_t loop_kf;          /* nLoopKF */
} orc_gba_map;

typedef struct {
  float* Tcw_out;            /* n_kf x 16: mTcwGBA where the call set it, else Tcw */
  float* points_out;         /* n_mp x 3: mPosGBA where the call set it, else mWorldPos */
  uint8_t* kf_gba;           /* n_kf: 1 = mTcwGBA was set */
  uint8_t* mp_gba;           /* n_mp: 1 = mPosGBA was set */
  uint64_t* kf_ba_global;    /* n_kf: mnBAGlobalForKF after the call */
  uint64_t* mp_ba_global;    /* n_mp */
  int32_t* mp_updates;       /* n_mp: UpdateNormalAndDepth() calls */
  int32_t* trace;            /* optional (>= 256), -1 terminated */
  int n_trials;
} orc_gba_map_result;

/* oracle/ref_gba_glue.cpp: the reference's Optimizer::GlobalBundleAdjustemnt (libref_gba.so) or the product's drop-in body
 * (libadapter_gba.so, entry point adp_global_ba) on the object graph.  Returns 0, < 0 if the map cannot be expressed. */
int ref_global_ba(const orc_gba_map* m, const volatile uint8_t* stop, orc_gba_map_result* r);

#ifdef __cplusplus
}
#endif
