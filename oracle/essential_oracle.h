/*
 * oracle/essential_oracle.h — the essential-graph optimisation for the CPU checkers (TEST INFRASTRUCTURE, see
 * orb_oracle.h).
 *
 * orc_sim3 / orc_sim3_edge / orc_eg_problem / orc_eg_result are layout-identical to b2s_sim3 / b2s_sim3_edge /
 * b2s_eg_problem / b2s_eg_result of include/b200slam.h.  orc_eg_map is the object graph ref_essential_graph builds for
 * the reference's own Optimizer::OptimizeEssentialGraph: keyframe k gets mnId k, map point m gets mnId m.
 */
#pragma once
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  double q[4]; /* qx qy qz qw */
  double t[3];
  double s;
} orc_sim3;
typedef struct {
  int32_t i, j;
  orc_sim3 meas;
} orc_sim3_edge;
typedef struct {
  int n_kf;
  const orc_sim3* Siw;
  int fixed_kf;
  int fix_scale;
  int n_edges;
  const orc_sim3_edge* edges;
  int n_mp;
  const float* points;
  const int32_t* ref_kf;
} orc_eg_problem;
typedef struct {
  float* Tcw_out;
  float* points_out;
  int32_t* trace;
  double chi2_initial, chi2_final;
  int n_trials;
} orc_eg_result;

/* oracle/essential.cpp: Optimizer::OptimizeEssentialGraph from the built graph on.  Returns 0. */
int orc_optimize_essential_graph(const orc_eg_problem* p, orc_eg_result* r);
/* its g2o::Sim3 operations (types/sim3.h), for the gather and the Sim3 test */
void orc_sim3_exp(const double* update7, orc_sim3* out);
void orc_sim3_log(const orc_sim3* a, double* out7);
void orc_sim3_mul(const orc_sim3* a, const orc_sim3* b, orc_sim3* out);
void orc_sim3_inverse(const orc_sim3* a, orc_sim3* out);
void orc_sim3_map(const orc_sim3* a, const double* xyz, double* out);
void orc_sim3_from_Rt(const double* R9, const double* t3, double s, orc_sim3* out); /* Sim3(Matrix3d R, t, s) */

typedef struct {
  int n_kf;                   /* keyframe k has mnId k */
  const float* Tcw;           /* n_kf x 16 */
  const uint8_t* kf_bad;      /* bad keyframes are not in the map; they are reachable only as covisible neighbours */
  const int32_t* parent;      /* n_kf: spanning-tree parent, -1 for none (children follow from it) */
  int n_loop;
  const int32_t* loop_edges;  /* n_loop pairs (a, b): b is in a's loop edges */
  int n_cov;
  const int32_t* cov;         /* n_cov triples (k, n, weight): n appended to k's covisible list (ordered by weight) */
  int loop_kf, cur_kf;
  int n_corr;
  const int32_t* corr_kf;     /* n_corr keyframes of CorrectedSim3 / NonCorrectedSim3 */
  const orc_sim3* corr_S;     /* n_corr: CorrectedSim3 */
  const orc_sim3* noncorr_S;  /* n_corr: NonCorrectedSim3 */
  int n_conn;
  const int32_t* conn;        /* n_conn pairs (k, j): j is in LoopConnections[k] */
  int n_mp;                   /* map point m has mnId m */
  const float* points;        /* n_mp x 3 */
  const uint8_t* mp_bad;      /* n_mp */
  const int32_t* mp_ref;      /* n_mp: reference keyframe */
  const int32_t* mp_corrected_by;   /* n_mp: mnCorrectedByKF */
  const int32_t* mp_corrected_ref;  /* n_mp: mnCorrectedReference */
  int fix_scale;
} orc_eg_map;
typedef struct {
  float* Tcw_out;             /* n_kf x 16: the keyframes' poses after the call */
  float* points_out;          /* n_mp x 3 */
  int32_t* mp_updates;        /* n_mp: UpdateNormalAndDepth() calls */
  int32_t* trace;             /* optional (>= 256), -1 terminated */
  int n_trials;
} orc_eg_map_result;

/* oracle/ref_essential_glue.cpp: the reference's Optimizer::OptimizeEssentialGraph (libref_essential.so) on the object
 * graph.  Returns 0, < 0 if the map cannot be expressed. */
int ref_essential_graph(const orc_eg_map* m, orc_eg_map_result* r);
/* the same glue around the product's drop-in body (libadapter_essential.so) */
int adp_essential_graph(const orc_eg_map* m, orc_eg_map_result* r);
/* g2o::Sim3 of the reference's header, for the Sim3 test */
void ref_sim3_exp(const double* update7, orc_sim3* out);
void ref_sim3_log(const orc_sim3* a, double* out7);
void ref_sim3_mul(const orc_sim3* a, const orc_sim3* b, orc_sim3* out);
void ref_sim3_inverse(const orc_sim3* a, orc_sim3* out);
void ref_sim3_map(const orc_sim3* a, const double* xyz, double* out);

#ifdef __cplusplus
}
#endif
