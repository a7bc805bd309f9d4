/*
 * oracle/gba.cpp — CPU restatement of Optimizer::BundleAdjustment (src/Optimizer.cc:86-341), the body of
 * GlobalBundleAdjustemnt, from the point where the graph is built (TEST INFRASTRUCTURE, see orb_oracle.h).
 *
 * The edges, Jacobians, Huber kernel, Schur solve, SE3 update and Levenberg control are exactly those of the LocalBA
 * oracle: struct BA of local_ba.cpp is compiled into this library unchanged and driven for one round.  What differs:
 *   - one optimize(nIterations) call, no outlier round (:279-280);
 *   - Huber deltas sqrt(5.99) / sqrt(7.815) as float (:141-142), only when bRobust;
 *   - a keyframe without an edge is an inactive vertex (sparse_optimizer.cpp:206-230): no block in H, its estimate is
 *     kept; it is held here as a fixed vertex, which is the same thing;
 *   - a point without an edge is removed from the graph (vbNotIncludedMP, :266-274) and not written back; kept here as
 *     an inert landmark (zero Hessian, zero step) and flagged in point_included;
 *   - every keyframe, fixed and inactive ones included, is written back through Converter (:294-308);
 *   - the stop flag only ends the LM loop (g2o's terminate()); the write-back always happens.
 */
#include "local_ba.cpp"

#include "gba_oracle.h"

extern "C" int orc_global_ba(const orc_gba_problem* g, const volatile uint8_t* stop, orc_gba_result* r) {
  const int nKF = g->n_kf, nMP = g->n_mp, nE = g->n_edges;
  std::vector<uint8_t> fixed(g->fixed, g->fixed + nKF), kfActive((size_t)nKF, 0);
  for (int m = 0; m < nMP; m++) r->point_included[m] = 0;
  for (int e = 0; e < nE; e++) {
    kfActive[(size_t)g->edges[e].kf] = 1;
    r->point_included[g->edges[e].mp] = 1;
  }
  for (int k = 0; k < nKF; k++)
    if (!kfActive[(size_t)k]) fixed[(size_t)k] = 1;
  orc_ba_problem p;
  p.n_kf = nKF;
  p.n_local = nKF;
  p.Tcw = g->Tcw;
  p.fixed = fixed.data();
  p.n_mp = nMP;
  p.points = g->points;
  p.n_edges = nE;
  p.edges = g->edges;
  p.fx = g->fx; p.fy = g->fy; p.cx = g->cx; p.cy = g->cy; p.bf = g->bf;
  p.its1 = g->iterations;
  p.its2 = 0;
  BA ba;
  ba.P = &p;
  ba.stop = stop;
  ba.init();
  ba.robust = g->robust != 0;
  ba.delta_mono = (double)(float)std::sqrt(5.99);  // const float thHuber2D = sqrt(5.99) (:141)
  ba.delta_stereo = (double)(float)std::sqrt(7.815);
  ba.optimize(g->iterations);
  for (int k = 0; k < nKF; k++) pose_to_Tcw(ba.poses[(size_t)k], r->Tcw_out + (size_t)k * 16);
  for (int m = 0; m < nMP; m++)
    if (r->point_included[m])
      for (int c = 0; c < 3; c++) r->points_out[(size_t)m * 3 + c] = (float)ba.pts[(size_t)m * 3 + c];
  ba.compute_errors();
  r->chi2_final = ba.active_robust_chi2();
  r->n_trials = ba.n_trials;
  if (r->trace) {
    size_t n = std::min<size_t>(ba.trace.size(), 255);
    for (size_t i = 0; i < n; i++) r->trace[i] = ba.trace[i];
    r->trace[n] = -1;
  }
  return 0;
}
