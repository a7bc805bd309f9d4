// levenberg_harness.cu — test-only C surface over csrc/levenberg.cuh (the Levenberg step control of LocalBA,
// PoseOptimization, the global bundle adjustment and the essential graph), for tests/test_levenberg.py.  Host code only;
// it is not part of libb200slam.so.
#include "levenberg.cuh"

using b2s::Levenberg;

extern "C" int lm_state_size() { return (int)sizeof(Levenberg); }
extern "C" void lm_init_lambda(Levenberg* s, double lambda0) { s->init_lambda(lambda0); }
extern "C" void lm_begin(Levenberg* s, double chi) { s->begin(chi); }
extern "C" int lm_trial(Levenberg* s, int solved, double tempChi, double scale, int* trace) {
  return s->trial(solved != 0, tempChi, scale, trace) ? 1 : 0;
}
extern "C" int lm_retry(const Levenberg* s, int stop) { return s->retry(stop != 0) ? 1 : 0; }
extern "C" int lm_end_iteration(Levenberg* s) { return s->end_iteration() ? 1 : 0; }
