// b2s_host.h — the one handle policy of the host layer (host/*.cc and host/adapters/*.cc): which device a handle is
// created on, how a long-lived handle grows, and how a library failure is reported.
#pragma once
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <stdexcept>

#include "../../include/b200slam.h"

namespace b2s_host {

// The device every handle is created on: $B2S_DEVICE, else 0.
inline int device() {
  const char* e = getenv("B2S_DEVICE");
  return e ? atoi(e) : 0;
}

// One stderr line for a failed library call.
inline void report(const char* who, int rc) {
  fprintf(stderr, "%s: libb200slam error %d: %s\n", who, rc, b2s_last_error());
}

// report(), then throw: for the entries whose callers expect an exception.
[[noreturn]] inline void fail(const char* who, int rc) {
  report(who, rc);
  throw std::runtime_error(b2s_last_error());
}

// One handle of type H with N capacities, kept for the process lifetime by the thread role that owns it: a handle owns
// device buffers and a stream, so creating one per call would put cudaMalloc / cudaFree on that thread's critical path.
// The caller holds `mutex` across get() and every use of `h`.  Capacities only grow: a regrowth takes, per dimension,
// the largest of what is needed, what the handle had and the floor, so problems of alternating shapes settle on one
// handle instead of recreating it on every call.
//
// There is no destructor: a process-wide slot would be freed at static destruction, possibly after the CUDA runtime has
// gone.  A slot that must free its handle (a thread-local one) destroys `h` itself.
template <class H, int N, void (*Destroy)(H*)>
struct Slot {
  H* h = nullptr;
  int cap[N] = {};
  std::mutex mutex;

  // B2S_OK with `h` able to hold `need`; `create(cap, &h)` makes a handle of capacities `cap`.  A failed create's code
  // is returned for the caller to report with the call it guards, with `h` null and the capacities zero, so that the
  // next call tries again.
  template <class Create>
  int get(const int (&need)[N], const int (&floor)[N], Create create) {
    bool fits = h != nullptr;
    for (int i = 0; i < N; i++) fits = fits && need[i] <= cap[i];
    if (fits) return B2S_OK;
    if (h) Destroy(h);
    h = nullptr;
    for (int i = 0; i < N; i++) cap[i] = std::max({need[i], cap[i], floor[i]});
    const int rc = create(static_cast<const int*>(cap), &h);
    if (rc != B2S_OK) {
      h = nullptr;
      for (int i = 0; i < N; i++) cap[i] = 0;
    }
    return rc;
  }
};

}  // namespace b2s_host
