// Drives b2s_host::Slot (self_commit_orb-slam2_b200/host/b2s_host.h) with a fake handle whose create and destroy count
// their calls, so that the growth rule and the failure path are checked without a device.  One scenario per run:
//   host_slot_harness <scenario>     prints "ok" and exits 0, or names the failed check and exits 1
//   host_slot_harness device         prints b2s_host::device()
//   host_slot_harness report         calls b2s_host::report("who", 3) (the line goes to stderr)
//   host_slot_harness fail           calls b2s_host::fail("who", 3) and prints what it threw
#include <cstdio>
#include <cstring>
#include <map>
#include <stdexcept>
#include <string>

#include "b2s_host.h"

extern "C" const char* b2s_last_error(void) { return "fake error"; }

namespace {

struct Fake {
  int cap[3];
};

int g_creates = 0, g_fail_rc = B2S_OK;
std::map<const Fake*, int> g_destroyed;  // every handle created, with the number of times it was destroyed

void destroy_fake(Fake* h) { g_destroyed[h]++; }

int create_fake(const int* cap, Fake** h) {
  g_creates++;
  if (g_fail_rc != B2S_OK) return g_fail_rc;
  *h = new Fake{{cap[0], cap[1], cap[2]}};  // never freed: a destroyed handle's address stays unique for the count
  g_destroyed[*h] = 0;
  return B2S_OK;
}

using FakeSlot = b2s_host::Slot<Fake, 3, destroy_fake>;

#define CHECK(c)                                              \
  do {                                                        \
    if (!(c)) {                                               \
      printf("check failed at line %d: %s\n", __LINE__, #c); \
      return 1;                                               \
    }                                                         \
  } while (0)

bool caps_are(const FakeSlot& s, int a, int b, int c) {
  return s.cap[0] == a && s.cap[1] == b && s.cap[2] == c && s.h && s.h->cap[0] == a && s.h->cap[1] == b &&
         s.h->cap[2] == c;
}

const int kFloor[3] = {64, 8192, 65536};

int first() {  // the first get creates at the floors
  FakeSlot s;
  CHECK(s.get({10, 100, 1000}, kFloor, create_fake) == B2S_OK);
  CHECK(g_creates == 1);
  CHECK(caps_are(s, 64, 8192, 65536));
  return 0;
}

int reuse() {  // a request within capacity keeps the handle
  FakeSlot s;
  CHECK(s.get({10, 100, 1000}, kFloor, create_fake) == B2S_OK);
  Fake* h = s.h;
  CHECK(s.get({64, 8192, 65536}, kFloor, create_fake) == B2S_OK);
  CHECK(s.get({0, 0, 0}, kFloor, create_fake) == B2S_OK);
  CHECK(s.h == h && g_creates == 1 && g_destroyed[h] == 0);
  return 0;
}

int grow() {  // an overflow grows every dimension to max(need, cap, floor)
  FakeSlot s;
  CHECK(s.get({100, 10, 10}, kFloor, create_fake) == B2S_OK);
  CHECK(caps_are(s, 100, 8192, 65536));
  CHECK(s.get({50, 9000, 70000}, kFloor, create_fake) == B2S_OK);
  CHECK(caps_are(s, 100, 9000, 70000));
  CHECK(s.get({101, 1, 1}, kFloor, create_fake) == B2S_OK);
  CHECK(caps_are(s, 101, 9000, 70000));
  CHECK(g_creates == 3);
  return 0;
}

int alternate() {  // two shapes, each overflowing the other's largest dimension: one regrowth, then none
  FakeSlot s;
  for (int i = 0; i < 10; i++) {
    CHECK(s.get({70, 5000, 65536}, kFloor, create_fake) == B2S_OK);
    CHECK(s.get({50, 9000, 65536}, kFloor, create_fake) == B2S_OK);
  }
  CHECK(g_creates == 2);
  CHECK(caps_are(s, 70, 9000, 65536));
  return 0;
}

int failed_create() {  // a failed create hands back its code, leaves no handle and no capacity; the next get retries
  FakeSlot s;
  CHECK(s.get({100, 10, 10}, kFloor, create_fake) == B2S_OK);
  g_fail_rc = B2S_ERR_CUDA;
  CHECK(s.get({200, 10, 10}, kFloor, create_fake) == B2S_ERR_CUDA);
  CHECK(s.h == nullptr && s.cap[0] == 0 && s.cap[1] == 0 && s.cap[2] == 0);
  CHECK(s.get({1, 1, 1}, kFloor, create_fake) == B2S_ERR_CUDA);  // still failing: tried again
  CHECK(g_creates == 3);
  g_fail_rc = B2S_OK;
  CHECK(s.get({1, 1, 1}, kFloor, create_fake) == B2S_OK);
  CHECK(g_creates == 4);
  CHECK(caps_are(s, 64, 8192, 65536));
  return 0;
}

int destroy_once() {  // each replaced handle is destroyed exactly once; the live one is not
  FakeSlot s;
  const int shapes[][3] = {{1, 1, 1}, {65, 1, 1}, {1, 9000, 1}, {2, 2, 2}, {1, 1, 70000}, {66, 9001, 70001}};
  for (const auto& n : shapes) CHECK(s.get({n[0], n[1], n[2]}, kFloor, create_fake) == B2S_OK);
  CHECK(g_creates == 5 && (int)g_destroyed.size() == 5);
  for (const auto& kv : g_destroyed) CHECK(kv.second == (kv.first == s.h ? 0 : 1));
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  if (argc != 2) return 2;
  const std::string what = argv[1];
  if (what == "device") {
    printf("%d\n", b2s_host::device());
    return 0;
  }
  if (what == "report") {
    b2s_host::report("who", 3);
    return 0;
  }
  if (what == "fail") {
    try {
      b2s_host::fail("who", 3);
    } catch (const std::runtime_error& e) {
      printf("%s\n", e.what());
    }
    return 0;
  }
  const std::map<std::string, int (*)()> scenarios = {{"first", first},   {"reuse", reuse},
                                                      {"grow", grow},     {"alternate", alternate},
                                                      {"failed_create", failed_create}, {"destroy_once", destroy_once}};
  const auto it = scenarios.find(what);
  if (it == scenarios.end()) return 2;
  const int rc = it->second();
  if (rc == 0) printf("ok\n");
  return rc;
}
