// batcher_test.cpp — the batching core of the broker (openh264_b200/wels/batcher.h) behind a fake coder, without a GPU.
// usage: batcher_test many | fail | lone | release      (exit status 0: every check held)
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <chrono>
#include <thread>
#include <vector>

#include "batcher.h"

#define CHECK(c)                                                                   \
  do {                                                                             \
    if (!(c)) { fprintf(stderr, "%s:%d: check failed: %s\n", __FILE__, __LINE__, #c); exit(1); } \
  } while (0)

namespace {

const int kFailed = -77;        // the result of every slot of the batch the coder is told to fail
const int kBatchStride = 1000;  // a successful result is batch number * kBatchStride + slot

// Records each batch, sleeps step_ms in it, and fails batch number fail_batch.  phase[s] follows slot s through one run():
// 0 outside, 1 pending (set by the owner before it joins), 2 coded (set here); the owner checks it went 0 -> 1 -> 2 -> 0.
struct FakeCoder : b2wels::Batcher {
  explicit FakeCoder(int cap) : Batcher(cap), phase(cap) {}
  void code_batch(const std::vector<int>& slots, int* result) override {
    const int n = (int)batches.size();
    for (int s : slots) CHECK(phase[s].exchange(2) == 1);    // only pending slots, each once
    batches.push_back(slots);                                // one batch at a time: no lock needed
    started = true;
    std::this_thread::sleep_for(std::chrono::milliseconds(step_ms));
    for (int s : slots) result[s] = n == fail_batch ? kFailed : n * kBatchStride + s;
    step_returned = true;
  }
  void reset_stream(int slot) override { resets.push_back(slot); }   // under the core's lock
  int call(int slot) {
    CHECK(phase[slot].exchange(1) == 0);
    const int rc = run(slot);
    CHECK(phase[slot].exchange(0) == 2);
    return rc;
  }
  std::vector<std::atomic<int>> phase;
  std::vector<std::vector<int>> batches;
  std::vector<int> resets;
  int step_ms = 1, fail_batch = -1;
  std::atomic<bool> started{false}, step_returned{false};
};

// T threads x P calls, each thread with its own slot, releasing it after its last call; returns every thread's results.
// Some calls come late, past the window, so that batches also form while other slots are idle
std::vector<std::vector<int>> run_threads(FakeCoder& c, int T, int P) {
  std::vector<int> slot(T);
  for (int t = 0; t < T; t++) CHECK((slot[t] = c.acquire()) >= 0);
  std::vector<std::vector<int>> rc(T);
  std::vector<std::thread> th;
  for (int t = 0; t < T; t++)
    th.emplace_back([&, t] {
      for (int p = 0; p < P; p++) {
        if ((p + t) % 7 == 0) std::this_thread::sleep_for(std::chrono::milliseconds(3));
        rc[t].push_back(c.call(slot[t]));
      }
      c.release(slot[t]);
    });
  for (auto& x : th) x.join();
  CHECK(c.registered() == 0 && (int)c.resets.size() == T);
  for (int t = 0; t < T; t++) CHECK(slot[t] == t);            // acquire hands out the lowest free slot
  return rc;
}

// every call returns its own slot's result from a batch that holds the slot, and T x P pictures are coded in all
void many() {
  const int T = 8, P = 200;
  FakeCoder c(16);
  const auto rc = run_threads(c, T, P);
  size_t coded = 0;
  for (auto& b : c.batches) coded += b.size();
  CHECK(coded == (size_t)T * P);
  for (int t = 0; t < T; t++) {
    int last = -1;
    for (int r : rc[t]) {
      const int n = r / kBatchStride;
      CHECK(r >= 0 && r % kBatchStride == t && n > last && n < (int)c.batches.size());
      bool held = false;
      for (int s : c.batches[n]) held |= s == t;
      CHECK(held);
      last = n;
    }
  }
}

// every caller of the failed batch gets the failure, and the callers of the next batch succeed
void fail() {
  const int T = 6, P = 20, bad = 3;
  FakeCoder c(8);
  c.fail_batch = bad;
  const auto rc = run_threads(c, T, P);
  CHECK((int)c.batches.size() > bad + 1);
  std::vector<int> failures(T, 0);
  for (int t = 0; t < T; t++)
    for (int r : rc[t]) {
      if (r == kFailed) failures[t]++;
      else CHECK(r >= 0 && r % kBatchStride == t);
    }
  std::vector<int> expect(T, 0);
  for (int s : c.batches[bad]) expect[s] = 1;
  CHECK(failures == expect);
  for (int s : c.batches[bad + 1]) {
    bool ok = false;
    for (int r : rc[s]) ok |= r == (bad + 1) * kBatchStride + s;
    CHECK(ok);
  }
}

// a lone registered slot never waits for the window (10 s here)
void lone() {
  const int P = 20;
  FakeCoder c(4);
  const int s = c.acquire();
  const auto t0 = std::chrono::steady_clock::now();
  for (int p = 0; p < P; p++) CHECK(c.call(s) == p * kBatchStride + s);
  const double secs = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  printf("%d calls of a lone slot: %.3f s\n", P, secs);
  CHECK(secs < 5.0);
  c.release(s);
}

// a release issued while a batch is in flight returns only after the batch's step has returned, and resets that stream
void release() {
  FakeCoder c(4);
  c.step_ms = 200;
  const int a = c.acquire(), b = c.acquire();
  int rc = -1;
  std::thread owner([&] { rc = c.call(a); });           // b is registered but idle: the batch {a} starts when the window expires
  while (!c.started) std::this_thread::sleep_for(std::chrono::milliseconds(1));
  c.release(b);
  CHECK(c.step_returned);
  owner.join();
  CHECK(rc == a && c.batches.size() == 1 && c.batches[0] == std::vector<int>{a});
  CHECK(c.resets == std::vector<int>{b} && c.registered() == 1);
  c.release(a);
}

}  // namespace

int main(int argc, char** argv) {
  const char* which = argc > 1 ? argv[1] : "";
  // the window the core reads: the default, except for the lone slot, which must not wait for it
  setenv("B2H264_BROKER_WAIT_US", strcmp(which, "lone") ? "2000" : "10000000", 1);
  if (!strcmp(which, "many")) many();
  else if (!strcmp(which, "fail")) fail();
  else if (!strcmp(which, "lone")) lone();
  else if (!strcmp(which, "release")) release();
  else { fprintf(stderr, "usage: %s many | fail | lone | release\n", argv[0]); return 2; }
  printf("%s: ok\n", which);
  return 0;
}
