// batcher.h — the batching core of the broker's encoder and decoder pools (broker.h).  Plain C++: no CUDA header, so that a
// test can put a fake coder behind it (tests/wels/batcher_test.cpp).
#pragma once
#include <condition_variable>
#include <mutex>
#include <vector>

namespace b2wels {

// the integer value of environment variable `name`, `dflt` when it is unset or empty
long env_long(const char* name, long dflt);

// Slots are the streams of one batched coder.  A slot's owner thread calls run(slot) once per unit; the callers that arrive within
// the window (B2H264_BROKER_WAIT_US, default 2000 µs, after a caller's arrival) are coded as one batch by the caller that
// completes the set of registered slots or whose wait expires, while the others sleep.  A lone slot never waits.  At most one batch
// is in flight at a time.
class Batcher {
 public:
  explicit Batcher(int capacity);
  virtual ~Batcher() = default;
  int acquire();                          // a free slot (fresh stream state) or -1
  void release(int slot);                 // waits out a batch in flight, resets the slot's stream and frees the slot
  int registered();
  // joins the next batch with `slot` and returns the result code_batch() wrote for it; -1 for a slot that is not registered
  int run(int slot);

  // runs f() under the lock once no batch is in flight, and returns what it returns
  template <class F>
  auto when_idle(F f) {
    std::unique_lock<std::mutex> lk(m_);
    cv_.wait(lk, [&] { return !flushing_; });
    return f();
  }

 protected:
  const int cap_;
  // codes one batch: `slots` lists its slots (each once, in increasing order); writes result[s] (indexed by slot) for each of them.
  // Called without the lock; a slot's owner does not touch the slot's data until run() returns
  virtual void code_batch(const std::vector<int>& slots, int* result) = 0;
  virtual void reset_stream(int slot) = 0;       // called under the lock, no batch in flight

 private:
  enum State { FREE, IDLE, PENDING, INFLIGHT, DONE };
  void flush_locked(std::unique_lock<std::mutex>& lk);
  const long wait_us_;
  std::mutex m_;
  std::condition_variable cv_;
  std::vector<State> state_;
  std::vector<int> result_;
  int n_registered_ = 0, n_pending_ = 0;
  bool flushing_ = false;
};

}  // namespace b2wels
