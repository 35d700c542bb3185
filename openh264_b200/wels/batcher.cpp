// batcher.cpp — see batcher.h
#include "batcher.h"

#include <stdlib.h>

#include <chrono>

namespace b2wels {

long env_long(const char* name, long dflt) {
  const char* v = getenv(name);
  return v && *v ? atol(v) : dflt;
}

Batcher::Batcher(int capacity)
    : cap_(capacity), wait_us_(env_long("B2H264_BROKER_WAIT_US", 2000)), state_(capacity, FREE), result_(capacity, 0) {}

int Batcher::acquire() {
  std::unique_lock<std::mutex> lk(m_);
  for (int s = 0; s < cap_; s++)
    if (state_[s] == FREE) { state_[s] = IDLE; n_registered_++; return s; }
  return -1;
}

void Batcher::release(int slot) {
  when_idle([&] {
    reset_stream(slot);
    state_[slot] = FREE;
    n_registered_--;
    cv_.notify_all();                                  // "everybody is waiting" may have become true
  });
}

int Batcher::registered() {
  std::unique_lock<std::mutex> lk(m_);
  return n_registered_;
}

// codes every PENDING slot as one batch; called with the lock held, returns with it held
void Batcher::flush_locked(std::unique_lock<std::mutex>& lk) {
  flushing_ = true;
  std::vector<int> slots;
  for (int s = 0; s < cap_; s++)
    if (state_[s] == PENDING) { state_[s] = INFLIGHT; slots.push_back(s); }
  n_pending_ = 0;
  lk.unlock();
  std::vector<int> rc(cap_, -1);
  code_batch(slots, rc.data());
  lk.lock();
  for (int s : slots) { result_[s] = rc[s]; state_[s] = DONE; }
  flushing_ = false;
  cv_.notify_all();
}

int Batcher::run(int slot) {
  std::unique_lock<std::mutex> lk(m_);
  if (slot < 0 || slot >= cap_ || state_[slot] != IDLE) return -1;
  state_[slot] = PENDING;
  n_pending_++;
  const auto deadline = std::chrono::steady_clock::now() + std::chrono::microseconds(wait_us_);
  while (state_[slot] != DONE) {
    if (state_[slot] == PENDING && !flushing_) {
      if (n_pending_ >= n_registered_ || std::chrono::steady_clock::now() >= deadline) { flush_locked(lk); continue; }
      cv_.wait_until(lk, deadline);
    } else {
      cv_.wait(lk);
    }
  }
  state_[slot] = IDLE;
  return result_[slot];
}

}  // namespace b2wels
