// broker.h — process-wide batching broker behind layer 3 (include/b2h264_wels_api.h).
//
// The reference's ISVCEncoder is one object per stream and EncodeFrame is synchronous
// (codec/encoder/plus/src/welsEncoderExt.cpp:375).  The GPU pipeline earns its throughput by coding MANY streams
// per kernel launch (include/b2h264_codec.h, layer 2).  The broker reconciles the two: ISVCEncoder objects with
// equal configuration register as streams (slots) of ONE shared b2h264_enc ("pool"); EncodeFrame stages its picture,
// and the callers that arrive within a short window are coded as one batch — the caller that completes the set
// (or whose wait expires) runs submit + collect for everybody, the others sleep on a condition variable.
//   * pool capacity: B2H264_BROKER_SLOTS streams (default 128); further objects of the class open another pool,
//     pools are placed round-robin over the visible CUDA devices;
//   * wait: B2H264_BROKER_WAIT_US (default 2000) after a caller's arrival, skipped when every registered stream
//     of the pool is already waiting (so a lone encoder never waits).
// Streams that do not take part in a batch are passed as NULL sources to b2h264_enc_submit and keep their state.
#pragma once
#include <stdint.h>

#include <chrono>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <vector>

#include "b2h264_codec.h"

namespace b2wels {

struct PoolKey {
  int width, height, qp, bitrate, strategy, complexity_low, entropy_cabac, profile_idc, intra_period, dbk_idc, dbk_alpha, dbk_beta;
  float fps;
  bool operator==(const PoolKey& o) const {
    return width == o.width && height == o.height && qp == o.qp && bitrate == o.bitrate && strategy == o.strategy && complexity_low == o.complexity_low && entropy_cabac == o.entropy_cabac &&
           profile_idc == o.profile_idc && intra_period == o.intra_period && dbk_idc == o.dbk_idc &&
           dbk_alpha == o.dbk_alpha && dbk_beta == o.dbk_beta && fps == o.fps;
  }
};

class Pool {
 public:
  Pool(const PoolKey& key, int capacity, int device);
  ~Pool();
  bool ok() const { return enc_ != nullptr; }
  const PoolKey& key() const { return key_; }
  int device() const { return device_; }
  int acquire();                     // a free slot (fresh stream state) or -1
  void release(int slot);
  int registered();
  // synchronous: codes `planes` (tightly packed I420 already gathered into the slot's staging picture by stage())
  // as the next picture of `slot`; *au receives the access unit, *idr its type.  0 or a negative / CUDA error.
  uint8_t* staging(int slot) { return pinned_ + (size_t)slot * frame_bytes_; }
  // starts the host -> device copy of the slot's staged picture right away (on the caller's thread): by the time the last
  // stream of a batch arrives the pictures of the others are already in HBM
  int upload(int slot);
  int encode(int slot, std::vector<uint8_t>* au, bool* idr);
  int force_idr(int slot);

 private:
  enum State { FREE, IDLE, PENDING, INFLIGHT, DONE, FAILED };
  void flush_locked(std::unique_lock<std::mutex>& lk);
  PoolKey key_;
  int cap_, device_;
  size_t frame_bytes_;
  b2h264_enc* enc_ = nullptr;
  uint8_t* pinned_ = nullptr;
  uint8_t* d_stage_ = nullptr;             // device copies of the staged pictures (what the batch reads)
  void* up_stream_ = nullptr;              // cudaStream_t of the early uploads
  std::mutex m_;
  std::condition_variable cv_;
  std::vector<State> state_;
  std::vector<std::vector<uint8_t>> au_;
  std::vector<uint8_t> idr_;
  int n_registered_ = 0, n_pending_ = 0, last_rc_ = 0;
  bool flushing_ = false;
  long wait_us_;
};

// The same for ISVCDecoder objects: decoders of one picture size are streams of ONE shared b2h264_dec.  DecodeFrame2 hands in its
// access unit (the caller's own buffer: the caller blocks until the batch is done) and gets its picture in the slot's page-locked
// output area; every stream of a batch has its own outcome (b2h264_dec_decode3), a broken stream does not disturb the others.
class DecPool {
 public:
  DecPool(int width, int height, int capacity, int device);
  ~DecPool();
  bool ok() const { return dec_ != nullptr; }
  int width() const { return w_; }
  int height() const { return h_; }
  int acquire();
  void release(int slot);
  int registered();
  uint8_t* picture(int slot) { return pinned_ + (size_t)slot * frame_bytes_; }
  // synchronous: decodes the access unit as the next unit of `slot`.  Returns the stream's status: 1 picture (in picture(slot)),
  // 0 no picture, < 0 the layer-2 error of this stream / the call
  int decode(int slot, const uint8_t* au, int32_t bytes);
  // of the picture `slot` decoded last (b2h264_dec_last_picture_order); only the slot's owner calls this, between its decode calls
  void picture_order(int slot, int32_t* poc, int32_t* flags, int32_t* depth) { b2h264_dec_last_picture_order(dec_, slot, poc, flags, depth); }

 private:
  enum State { FREE, IDLE, PENDING, INFLIGHT, DONE };
  void flush_locked(std::unique_lock<std::mutex>& lk);
  int w_, h_, cap_, device_;
  size_t frame_bytes_;
  b2h264_dec* dec_ = nullptr;
  uint8_t* pinned_ = nullptr;
  std::mutex m_;
  std::condition_variable cv_;
  std::vector<State> state_;
  std::vector<const uint8_t*> au_;
  std::vector<int32_t> bytes_, status_;
  int n_registered_ = 0, n_pending_ = 0;
  bool flushing_ = false;
  long wait_us_;
};

// the pools of the process
class Broker {
 public:
  static Broker& get();
  // registers a stream; returns its pool + slot (nullptr on failure)
  std::shared_ptr<Pool> attach(const PoolKey& key, int* slot);
  void detach(const std::shared_ptr<Pool>& pool, int slot);
  std::shared_ptr<DecPool> attach_decoder(int width, int height, int* slot);
  void detach_decoder(const std::shared_ptr<DecPool>& pool, int slot);

 private:
  std::mutex m_;
  std::vector<std::shared_ptr<Pool>> pools_;
  std::vector<std::shared_ptr<DecPool>> dec_pools_;
  int next_device_ = 0;
};

}  // namespace b2wels
