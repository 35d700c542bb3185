// broker.h — process-wide batching broker behind layer 3 (include/b2h264_wels_api.h).
//
// The reference's ISVCEncoder and ISVCDecoder are one object per stream with synchronous calls
// (codec/encoder/plus/src/welsEncoderExt.cpp:375).  The GPU pipeline earns its throughput by coding MANY streams per kernel
// launch (include/b2h264_codec.h, layer 2).  The broker reconciles the two: objects of one class register as streams (slots) of
// ONE shared batched coder ("pool"), and the calls that arrive within a short window are coded as one batch (Batcher, batcher.h:
// the caller that completes the set, or whose wait expires, codes for everybody, the others sleep on a condition variable).
//   * EncPool: ISVCEncoder objects of equal configuration (PoolKey) share one b2h264_enc.  EncodeFrame stages its picture and
//     starts its upload on the caller's thread; streams that do not take part in a batch are passed as NULL sources to
//     b2h264_enc_submit and keep their state.
//   * DecPool: ISVCDecoder objects of one picture size share one b2h264_dec.  DecodeFrame2 hands in its access unit (the caller's
//     own buffer: the caller blocks until the batch is done) and gets its picture in the slot's page-locked output area; every
//     stream of a batch has its own outcome (b2h264_dec_decode3), a broken stream does not disturb the others.
//   * pool capacity: B2H264_BROKER_SLOTS streams, else 4, 16, 64, 128, 128, ... for successive pools of a class; pools are
//     placed round-robin over the visible CUDA devices (B2H264_DEVICE pins one);
//   * wait: B2H264_BROKER_WAIT_US (default 2000) after a caller's arrival, skipped when every registered stream of the pool is
//     already waiting (so a lone stream never waits).
#pragma once
#include <stdint.h>
#include <string.h>

#include <memory>
#include <mutex>
#include <vector>

#include "../csrc/cuda_owned.h"
#include "../csrc/enc_slices.h"
#include "b2h264_codec.h"
#include "batcher.h"

namespace b2wels {

struct PoolKey {
  int width, height, qp, bitrate, strategy, complexity_low, entropy_cabac, profile_idc, intra_period, dbk_idc, dbk_alpha, dbk_beta;
  // resolved reference configuration (max_num_ref_frames of the SPS, LTR on / off): every stream of a pool has the same picture
  // store; the LTR marking period is per stream (EncPool::ltr_mark_period)
  int num_ref_frames = 1, ltr = 0;
  // resolved slice partition (enc_slices.h): the run length of every slice; dbk_idc above is the idc as coded
  int slice_num = 1;
  uint32_t slice_mb[b2h264::kMaxSlicesNum] = {};
  float fps;
  bool operator==(const PoolKey& o) const {
    return width == o.width && height == o.height && qp == o.qp && bitrate == o.bitrate && strategy == o.strategy && complexity_low == o.complexity_low && entropy_cabac == o.entropy_cabac &&
           profile_idc == o.profile_idc && intra_period == o.intra_period && dbk_idc == o.dbk_idc &&
           dbk_alpha == o.dbk_alpha && dbk_beta == o.dbk_beta && num_ref_frames == o.num_ref_frames && ltr == o.ltr && fps == o.fps &&
           slice_num == o.slice_num && memcmp(slice_mb, o.slice_mb, sizeof(slice_mb)) == 0;
  }
};

class EncPool : public Batcher {
 public:
  EncPool(const PoolKey& key, int capacity, int device);
  ~EncPool() override;
  bool ok() const { return enc_ != nullptr; }
  bool serves(const PoolKey& key) const { return key == key_; }
  // the slot's page-locked staging picture: the caller gathers its planes here (tightly packed I420) before upload()
  uint8_t* staging(int slot) { return pinned_.get() + (size_t)slot * frame_bytes_; }
  // starts the host -> device copy of the slot's staged picture right away (on the caller's thread): by the time the last
  // stream of a batch arrives the pictures of the others are already in HBM
  int upload(int slot);
  // synchronous: codes the uploaded picture as the next picture of `slot`; *au receives the access unit, *idr its type.
  // 0 or a negative / CUDA error
  int encode(int slot, std::vector<uint8_t>* au, bool* idr);
  int force_idr(int slot);
  // loss-recovery feedback and the marking period of the slot's stream: they take effect on its next picture
  int ltr_recovery_request(int slot, int type, int idr_pic_id, int cur_frame_num, int last_correct_frame_num);
  int ltr_marking_feedback(int slot, int type, int idr_pic_id, int ltr_frame_num);
  int ltr_mark_period(int slot, int period);
  // the resolved reference configuration (b2h264_enc_get_references)
  int references(int32_t* out4) { return b2h264_enc_get_references(enc_, out4); }

 private:
  void code_batch(const std::vector<int>& slots, int* result) override;
  void reset_stream(int slot) override { b2h264_enc_reset_stream(enc_, slot); }
  PoolKey key_;
  int device_;
  size_t frame_bytes_;
  b2h264_enc* enc_ = nullptr;
  b2h264::Stream up_stream_;               // the early uploads; released after the buffers below
  b2h264::HostBuf<uint8_t> pinned_;
  b2h264::DeviceBuf<uint8_t> d_stage_;     // device copies of the staged pictures (what the batch reads)
  std::vector<std::vector<uint8_t>> au_;
  std::vector<uint8_t> idr_;
};

class DecPool : public Batcher {
 public:
  DecPool(int width, int height, int capacity, int device);
  ~DecPool() override;
  bool ok() const { return dec_ != nullptr; }
  bool serves(int width, int height) const { return width == w_ && height == h_; }
  uint8_t* picture(int slot) { return pinned_ + (size_t)slot * frame_bytes_; }
  // synchronous: decodes the access unit as the next unit of `slot`.  Returns the stream's status: 1 picture (in picture(slot)),
  // 0 no picture, < 0 the layer-2 error of this stream / the call
  int decode(int slot, const uint8_t* au, int32_t bytes);
  // of the picture `slot` decoded last (b2h264_dec_last_picture_order); only the slot's owner calls this, between its decode calls
  void picture_order(int slot, int32_t* poc, int32_t* flags, int32_t* depth) { b2h264_dec_last_picture_order(dec_, slot, poc, flags, depth); }

 private:
  void code_batch(const std::vector<int>& slots, int* result) override;
  void reset_stream(int slot) override { b2h264_dec_reset_stream(dec_, slot); }
  int w_, h_;
  size_t frame_bytes_;
  b2h264_dec* dec_ = nullptr;
  uint8_t* pinned_ = nullptr;
  std::vector<const uint8_t*> au_;         // the owner's access unit of each slot, written before it joins a batch
  std::vector<int32_t> bytes_;
};

// the pools of the process
class Broker {
 public:
  static Broker& get();
  // registers a stream; returns its pool + slot (nullptr on failure)
  std::shared_ptr<EncPool> attach(const PoolKey& key, int* slot);
  std::shared_ptr<DecPool> attach_decoder(int width, int height, int* slot);
  void detach(const std::shared_ptr<Batcher>& pool, int slot);

 private:
  // a free slot of a pool of type P that serves(args...), else the first slot of a new such pool, made as P(args..., capacity, device)
  template <class P, class... Args>
  std::shared_ptr<P> attach_pool(int* slot, const Args&... args);
  std::mutex m_;
  std::vector<std::shared_ptr<Batcher>> pools_;
  int next_device_ = 0;                    // shared by encoder and decoder pools
};

}  // namespace b2wels
