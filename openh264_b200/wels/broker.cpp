// broker.cpp — see broker.h
#include "broker.h"

#include <cuda_runtime_api.h>
#include <string.h>

namespace b2wels {

EncPool::EncPool(const PoolKey& key, int capacity, int device) : Batcher(capacity), key_(key), device_(device) {
  frame_bytes_ = (size_t)key.width * key.height * 3 / 2;
  b2h264_enc_config cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.width = key.width; cfg.height = key.height; cfg.qp = key.qp; cfg.fps = key.fps;
  cfg.target_bitrate = key.bitrate;
  cfg.n_streams = capacity;
  cfg.entropy_threads = 0;
  cfg.device = device;
  cfg.sps_pps_id_strategy = key.strategy;
  cfg.complexity_low = key.complexity_low;
  cfg.entropy_cabac = key.entropy_cabac;
  cfg.profile_idc = key.profile_idc;
  cfg.intra_period = key.intra_period;
  cfg.loop_filter_idc = key.dbk_idc; cfg.loop_filter_alpha_c0_offset = key.dbk_alpha; cfg.loop_filter_beta_offset = key.dbk_beta;
  if (b2h264_enc_create(&cfg, &enc_) != 0) { enc_ = nullptr; return; }
  // on failure ok() is false and the destructor releases what was acquired
  // the resolved partition, handed back as a raster request that resolves to it: one slice per row (which a picture of at most
  // 48 macroblocks keeps), or explicit runs
  const int mb_w = (key.width + 15) >> 4, mb_h = (key.height + 15) >> 4;
  bool rows = key.slice_num > 1 && key.slice_num == mb_h;
  for (int k = 0; rows && k < key.slice_num; k++) rows = key.slice_mb[k] == (uint32_t)mb_w;
  const uint32_t no_runs[b2h264::kMaxSlicesNum] = {};
  if (b2h264_enc_set_references(enc_, key.num_ref_frames, key.ltr, 30) != 0 ||
      b2h264_enc_set_slices(enc_, key.slice_num > 1 ? b2h264::kSmRaster : b2h264::kSmSingle, key.slice_num,
                            rows ? no_runs : key.slice_mb) != 0 ||
      cudaSetDevice(device) != cudaSuccess ||
      pinned_.alloc(frame_bytes_ * capacity, cudaHostAllocPortable) != cudaSuccess || d_stage_.alloc(frame_bytes_ * capacity) != cudaSuccess ||
      up_stream_.create(cudaStreamNonBlocking) != cudaSuccess) {
    b2h264_enc_destroy(enc_);
    enc_ = nullptr;
    return;
  }
  au_.resize(capacity);
  idr_.assign(capacity, 0);
}

EncPool::~EncPool() {
  cudaSetDevice(device_);
  if (up_stream_.get()) cudaStreamSynchronize(up_stream_.get());
  if (enc_) b2h264_enc_destroy(enc_);
}

int EncPool::upload(int slot) {
  if (cudaSetDevice(device_) != cudaSuccess) return -1;
  return cudaMemcpyAsync(d_stage_.get() + (size_t)slot * frame_bytes_, pinned_.get() + (size_t)slot * frame_bytes_, frame_bytes_, cudaMemcpyHostToDevice,
                         up_stream_.get()) == cudaSuccess ? 0 : -1;
}

int EncPool::force_idr(int slot) {
  return when_idle([&] { return b2h264_enc_force_idr(enc_, slot); });
}

int EncPool::ltr_recovery_request(int slot, int type, int idr_pic_id, int cur_frame_num, int last_correct_frame_num) {
  return when_idle([&] { return b2h264_enc_ltr_recovery_request(enc_, slot, type, idr_pic_id, cur_frame_num, last_correct_frame_num); });
}

int EncPool::ltr_marking_feedback(int slot, int type, int idr_pic_id, int ltr_frame_num) {
  return when_idle([&] { return b2h264_enc_ltr_marking_feedback(enc_, slot, type, idr_pic_id, ltr_frame_num); });
}

int EncPool::ltr_mark_period(int slot, int period) {
  return when_idle([&] { return b2h264_enc_ltr_mark_period(enc_, slot, period); });
}

void EncPool::code_batch(const std::vector<int>& slots, int* result) {
  std::vector<const uint8_t*> src(cap_, nullptr), bs(cap_, nullptr);
  std::vector<int32_t> nb(cap_, 0), ft(cap_, 0);
  for (int s : slots) src[s] = d_stage_.get() + (size_t)s * frame_bytes_;
  // every stream of the batch enqueued its upload before it joined: one wait covers them all
  int rc = cudaSetDevice(device_) == cudaSuccess && cudaStreamSynchronize(up_stream_.get()) == cudaSuccess ? 0 : -1;
  if (rc == 0) rc = b2h264_enc_submit(enc_, src.data(), 1);
  if (rc == 0) rc = b2h264_enc_collect(enc_, bs.data(), nb.data(), ft.data());
  for (int s : slots) {
    if (rc == 0 && bs[s]) { au_[s].assign(bs[s], bs[s] + nb[s]); idr_[s] = ft[s] == 1; }
    result[s] = rc ? rc : (bs[s] ? 0 : -1);
  }
}

int EncPool::encode(int slot, std::vector<uint8_t>* au, bool* idr) {
  const int rc = run(slot);
  if (rc == 0) { au->swap(au_[slot]); *idr = idr_[slot] != 0; }
  return rc;
}

// ---------------------------------------------------------------------------------------------------------------------
DecPool::DecPool(int width, int height, int capacity, int device) : Batcher(capacity), w_(width), h_(height) {
  frame_bytes_ = (size_t)width * height * 3 / 2;
  b2h264_dec_config cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.width = width; cfg.height = height; cfg.n_streams = capacity; cfg.device = device;
  if (b2h264_dec_create(&cfg, &dec_) != 0) { dec_ = nullptr; return; }
  pinned_ = static_cast<uint8_t*>(b2h264_host_alloc(frame_bytes_ * capacity));
  if (!pinned_) { b2h264_dec_destroy(dec_); dec_ = nullptr; return; }
  au_.assign(capacity, nullptr);
  bytes_.assign(capacity, 0);
}

DecPool::~DecPool() {
  if (dec_) b2h264_dec_destroy(dec_);
  if (pinned_) b2h264_host_free(pinned_);
}

void DecPool::code_batch(const std::vector<int>& slots, int* result) {
  std::vector<const uint8_t*> au(cap_, nullptr);
  std::vector<int32_t> nb(cap_, 0), st(cap_, 0);
  std::vector<uint8_t*> out(cap_);
  for (int s = 0; s < cap_; s++) out[s] = picture(s);
  for (int s : slots) { au[s] = au_[s]; nb[s] = bytes_[s]; }
  const int rc = b2h264_dec_decode3(dec_, au.data(), nb.data(), out.data(), st.data());
  for (int s : slots) result[s] = rc ? (rc > 0 ? -1000 - rc : rc) : st[s];   // a failure of the call as a whole fails every stream of the batch
}

int DecPool::decode(int slot, const uint8_t* au, int32_t bytes) {
  if (slot < 0 || slot >= cap_) return -1;
  au_[slot] = au; bytes_[slot] = bytes;
  return run(slot);
}

// ---------------------------------------------------------------------------------------------------------------------
Broker& Broker::get() {
  static Broker* b = new Broker();       // never destroyed: encoder objects may outlive static destruction order
  return *b;
}

template <class P, class... Args>
std::shared_ptr<P> Broker::attach_pool(int* slot, const Args&... args) {
  std::lock_guard<std::mutex> g(m_);
  int same_class = 0;
  for (auto& b : pools_) {
    auto p = std::dynamic_pointer_cast<P>(b);
    if (!p || !p->serves(args...)) continue;
    same_class++;
    const int s = p->acquire();
    if (s >= 0) { *slot = s; return p; }
  }
  // capacity: B2H264_BROKER_SLOTS, else 4, 16, 64, 128, 128, ... for successive pools of a class (a lone stream stays
  // small: an encoder slot costs ~30 MB of HBM and ~25 MB of pinned host memory at 1080p)
  long cap = env_long("B2H264_BROKER_SLOTS", 0);
  if (cap <= 0) { cap = 4L << (2 * (same_class < 3 ? same_class : 3)); if (cap > 128) cap = 128; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) return nullptr;
  const long dev_env = env_long("B2H264_DEVICE", -1);
  const int device = dev_env >= 0 ? (int)(dev_env % ndev) : (next_device_++ % ndev);
  auto p = std::make_shared<P>(args..., (int)cap, device);
  if (!p->ok()) return nullptr;
  pools_.push_back(p);
  *slot = p->acquire();
  return p;
}

std::shared_ptr<EncPool> Broker::attach(const PoolKey& key, int* slot) { return attach_pool<EncPool>(slot, key); }

std::shared_ptr<DecPool> Broker::attach_decoder(int width, int height, int* slot) { return attach_pool<DecPool>(slot, width, height); }

void Broker::detach(const std::shared_ptr<Batcher>& pool, int slot) {
  pool->release(slot);
  std::lock_guard<std::mutex> g(m_);
  if (pool->registered() == 0)
    for (size_t i = 0; i < pools_.size(); i++)
      if (pools_[i] == pool) { pools_.erase(pools_.begin() + i); break; }     // the last reference frees the coder
}

}  // namespace b2wels
