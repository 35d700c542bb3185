// enc_batch.cu — layer-2 batched frame encoder (include/b2h264_codec.h): device buffers, the asynchronous
// H2D -> kernels -> D2H pipeline on one CUDA stream, and host entropy coding on a small thread pool.
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <string.h>
#include <thread>
#include <vector>

#include "../../include/b2h264_codec.h"
#include "b2h264_internal.h"
#include "cuda_owned.h"
#include "enc_host.h"
#include "enc_launch.h"
#include "enc_slices.h"
#include "host_pool.h"

using b2h264::StreamCtl;
using b2h264::StreamRefs;
using b2h264::RefConfig;
using b2h264::RefDecision;
using b2h264::Pool;
using b2h264::PicLayout;
using b2h264::SliceConfig;
using b2h264::DeviceBuf;
using b2h264::HostBuf;
using b2h264::Event;
using b2h264::Stream;
using b2h264::usable_cores;

namespace {

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return (int)e_; } while (0)


}  // namespace

struct b2h264_enc {
  b2h264_enc_config cfg;
  int S = 0, n_mb = 0;
  std::vector<StreamCtl> ctl;
  std::vector<uint8_t> idr_next;          // per stream: code next picture as IDR
  std::vector<int32_t> p_since_idr;       // per stream: P pictures since the last IDR (SSpatialLayerInternal::iFrameIndex)
  std::vector<StreamRefs> refs;           // per stream: reference lists, long-term state, slots of its pictures (enc_refs.h)
  RefConfig refcfg;                       // b2h264_enc_set_references; the default is one reference, no LTR
  SliceConfig slices;                     // b2h264_enc_set_slices; the default is one slice per picture
  std::vector<int32_t> slice_first;       // first macroblock of each slice (more than one slice only)
  bool started = false;                   // a picture has been submitted: the picture store is fixed
  // the CUDA resources are released in the reverse order of their declaration: the buffers and events before the streams
  Stream own_st;                          // the encoder's kernel stream until b2h264_enc_set_stream lends it the caller's
  cudaStream_t st = nullptr;              // kernels: own_st or the caller's stream
  Stream st_in;                           // source uploads: overlap the previous picture's kernels
  Stream st_out;                          // record downloads: overlap deblocking and the next picture's kernels
  // device memory
  DeviceBuf<uint8_t> d_cur;               // refcfg.src_slots() x S x (Y,U,V) MB-aligned source pictures (current, previous and
                                          // long-term sources: VAA statistics), set * S + stream
  DeviceBuf<int32_t> d_vaa;               // S x n_mb x 4: 8x8 SADs against the previous source picture (LOW_COMPLEXITY)
  DeviceBuf<uint8_t> d_pic_all;           // picture store: refcfg.slots() x S x padded (Y,U,V), slot * S + stream
  DeviceBuf<uint8_t> d_src;               // S x raw I420 staging (2 slots)
  DeviceBuf<MbInfo> d_mbi;
  DeviceBuf<RefMbInfo> d_rinfo;           // co-located records of every stored picture: (slot * S + stream) x n_mb
  DeviceBuf<MbOut> d_out[2];
  DeviceBuf<int32_t> d_sad;
  DeviceBuf<int32_t> d_bits;              // S x n_mb: exact CAVLC bits per macroblock (when enabled)
  DeviceBuf<int32_t> d_slice_first;       // n_mb: first macroblock of each macroblock's slice (several slices only; EncFramePtrs)
  bool mb_bits_on = false;
  DeviceBuf<int> d_tickets;
  DeviceBuf<uint8_t> d_stash;             // parked macroblock scratches of the staged scheduler
  DeviceBuf<StreamFrame> d_sf[2];
  alignas(64) unsigned char tmap_pic[128];      // CUtensorMap of the luma planes of every slot of all streams
  bool have_tmap = false;
  DeviceBuf<const uint8_t*> d_srcptr[2];
  // pinned host memory
  HostBuf<uint8_t> h_src;                 // 2 slots x S x frame
  HostBuf<MbOut> h_out[2];                // mapped pinned: coded records, packed per stream (worst case sized)
  HostBuf<int32_t> h_idx[2];              // mapped pinned: per MB offset of its compact record (32-byte units) or -1
  HostBuf<int32_t> h_cnt[2];              // mapped pinned: 32-byte units written per stream
  unsigned long long last_d2h = 0;
  HostBuf<StreamFrame> h_sf[2];
  HostBuf<const uint8_t*> h_srcptr[2];
  // in-flight bookkeeping
  struct Slot { bool busy = false; std::vector<uint8_t> idr; std::vector<int> act;   // act: streams of this batch (compact order)
                std::vector<RefDecision> rd;                                       // per stream: reference decisions of its picture
                std::vector<int> dropped;                                          // streams whose picture was not coded (RefDecision::not_coded)
                Event ev0, ev1, ev2, done, in_done; };
  Slot slot[2];
  int submit_idx = 0, collect_idx = 0;
  std::vector<std::vector<uint8_t>> bs;   // per stream output of the last collect
  float last_us[4] = {0, 0, 0, 0};
  size_t frame_bytes = 0, cur_bytes = 0, pic_bytes = 0;
  PicLayout lay;                          // of each picture in the store; pic_bytes is its slot pitch, rounded up to 256 bytes
  std::unique_ptr<Pool> pool;             // declared last: its threads stop before anything they use is released

  uint8_t* pic_plane0(int slot, int s, int pl) const {   // pixel (0,0) of plane pl of stream s's picture in `slot`
    return d_pic_all.get() + ((size_t)slot * S + s) * pic_bytes + lay.plane0(pl);
  }
  // stream s's parameter sets and numbering as a fresh encoder starts them; false if cfg's loop-filter values are out of range
  bool init_stream(int s) {
    StreamCtl& c = ctl[s] = StreamCtl();
    c.init(cfg.width, cfg.height, cfg.qp, cfg.fps, cfg.target_bitrate, cfg.entropy_cabac, cfg.profile_idc);
    c.increasing_ids = cfg.sps_pps_id_strategy != 0;
    c.fast_mode = cfg.complexity_low != 0;
    c.record_mb_bits = mb_bits_on;
    c.set_num_ref_frames(refcfg.sps_num_ref_frames, cfg.target_bitrate);
    c.slice_first = slice_first;
    return c.set_loop_filter(cfg.loop_filter_idc, cfg.loop_filter_alpha_c0_offset, cfg.loop_filter_beta_offset);
  }
  // allocates the picture store, its co-located records and the source pictures for configuration c, zero-filled, and
  // replaces the current ones only when every allocation succeeded
  int alloc_store(const RefConfig& c) {
    const size_t K = c.slots(), KS = c.src_slots();
    DeviceBuf<uint8_t> np, ncur;
    DeviceBuf<RefMbInfo> nrinfo;
    CK(np.alloc(K * S * pic_bytes + 256));
    CK(cudaMemset(np.get(), 0, K * S * pic_bytes + 256));
    CK(nrinfo.alloc(K * S * n_mb * sizeof(RefMbInfo)));
    CK(cudaMemset(nrinfo.get(), 0, K * S * n_mb * sizeof(RefMbInfo)));
    CK(ncur.alloc(KS * S * cur_bytes + 256));
    CK(cudaMemset(ncur.get(), 0, KS * S * cur_bytes + 256));
    d_pic_all = std::move(np); d_rinfo = std::move(nrinfo); d_cur = std::move(ncur);
    // TMA descriptor of the store: (x, y) from the padded origin of the luma plane, z = slot * S + stream
    have_tmap = b2h264_make_tmap_planes(tmap_pic, d_pic_all.get(), (uint64_t)lay.stride_y, (uint64_t)lay.rows_y, K * S,
                                        (uint64_t)lay.stride_y, (uint64_t)pic_bytes, 64, 48) == 0;
    return 0;
  }
};

extern "C" {

static int enc_create(const b2h264_enc_config* cfg, b2h264_enc** out) {
  if (cfg->width < 16 || cfg->height < 16 || (cfg->width & 3) || (cfg->height & 1) || cfg->qp < 0 || cfg->qp > 51 ||
      cfg->n_streams < 1)
    return -2;
  int rc = b2h264_init(cfg->device);
  if (rc) return rc;
  if ((rc = enc_upload_deblock_tables())) return rc;
  std::unique_ptr<b2h264_enc> e(new b2h264_enc());
  e->cfg = *cfg;
  e->S = cfg->n_streams;
  e->ctl.resize(e->S);
  for (int s = 0; s < e->S; s++)
    if (!e->init_stream(s)) return -1;
  e->idr_next.assign(e->S, 1);
  e->p_since_idr.assign(e->S, 0);
  e->refs.assign(e->S, StreamRefs());
  const int mbw = e->ctl[0].sp.mb_w, mbh = e->ctl[0].sp.mb_h;
  e->n_mb = mbw * mbh;
  e->frame_bytes = (size_t)cfg->width * cfg->height * 3 / 2;
  e->cur_bytes = (size_t)e->n_mb * 384;
  e->lay = PicLayout(mbw, mbh);
  e->pic_bytes = (e->lay.bytes() + 255) & ~(size_t)255;
  const size_t S = e->S;
  CK(e->own_st.create(cudaStreamNonBlocking));
  e->st = e->own_st.get();
  CK(e->st_in.create(cudaStreamNonBlocking));
  {
    int lo = 0, hi = 0;                       // record hand-over runs behind the kernels of the pictures
    cudaDeviceGetStreamPriorityRange(&lo, &hi);
    CK(e->st_out.create(cudaStreamNonBlocking, lo));
  }
  if ((rc = e->alloc_store(e->refcfg))) return rc;
  CK(e->d_vaa.alloc(S * e->n_mb * 4 * sizeof(int32_t)));
  CK(cudaMemset(e->d_vaa.get(), 0, S * e->n_mb * 4 * sizeof(int32_t)));
  for (int i = 0; i < 2; i++) {
    CK(e->d_out[i].alloc(S * e->n_mb * sizeof(MbOut)));
    CK(e->d_sf[i].alloc(S * sizeof(StreamFrame)));
    CK(e->d_srcptr[i].alloc(S * sizeof(uint8_t*)));
    CK(e->h_out[i].alloc(S * e->n_mb * sizeof(MbOut), cudaHostAllocMapped));
    CK(e->h_idx[i].alloc(S * e->n_mb * sizeof(int32_t), cudaHostAllocMapped));
    CK(e->h_cnt[i].alloc(S * sizeof(int32_t), cudaHostAllocMapped));
    CK(e->h_sf[i].alloc(S * sizeof(StreamFrame)));
    CK(e->h_srcptr[i].alloc(S * sizeof(uint8_t*)));
    b2h264_enc::Slot& sl = e->slot[i];
    CK(sl.ev0.create()); CK(sl.ev1.create()); CK(sl.ev2.create());
    CK(sl.done.create(cudaEventDisableTiming));
    CK(sl.in_done.create(cudaEventDisableTiming));
  }
  CK(e->d_src.alloc(2 * S * e->frame_bytes + 256));
  CK(e->h_src.alloc(2 * S * e->frame_bytes));
  CK(e->d_mbi.alloc(S * e->n_mb * sizeof(MbInfo)));
  CK(cudaMemset(e->d_mbi.get(), 0, S * e->n_mb * sizeof(MbInfo)));
  CK(e->d_sad.alloc(S * e->n_mb * sizeof(int32_t)));
  CK(cudaMemset(e->d_sad.get(), 0, S * e->n_mb * sizeof(int32_t)));
  CK(e->d_bits.alloc(S * e->n_mb * sizeof(int32_t)));
  CK(e->d_tickets.alloc(enc_sched_ints((int)S, mbw, mbh) * sizeof(int)));
  CK(e->d_stash.alloc(enc_stash_bytes((int)S, mbh)));
  e->bs.resize(S);
  int nt = cfg->entropy_threads;
  if (nt <= 0) { nt = usable_cores(); if (nt > (int)S) nt = (int)S; if (nt < 1) nt = 1; }
  e->pool.reset(new Pool(nt));
  *out = e.release();
  return 0;
}

int b2h264_enc_create(const b2h264_enc_config* cfg, b2h264_enc** out) {
  if (!cfg || !out) return -1;
  const int rc = enc_create(cfg, out);
  if (rc > 0) (void)cudaGetLastError();    // the failure is returned here: later launch checks must not see it
  return rc;
}

void b2h264_enc_destroy(b2h264_enc* e) {
  if (!e) return;
  cudaSetDevice(e->cfg.device);
  cudaStreamSynchronize(e->st); cudaStreamSynchronize(e->st_in.get()); cudaStreamSynchronize(e->st_out.get());
  delete e;
}

int b2h264_enc_force_idr(b2h264_enc* e, int stream) {
  if (!e || stream >= e->S) return -1;
  for (int s = 0; s < e->S; s++) if (stream < 0 || stream == s) e->idr_next[s] = 1;
  return 0;
}

int b2h264_enc_set_references(b2h264_enc* e, int num_ref_frames, int ltr_enable, int ltr_mark_period) {
  if (!e) return -1;
  RefConfig c;
  if (ltr_mark_period < 0 || !RefConfig::resolve(num_ref_frames, ltr_enable != 0, ltr_mark_period, e->cfg.intra_period, &c)) return -2;
  if (e->started) return -3;
  CK(cudaSetDevice(e->cfg.device));
  CK(cudaStreamSynchronize(e->st));
  if (c.slots() != e->refcfg.slots() || c.src_slots() != e->refcfg.src_slots()) {
    const int rc = e->alloc_store(c);
    if (rc) return rc;                          // the encoder keeps its previous store and configuration
  }
  e->refcfg = c;
  for (int s = 0; s < e->S; s++) {
    e->ctl[s].set_num_ref_frames(c.sps_num_ref_frames, e->cfg.target_bitrate);
    e->refs[s].cfg = c;
    e->refs[s].reset();
  }
  return 0;
}

int b2h264_enc_get_references(b2h264_enc* e, int32_t* out4) {
  if (!e || !out4) return -1;
  out4[0] = e->refcfg.num_ref_frames; out4[1] = e->refcfg.sps_num_ref_frames; out4[2] = e->refcfg.ltr_ref_num; out4[3] = e->refcfg.slots();
  return 0;
}

int b2h264_enc_set_slices(b2h264_enc* e, int mode, int num, const uint32_t* mb_num) {
  if (!e) return -1;
  SliceConfig c;
  const char* why = nullptr;
  if (num < 0 || !SliceConfig::resolve(mode, num, mb_num, e->ctl[0].sp.mb_w, e->ctl[0].sp.mb_h, &c, &why)) return -2;
  if (e->started) return -3;
  CK(cudaSetDevice(e->cfg.device));
  std::vector<int32_t> first(c.slices() + 1);
  c.starts(e->n_mb, first.data());
  if (c.slices() > 1) {
    // every macroblock carries its slice's first address: availability is one load and two compares (enc_frame.cuh: mb_ctx)
    std::vector<int32_t> per_mb(e->n_mb);
    for (int k = 0; k < c.slices(); k++)
      for (int i = first[k]; i < first[k + 1]; i++) per_mb[i] = first[k];
    DeviceBuf<int32_t> d;
    CK(d.alloc(e->n_mb * sizeof(int32_t)));
    CK(cudaMemcpy(d.get(), per_mb.data(), e->n_mb * sizeof(int32_t), cudaMemcpyHostToDevice));
    e->d_slice_first = std::move(d);
    first.pop_back();
    e->slice_first.swap(first);
  } else {
    e->slice_first.clear();
  }
  e->slices = c;
  for (int s = 0; s < e->S; s++) e->init_stream(s);   // cannot fail: create accepted the loop-filter values
  return 0;
}

int b2h264_enc_get_slices(b2h264_enc* e, int32_t* mode, int32_t* num, uint32_t* mb_num) {
  if (!e) return -1;
  if (mode) *mode = e->slices.mode;
  if (num) *num = e->slices.num;
  if (mb_num) memcpy(mb_num, e->slices.mb_num, sizeof(e->slices.mb_num));
  return 0;
}

int b2h264_enc_ltr_recovery_request(b2h264_enc* e, int stream, int feedback_type, int idr_pic_id, int cur_frame_num,
                                    int last_correct_frame_num) {
  if (!e || stream < 0 || stream >= e->S) return -1;
  e->refs[stream].recovery_request(feedback_type, idr_pic_id, cur_frame_num, last_correct_frame_num);
  return 0;
}

int b2h264_enc_ltr_marking_feedback(b2h264_enc* e, int stream, int feedback_type, int idr_pic_id, int ltr_frame_num) {
  if (!e || stream < 0 || stream >= e->S) return -1;
  e->refs[stream].marking_feedback(feedback_type, idr_pic_id, ltr_frame_num);
  return 0;
}

int b2h264_enc_ltr_mark_period(b2h264_enc* e, int stream, int period) {
  if (!e || stream < 0 || stream >= e->S || period < 0) return -1;
  e->refs[stream].set_mark_period(period);
  return 0;
}

int b2h264_enc_submit(b2h264_enc* e, const uint8_t* const* src, int src_on_device) {
  if (!e || !src) return -1;
  CK(cudaSetDevice(e->cfg.device));
  const int k = e->submit_idx & 1;
  b2h264_enc::Slot& sl = e->slot[k];
  if (sl.busy) return -3;                       // two batches already in flight
  const int S = e->S, mbw = e->ctl[0].sp.mb_w, mbh = e->ctl[0].sp.mb_h;
  // streams with a NULL source sit this batch out (their state does not change); the kernels see the others as a
  // compact list of n streams, each carrying its slot index (EncFrameParams::stream) for the reference tensor map
  sl.act.clear();
  for (int s = 0; s < S; s++) if (src[s]) sl.act.push_back(s);
  if (sl.act.empty()) return -5;
  // reference decisions first: a stream whose picture cannot be coded (no reference picture left after a recovery request)
  // leaves the batch, and its next picture is an IDR
  sl.idr.assign(S, 0);
  sl.rd.resize(S);
  sl.dropped.clear();
  {
    std::vector<int> coded;
    for (int s : sl.act) {
      // uiIntraPeriod: bIdrPeriodFlag = 1 + iFrameIndex >= uiIntraPeriod (wels_preprocess.cpp:369-371); iFrameIndex counts the P
      // pictures since the last IDR (encoder.cpp:284,301)
      const bool want = e->idr_next[s] != 0 || e->refs[s].idr_wanted() ||
                        (e->cfg.intra_period > 0 && 1 + e->p_since_idr[s] >= e->cfg.intra_period);
      const RefDecision& d = sl.rd[s] = e->refs[s].code_picture(want);
      if (d.not_coded) { sl.dropped.push_back(s); e->idr_next[s] = 1; e->p_since_idr[s] = 0; continue; }
      e->p_since_idr[s] = d.idr ? 0 : e->p_since_idr[s] + 1;
      sl.idr[s] = d.idr;
      e->idr_next[s] = 0;
      coded.push_back(s);
    }
    sl.act.swap(coded);
  }
  const int n = (int)sl.act.size();
  // stage sources: page-locked caller memory is DMA'd from where it lies (the caller keeps it untouched until the
  // matching collect: include/b2h264_codec.h), pageable memory goes through the encoder's pinned ring
  for (int i = 0; i < n; i++) {
    const int s = sl.act[i];
    if (src_on_device) { e->h_srcptr[k].get()[i] = src[s]; continue; }
    uint8_t* dd = e->d_src.get() + ((size_t)k * S + s) * e->frame_bytes;
    e->h_srcptr[k].get()[i] = dd;
    cudaPointerAttributes at;
    const bool pinned = cudaPointerGetAttributes(&at, src[s]) == cudaSuccess && at.type == cudaMemoryTypeHost;
    const uint8_t* from = src[s];
    if (!pinned) {
      (void)cudaGetLastError();
      uint8_t* hs = e->h_src.get() + ((size_t)k * S + s) * e->frame_bytes;
      memcpy(hs, src[s], e->frame_bytes);
      from = hs;
    }
    CK(cudaMemcpyAsync(dd, from, e->frame_bytes, cudaMemcpyHostToDevice, e->st_in.get()));
  }
  // per-stream frame descriptors; every stream has its OWN picture slots (a stream that sat a batch out keeps its references
  // where they are)
  for (int i = 0; i < n; i++) {
    const int s = sl.act[i];
    const RefDecision& d = sl.rd[s];
    const bool idr = d.idr;
    StreamFrame& F = e->h_sf[k].get()[i];
    F.p = e->ctl[s].frame_params(idr, d.ref_is_p);
    uint8_t* cur = e->d_cur.get() + ((size_t)d.cur_src * S + s) * e->cur_bytes;
    F.f.prev_luma = e->cfg.complexity_low ? e->d_cur.get() + ((size_t)d.vaa_src * S + s) * e->cur_bytes : nullptr;
    F.f.vaa_sad8x8 = e->cfg.complexity_low ? e->d_vaa.get() + (size_t)s * e->n_mb * 4 : nullptr;
    F.f.cur[0] = cur; F.f.cur[1] = cur + (size_t)e->n_mb * 256; F.f.cur[2] = cur + (size_t)e->n_mb * 320;
    const int rec = d.rec_slot, ref = idr ? (rec == 0 ? 1 : 0) : d.ref_slot;   // an IDR reads no reference: any other slot
    F.p.ref_plane = ref * S + s;
    for (int pl = 0; pl < 3; pl++) { F.f.rec[pl] = e->pic_plane0(rec, s, pl); F.f.ref[pl] = e->pic_plane0(ref, s, pl); }
    F.f.mbi = e->d_mbi.get() + (size_t)s * e->n_mb;
    F.f.rec_info = e->d_rinfo.get() + ((size_t)rec * S + s) * e->n_mb;
    F.f.ref_info = e->d_rinfo.get() + ((size_t)ref * S + s) * e->n_mb;
    F.f.out = e->d_out[k].get() + (size_t)i * e->n_mb;
    F.f.sad_cost = e->d_sad.get() + (size_t)s * e->n_mb;
    F.f.mb_bits = e->mb_bits_on ? e->d_bits.get() + (size_t)s * e->n_mb : nullptr;
    F.f.slice_first = e->slice_first.empty() ? nullptr : e->d_slice_first.get();
  }
  e->started = true;
  if (!src_on_device) {                        // the kernels of this picture wait for its uploads only
    CK(cudaEventRecord(sl.in_done.get(), e->st_in.get()));
    CK(cudaStreamWaitEvent(e->st, sl.in_done.get(), 0));
  }
  if (n == 0) {                                // every picture of the call was dropped: nothing to launch
    CK(cudaEventRecord(sl.ev0.get(), e->st)); CK(cudaEventRecord(sl.ev1.get(), e->st)); CK(cudaEventRecord(sl.ev2.get(), e->st));
    CK(cudaStreamWaitEvent(e->st_out.get(), sl.ev1.get(), 0));
    CK(cudaEventRecord(sl.done.get(), e->st_out.get()));
    sl.busy = true;
    e->submit_idx++;
    return 0;
  }
  CK(cudaMemcpyAsync(e->d_sf[k].get(), e->h_sf[k].get(), n * sizeof(StreamFrame), cudaMemcpyHostToDevice, e->st));
  CK(cudaMemcpyAsync(e->d_srcptr[k].get(), e->h_srcptr[k].get(), n * sizeof(uint8_t*), cudaMemcpyHostToDevice, e->st));
  CK(cudaEventRecord(sl.ev0.get(), e->st));
  int rc = enc_launch_frame(e->d_sf[k].get(), e->d_srcptr[k].get(), n, e->cfg.width, e->cfg.height, mbw, mbh, e->d_tickets.get(), e->d_stash.get(),
                            e->have_tmap ? e->tmap_pic : nullptr, e->cfg.complexity_low != 0, e->st);
  if (rc) return rc;
  CK(cudaEventRecord(sl.ev1.get(), e->st));
  rc = enc_launch_deblock_expand(e->d_sf[k].get(), n, mbw, mbh, e->st);
  if (rc) return rc;
  CK(cudaEventRecord(sl.ev2.get(), e->st));
  // the macroblock records are final once the encode kernel is done (deblocking does not touch them)
  CK(cudaStreamWaitEvent(e->st_out.get(), sl.ev1.get(), 0));
  rc = enc_launch_pack(e->d_sf[k].get(), n, e->n_mb, e->h_out[k].get(), e->h_idx[k].get(), e->h_cnt[k].get(), e->st_out.get());
  if (rc) return rc;
  CK(cudaEventRecord(sl.done.get(), e->st_out.get()));
  sl.busy = true;
  e->submit_idx++;
  return 0;
}

int b2h264_enc_collect(b2h264_enc* e, const uint8_t** bs, int32_t* bs_bytes, int32_t* frame_type) {
  if (!e) return -1;
  CK(cudaSetDevice(e->cfg.device));
  const int k = e->collect_idx & 1;
  b2h264_enc::Slot& sl = e->slot[k];
  if (!sl.busy) return -4;
  CK(cudaEventSynchronize(sl.done.get()));
  float ms = 0;
  cudaEventElapsedTime(&ms, sl.ev0.get(), sl.ev1.get());
  e->last_us[0] = ms * 1000.f;               // source padding + macroblock wavefront kernel
  // deblocking of this picture may still be running (the records were downloaded as soon as the encode kernel
  // finished): report it when it is done, otherwise keep the previous picture's figure
  if (cudaEventQuery(sl.ev2.get()) == cudaSuccess && cudaEventElapsedTime(&ms, sl.ev1.get(), sl.ev2.get()) == cudaSuccess)
    e->last_us[1] = ms * 1000.f;             // deblocking wavefront + border expansion
  (void)cudaGetLastError();
  const auto t0 = std::chrono::steady_clock::now();
  const int n_mb = e->n_mb, n = (int)sl.act.size();
  e->last_d2h = (unsigned long long)n * (n_mb + 1) * sizeof(int32_t);
  for (int i = 0; i < n; i++) e->last_d2h += (unsigned long long)e->h_cnt[k].get()[i] * 32;
  for (int s = 0; s < e->S; s++) e->bs[s].clear();
  std::function<void(int)> job = [&](int i) {
    const int s = sl.act[i];
    e->ctl[s].write_access_unit_packed(sl.idr[s] != 0, e->h_out[k].get() + (size_t)i * n_mb, e->h_idx[k].get() + (size_t)i * n_mb, &e->bs[s], &sl.rd[s]);
  };
  e->pool->run(n, job);
  e->last_us[2] = std::chrono::duration<float, std::micro>(std::chrono::steady_clock::now() - t0).count();
  std::vector<int8_t> active(e->S, 0);
  for (int i = 0; i < n; i++) active[sl.act[i]] = 1;
  for (int s : sl.dropped) active[s] = -1;
  for (int s = 0; s < e->S; s++) {
    if (bs) bs[s] = active[s] == 1 ? e->bs[s].data() : nullptr;
    if (bs_bytes) bs_bytes[s] = (int32_t)e->bs[s].size();
    if (frame_type) frame_type[s] = active[s] == 0 ? 0 : active[s] < 0 ? -1 : sl.idr[s] ? 1 : 2;
  }
  sl.busy = false;
  e->collect_idx++;
  return 0;
}

int b2h264_enc_reset_stream(b2h264_enc* e, int stream) {
  if (!e || stream < 0 || stream >= e->S) return -1;
  if (e->slot[0].busy || e->slot[1].busy) return -3;
  CK(cudaSetDevice(e->cfg.device));
  e->init_stream(stream);                    // cannot fail: create accepted the same configuration
  e->idr_next[stream] = 1;
  e->p_since_idr[stream] = 0;
  e->refs[stream].cfg = e->refcfg;           // the marking period a previous owner set does not carry over
  e->refs[stream].reset();
  // what a fresh encoder starts from: no SAD history, no reference-picture records
  CK(cudaMemsetAsync(e->d_sad.get() + (size_t)stream * e->n_mb, 0, e->n_mb * sizeof(int32_t), e->st));
  for (int i = 0; i < e->refcfg.slots(); i++)
    CK(cudaMemsetAsync(e->d_rinfo.get() + ((size_t)i * e->S + stream) * e->n_mb, 0, e->n_mb * sizeof(RefMbInfo), e->st));
  CK(cudaMemsetAsync(e->d_mbi.get() + (size_t)stream * e->n_mb, 0, e->n_mb * sizeof(MbInfo), e->st));
  CK(cudaStreamSynchronize(e->st));
  return 0;
}

int b2h264_enc_set_mb_bits(b2h264_enc* e, int on) {
  if (!e) return -1;
  if (e->slot[0].busy || e->slot[1].busy) return -3;
  e->mb_bits_on = on != 0;
  for (auto& c : e->ctl) c.record_mb_bits = on != 0;
  return 0;
}

int b2h264_enc_get_mb_bits(b2h264_enc* e, int stream, int32_t* device_bits, int32_t* host_bits) {
  if (!e || stream < 0 || stream >= e->S || !e->mb_bits_on) return -1;
  if (e->slot[0].busy || e->slot[1].busy) return -3;
  CK(cudaSetDevice(e->cfg.device));
  CK(cudaStreamSynchronize(e->st));
  if (device_bits) CK(cudaMemcpy(device_bits, e->d_bits.get() + (size_t)stream * e->n_mb, e->n_mb * sizeof(int32_t), cudaMemcpyDeviceToHost));
  if (host_bits) {
    if ((int)e->ctl[stream].last_mb_bits.size() != e->n_mb) return -1;
    memcpy(host_bits, e->ctl[stream].last_mb_bits.data(), e->n_mb * sizeof(int32_t));
  }
  return 0;
}

// macroblocks of the last collected batch that were coded (not P_SKIP), summed over its streams
int b2h264_enc_last_coded_mbs(b2h264_enc* e, unsigned long long* count) {
  if (!e || !count) return -1;
  unsigned long long n = 0;
  for (const auto& c : e->ctl) n += (unsigned long long)c.last_coded_mbs;
  *count = n;
  return 0;
}
int b2h264_enc_last_d2h_bytes(b2h264_enc* e, unsigned long long* bytes) {
  if (!e || !bytes) return -1;
  *bytes = e->last_d2h;
  return 0;
}

int b2h264_enc_get_recon(b2h264_enc* e, int stream, uint8_t* dst) {
  if (!e || stream < 0 || stream >= e->S || !dst) return -1;
  CK(cudaSetDevice(e->cfg.device));
  CK(cudaStreamSynchronize(e->st));
  const int set = e->refs[stream].last_rec_slot();
  const int w = e->cfg.width, h = e->cfg.height;
  for (int pl = 0; pl < 3; pl++) {
    const int pw = pl ? w / 2 : w, ph = pl ? h / 2 : h;
    CK(cudaMemcpy2D(dst, pw, e->pic_plane0(set, stream, pl), e->lay.stride(pl), pw, ph, cudaMemcpyDeviceToHost));
    dst += (size_t)pw * ph;
  }
  return 0;
}

int b2h264_enc_last_timing(b2h264_enc* e, float* us3) {
  if (!e || !us3) return -1;
  us3[0] = e->last_us[0]; us3[1] = e->last_us[1]; us3[2] = e->last_us[2];
  return 0;
}

int b2h264_enc_set_stream(b2h264_enc* e, void* stream) {
  if (!e) return -1;
  if (e->slot[0].busy || e->slot[1].busy) return -3;
  CK(cudaSetDevice(e->cfg.device));
  CK(cudaStreamSynchronize(e->st));
  e->own_st = Stream();
  e->st = (cudaStream_t)stream;
  return 0;
}

}  // extern "C"
