// enc_batch.cu — layer-2 batched frame encoder (include/b2h264_codec.h): device buffers, the asynchronous
// H2D -> kernels -> D2H pipeline on one CUDA stream, and host entropy coding on a small thread pool.
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <string.h>
#include <thread>
#include <vector>

#include "../../include/b2h264_codec.h"
#include "b2h264_internal.h"
#include "enc_host.h"
#include "enc_launch.h"
#include "host_pool.h"

using b2h264::StreamCtl;
using b2h264::StreamRefs;
using b2h264::RefConfig;
using b2h264::RefDecision;
using b2h264::Pool;
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
  bool started = false;                   // a picture has been submitted: the picture store is fixed
  cudaStream_t st = nullptr;        // kernels (may be the caller's stream, b2h264_enc_set_stream)
  cudaStream_t st_in = nullptr;     // source uploads: overlap the previous picture's kernels
  cudaStream_t st_out = nullptr;    // record downloads: overlap deblocking and the next picture's kernels
  // device memory
  uint8_t* d_cur = nullptr;               // refcfg.src_slots() x S x (Y,U,V) MB-aligned source pictures (current, previous and
                                          // long-term sources: VAA statistics), set * S + stream
  int32_t* d_vaa = nullptr;               // S x n_mb x 4: 8x8 SADs against the previous source picture (LOW_COMPLEXITY)
  uint8_t* d_pic_all = nullptr;           // picture store: refcfg.slots() x S x padded (Y,U,V), slot * S + stream
  uint8_t* d_src = nullptr;               // S x raw I420 staging (2 slots)
  MbInfo* d_mbi = nullptr;
  RefMbInfo* d_rinfo = nullptr;           // co-located records of every stored picture: (slot * S + stream) x n_mb
  MbOut* d_out[2] = {nullptr, nullptr};
  int32_t* d_sad = nullptr;
  int32_t* d_bits = nullptr;              // S x n_mb: exact CAVLC bits per macroblock (when enabled)
  bool mb_bits_on = false;
  int* d_tickets = nullptr;
  void* d_stash = nullptr;          // parked macroblock scratches of the staged scheduler
  StreamFrame* d_sf[2] = {nullptr, nullptr};
  alignas(64) unsigned char tmap_pic[128];      // CUtensorMap of the luma planes of every slot of all streams
  bool have_tmap = false;
  const uint8_t** d_srcptr[2] = {nullptr, nullptr};
  // pinned host memory
  uint8_t* h_src = nullptr;               // 2 slots x S x frame
  MbOut* h_out[2] = {nullptr, nullptr};      // mapped pinned: coded records, packed per stream (worst case sized)
  int32_t* h_idx[2] = {nullptr, nullptr};    // mapped pinned: per MB offset of its compact record (32-byte units) or -1
  int32_t* h_cnt[2] = {nullptr, nullptr};    // mapped pinned: 32-byte units written per stream
  unsigned long long last_d2h = 0;
  StreamFrame* h_sf[2] = {nullptr, nullptr};
  const uint8_t** h_srcptr[2] = {nullptr, nullptr};
  // in-flight bookkeeping
  struct Slot { bool busy = false; std::vector<uint8_t> idr; std::vector<int> act;   // act: streams of this batch (compact order)
                std::vector<RefDecision> rd;                                       // per stream: reference decisions of its picture
                std::vector<int> dropped;                                          // streams whose picture was not coded (RefDecision::not_coded)
                cudaEvent_t ev0, ev1, ev2, done, in_done, enc_done; };
  Slot slot[2];
  int submit_idx = 0, collect_idx = 0;
  std::vector<std::vector<uint8_t>> bs;   // per stream output of the last collect
  Pool* pool = nullptr;
  float last_us[4] = {0, 0, 0, 0};
  bool own_stream = true;
  size_t frame_bytes = 0, cur_bytes = 0, pic_bytes = 0, pic_y_bytes = 0, pic_c_bytes = 0;

  uint8_t* pic_plane0(int slot, int s, int pl) const {   // pixel (0,0) of plane pl of stream s's picture in `slot`
    const int sty = ctl[0].rec_stride_y(), stc = ctl[0].rec_stride_c();
    uint8_t* base = d_pic_all + ((size_t)slot * S + s) * pic_bytes;
    if (pl == 0) return base + (size_t)32 * sty + 32;
    return base + pic_y_bytes + (size_t)(pl - 1) * pic_c_bytes + (size_t)16 * stc + 16;
  }
  // allocates the picture store, its co-located records and the source pictures for configuration c, zero-filled, and
  // replaces the current ones only when every allocation succeeded
  int alloc_store(const RefConfig& c) {
    const size_t K = c.slots(), KS = c.src_slots();
    uint8_t* pic = nullptr; RefMbInfo* rinfo = nullptr; uint8_t* cur = nullptr;
    cudaError_t err = cudaMalloc(&pic, K * S * pic_bytes + 256);
    if (err == cudaSuccess) err = cudaMemset(pic, 0, K * S * pic_bytes + 256);
    if (err == cudaSuccess) err = cudaMalloc(&rinfo, K * S * n_mb * sizeof(RefMbInfo));
    if (err == cudaSuccess) err = cudaMemset(rinfo, 0, K * S * n_mb * sizeof(RefMbInfo));
    if (err == cudaSuccess) err = cudaMalloc(&cur, KS * S * cur_bytes + 256);
    if (err == cudaSuccess) err = cudaMemset(cur, 0, KS * S * cur_bytes + 256);
    if (err != cudaSuccess) { cudaFree(pic); cudaFree(rinfo); cudaFree(cur); return (int)err; }
    cudaFree(d_pic_all); cudaFree(d_rinfo); cudaFree(d_cur);
    d_pic_all = pic; d_rinfo = rinfo; d_cur = cur;
    // TMA descriptor of the store: (x, y) from the padded origin of the luma plane, z = slot * S + stream
    const StreamCtl& c0 = ctl[0];
    have_tmap = b2h264_make_tmap_planes(tmap_pic, d_pic_all, (uint64_t)c0.rec_stride_y(), (uint64_t)c0.rec_rows_y(), K * S,
                                        (uint64_t)c0.rec_stride_y(), (uint64_t)pic_bytes, 64, 48) == 0;
    return 0;
  }
};

extern "C" {

int b2h264_enc_create(const b2h264_enc_config* cfg, b2h264_enc** out) {
  if (!cfg || !out) return -1;
  if (cfg->width < 16 || cfg->height < 16 || (cfg->width & 3) || (cfg->height & 1) || cfg->qp < 0 || cfg->qp > 51 ||
      cfg->n_streams < 1)
    return -2;
  int rc = b2h264_init(cfg->device);
  if (rc) return rc;
  if ((rc = enc_upload_deblock_tables())) return rc;
  b2h264_enc* e = new b2h264_enc();
  e->cfg = *cfg;
  e->S = cfg->n_streams;
  e->ctl.resize(e->S);
  for (auto& c : e->ctl) {
    c.init(cfg->width, cfg->height, cfg->qp, cfg->fps, cfg->target_bitrate, cfg->entropy_cabac, cfg->profile_idc);
    c.fast_mode = cfg->complexity_low != 0;
    if (!c.set_loop_filter(cfg->loop_filter_idc, cfg->loop_filter_alpha_c0_offset, cfg->loop_filter_beta_offset)) { delete e; return -1; }
    c.increasing_ids = cfg->sps_pps_id_strategy != 0;
  }
  e->idr_next.assign(e->S, 1);
  e->p_since_idr.assign(e->S, 0);
  e->refs.assign(e->S, StreamRefs());
  const StreamCtl& c0 = e->ctl[0];
  const int mbw = c0.sp.mb_w, mbh = c0.sp.mb_h;
  e->n_mb = mbw * mbh;
  e->frame_bytes = (size_t)cfg->width * cfg->height * 3 / 2;
  e->cur_bytes = (size_t)e->n_mb * 384;
  e->pic_y_bytes = (size_t)c0.rec_stride_y() * c0.rec_rows_y();
  e->pic_c_bytes = (size_t)c0.rec_stride_c() * c0.rec_rows_c();
  e->pic_bytes = (e->pic_y_bytes + 2 * e->pic_c_bytes + 255) & ~(size_t)255;
  const size_t S = e->S;
  CK(cudaStreamCreateWithFlags(&e->st, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&e->st_in, cudaStreamNonBlocking));
  {
    int lo = 0, hi = 0;                       // record hand-over runs behind the kernels of the pictures
    cudaDeviceGetStreamPriorityRange(&lo, &hi);
    CK(cudaStreamCreateWithPriority(&e->st_out, cudaStreamNonBlocking, lo));
  }
  if ((rc = e->alloc_store(e->refcfg))) return rc;
  CK(cudaMalloc(&e->d_vaa, S * e->n_mb * 4 * sizeof(int32_t)));
  CK(cudaMemset(e->d_vaa, 0, S * e->n_mb * 4 * sizeof(int32_t)));
  for (int i = 0; i < 2; i++) {
    CK(cudaMalloc(&e->d_out[i], S * e->n_mb * sizeof(MbOut)));
    CK(cudaMalloc(&e->d_sf[i], S * sizeof(StreamFrame)));
    CK(cudaMalloc(&e->d_srcptr[i], S * sizeof(uint8_t*)));
    CK(cudaHostAlloc(&e->h_out[i], S * e->n_mb * sizeof(MbOut), cudaHostAllocMapped));
    CK(cudaHostAlloc(&e->h_idx[i], S * e->n_mb * sizeof(int32_t), cudaHostAllocMapped));
    CK(cudaHostAlloc(&e->h_cnt[i], S * sizeof(int32_t), cudaHostAllocMapped));
    CK(cudaMallocHost(&e->h_sf[i], S * sizeof(StreamFrame)));
    CK(cudaMallocHost(&e->h_srcptr[i], S * sizeof(uint8_t*)));
    CK(cudaEventCreate(&e->slot[i].ev0));
    CK(cudaEventCreate(&e->slot[i].ev1));
    CK(cudaEventCreate(&e->slot[i].ev2));
    CK(cudaEventCreateWithFlags(&e->slot[i].done, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&e->slot[i].in_done, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&e->slot[i].enc_done, cudaEventDisableTiming));
  }
  CK(cudaMalloc(&e->d_src, 2 * S * e->frame_bytes + 256));
  CK(cudaMallocHost(&e->h_src, 2 * S * e->frame_bytes));
  CK(cudaMalloc(&e->d_mbi, S * e->n_mb * sizeof(MbInfo)));
  CK(cudaMemset(e->d_mbi, 0, S * e->n_mb * sizeof(MbInfo)));
  CK(cudaMalloc(&e->d_sad, S * e->n_mb * sizeof(int32_t)));
  CK(cudaMemset(e->d_sad, 0, S * e->n_mb * sizeof(int32_t)));
  CK(cudaMalloc(&e->d_bits, S * e->n_mb * sizeof(int32_t)));
  CK(cudaMalloc(&e->d_tickets, enc_sched_ints((int)S, mbw, mbh) * sizeof(int)));
  CK(cudaMalloc(&e->d_stash, enc_stash_bytes((int)S, mbh)));
  e->bs.resize(S);
  int nt = cfg->entropy_threads;
  if (nt <= 0) { nt = usable_cores(); if (nt > (int)S) nt = (int)S; if (nt < 1) nt = 1; }
  e->pool = new Pool(nt);
  *out = e;
  return 0;
}

void b2h264_enc_destroy(b2h264_enc* e) {
  if (!e) return;
  cudaSetDevice(e->cfg.device);
  cudaStreamSynchronize(e->st);
  delete e->pool;
  cudaFree(e->d_pic_all); cudaFree(e->d_rinfo); cudaFree(e->d_cur); cudaFree(e->d_vaa); cudaFree(e->d_src); cudaFree(e->d_mbi); cudaFree(e->d_sad); cudaFree(e->d_bits); cudaFree(e->d_tickets); cudaFree(e->d_stash);
  cudaFreeHost(e->h_src);
  for (int i = 0; i < 2; i++) {
    cudaFree(e->d_out[i]); cudaFree(e->d_sf[i]); cudaFree(e->d_srcptr[i]);
    cudaFreeHost(e->h_out[i]); cudaFreeHost(e->h_idx[i]); cudaFreeHost(e->h_cnt[i]); cudaFreeHost(e->h_sf[i]); cudaFreeHost(e->h_srcptr[i]);
    cudaEventDestroy(e->slot[i].ev0); cudaEventDestroy(e->slot[i].ev1); cudaEventDestroy(e->slot[i].ev2); cudaEventDestroy(e->slot[i].done); cudaEventDestroy(e->slot[i].in_done); cudaEventDestroy(e->slot[i].enc_done);
  }
  if (e->own_stream) cudaStreamDestroy(e->st);
  cudaStreamDestroy(e->st_in); cudaStreamDestroy(e->st_out);
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
    if (src_on_device) { e->h_srcptr[k][i] = src[s]; continue; }
    uint8_t* dd = e->d_src + ((size_t)k * S + s) * e->frame_bytes;
    e->h_srcptr[k][i] = dd;
    cudaPointerAttributes at;
    const bool pinned = cudaPointerGetAttributes(&at, src[s]) == cudaSuccess && at.type == cudaMemoryTypeHost;
    const uint8_t* from = src[s];
    if (!pinned) {
      (void)cudaGetLastError();
      uint8_t* hs = e->h_src + ((size_t)k * S + s) * e->frame_bytes;
      memcpy(hs, src[s], e->frame_bytes);
      from = hs;
    }
    CK(cudaMemcpyAsync(dd, from, e->frame_bytes, cudaMemcpyHostToDevice, e->st_in));
  }
  // per-stream frame descriptors; every stream has its OWN picture slots (a stream that sat a batch out keeps its references
  // where they are)
  for (int i = 0; i < n; i++) {
    const int s = sl.act[i];
    const RefDecision& d = sl.rd[s];
    const bool idr = d.idr;
    StreamFrame& F = e->h_sf[k][i];
    F.p = e->ctl[s].frame_params(idr, d.ref_is_p);
    uint8_t* cur = e->d_cur + ((size_t)d.cur_src * S + s) * e->cur_bytes;
    F.f.prev_luma = e->cfg.complexity_low ? e->d_cur + ((size_t)d.vaa_src * S + s) * e->cur_bytes : nullptr;
    F.f.vaa_sad8x8 = e->cfg.complexity_low ? e->d_vaa + (size_t)s * e->n_mb * 4 : nullptr;
    F.f.cur[0] = cur; F.f.cur[1] = cur + (size_t)e->n_mb * 256; F.f.cur[2] = cur + (size_t)e->n_mb * 320;
    const int rec = d.rec_slot, ref = idr ? (rec == 0 ? 1 : 0) : d.ref_slot;   // an IDR reads no reference: any other slot
    F.p.ref_plane = ref * S + s;
    for (int pl = 0; pl < 3; pl++) { F.f.rec[pl] = e->pic_plane0(rec, s, pl); F.f.ref[pl] = e->pic_plane0(ref, s, pl); }
    F.f.mbi = e->d_mbi + (size_t)s * e->n_mb;
    F.f.rec_info = e->d_rinfo + ((size_t)rec * S + s) * e->n_mb;
    F.f.ref_info = e->d_rinfo + ((size_t)ref * S + s) * e->n_mb;
    F.f.out = e->d_out[k] + (size_t)i * e->n_mb;
    F.f.sad_cost = e->d_sad + (size_t)s * e->n_mb;
    F.f.mb_bits = e->mb_bits_on ? e->d_bits + (size_t)s * e->n_mb : nullptr;
  }
  e->started = true;
  if (!src_on_device) {                        // the kernels of this picture wait for its uploads only
    CK(cudaEventRecord(sl.in_done, e->st_in));
    CK(cudaStreamWaitEvent(e->st, sl.in_done, 0));
  }
  if (n == 0) {                                // every picture of the call was dropped: nothing to launch
    CK(cudaEventRecord(sl.ev0, e->st)); CK(cudaEventRecord(sl.ev1, e->st)); CK(cudaEventRecord(sl.ev2, e->st));
    CK(cudaStreamWaitEvent(e->st_out, sl.ev1, 0));
    CK(cudaEventRecord(sl.done, e->st_out));
    sl.busy = true;
    e->submit_idx++;
    return 0;
  }
  CK(cudaMemcpyAsync(e->d_sf[k], e->h_sf[k], n * sizeof(StreamFrame), cudaMemcpyHostToDevice, e->st));
  CK(cudaMemcpyAsync(e->d_srcptr[k], e->h_srcptr[k], n * sizeof(uint8_t*), cudaMemcpyHostToDevice, e->st));
  CK(cudaEventRecord(sl.ev0, e->st));
  int rc = enc_launch_frame(e->d_sf[k], e->d_srcptr[k], n, e->cfg.width, e->cfg.height, mbw, mbh, e->d_tickets, e->d_stash,
                            e->have_tmap ? e->tmap_pic : nullptr, e->cfg.complexity_low != 0, e->st);
  if (rc) return rc;
  CK(cudaEventRecord(sl.ev1, e->st));
  rc = enc_launch_deblock_expand(e->d_sf[k], n, mbw, mbh, e->st);
  if (rc) return rc;
  CK(cudaEventRecord(sl.ev2, e->st));
  // the macroblock records are final once the encode kernel is done (deblocking does not touch them)
  CK(cudaStreamWaitEvent(e->st_out, sl.ev1, 0));
  rc = enc_launch_pack(e->d_sf[k], n, e->n_mb, e->h_out[k], e->h_idx[k], e->h_cnt[k], e->st_out);
  if (rc) return rc;
  CK(cudaEventRecord(sl.done, e->st_out));
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
  CK(cudaEventSynchronize(sl.done));
  float ms = 0;
  cudaEventElapsedTime(&ms, sl.ev0, sl.ev1);
  e->last_us[0] = ms * 1000.f;               // source padding + macroblock wavefront kernel
  // deblocking of this picture may still be running (the records were downloaded as soon as the encode kernel
  // finished): report it when it is done, otherwise keep the previous picture's figure
  if (cudaEventQuery(sl.ev2) == cudaSuccess && cudaEventElapsedTime(&ms, sl.ev1, sl.ev2) == cudaSuccess)
    e->last_us[1] = ms * 1000.f;             // deblocking wavefront + border expansion
  (void)cudaGetLastError();
  const auto t0 = std::chrono::steady_clock::now();
  const int n_mb = e->n_mb, n = (int)sl.act.size();
  e->last_d2h = (unsigned long long)n * (n_mb + 1) * sizeof(int32_t);
  for (int i = 0; i < n; i++) e->last_d2h += (unsigned long long)e->h_cnt[k][i] * 32;
  for (int s = 0; s < e->S; s++) e->bs[s].clear();
  std::function<void(int)> job = [&](int i) {
    const int s = sl.act[i];
    e->ctl[s].write_access_unit_packed(sl.idr[s] != 0, e->h_out[k] + (size_t)i * n_mb, e->h_idx[k] + (size_t)i * n_mb, &e->bs[s], &sl.rd[s]);
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
  e->ctl[stream] = StreamCtl();
  e->ctl[stream].init(e->cfg.width, e->cfg.height, e->cfg.qp, e->cfg.fps, e->cfg.target_bitrate, e->cfg.entropy_cabac, e->cfg.profile_idc);
  e->ctl[stream].increasing_ids = e->cfg.sps_pps_id_strategy != 0;
  e->ctl[stream].fast_mode = e->cfg.complexity_low != 0;
  e->ctl[stream].set_loop_filter(e->cfg.loop_filter_idc, e->cfg.loop_filter_alpha_c0_offset, e->cfg.loop_filter_beta_offset);
  e->ctl[stream].record_mb_bits = e->mb_bits_on;
  e->ctl[stream].set_num_ref_frames(e->refcfg.sps_num_ref_frames, e->cfg.target_bitrate);
  e->idr_next[stream] = 1;
  e->p_since_idr[stream] = 0;
  e->refs[stream].cfg = e->refcfg;           // the marking period a previous owner set does not carry over
  e->refs[stream].reset();
  // what a fresh encoder starts from: no SAD history, no reference-picture records
  CK(cudaMemsetAsync(e->d_sad + (size_t)stream * e->n_mb, 0, e->n_mb * sizeof(int32_t), e->st));
  for (int i = 0; i < e->refcfg.slots(); i++)
    CK(cudaMemsetAsync(e->d_rinfo + ((size_t)i * e->S + stream) * e->n_mb, 0, e->n_mb * sizeof(RefMbInfo), e->st));
  CK(cudaMemsetAsync(e->d_mbi + (size_t)stream * e->n_mb, 0, e->n_mb * sizeof(MbInfo), e->st));
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
  if (device_bits) CK(cudaMemcpy(device_bits, e->d_bits + (size_t)stream * e->n_mb, e->n_mb * sizeof(int32_t), cudaMemcpyDeviceToHost));
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
    const int st = pl ? e->ctl[0].rec_stride_c() : e->ctl[0].rec_stride_y();
    CK(cudaMemcpy2D(dst, pw, e->pic_plane0(set, stream, pl), st, pw, ph, cudaMemcpyDeviceToHost));
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
  CK(cudaStreamSynchronize(e->st));
  if (e->own_stream) cudaStreamDestroy(e->st);
  e->st = (cudaStream_t)stream;
  e->own_stream = false;
  return 0;
}

}  // extern "C"
