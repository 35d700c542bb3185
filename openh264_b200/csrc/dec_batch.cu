// dec_batch.cu — layer-2 batched decoder: S independent streams, one access unit per stream per call.
// Host: Annex-B parsing (h264_parse.cpp, like the reference parses on the host: codec/decoder/core/src/au_parser.cpp,
// parse_mb_syn_cavlc.cpp), device: reconstruction of every macroblock by one warp (dec_mb.cuh, k_decode_mbs),
// in-loop deblocking and border replication (the encoder's kernels).  Replaces, for the supported stream class,
// CWelsDecoder::DecodeFrameNoDelay -> WelsDecodeBs -> DecodeCurrentAccessUnit -> WelsTargetSliceConstruction /
// WelsTargetMbConstruction (codec/decoder/core/src/decoder_core.cpp, decode_slice.cpp:~100) and
// WelsDeblockingFilterSlice (deblocking.cpp).  Streams outside the class are rejected with the parser's error
// code; there is no CPU reconstruction path in this library.
// Host output: synchronous per call (parse -> H2D -> kernels -> D2H).  Device output (b2h264_dec_decode_device): the call
// returns once its work is enqueued, and k_dec_output crops the pictures into the caller's HBM.  Streams without a slice in
// their access unit sit the call out.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <chrono>
#include <memory>
#include <type_traits>

#include <vector>

#include "../../include/b2h264_codec.h"
#include "b2h264_internal.h"
#include "cuda_owned.h"
#include "enc_host.h"
#include "enc_launch.h"
#include "h264_parse.h"
#include "host_pool.h"

using namespace b2h264;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return (int)e_; } while (0)

struct DecOutPic {                        // b2h264_dec_decode_device: one active stream's output
  const uint8_t* src[3];                  // first sample of each plane inside the crop window of the picture's DPB slot
  uint8_t* dst;                           // the caller's I420 picture (w*h*3/2 bytes, any alignment)
};

struct b2h264_dec {
  b2h264_dec_config cfg;
  int S = 0, mb_w = 0, mb_h = 0, n_mb = 0;
  PicLayout lay;                          // of each picture slot; pic_bytes = lay.bytes() is the slot pitch
  std::vector<ParserState> parser;
  std::vector<ParsedPicture> parsed;      // per stream: the access unit of the running call
  std::vector<int> parse_rc;
  int slots = 2;                          // picture slots per stream (num_ref_frames + 1 of the most demanding stream so far)
  std::vector<int> out_cx, out_cy;        // per active stream: luma samples cropped at the left / top of the output
  std::vector<int> out_slot;              // per active stream: slot of the picture decoded in this call
  std::vector<int> act;
  std::vector<uint8_t> act_ref;           // is the picture of act[i] a reference picture
  // the CUDA resources are released in the reverse order of their declaration: the buffers and the event before the stream
  Stream own_st;                          // the decoder's stream until b2h264_dec_set_stream lends it the caller's
  cudaStream_t st = nullptr;              // own_st or the caller's stream
  Event staged;                           // after the last host-to-device copy of a call: the pinned buffers may be rewritten
  DeviceBuf<uint8_t> d_pic;               // S x slots padded pictures: picture (s, slot) at (s * slots + slot) * pic_bytes
  DeviceBuf<MbInfo> d_mbi;
  DeviceBuf<MbOut> d_recs;
  HostBuf<MbOut> h_recs;                  // pinned: COMPACT records (pack_records_compact), one worst-case slot per stream
  DeviceBuf<uint8_t> d_pack;              // device copy of the compact records (same slots)
  HostBuf<int32_t> h_idx;                 // pinned: per macroblock offset of its compact record or -1 - qp (skipped)
  DeviceBuf<int32_t> d_idx;
  std::vector<int> units;                 // 32-byte units packed per active stream
  DeviceBuf<DecMbAux> d_aux;
  HostBuf<DecMbAux> h_aux;                // pinned
  DeviceBuf<DecMbAuxB> d_aux_b;           // list 1 of B macroblocks: allocated when the first picture with B slices arrives
  HostBuf<DecMbAuxB> h_aux_b;             // pinned
  std::vector<int> last_poc, last_idr, last_reorder;   // per stream: picture order count / IDR flag / reorder depth of the last decoded picture
  DeviceBuf<StreamFrame> d_sf;
  HostBuf<StreamFrame> h_sf;              // pinned
  DeviceBuf<DecOutPic> d_out;             // device output: per active stream, the sources and the destination of its planes
  HostBuf<DecOutPic> h_out;               // pinned
  DeviceBuf<int> d_ws;
  size_t pic_bytes = 0;
  int last_error_stream = -1;
  std::unique_ptr<Pool> pool;             // the streams are parsed side by side (the parser is the decoder's host cost); declared
                                          // last: its threads stop before anything else is released

  uint8_t* plane0(int slot, int s, int pl) const { return d_pic.get() + ((size_t)s * slots + slot) * pic_bytes + lay.plane0(pl); }
};

// ---- device output: the cropped pictures of one call into the caller's HBM, every active stream and plane in one launch ----
// One warp per row of a plane.  A row is copied in the widest words (16, 8, 4 or 1 bytes) that its source and destination
// share an alignment for: the destination's head bytes go one by one, then whole words, then the tail.
template <int V>
__device__ __forceinline__ void out_row(const uint8_t* src, uint8_t* dst, int n, int lane) {
  int head = (int)((0u - (unsigned)(uintptr_t)dst) & (V - 1));
  if (head > n) head = n;
  if (lane < head) dst[lane] = src[lane];
  const int words = (n - head) / V;
  // word-aligned because source and destination agree modulo V; rounding the source down only makes that explicit
  typedef typename std::conditional<V == 16, uint4, typename std::conditional<V == 8, uint2, uint32_t>::type>::type W;
  const W* s = reinterpret_cast<const W*>((uintptr_t)(src + head) & ~(uintptr_t)(V - 1));
  W* d = reinterpret_cast<W*>(dst + head);
  for (int k = lane; k < words; k += 32) d[k] = __ldg(s + k);
  const int t = head + words * V + lane;
  if (t < n) dst[t] = src[t];
}

__global__ void __launch_bounds__(256) k_dec_output(const DecOutPic* __restrict__ pics, int w, int h, int sty, int stc) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);   // row over the three planes: h luma rows, then h / 2 of each chroma plane
  if (r >= 2 * h) return;
  const DecOutPic& P = pics[blockIdx.y];
  const int pl = r < h ? 0 : r < h + h / 2 ? 1 : 2;
  const int y = pl == 0 ? r : r - h - (pl - 1) * (h / 2);
  const int n = pl ? w / 2 : w;
  const uint8_t* src = P.src[pl] + (size_t)y * (pl ? stc : sty);
  uint8_t* dst = P.dst + (pl ? (size_t)w * h + (size_t)(pl - 1) * (w / 2) * (h / 2) : 0) + (size_t)y * n;
  const unsigned mis = (unsigned)(((uintptr_t)src ^ (uintptr_t)dst) & 15);
  if (mis == 0) out_row<16>(src, dst, n, lane);
  else if ((mis & 7) == 0) out_row<8>(src, dst, n, lane);
  else if ((mis & 3) == 0) out_row<4>(src, dst, n, lane);
  else for (int x = lane; x < n; x += 32) dst[x] = src[x];
}

extern "C" {

static int dec_create(const b2h264_dec_config* cfg, b2h264_dec** out) {
  if (cfg->width < 16 || cfg->height < 16 || (cfg->width & 1) || (cfg->height & 1) || cfg->n_streams < 1) return -2;
  int rc = b2h264_init(cfg->device);
  if (rc) return rc;
  if ((rc = enc_upload_deblock_tables())) return rc;
  std::unique_ptr<b2h264_dec> d(new b2h264_dec());
  d->cfg = *cfg;
  d->S = cfg->n_streams;
  d->mb_w = (cfg->width + 15) >> 4; d->mb_h = (cfg->height + 15) >> 4; d->n_mb = d->mb_w * d->mb_h;
  d->parser.resize(d->S);
  d->parsed.resize(d->S);
  d->parse_rc.assign(d->S, 0);
  d->lay = PicLayout(d->mb_w, d->mb_h);
  d->pic_bytes = d->lay.bytes();
  const size_t S = d->S;
  CK(d->own_st.create(cudaStreamNonBlocking));
  d->st = d->own_st.get();
  CK(d->d_pic.alloc(S * d->slots * d->pic_bytes + 256));
  CK(cudaMemset(d->d_pic.get(), 0, S * d->slots * d->pic_bytes + 256));
  CK(d->d_mbi.alloc(S * d->n_mb * sizeof(MbInfo)));
  CK(cudaMemset(d->d_mbi.get(), 0, S * d->n_mb * sizeof(MbInfo)));
  CK(d->d_recs.alloc(S * d->n_mb * sizeof(MbOut)));
  CK(d->h_recs.alloc(S * d->n_mb * sizeof(MbOut)));
  CK(d->d_pack.alloc(S * d->n_mb * sizeof(MbOut)));
  CK(d->h_idx.alloc(S * d->n_mb * sizeof(int32_t)));
  CK(d->d_idx.alloc(S * d->n_mb * sizeof(int32_t)));
  d->units.assign(d->S, 0);
  d->last_poc.assign(d->S, 0); d->last_idr.assign(d->S, 0); d->last_reorder.assign(d->S, 0);
  CK(d->d_aux.alloc(S * d->n_mb * sizeof(DecMbAux)));
  CK(d->h_aux.alloc(S * d->n_mb * sizeof(DecMbAux)));
  CK(d->d_sf.alloc(S * sizeof(StreamFrame)));
  CK(d->h_sf.alloc(S * sizeof(StreamFrame)));
  CK(d->d_out.alloc(S * sizeof(DecOutPic)));
  CK(d->h_out.alloc(S * sizeof(DecOutPic)));
  CK(d->staged.create(cudaEventDisableTiming));
  CK(d->d_ws.alloc(dec_sched_ints((int)S, d->mb_w, d->mb_h) * sizeof(int)));
  { int nt = usable_cores(); if (nt > d->S) nt = d->S; d->pool.reset(new Pool(nt < 1 ? 1 : nt)); }
  *out = d.release();
  return 0;
}

int b2h264_dec_create(const b2h264_dec_config* cfg, b2h264_dec** out) {
  if (!cfg || !out) return -1;
  const int rc = dec_create(cfg, out);
  if (rc > 0) (void)cudaGetLastError();    // the failure is returned here: later launch checks must not see it
  return rc;
}

void b2h264_dec_destroy(b2h264_dec* d) {
  if (!d) return;
  cudaSetDevice(d->cfg.device);
  cudaStreamSynchronize(d->st);
  delete d;
}

// got_picture (may be NULL): per stream 1 = a picture was decoded into yuv[s], 0 = the access unit carried no slice
// (parameter sets only / au[s] == NULL).  With got_picture == NULL an access unit without a slice is an error.
// status (may be NULL): per-stream outcome for callers that batch UNRELATED streams (the ISVCDecoder broker): 1 = picture, 0 = no slice in
// the unit, < 0 = this stream's error (-101 .. -105, -2) — such a stream sits the batch out and the others are decoded; without
// `status` the first stream error ends the call (the streams of one application stand or fall together).
// on_device: yuv[s] are device pointers on the decoder's device, written by k_dec_output; the call returns once its work is enqueued.
static int dec_decode_impl(b2h264_dec* d, const uint8_t* const* au, const int32_t* au_bytes, uint8_t* const* yuv, int32_t* got_picture, int32_t* status,
                           bool on_device = false) {
  if (!d || !au || !au_bytes || !yuv) return -1;
  CK(cudaSetDevice(d->cfg.device));
  const int S = d->S;
  int deblock = 1;
  static const bool timing = getenv("B2H264_DEC_TIMING") != nullptr;          // debug: host phases of the call on stderr
  const auto t0 = std::chrono::steady_clock::now();
  auto ms_since = [&](std::chrono::steady_clock::time_point a) { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a).count(); };
  d->act.clear(); d->act_ref.clear(); d->out_slot.clear(); d->out_cx.clear(); d->out_cy.clear();
  // 1. parse: every stream's access unit on the pool (streams are independent; a stream's parser state is its own)
  {
    std::function<void(int)> job = [&](int s) {
      d->parse_rc[s] = (!au[s] || au_bytes[s] <= 0) ? PARSE_NO_PICTURE : parse_access_unit(au[s], (size_t)au_bytes[s], &d->parser[s], &d->parsed[s]);
    };
    d->pool->run(S, job);
  }
  const double t_parse = ms_since(t0);
  // the pinned staging buffers still feed the previous call's copies until they are issued: the parse above overlapped them
  CK(cudaEventSynchronize(d->staged.get()));
  // 2. the batch: descriptors and records of the streams that carry a picture, in stream order
#define STREAM_FAIL(code) { d->last_error_stream = s; if (status) { status[s] = (code); continue; } return (code); }
  if (status) for (int s = 0; s < S; s++) status[s] = 0;
  for (int s = 0; s < S; s++) {
    if (got_picture) got_picture[s] = 0;
    if (!au[s] || au_bytes[s] <= 0) {
      if (!got_picture && !status) { d->last_error_stream = s; return -1; }
      continue;
    }
    ParsedPicture& pic = d->parsed[s];
    const int rc = d->parse_rc[s];
    if (rc == PARSE_NO_PICTURE && (got_picture || status)) continue;
    if (rc != PARSE_OK) STREAM_FAIL(-100 + (rc == PARSE_NO_PICTURE ? PARSE_INVALID : rc))   // -101 truncated, -102 unsupported, -103 invalid, -104 no parameter sets, -105 picture incomplete
    const StreamParams& sp = d->parser[s].sp;
    if (sp.mb_w != d->mb_w || sp.mb_h != d->mb_h || sp.width != d->cfg.width || sp.height != d->cfg.height) STREAM_FAIL(-2)
    if ((int)pic.mbs.size() != d->n_mb) STREAM_FAIL(-103)
    if ((int)pic.aux.size() != d->n_mb) STREAM_FAIL(-103)
    if (pic.has_b && (int)pic.aux_b.size() != d->n_mb) STREAM_FAIL(-103)
    if (pic.n_slots > d->slots) {                   // a stream with more reference frames: widen every stream's slot array, keeping the pictures
      if (pic.n_slots > 17) STREAM_FAIL(-103)
      DeviceBuf<uint8_t> np;
      CK(np.alloc((size_t)S * pic.n_slots * d->pic_bytes + 256));
      CK(cudaMemsetAsync(np.get(), 0, (size_t)S * pic.n_slots * d->pic_bytes + 256, d->st));
      for (int q = 0; q < S; q++)
        CK(cudaMemcpyAsync(np.get() + (size_t)q * pic.n_slots * d->pic_bytes, d->d_pic.get() + (size_t)q * d->slots * d->pic_bytes,
                           (size_t)d->slots * d->pic_bytes, cudaMemcpyDeviceToDevice, d->st));
      CK(cudaStreamSynchronize(d->st));
      d->d_pic = std::move(np); d->slots = pic.n_slots;
      for (int q = 0; q < (int)d->act.size(); q++) {      // descriptors built before the move
        StreamFrame& G = d->h_sf.get()[q];
        const int qs = d->act[q];
        for (int pl = 0; pl < 3; pl++) { G.f.rec[pl] = d->plane0(d->out_slot[q], qs, pl); G.f.ref[pl] = G.f.dpb0[pl] = d->plane0(0, qs, pl); }
      }
    }
    if (d->act.empty()) deblock = 0;
    if (pic.any_deblock) deblock = 1;               // the filter kernel runs if any slice of any stream wants it (per-MB control inside)
    const int i = (int)d->act.size();
    d->act.push_back(s); d->act_ref.push_back(pic.is_ref ? 1 : 0); d->out_slot.push_back(pic.cur_slot); d->out_cx.push_back(pic.crop_left); d->out_cy.push_back(pic.crop_top);
    StreamFrame& F = d->h_sf.get()[i];
    memset(&F, 0, sizeof(F));
    F.p.mb_w = d->mb_w; F.p.mb_h = d->mb_h;
    F.p.rec_stride_y = d->lay.stride_y; F.p.rec_stride_c = d->lay.stride_c;
    F.p.dec_cqp_off = pic.chroma_qp_offset;
    F.p.qp = pic.ss.qp; F.p.is_idr = pic.ss.idr; F.p.ref_is_p = !pic.ss.idr; F.p.mv_range = 64; F.p.dec_mode = 1;
    if (pic.cur_slot >= d->slots) STREAM_FAIL(-103)
    for (int pl = 0; pl < 3; pl++) { F.f.rec[pl] = d->plane0(pic.cur_slot, s, pl); F.f.ref[pl] = F.f.dpb0[pl] = d->plane0(0, s, pl); }
    F.f.dpb_stride = (int64_t)d->pic_bytes;
    F.f.mbi = d->d_mbi.get() + (size_t)s * d->n_mb;
    d->last_poc[s] = pic.poc; d->last_idr[s] = (pic.ss.idr ? 1 : 0) | (pic.has_b ? 2 : 0); d->last_reorder[s] = pic.max_reorder;
    if (pic.has_b) {                                // list-1 records of the picture's B macroblocks travel beside the aux records
      if (!d->d_aux_b.get()) {
        DeviceBuf<DecMbAuxB> db;
        HostBuf<DecMbAuxB> hb;
        CK(db.alloc((size_t)S * d->n_mb * sizeof(DecMbAuxB)));
        CK(hb.alloc((size_t)S * d->n_mb * sizeof(DecMbAuxB)));
        d->d_aux_b = std::move(db); d->h_aux_b = std::move(hb);
      }
      F.f.dec_aux_b = d->d_aux_b.get() + (size_t)i * d->n_mb;
    }
  }
  const int n = (int)d->act.size();
  if (n == 0) return 0;
  {
    std::function<void(int)> job = [&](int i) {          // compact records + index table into the stream's pinned slot
      const ParsedPicture& pic = d->parsed[d->act[i]];
      d->units[i] = pack_records_compact(pic.mbs.data(), d->n_mb, reinterpret_cast<uint8_t*>(d->h_recs.get() + (size_t)i * d->n_mb), d->h_idx.get() + (size_t)i * d->n_mb);
      memcpy(d->h_aux.get() + (size_t)i * d->n_mb, pic.aux.data(), (size_t)d->n_mb * sizeof(DecMbAux));
      if (pic.has_b) memcpy(d->h_aux_b.get() + (size_t)i * d->n_mb, pic.aux_b.data(), (size_t)d->n_mb * sizeof(DecMbAuxB));
    };
    d->pool->run(n, job);
  }
  const double t_pack = ms_since(t0);
  for (int i = 0; i < n; i++)                            // only what was packed crosses PCIe
    if (d->units[i] > 0)
      CK(cudaMemcpyAsync(d->d_pack.get() + (size_t)i * d->n_mb * sizeof(MbOut), d->h_recs.get() + (size_t)i * d->n_mb, (size_t)d->units[i] * 32, cudaMemcpyHostToDevice, d->st));
  CK(cudaMemcpyAsync(d->d_idx.get(), d->h_idx.get(), (size_t)n * d->n_mb * sizeof(int32_t), cudaMemcpyHostToDevice, d->st));
  { const int rcu = dec_launch_unpack(d->d_pack.get(), (size_t)d->n_mb * sizeof(MbOut), d->d_idx.get(), d->d_recs.get(), n, d->n_mb, d->st); if (rcu) return rcu; }
  CK(cudaMemcpyAsync(d->d_aux.get(), d->h_aux.get(), (size_t)n * d->n_mb * sizeof(DecMbAux), cudaMemcpyHostToDevice, d->st));
  for (int i = 0; i < n; i++)
    if (d->parsed[d->act[i]].has_b)
      CK(cudaMemcpyAsync(d->d_aux_b.get() + (size_t)i * d->n_mb, d->h_aux_b.get() + (size_t)i * d->n_mb, (size_t)d->n_mb * sizeof(DecMbAuxB), cudaMemcpyHostToDevice, d->st));
  CK(cudaMemcpyAsync(d->d_sf.get(), d->h_sf.get(), (size_t)n * sizeof(StreamFrame), cudaMemcpyHostToDevice, d->st));
  const int w = d->cfg.width, h = d->cfg.height;
  if (on_device) {
    for (int i = 0; i < n; i++) {
      DecOutPic& O = d->h_out.get()[i];
      for (int pl = 0; pl < 3; pl++) {
        const int c = pl ? 1 : 0;
        O.src[pl] = d->plane0(d->out_slot[i], d->act[i], pl) + (size_t)(d->out_cy[i] >> c) * d->lay.stride(pl) + (d->out_cx[i] >> c);
      }
      O.dst = yuv[d->act[i]];
    }
    CK(cudaMemcpyAsync(d->d_out.get(), d->h_out.get(), (size_t)n * sizeof(DecOutPic), cudaMemcpyHostToDevice, d->st));
  }
  CK(cudaEventRecord(d->staged.get(), d->st));
  int b_slices = 0;
  for (int i = 0; i < n; i++) b_slices |= (d->parsed[d->act[i]].has_b || d->parsed[d->act[i]].has_t8) ? 1 : 0;   // Main / High tools: the wider filter kernel
  const int rc = dec_launch_frame(d->d_sf.get(), n, d->mb_w, d->mb_h, d->d_ws.get(), d->d_recs.get(), d->d_aux.get(), deblock, d->st, b_slices);
  if (rc) return rc;
  const double t_launch = ms_since(t0);
  if (timing) cudaStreamSynchronize(d->st);
  const double t_kernels = ms_since(t0);
  if (on_device) {
    k_dec_output<<<dim3((2 * h + 7) / 8, n), 256, 0, d->st>>>(d->d_out.get(), w, h, d->lay.stride_y, d->lay.stride_c);
    const int rco = b2h264_launched();
    if (rco) return rco;
    for (int i = 0; i < n; i++) status[d->act[i]] = 1;
    return 0;
  }
  for (int i = 0; i < n; i++) {
    const int s = d->act[i], rec = d->out_slot[i];
    uint8_t* dst = yuv[s];
    for (int pl = 0; pl < 3; pl++) {
      const int pw = pl ? w / 2 : w, ph = pl ? h / 2 : h;
      const int stp = d->lay.stride(pl);
      const uint8_t* from = d->plane0(rec, s, pl) + (size_t)(d->out_cy[i] >> (pl ? 1 : 0)) * stp + (d->out_cx[i] >> (pl ? 1 : 0));
      CK(cudaMemcpy2DAsync(dst, pw, from, stp, pw, ph, cudaMemcpyDeviceToHost, d->st));
      dst += (size_t)pw * ph;
    }
    if (got_picture) got_picture[s] = 1;
    if (status) status[s] = 1;
  }
  CK(cudaStreamSynchronize(d->st));
  if (timing) {
    long long units = 0;
    for (int i = 0; i < n; i++) units += d->units[i];
    fprintf(stderr, "b2h264_dec_decode: %d pictures: parse %.2f ms, pack %.2f, launches issued %.2f, kernels done %.2f, pictures on the host %.2f; %.2f MB of records\n", n, t_parse,
            t_pack - t_parse, t_launch - t_pack, t_kernels - t_launch, ms_since(t0) - t_kernels, units * 32 / 1e6);
  }
  return 0;
}

#undef STREAM_FAIL

int b2h264_dec_decode2(b2h264_dec* d, const uint8_t* const* au, const int32_t* au_bytes, uint8_t* const* yuv, int32_t* got_picture) {
  return dec_decode_impl(d, au, au_bytes, yuv, got_picture, nullptr);
}
int b2h264_dec_decode3(b2h264_dec* d, const uint8_t* const* au, const int32_t* au_bytes, uint8_t* const* yuv, int32_t* status) {
  if (!status) return -1;
  return dec_decode_impl(d, au, au_bytes, yuv, nullptr, status);
}
int b2h264_dec_decode(b2h264_dec* d, const uint8_t* const* au, const int32_t* au_bytes, uint8_t* const* yuv) {
  return dec_decode_impl(d, au, au_bytes, yuv, nullptr, nullptr);
}
int b2h264_dec_decode_device(b2h264_dec* d, const uint8_t* const* au, const int32_t* au_bytes, uint8_t* const* yuv_dev, int32_t* status) {
  if (!d || !au || !au_bytes || !yuv_dev || !status) return -1;
  CK(cudaSetDevice(d->cfg.device));
  for (int s = 0; s < d->S; s++) {                       // every destination that may be written: HBM of the decoder's device
    if (!au[s]) continue;
    cudaPointerAttributes at;
    if (!yuv_dev[s] || cudaPointerGetAttributes(&at, yuv_dev[s]) != cudaSuccess || at.type != cudaMemoryTypeDevice || at.device != d->cfg.device) {
      (void)cudaGetLastError();
      return -1;
    }
  }
  return dec_decode_impl(d, au, au_bytes, yuv_dev, nullptr, status, true);
}

int b2h264_dec_set_stream(b2h264_dec* d, void* stream) {
  if (!d) return -1;
  CK(cudaSetDevice(d->cfg.device));
  CK(cudaStreamSynchronize(d->st));
  d->own_st = Stream();
  d->st = (cudaStream_t)stream;
  return 0;
}

// Looks at an access unit without a decoder: *has_slice = a coded slice NAL is present; if it carries an SPS of the
// supported class, *width / *height = the cropped picture size (else left untouched).  0, or a parser error (-10x).
int b2h264_dec_probe(const uint8_t* au, int32_t au_bytes, int32_t* width, int32_t* height, int32_t* has_slice) {
  if (!au || au_bytes <= 0) return -1;
  int w = 0, h = 0, sl = 0;
  const int rc = probe_access_unit(au, (size_t)au_bytes, &w, &h, &sl);
  if (has_slice) *has_slice = sl;
  if (rc != PARSE_OK) return -100 + rc;
  if (w > 0 && width) *width = w;
  if (h > 0 && height) *height = h;
  return 0;
}

// Output order: the decoder hands every picture back in DECODING order; *poc is its picture order count inside its coded video sequence
// (*flags: bit 0 = IDR picture, a new sequence starts; bit 1 = the picture holds B slices), *reorder_depth how many later-decoded pictures may precede it on output (0: the stream class has no
// reordering — Baseline — and decoding order is output order).  Layer 3 (ISVCDecoder) reorders with these.
int b2h264_dec_last_picture_order(b2h264_dec* d, int stream, int32_t* poc, int32_t* flags, int32_t* reorder_depth) {
  if (!d || stream < 0 || stream >= d->S) return -1;
  if (poc) *poc = d->last_poc[stream];
  if (flags) *flags = d->last_idr[stream];
  if (reorder_depth) *reorder_depth = d->last_reorder[stream];
  return 0;
}

// a stream slot starts over (a new ISVCDecoder object takes it): parser state, parameter sets and reference pictures are forgotten
int b2h264_dec_reset_stream(b2h264_dec* d, int stream) {
  if (!d || stream < 0 || stream >= d->S) return -1;
  d->parser[stream] = ParserState();
  d->parsed[stream] = ParsedPicture();
  return 0;
}

void* b2h264_host_alloc(size_t bytes) {
  void* p = nullptr;
  return cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocPortable) == cudaSuccess ? p : nullptr;
}
void b2h264_host_free(void* p) { if (p) cudaFreeHost(p); }

}  // extern "C"
