// tests/emu/emu.cu — HOST EMULATION BUILD of the device macroblock pipeline (debugging aid).
//
// TEST INFRASTRUCTURE ONLY.  The macroblock code in openh264_b200/csrc/enc_*.cuh is written once as
// __host__ __device__; this file compiles its HOST instantiation ("1-lane warp", see mbk_common.cuh)
// and drives it in plain raster order, so that bit-exactness against the reference can be debugged in a
// container without a GPU.  It is built into tests/emu/libb2h264_emu.so, which the product library
// never links or loads; the shipped path is the CUDA one (enc_kernels.cu) and fails without a device.
#include <stddef.h>
#include <stdio.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <chrono>
#include <array>
#include <algorithm>
#include <vector>

#include "../../openh264_b200/csrc/enc_frame.cuh"
#include "../../openh264_b200/csrc/enc_deblock.cuh"
#include "../../openh264_b200/csrc/h264_bitstream.h"

#include "../../openh264_b200/csrc/enc_host.h"
#include "../../openh264_b200/csrc/h264_parse.h"
#include "../../openh264_b200/csrc/dec_mb.cuh"

using namespace mbk;

extern "C" void b2h264_build_host_tables();

static bool same_record(const MbOut& a, const MbOut& b);

namespace {

// host-memory twin of the product's device-side frame buffers
static int g_emu_time_writer = 0;                     // > 0: time that many extra write_access_unit calls per picture
static double g_emu_writer_us = 0, g_emu_parser_us = 0;
static int g_emu_dbk[3] = {0, 0, 0};                  // iLoopFilterDisableIdc, alpha / beta offsets
static int g_emu_intra_period = 0;                    // uiIntraPeriod, the rule of csrc/enc_batch.cu (b2h264_enc_submit)
static int g_emu_cabac = 0, g_emu_profile = 0;       // entropy coder of the host writer (the macroblock decisions do not depend on it)
struct HostFrameEncoder {
  b2h264::StreamCtl ctl;
  EncFrameParams p;
  std::vector<uint8_t> cur[3], pic[2][3];
  std::vector<MbInfo> mbi;
  std::vector<RefMbInfo> rinfo[2];
  std::vector<MbOut> out;
  std::vector<uint8_t> prev_y;                // previous SOURCE luma (MB-aligned), reference of the VAA statistics
  std::vector<int32_t> vaa;                   // pSad8x8, indexed [iMbXY * 4 + k] as the reference does
  std::vector<int32_t> sad_cost, mb_bits;     // mb_bits: the macroblock code's own CAVLC bit count (enc_cavlc_bits.cuh)
  bool mb_bits_ok = true;
  MbScratch scratch;
  int cur_rec = 0;
  bool idr = true, have_ref_p = false;
  int p_since_idr = 0;

  HostFrameEncoder(int w, int h, int qp, float fps) {
    ctl.init(w, h, qp, fps, 5000000, g_emu_cabac, g_emu_profile);
    ctl.set_loop_filter(g_emu_dbk[0], g_emu_dbk[1], g_emu_dbk[2]);
    const int n = ctl.sp.mb_w * ctl.sp.mb_h;
    cur[0].resize((size_t)n * 256 + 64); cur[1].resize((size_t)n * 64 + 64); cur[2].resize((size_t)n * 64 + 64);
    for (int b = 0; b < 2; b++) {
      pic[b][0].assign((size_t)ctl.rec_stride_y() * ctl.rec_rows_y() + 64, 0);
      pic[b][1].assign((size_t)ctl.rec_stride_c() * ctl.rec_rows_c() + 64, 0);
      pic[b][2].assign((size_t)ctl.rec_stride_c() * ctl.rec_rows_c() + 64, 0);
      rinfo[b].resize(n);
    }
    mbi.resize(n); out.resize(n); sad_cost.assign(n, 0); mb_bits.assign(n, -1);
    prev_y.assign(cur[0].size(), 0); vaa.assign((size_t)n * 4, 0);
    ctl.record_mb_bits = true;
    memset(&scratch, 0, sizeof(scratch));
  }
  void load_source(const uint8_t* yuv) {
    b2h264::pad_source(yuv, ctl.sp.width, ctl.sp.height, ctl.sp.mb_w, ctl.sp.mb_h, cur[0].data(), cur[1].data(), cur[2].data());
  }
  void begin_frame() {
    idr = ctl.next_is_idr() || (g_emu_intra_period > 0 && 1 + p_since_idr >= g_emu_intra_period);
    p_since_idr = idr ? 0 : p_since_idr + 1;
    p = ctl.frame_params(idr, have_ref_p);
    if (ctl.fast_mode) {
      // VAACalcSad_c (codec/processing/src/vaacalc/vaacalcfuncs.cpp:254): 8x8 SADs of the (w >> 4) x (h >> 4) whole macroblocks
      // of the picture against the previous source picture, stored with a running macroblock index of THAT width
      const int st = ctl.sp.mb_w * 16, vw = ctl.sp.mb_w, vh = ctl.sp.mb_h;
      int mb_index = 0;
      for (int i = 0; i < vh; i++)
        for (int j = 0; j < vw; j++, mb_index++)
          for (int k = 0; k < 4; k++) {
            const uint8_t* a = cur[0].data() + (size_t)(i * 16 + (k >> 1) * 8) * st + j * 16 + (k & 1) * 8;
            const uint8_t* b = prev_y.data() + (a - cur[0].data());
            int sad = 0;
            for (int y = 0; y < 8; y++) for (int x = 0; x < 8; x++) sad += abs((int)a[y * st + x] - (int)b[y * st + x]);
            vaa[(size_t)mb_index * 4 + k] = sad;
          }
    }
  }
  uint8_t* plane0(int b, int pl) {   // pixel (0,0) inside the padding
    const int pad = pl ? 16 : 32, st = pl ? ctl.rec_stride_c() : ctl.rec_stride_y();
    return pic[b][pl].data() + (size_t)pad * st + pad;
  }
  EncFramePtrs ptrs() {
    EncFramePtrs f;
    memset(&f, 0, sizeof(f));
    for (int pl = 0; pl < 3; pl++) { f.cur[pl] = cur[pl].data(); f.rec[pl] = plane0(cur_rec, pl); f.ref[pl] = plane0(1 - cur_rec, pl); }
    f.mbi = mbi.data(); f.rec_info = rinfo[cur_rec].data(); f.ref_info = rinfo[1 - cur_rec].data(); f.out = out.data();
    f.sad_cost = sad_cost.data();
    f.mb_bits = mb_bits.data();
    f.vaa_sad8x8 = vaa.data();
    return f;
  }
  bool packed_writer_ok = true;
  // parser round trip (h264_parse.h): parse(write(records)) must give the records back
  b2h264::ParserState parser;
  int parse_status = 0;              // 0 ok, <0 ParseError, >0 = 1 + index of the first macroblock that differs
  void check_parse(const std::vector<uint8_t>& au) {
    b2h264::ParsedPicture pic;
    if (g_emu_time_writer > 0) {                      // microbenchmark of the parser on the same access unit
      b2h264::ParsedPicture tp;
      { b2h264::ParserState ps = parser; b2h264::parse_access_unit(au.data(), au.size(), &ps, &tp); }
      double us = 0;
      for (int r = 0; r < g_emu_time_writer; r++) {
        b2h264::ParserState ps = parser;
        const auto t0 = std::chrono::steady_clock::now();
        b2h264::parse_access_unit(au.data(), au.size(), &ps, &tp);
        us += std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count();
      }
      g_emu_parser_us = us / g_emu_time_writer;
    }
    const int rc = b2h264::parse_access_unit(au.data(), au.size(), &parser, &pic);
    if (rc != 0) { parse_status = rc; return; }
    if (pic.ss.idr != idr || pic.mbs.size() != out.size() || parser.sp.mb_w != ctl.sp.mb_w || parser.sp.width != ctl.sp.width ||
        parser.sp.height != ctl.sp.height) { parse_status = -100; return; }
    for (size_t i = 0; i < out.size(); i++) {
      const bool same = same_record(out[i], pic.mbs[i]);
      if (!same) { parse_status = 1 + (int)i; return; }
    }
  }
  void finish_frame(std::vector<uint8_t>* bs) {
    // the product hands the host only the coded macroblocks' records plus an index table (k_pack_records):
    // write the access unit through that form too and insist on the same bytes
    if (g_emu_time_writer > 0) {                      // microbenchmark of the host entropy coder (tools/time_writer.py)
      b2h264::StreamCtl c2 = ctl;
      std::vector<uint8_t> tmp;
      c2.write_access_unit(idr, out.data(), &tmp);      // warm: buffers at their final capacity
      const auto t0 = std::chrono::steady_clock::now();
      for (int r = 0; r < g_emu_time_writer; r++) { tmp.clear(); c2.write_access_unit(idr, out.data(), &tmp); }
      g_emu_writer_us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count() / g_emu_time_writer;
    }
    {
      b2h264::StreamCtl twin = ctl;
      // the host twin of k_pack_records (the decoder's hand-over uses it; the encoder's device kernel follows the same rules)
      std::vector<uint8_t> packed(out.size() * sizeof(MbOut));
      std::vector<int32_t> index(out.size());
      b2h264::pack_records_compact(out.data(), (int)out.size(), packed.data(), index.data());
      std::vector<uint8_t> a, b;
      b2h264::StreamCtl plain = ctl;
      plain.write_access_unit(idr, out.data(), &a);
      twin.write_access_unit_packed(idr, reinterpret_cast<const MbOut*>(packed.data()), index.data(), &b);
      if (a != b) packed_writer_ok = false;
    }
    ctl.write_access_unit(idr, out.data(), bs);
    // the bit count the macroblock code computed without writing must equal what the writer spent, macroblock by macroblock
    if (!ctl.sp.entropy_cabac && ctl.last_mb_bits != mb_bits) mb_bits_ok = false;
    if (parse_status == 0) check_parse(*bs);                                  // CAVLC and CABAC alike
    have_ref_p = !idr;
    prev_y = cur[0];
    cur_rec = 1 - cur_rec;            // the picture just reconstructed becomes the reference
  }
  void copy_recon(uint8_t* dst) {     // cropped I420 of the picture just finished (now the reference)
    const int b = 1 - cur_rec;
    for (int pl = 0; pl < 3; pl++) {
      const int w = pl ? ctl.sp.width / 2 : ctl.sp.width, h = pl ? ctl.sp.height / 2 : ctl.sp.height;
      const int st = pl ? ctl.rec_stride_c() : ctl.rec_stride_y();
      for (int y = 0; y < h; y++) { memcpy(dst, plane0(b, pl) + (size_t)y * st, w); dst += w; }
    }
  }
};

void deblock_frame_host(const EncFrameParams& p, const EncFramePtrs& f);
void expand_frame_host(const EncFrameParams& p, const EncFramePtrs& f) {
  for (int pl = 0; pl < 3; pl++) {
    const int pad = pl ? 16 : 32, st = pl ? p.rec_stride_c : p.rec_stride_y;
    const int w = (pl ? 8 : 16) * p.mb_w, h = (pl ? 8 : 16) * p.mb_h;
    uint8_t* pic = f.rec[pl];
    for (int y = 0; y < h; y++) { memset(pic + (size_t)y * st - pad, pic[(size_t)y * st], pad); memset(pic + (size_t)y * st + w, pic[(size_t)y * st + w - 1], pad); }
    for (int y = 1; y <= pad; y++) {
      memcpy(pic - (ptrdiff_t)y * st - pad, pic - pad, w + 2 * pad);
      memcpy(pic + (size_t)(h - 1 + y) * st - pad, pic + (size_t)(h - 1) * st - pad, w + 2 * pad);
    }
  }
}
void deblock_frame_host(const EncFrameParams& p, const EncFramePtrs& f) {
  for (int mby = 0; mby < p.mb_h; mby++)
    for (int mbx = 0; mbx < p.mb_w; mbx++) {
      static DbkTileB tile;
      if (p.dec_mode) deblock_one_mb_b(p, f, mbx, mby, tile);      // decoded pictures: B slices / the 8x8 transform may occur
      else deblock_one_mb(p, f, mbx, mby, tile);
    }
}

}  // namespace

// the border replication of expand_frame_host, for the hooks built beside this file (decode_records_hooks.cu)
void emu_expand_frame(const EncFrameParams& p, const EncFramePtrs& f) { expand_frame_host(p, f); }

// do two records describe the same coded macroblock?  (only what the bitstream carries is compared)
static bool same_record(const MbOut& a, const MbOut& b) {
  bool same = a.mb_type == b.mb_type;
  if (same && a.mb_type != MBT_PSKIP) {
    same = a.cbp == b.cbp && memcmp(a.nnz, b.nnz, 24) == 0;
    if (a.cbp > 0 || a.mb_type == MBT_I16x16) same = same && a.qp == b.qp;
    if (MBT_IS_INTRA(a.mb_type)) same = same && a.chroma_mode == b.chroma_mode;
    if (a.mb_type == MBT_I16x16) same = same && a.i16_mode == b.i16_mode && memcmp(a.luma_dc, b.luma_dc, 32) == 0;
    if (a.mb_type == MBT_I4x4)
      for (int k = 0; k < 16; k++) same = same && a.prev_i4_flag[k] == b.prev_i4_flag[k] && (a.prev_i4_flag[k] || a.rem_i4_mode[k] == b.rem_i4_mode[k]);
    const int nparts = a.mb_type == MBT_P16x16 ? 1 : (a.mb_type == MBT_P16x8 || a.mb_type == MBT_P8x16) ? 2 : a.mb_type == MBT_P8x8 ? 4 : 0;
    for (int k = 0; k < nparts; k++) same = same && a.mvd[k][0] == b.mvd[k][0] && a.mvd[k][1] == b.mvd[k][1];
    for (int k = 0; k < 16 && same; k++) {
      const int bx = (k & 1) | ((k >> 1) & 2), by = ((k >> 1) & 1) | ((k >> 2) & 2);
      if (!(a.cbp & (1 << (k >> 2))) || a.nnz[by * 4 + bx] == 0) continue;     // not coded / written as empty
      same = memcmp(a.luma[k], b.luma[k], (a.mb_type == MBT_I16x16 ? 15 : 16) * 2) == 0;
    }
    if (same && (a.cbp >> 4)) same = memcmp(a.chroma_dc, b.chroma_dc, 16) == 0;
    if (same && (a.cbp >> 4) == 2)
      for (int j = 0; j < 8 && same; j++)
        if (a.nnz[16 + j] > 0) same = memcmp(a.chroma_ac[j], b.chroma_ac[j], 30) == 0;
  }
  return same;
}

static std::vector<uint8_t> g_last_path;     // per macroblock of the last picture: bit s = stage s ran
static unsigned g_stages_run;                 // the same bits over every macroblock of every picture of the last emu_encode
extern "C" int emu_last_path(uint8_t* path, int n) {
  if ((int)g_last_path.size() < n) return -1;
  memcpy(path, g_last_path.data(), n);
  return 0;
}
extern "C" unsigned emu_stages_run() { return g_stages_run; }
static std::vector<MbOut> g_last_out;
static std::vector<MbInfo> g_last_info;
extern "C" int emu_last(MbOut* out, MbInfo* info, int n) {
  if ((int)g_last_out.size() < n) return -1;
  if (out) memcpy(out, g_last_out.data(), sizeof(MbOut) * n);
  if (info) memcpy(info, g_last_info.data(), sizeof(MbInfo) * n);
  return 0;
}
static int g_emu_fast_mode = 0;
extern "C" void emu_set_entropy(int cabac, int profile_idc) { g_emu_cabac = cabac; g_emu_profile = profile_idc; }
extern "C" void emu_set_time_writer(int reps) { g_emu_time_writer = reps; }
extern "C" double emu_last_writer_us() { return g_emu_writer_us; }
extern "C" double emu_last_parser_us() { return g_emu_parser_us; }
extern "C" void emu_set_loop_filter(int idc, int a, int b) { g_emu_dbk[0] = idc; g_emu_dbk[1] = a; g_emu_dbk[2] = b; }
extern "C" void emu_set_intra_period(int n) { g_emu_intra_period = n; }
extern "C" void emu_set_complexity_low(int on) { g_emu_fast_mode = on; }
extern "C" long emu_encode(const uint8_t* yuv, int w, int h, int nframes, int qp, float fps, uint8_t* out, long cap,
                           int32_t* frame_bytes, uint8_t* recon_out /* nframes * w*h*3/2 or NULL */) {
  b2h264_build_host_tables();
  HostFrameEncoder enc(w, h, qp, fps);
  enc.ctl.fast_mode = g_emu_fast_mode != 0;
  long total = 0;
  const size_t fsz = (size_t)w * h * 3 / 2;
  g_stages_run = 0;
  for (int i = 0; i < nframes; i++) {
    std::vector<uint8_t> bs;
    enc.load_source(yuv + i * fsz);
    enc.begin_frame();
    // --- the part the GPU does in the product: macroblocks (raster order here), deblocking, expansion
    g_last_path.assign((size_t)enc.p.mb_w * enc.p.mb_h, 0);
    for (int mby = 0; mby < enc.p.mb_h; mby++)
      for (int mbx = 0; mbx < enc.p.mb_w; mbx++) {
        // the stages of the macroblock back to back, each recorded (bit s = stage s ran): the device scheduler runs
        // them as separate tasks (tools/sched_sim.py replays these paths)
        const EncFramePtrs f = enc.ptrs();
        mb_ctx(enc.scratch.ctx, enc.p, f, mbx, mby);
        int stage = enc.p.is_idr ? MBS_I : MBS_A;
        while (stage != MBS_DONE) {
          g_last_path[(size_t)mby * enc.p.mb_w + mbx] |= (uint8_t)(1u << stage);
          g_stages_run |= 1u << stage;
          stage = mb_run_stage(enc.scratch.ctx, enc.scratch, stage);
        }
      }
    deblock_frame_host(enc.p, enc.ptrs());
    expand_frame_host(enc.p, enc.ptrs());
    // --- host entropy coding
    g_last_out = enc.out; g_last_info = enc.mbi;
    enc.finish_frame(&bs);
    if (!enc.packed_writer_ok) return -9;          // packed hand-over form wrote different bytes
    if (!enc.mb_bits_ok) return -8;                // exact CAVLC bit count differs from the writer
    if (enc.parse_status != 0) return -1000 - (enc.parse_status < 0 ? -enc.parse_status : 100 + enc.parse_status);   // parser round trip failed
    if (total + (long)bs.size() > cap) return -1;
    memcpy(out + total, bs.data(), bs.size());
    total += bs.size();
    if (frame_bytes) frame_bytes[i] = (int32_t)bs.size();
    if (recon_out) enc.copy_recon(recon_out + i * fsz);
  }
  return total;
}


// ---- decoder construct path, host build (groundwork: dec_mb.cuh + h264_parse.h) ---------------------------------------
// Decodes an Annex-B stream of the supported class; writes the cropped I420 pictures back to back into out.
// Returns the number of pictures, or a negative error (-1000 - k: parse error k).
extern "C" int emu_decode(const uint8_t* bs, long len, uint8_t* out, long cap, int* w, int* h) {
  b2h264_build_host_tables();
  b2h264::ParserState st;
  // picture slots (decoded picture buffer): one contiguous buffer per plane, slot k at k * slot_bytes[pl]
  std::vector<uint8_t> dpb;                 // slot k = one whole padded picture (Y, U, V) at k * pic_bytes, like the device layout
  size_t pic_bytes = 0, y_bytes = 0, c_bytes = 0;
  int n_slots = 0;
  std::vector<MbInfo> mbi;
  static MbScratch scratch;
  int frames = 0, seq = 0;
  std::vector<std::array<int, 3>> order;      // (coded video sequence, picture order count, position in `out`) of every picture
  long outpos = 0;
  bool have_buffers = false;
  auto is_start = [&](long k) { return k + 2 < len && bs[k] == 0 && bs[k + 1] == 0 && bs[k + 2] == 1; };
  long pos = 0;
  while (pos + 3 < len && !is_start(pos)) pos++;
  long au_begin = pos > 0 && bs[pos - 1] == 0 ? pos - 1 : pos;
  while (pos + 3 < len) {
    // walk NAL by NAL; an access unit ends with its (single) slice NAL
    const int type = bs[pos + 3] & 31;
    long next = pos + 3;
    while (next + 3 < len && !is_start(next)) next++;
    if (next + 3 >= len) next = len;
    // an access unit ends with its last slice NAL: the NAL that follows is not a slice, or is a slice that starts a new
    // picture (first_mb_in_slice == 0: its ue(v) is the single bit 1 right after the NAL header)
    bool last_slice = false;
    if (type == 1 || type == 5) {
      last_slice = true;
      if (next + 4 < len) {
        const long hdr = next + 3;                      // NAL header byte of the next unit
        const int ntype = bs[hdr] & 31;
        if ((ntype == 1 || ntype == 5) && !(bs[hdr + 1] & 0x80)) last_slice = false;   // next slice continues this picture
      }
    }
    if (last_slice) {
      long au_end = next;
      if (au_end < len && au_end > 0 && bs[au_end - 1] == 0) au_end--;        // zero_byte of the next 4-byte start code
      b2h264::ParsedPicture pp;
      const int rc = b2h264::parse_access_unit(bs + au_begin, (size_t)(au_end - au_begin), &st, &pp);
      if (rc != 0 && getenv("EMU_MAX_FRAMES")) { fprintf(stderr, "parse error %d at picture %d\n", rc, frames); break; }
      if (rc != 0) return -1000 + rc;
      b2h264::StreamCtl geo;                                                    // picture geometry helpers
      geo.sp = st.sp;
      if (have_buffers && (int)mbi.size() != st.sp.mb_w * st.sp.mb_h) return -4;   // picture size changed mid-stream
      if (!have_buffers || pp.n_slots > n_slots) {
        if (have_buffers && !pp.ss.idr) return -5;                               // more slots needed mid-sequence
        n_slots = pp.n_slots;
        y_bytes = (size_t)geo.rec_stride_y() * geo.rec_rows_y() + 64;
        c_bytes = (size_t)geo.rec_stride_c() * geo.rec_rows_c() + 64;
        pic_bytes = y_bytes + 2 * c_bytes;
        dpb.assign(pic_bytes * n_slots, 0);
        mbi.assign((size_t)st.sp.mb_w * st.sp.mb_h, MbInfo());
        have_buffers = true;
      }
      EncFrameParams p;
      memset(&p, 0, sizeof(p));
      p.mb_w = st.sp.mb_w; p.mb_h = st.sp.mb_h;
      p.rec_stride_y = geo.rec_stride_y(); p.rec_stride_c = geo.rec_stride_c();
      p.qp = pp.ss.qp; p.is_idr = pp.ss.idr; p.ref_is_p = !pp.ss.idr; p.mv_range = 64; p.dec_mode = 1;
      p.dec_cqp_off = pp.chroma_qp_offset;
      EncFramePtrs f;
      memset(&f, 0, sizeof(f));
      for (int pl = 0; pl < 3; pl++) {
        const int pad = pl ? 16 : 32, stp = pl ? p.rec_stride_c : p.rec_stride_y;
        f.dpb0[pl] = dpb.data() + (pl == 0 ? 0 : y_bytes + (pl - 1) * c_bytes) + (size_t)pad * stp + pad;
        f.rec[pl] = const_cast<uint8_t*>(f.dpb0[pl]) + (size_t)pp.cur_slot * pic_bytes;
        f.ref[pl] = f.dpb0[pl];
      }
      f.dpb_stride = (int64_t)pic_bytes;
      f.mbi = mbi.data();
      f.dec_aux_b = pp.has_b ? pp.aux_b.data() : nullptr;
      if (const char* dbg = getenv("EMU_DUMP_MB")) {            // debugging aid: "frame,mbx,mby"
        int df = 0, dx = 0, dy = 0;
        if (sscanf(dbg, "%d,%d,%d", &df, &dx, &dy) == 3 && df == frames && dx < p.mb_w && dy < p.mb_h) {
          const MbOut& m = pp.mbs[(size_t)dy * p.mb_w + dx];
          const DecMbAux& a = pp.aux[(size_t)dy * p.mb_w + dx];
          fprintf(stderr, "mb (%d,%d) frame %d: type %d cbp %d qp %d i16 %d chroma %d avail %d flags %d poc %d\n", dx, dy, df, m.mb_type, m.cbp, m.qp, m.i16_mode, m.chroma_mode, a.avail, a.flags, pp.poc);
          fprintf(stderr, "  i4 prev/rem:");
          for (int k = 0; k < 16; k++) fprintf(stderr, " %d/%d", m.prev_i4_flag[k], m.rem_i4_mode[k]);
          fprintf(stderr, "\n  ref0 %d %d %d %d", a.ref_idx[0], a.ref_idx[1], a.ref_idx[2], a.ref_idx[3]);
          if (pp.has_b) { const DecMbAuxB& b = pp.aux_b[(size_t)dy * p.mb_w + dx]; fprintf(stderr, " ref1 %d %d %d %d w1 %d", b.ref_idx[0], b.ref_idx[1], b.ref_idx[2], b.ref_idx[3], b.w1[0]);
            fprintf(stderr, "\n  mv0:"); for (int k = 0; k < 16; k++) fprintf(stderr, " (%d,%d)", a.mvd[k][0], a.mvd[k][1]);
            fprintf(stderr, "\n  mv1:"); for (int k = 0; k < 16; k++) fprintf(stderr, " (%d,%d)", b.mv[k][0], b.mv[k][1]); }
          fprintf(stderr, "\n");
        }
      }
      for (int mby = 0; mby < p.mb_h; mby++)
        for (int mbx = 0; mbx < p.mb_w; mbx++) dec_one_mb(p, f, scratch, mbx, mby, pp.mbs[(size_t)mby * p.mb_w + mbx], pp.aux[(size_t)mby * p.mb_w + mbx]);
      if (pp.any_deblock) deblock_frame_host(p, f);
      expand_frame_host(p, f);
      const int W = st.sp.width, H = st.sp.height;
      *w = W; *h = H;
      if (outpos + (long)W * H * 3 / 2 > cap) return -2;
      for (int pl = 0; pl < 3; pl++) {
        const int pw = pl ? W / 2 : W, ph = pl ? H / 2 : H, stp = pl ? p.rec_stride_c : p.rec_stride_y;
        const int cx = pp.crop_left >> (pl ? 1 : 0), cy = pp.crop_top >> (pl ? 1 : 0);
        for (int y = 0; y < ph; y++) { memcpy(out + outpos, f.rec[pl] + (size_t)(y + cy) * stp + cx, pw); outpos += pw; }
      }
      if (pp.ss.idr) seq++;
      order.push_back({seq, pp.poc, frames});
      frames++;
      if (const char* mf = getenv("EMU_MAX_FRAMES")) if (frames >= atoi(mf)) break;   // debugging aid: stop after N pictures
      au_begin = au_end;
    }
    pos = next;
  }
  // output order: by picture order count inside every coded video sequence (an IDR picture starts a new one); decoding order for
  // streams without B slices (their counts rise with the decoding order)
  bool sorted = true;
  for (size_t i = 1; i < order.size(); i++) sorted = sorted && !(order[i] < order[i - 1]);
  if (!sorted) {
    std::vector<std::array<int, 3>> o2 = order;
    std::stable_sort(o2.begin(), o2.end(), [](const std::array<int, 3>& a, const std::array<int, 3>& b) { return a[0] != b[0] ? a[0] < b[0] : a[1] < b[1]; });
    const size_t fsz = (size_t)*w * *h * 3 / 2;
    std::vector<uint8_t> tmp(out, out + fsz * frames);
    for (int i = 0; i < frames; i++) memcpy(out + fsz * i, tmp.data() + fsz * o2[i][2], fsz);
  }
  return frames > 0 ? frames : -3;          // nothing decodable is an error, not an empty success
}


// ---- whole-picture deblocking of given records, the host build of the device filter (deblock_frame_host) ----------------
// Planes point at sample (0,0); mbi / aux_b hold mb_w * mb_h records as the decoder (dec_mode 1) or the encoder (dec_mode 0)
// leaves them; aux_b may be NULL.  idc / off_a / off_b: the encoder's per-picture control (the decoder's travels in mbi).
// tests/test_deblock_oracle_emu.py compares the result with oracle/orc_deblock_picture.
extern "C" int emu_deblock_picture(uint8_t* y, uint8_t* cb, uint8_t* cr, int stride_y, int stride_c, int mb_w, int mb_h, MbInfo* mbi,
                                   const DecMbAuxB* aux_b, int dec_mode, int idc, int off_a, int off_b) {
  if (mb_w < 1 || mb_h < 1 || !mbi || (aux_b && !dec_mode)) return -1;
  b2h264_build_host_tables();
  EncFrameParams p;
  memset(&p, 0, sizeof(p));
  p.mb_w = mb_w; p.mb_h = mb_h;
  p.rec_stride_y = stride_y; p.rec_stride_c = stride_c;
  p.dec_mode = dec_mode; p.dbk_idc = idc; p.dbk_off_a = off_a; p.dbk_off_b = off_b;
  EncFramePtrs f;
  memset(&f, 0, sizeof(f));
  f.rec[0] = y; f.rec[1] = cb; f.rec[2] = cr;
  f.mbi = mbi;
  f.dec_aux_b = aux_b;
  deblock_frame_host(p, f);
  return 0;
}

// ---- randomized writer <-> parser round trip (levels up to the Baseline escape range, every macroblock type) -----------
// Returns 0, a negative ParseError, or 1 + index of the first macroblock that came back different.
static int random_pictures(unsigned seed, int pictures, bool decodable, uint8_t* stream_out, long cap, long* stream_len,
                           bool loop_filter_off = false, std::vector<b2h264::ParsedPicture>* parsed = nullptr);
extern "C" int emu_roundtrip_random(unsigned seed, int pictures) { return random_pictures(seed, pictures, false, nullptr, 0, nullptr); }
// the same generator restricted to streams every conforming decoder reconstructs identically (DC intra prediction only,
// bounded coefficient energy, bounded vectors): the Annex-B stream is returned for tests/test_decoder_emu.py, which
// decodes it with the host construct path AND with the reference decoder
extern "C" long emu_random_stream(unsigned seed, int pictures, uint8_t* out, long cap) {
  long len = 0;
  const int rc = random_pictures(seed, pictures, true, out, cap, &len);
  return rc == 0 ? len : (long)rc;
}
// the same decodable streams written with the loop filter off (disable_deblocking_filter_idc 1), and what the parser made of each
// picture: recs / aux = pictures * 20 records (5 x 4 macroblocks, raster), info[3 * p] = the picture's slot, the stream's slot
// count and its chroma_qp_index_offset.  tests/test_decode_records_emu.py reconstructs these pictures with the spec oracle and
// compares them with the reference decoder's.  Returns the stream's length or a negative error as emu_random_stream does.
extern "C" long emu_random_stream_records(unsigned seed, int pictures, uint8_t* out, long cap, MbOut* recs, DecMbAux* aux, int32_t* info) {
  long len = 0;
  std::vector<b2h264::ParsedPicture> parsed;
  const int rc = random_pictures(seed, pictures, true, out, cap, &len, true, &parsed);
  if (rc != 0) return (long)rc;
  for (size_t p = 0; p < parsed.size(); p++) {
    if (parsed[p].mbs.size() != 20 || parsed[p].aux.size() != 20) return -300;
    memcpy(recs + 20 * p, parsed[p].mbs.data(), 20 * sizeof(MbOut));
    memcpy(aux + 20 * p, parsed[p].aux.data(), 20 * sizeof(DecMbAux));
    info[3 * p] = parsed[p].cur_slot; info[3 * p + 1] = parsed[p].n_slots; info[3 * p + 2] = parsed[p].chroma_qp_offset;
  }
  return len;
}
static int random_pictures(unsigned seed, int pictures, bool decodable, uint8_t* stream_out, long cap, long* stream_len,
                           bool loop_filter_off, std::vector<b2h264::ParsedPicture>* parsed) {
  uint32_t x = seed * 2654435761u + 12345u;
  auto rnd = [&](uint32_t n) { x = x * 1664525u + 1013904223u; return (x >> 8) % n; };
  const int W = 5, H = 4;
  b2h264::StreamCtl ctl;
  ctl.init(W * 16, H * 16, 26, 30.0f, 0);
  if (loop_filter_off && !ctl.set_loop_filter(1, 0, 0)) return -400;
  b2h264::ParserState st;
  int cur_qp = 26;                                            // qp the block being filled will be dequantised with
  auto rand_level = [&]() {
    const uint32_t c = rnd(100);
    int v = c < 60 ? 1 : c < 85 ? 2 + (int)rnd(6) : c < 97 ? 8 + (int)rnd(120) : 128 + (int)rnd(1872);
    return (int16_t)(rnd(2) ? -v : v);
  };
  auto fill_block = [&](int16_t* lv, int max_coef) {          // returns the number of non-zero levels
    for (int i = 0; i < 16; i++) lv[i] = 0;
    const uint32_t style = rnd(10);
    int nz = 0;
    // decodable streams keep the residual inside the range real encoders produce: one larger level at most, bounded by
    // the quantiser step, the rest small (a conforming stream never overflows the 16-bit transform path)
    const int big_cap = 1 + (1500 >> (cur_qp / 6));
    bool big_used = false;
    for (int i = 0; i < max_coef; i++) {
      const bool on = style == 0 ? true : style < 4 ? rnd(2) == 0 : rnd(8) == 0;
      if (!on) continue;
      int16_t v = rand_level();
      if (decodable) {
        int a = v < 0 ? -v : v;
        if (a > 2) { if (big_used) a = 1 + (int)rnd(2); else { a = a > big_cap ? big_cap : a; big_used = true; } }
        v = (int16_t)(v < 0 ? -a : a);
      }
      lv[i] = v; nz++;
    }
    if (loop_filter_off) {
      // the streams written with the loop filter off must also meet 8.5.10 to 8.5.12 exactly: every value of the inverse
      // transforms is bounded by the sum of the scaled coefficients' magnitudes, and a scaled level is at most |level| x 29 x
      // 2^(qp / 6) (normAdjust4x4 <= 29); a block's levels keep that sum under 16000 (room for a luma / chroma DC of a
      // quarter of it), so the spec oracle reconstructs them as the standard defines
      const int budget = 16000 / (29 << (cur_qp / 6));
      int sum = 0;
      for (int i = 0; i < max_coef; i++) sum += lv[i] < 0 ? -lv[i] : lv[i];
      while (sum > budget) {
        int k = 0;
        for (int i = 1; i < max_coef; i++) if (abs(lv[i]) > abs(lv[k])) k = i;
        lv[k] = (int16_t)(lv[k] < 0 ? lv[k] + 1 : lv[k] - 1);
        if (lv[k] == 0) nz--;
        sum--;
      }
    }
    return nz;
  };
  for (int pic = 0; pic < pictures; pic++) {
    const bool idr = pic == 0 || rnd(8) == 0;
    if (idr) ctl.force_idr = true;
    std::vector<MbOut> recs((size_t)W * H);
    std::vector<int8_t> i4modes((size_t)W * H * 16, 2);         // final I4x4 modes per MB (raster blocks), for mode prediction
    int qp = 26;
    for (size_t mi = 0; mi < recs.size(); mi++) {
      MbOut& m = recs[mi];
      const int mbx = (int)mi % W, mby = (int)mi / W;
      const int nbav = (mbx > 0 ? NB_LEFT : 0) | (mby > 0 ? NB_TOP : 0) | (mbx > 0 && mby > 0 ? NB_TOPLEFT : 0) | (mby > 0 && mbx < W - 1 ? NB_TOPRIGHT : 0);
      memset(&m, 0, sizeof(m));
      const uint32_t t = rnd(idr ? 2 : 8);
      m.mb_type = (uint8_t)(idr ? (t ? MBT_I16x16 : MBT_I4x4)
                                : t == 0 ? MBT_I4x4 : t == 1 ? MBT_I16x16 : t == 2 ? MBT_P16x16 : t == 3 ? MBT_P16x8 : t == 4 ? MBT_P8x16
                                  : t == 5 ? MBT_P8x8 : MBT_PSKIP);
      if (m.mb_type == MBT_PSKIP) { m.qp = (uint8_t)qp; continue; }
      int cbp_l = m.mb_type == MBT_I16x16 ? (rnd(2) ? 15 : 0) : (int)rnd(16);
      const int cbp_c = (int)rnd(3);
      // the quantiser this macroblock will carry is drawn first so that the level generator can respect it
      if ((cbp_l | cbp_c) > 0 || m.mb_type == MBT_I16x16) {
        qp += (int)rnd(41) - 20;                               // mb_qp_delta stays inside [-26, 25]
        qp = qp < 10 ? 10 : qp > 45 ? 45 : qp;
      }
      cur_qp = qp;
      // intra 16x16 / chroma modes: only modes whose neighbours exist (the parser rejects others as invalid); I4x4 modes
      // likewise in decodable streams;
      // DDL / VL without a top-right neighbour ARE allowed (8.3.1.2 substitutes samples) and are generated on purpose
      const bool L = (nbav & NB_LEFT) != 0, T = (nbav & NB_TOP) != 0, TL = (nbav & NB_TOPLEFT) != 0;
      if (MBT_IS_INTRA(m.mb_type)) {
        int cm = (int)rnd(4);                                    // 0 DC, 1 H, 2 V, 3 plane
        if (((cm == 1 && !L) || (cm == 2 && !T) || (cm == 3 && !(L && T && TL)))) cm = 0;
        m.chroma_mode = (uint8_t)cm;
      }
      if (m.mb_type == MBT_I16x16) {
        int im = (int)rnd(4);                                    // 0 V, 1 H, 2 DC, 3 plane
        if (((im == 0 && !T) || (im == 1 && !L) || (im == 3 && !(L && T && TL)))) im = 2;
        m.i16_mode = (uint8_t)im;
        fill_block(m.luma_dc, 16);
      }
      if (m.mb_type == MBT_I4x4) {
        for (int k = 0; k < 16; k++) {
          if (!decodable) { m.prev_i4_flag[k] = (int8_t)rnd(2); m.rem_i4_mode[k] = m.prev_i4_flag[k] ? 0 : (int8_t)rnd(8); continue; }
          const int bx = (k & 1) | ((k >> 1) & 2), by = ((k >> 1) & 1) | ((k >> 2) & 2);
          const int av = i4_avail(nbav, k);
          const bool l = av & 1, t = av & 2, tl = av & 4;
          int mode = (int)rnd(9);                                // 0 V 1 H 2 DC 3 DDL 4 DDR 5 VR 6 HD 7 VL 8 HU
          const bool need_t = mode == 0 || mode == 3 || mode == 7, need_l = mode == 1 || mode == 8;
          const bool need_all = mode == 4 || mode == 5 || mode == 6;
          if ((need_t && !t) || (need_l && !l) || (need_all && !(l && t && tl))) mode = 2;
          // predicted mode from the neighbours' final modes (DC for non-I4x4 / missing neighbours)
          auto mode_at = [&](int x, int y) -> int {            // block coordinates relative to this MB, may be -1
            int mx = mbx, my = mby;
            if (x < 0) { mx--; x += 4; }
            if (y < 0) { my--; y += 4; }
            if (mx < 0 || my < 0) return -1;
            const size_t ni = (size_t)my * W + mx;
            if (ni == mi) return i4modes[ni * 16 + y * 4 + x];
            return recs[ni].mb_type == MBT_I4x4 ? i4modes[ni * 16 + y * 4 + x] : 2;
          };
          const int lm = mode_at(bx - 1, by), tm = mode_at(bx, by - 1);
          const int pm = (lm < 0 || tm < 0) ? 2 : (lm < tm ? lm : tm);
          m.prev_i4_flag[k] = (int8_t)(mode == pm);
          m.rem_i4_mode[k] = (int8_t)(mode == pm ? 0 : (mode < pm ? mode : mode - 1));
          i4modes[mi * 16 + by * 4 + bx] = (int8_t)mode;
        }
      }
      const int nparts = m.mb_type == MBT_P16x16 ? 1 : (m.mb_type == MBT_P16x8 || m.mb_type == MBT_P8x16) ? 2 : m.mb_type == MBT_P8x8 ? 4 : 0;
      const int mr = decodable ? 300 : 2000;
      for (int k = 0; k < nparts; k++) { m.mvd[k][0] = (int16_t)((int)rnd(2 * mr + 1) - mr); m.mvd[k][1] = (int16_t)((int)rnd(401) - 200); }
      for (int k = 0; k < 16; k++) {
        if (!(cbp_l & (1 << (k >> 2)))) continue;
        const int bx = (k & 1) | ((k >> 1) & 2), by = ((k >> 1) & 1) | ((k >> 2) & 2);
        m.nnz[by * 4 + bx] = (int8_t)fill_block(m.luma[k], m.mb_type == MBT_I16x16 ? 15 : 16);
      }
      if (cbp_c) { fill_block(m.chroma_dc[0], 4); fill_block(m.chroma_dc[1], 4); }
      if (cbp_c == 2) for (int j = 0; j < 8; j++) m.nnz[16 + j] = (int8_t)fill_block(m.chroma_ac[j], 15);
      m.cbp = (uint8_t)(cbp_l | (cbp_c << 4));
      m.qp = (uint8_t)qp;
    }
    std::vector<uint8_t> au;
    ctl.write_access_unit(ctl.next_is_idr(), recs.data(), &au);
    b2h264::ParsedPicture got;
    const int rc = b2h264::parse_access_unit(au.data(), au.size(), &st, &got);
    if (rc != 0) return rc;
    if (got.mbs.size() != recs.size()) return -100;
    for (size_t i = 0; i < recs.size(); i++)
      if (!same_record(recs[i], got.mbs[i])) return 1 + (int)i;
    if (parsed) parsed->push_back(got);
    if (stream_out) {
      if (*stream_len + (long)au.size() > cap) return -200;
      memcpy(stream_out + *stream_len, au.data(), au.size());
      *stream_len += (long)au.size();
    }
  }
  return 0;
}

namespace b2h264 { extern thread_local int g_reject_line; }
extern "C" int emu_last_reject_line() { return b2h264::g_reject_line; }
