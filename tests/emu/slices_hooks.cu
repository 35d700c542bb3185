// tests/emu/slices_hooks.cu — host emulation build of the encoder with several slices per picture (TEST INFRASTRUCTURE ONLY).
// The macroblock code (enc_frame.cuh), the deblocking filter (enc_deblock.cuh) and the slice writers (enc_host.h) run in raster
// order on one reference picture, with the slice partition resolved by enc_slices.h and handed to the macroblock code the way
// the product does (EncFramePtrs::slice_first).  tests/test_encoder_slices_emu.py compares the output with the reference's.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#include "../../openh264_b200/csrc/enc_frame.cuh"
#include "../../openh264_b200/csrc/enc_deblock.cuh"
#include "../../openh264_b200/csrc/enc_host.h"
#include "../../openh264_b200/csrc/enc_slices.h"
#include "../../openh264_b200/csrc/h264_parse.h"

using namespace mbk;

extern "C" void b2h264_build_host_tables();
void emu_expand_frame(const EncFrameParams& p, const EncFramePtrs& f);   // emu.cu

// cfg: entropy_cabac, profile_idc, complexity_low, intra_period, loop-filter idc (as coded), alpha, beta, slice mode, slice num;
// runs: 35 uiSliceMbNum entries.  Returns the bytes written to out, -2 for a refused partition, -8 when the macroblock code's
// CAVLC bit count differs from the writer's, -7 when the decoder's parser does not read the access unit back.
extern "C" long emu_encode_slices(const uint8_t* yuv, int w, int h, int nframes, int qp, const int32_t* cfg, const uint32_t* runs,
                                  uint8_t* out, long cap, int32_t* frame_bytes, uint8_t* recon_out) {
  b2h264_build_host_tables();
  b2h264::StreamCtl ctl;
  ctl.init(w, h, qp, 30.0f, 5000000, cfg[0], cfg[1]);
  ctl.fast_mode = cfg[2] != 0;
  ctl.record_mb_bits = true;
  const int mbw = ctl.sp.mb_w, mbh = ctl.sp.mb_h, n = mbw * mbh;
  b2h264::SliceConfig sc;
  const char* why = nullptr;
  if (!b2h264::SliceConfig::resolve(cfg[7], cfg[8], runs, mbw, mbh, &sc, &why)) return -2;
  std::vector<int32_t> first(sc.slices() + 1), per_mb(n);
  sc.starts(n, first.data());
  for (int k = 0; k < sc.slices(); k++) for (int i = first[k]; i < first[k + 1]; i++) per_mb[i] = first[k];
  if (sc.slices() > 1) ctl.slice_first.assign(first.begin(), first.end() - 1);
  if (!ctl.set_loop_filter(cfg[4], cfg[5], cfg[6])) return -2;
  const b2h264::PicLayout lay(mbw, mbh);
  std::vector<uint8_t> cur((size_t)n * 384 + 64), prev_y((size_t)n * 256 + 64, 0), pic[2];
  for (auto& b : pic) b.assign(lay.bytes() + 64, 0);
  std::vector<MbInfo> mbi(n);
  std::vector<RefMbInfo> rinfo[2] = {std::vector<RefMbInfo>(n), std::vector<RefMbInfo>(n)};
  std::vector<MbOut> recs(n);
  std::vector<int32_t> sad(n, 0), bits(n, 0), vaa((size_t)n * 4, 0);
  static MbScratch scratch;
  memset(&scratch, 0, sizeof(scratch));
  b2h264::ParserState parser;
  int cur_rec = 0, p_since_idr = 0;
  bool have_ref_p = false;
  long total = 0;
  const size_t fsz = (size_t)w * h * 3 / 2;
  for (int i = 0; i < nframes; i++) {
    uint8_t* cy = cur.data();
    b2h264::pad_source(yuv + i * fsz, w, h, mbw, mbh, cy, cy + (size_t)n * 256, cy + (size_t)n * 320);
    const bool idr = ctl.next_is_idr() || (cfg[3] > 0 && 1 + p_since_idr >= cfg[3]);
    p_since_idr = idr ? 0 : p_since_idr + 1;
    const EncFrameParams p = ctl.frame_params(idr, have_ref_p);
    if (ctl.fast_mode)                         // VAACalcSad_c: 8x8 SADs against the previous source picture
      for (int mb = 0; mb < n; mb++)
        for (int k = 0; k < 4; k++) {
          const size_t o = (size_t)((mb / mbw) * 16 + (k >> 1) * 8) * mbw * 16 + (mb % mbw) * 16 + (k & 1) * 8;
          int s = 0;
          for (int y = 0; y < 8; y++) for (int x = 0; x < 8; x++) s += abs((int)cy[o + y * mbw * 16 + x] - (int)prev_y[o + y * mbw * 16 + x]);
          vaa[(size_t)mb * 4 + k] = s;
        }
    EncFramePtrs f;
    memset(&f, 0, sizeof(f));
    f.cur[0] = cy; f.cur[1] = cy + (size_t)n * 256; f.cur[2] = cy + (size_t)n * 320;
    for (int pl = 0; pl < 3; pl++) { f.rec[pl] = pic[cur_rec].data() + lay.plane0(pl); f.ref[pl] = pic[1 - cur_rec].data() + lay.plane0(pl); }
    f.mbi = mbi.data(); f.rec_info = rinfo[cur_rec].data(); f.ref_info = rinfo[1 - cur_rec].data(); f.out = recs.data();
    f.sad_cost = sad.data(); f.mb_bits = bits.data(); f.vaa_sad8x8 = vaa.data(); f.prev_luma = prev_y.data();
    f.slice_first = sc.slices() > 1 ? per_mb.data() : nullptr;
    for (int mby = 0; mby < mbh; mby++)
      for (int mbx = 0; mbx < mbw; mbx++) {
        mb_ctx(scratch.ctx, p, f, mbx, mby);
        for (int stage = idr ? MBS_I : MBS_A; stage != MBS_DONE;) stage = mb_run_stage(scratch.ctx, scratch, stage);
      }
    static DbkTile tile;
    for (int mby = 0; mby < mbh; mby++)
      for (int mbx = 0; mbx < mbw; mbx++) deblock_one_mb(p, f, mbx, mby, tile);
    emu_expand_frame(p, f);
    std::vector<uint8_t> au;
    ctl.write_access_unit(idr, recs.data(), &au);
    if (!ctl.sp.entropy_cabac && ctl.last_mb_bits != bits) return -8;
    b2h264::ParsedPicture parsed;
    if (b2h264::parse_access_unit(au.data(), au.size(), &parser, &parsed) != 0 || (int)parsed.mbs.size() != n) return -7;
    for (int mb = 0; mb < n; mb++)
      if (parsed.mbs[mb].mb_type != recs[mb].mb_type || (recs[mb].mb_type != MBT_PSKIP && parsed.mbs[mb].cbp != recs[mb].cbp)) return -7;
    if (total + (long)au.size() > cap) return -1;
    memcpy(out + total, au.data(), au.size());
    total += (long)au.size();
    if (frame_bytes) frame_bytes[i] = (int32_t)au.size();
    if (recon_out)
      for (int pl = 0; pl < 3; pl++) {
        const int pw = pl ? w / 2 : w, ph = pl ? h / 2 : h;
        for (int y = 0; y < ph; y++) memcpy(recon_out + i * fsz + (pl ? (size_t)w * h + (pl - 1) * (size_t)pw * ph : 0) + (size_t)y * pw,
                                            f.rec[pl] + (size_t)y * lay.stride(pl), pw);
      }
    memcpy(prev_y.data(), cy, (size_t)n * 256);
    have_ref_p = !idr;
    cur_rec = 1 - cur_rec;
  }
  return total;
}
