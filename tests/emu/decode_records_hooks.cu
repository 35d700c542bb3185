// tests/emu/decode_records_hooks.cu — test hook of the decoder's construct stage for the host emulation build (TEST
// INFRASTRUCTURE ONLY).  Linked with emu.cu into the library tests/test_decode_records_emu.py builds.  emu_decode_records runs
// the host build of dec_one_mb in raster order on given records, with the argument layout, the refusals and the output of the
// device hook b2h264_debug_decode_records (enc_kernels.cu): the reference pictures go into picture slots 0 .. n_refs - 1 and
// get their borders replicated, the picture is decoded into slot n_refs without deblocking and its borders are replicated.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../openh264_b200/csrc/enc_frame.cuh"
#include "../../openh264_b200/csrc/dec_mb.cuh"
#include "../../openh264_b200/csrc/dec_records_check.h"
#include "../../openh264_b200/csrc/enc_host.h"

using namespace mbk;

extern "C" void b2h264_build_host_tables();
void emu_expand_frame(const EncFrameParams& p, const EncFramePtrs& f);     // emu.cu

extern "C" int emu_decode_records(int n, int mb_w, int mb_h, const int* cqp_off, const MbOut* recs, const DecMbAux* aux,
                                  const DecMbAuxB* aux_b, int n_refs, const uint8_t* refs, uint8_t* planes, MbInfo* mbi) {
  if (!dec_records_ok(n, mb_w, mb_h, cqp_off, recs, aux, aux_b, n_refs, refs, planes, mbi)) return -1;
  const int n_mb = mb_w * mb_h;
  b2h264_build_host_tables();
  const b2h264::PicLayout lay(mb_w, mb_h);
  const size_t pic_bytes = lay.bytes();
  const size_t dense = (size_t)n_mb * 384;
  std::vector<uint8_t> dpb(((size_t)n_refs + 1) * pic_bytes + 256);
  static MbScratch scratch;
  for (int s = 0; s < n; s++) {
    EncFrameParams p;
    memset(&p, 0, sizeof(p));
    p.mb_w = mb_w; p.mb_h = mb_h; p.rec_stride_y = lay.stride_y; p.rec_stride_c = lay.stride_c;
    p.mv_range = 64; p.dec_mode = 1; p.dec_cqp_off = cqp_off[s];
    EncFramePtrs f;
    memset(&f, 0, sizeof(f));
    std::fill(dpb.begin(), dpb.end(), 0);
    auto plane0 = [&](int slot, int pl) { return dpb.data() + (size_t)slot * pic_bytes + lay.plane0(pl); };
    for (int r = 0; r < n_refs; r++) {
      const uint8_t* src = refs + ((size_t)s * n_refs + r) * dense;
      for (int pl = 0; pl < 3; pl++) {
        const int w = pl ? 8 * mb_w : 16 * mb_w, h = pl ? 8 * mb_h : 16 * mb_h;
        const uint8_t* from = src + (pl ? (size_t)n_mb * 256 + (size_t)(pl - 1) * n_mb * 64 : 0);
        for (int y = 0; y < h; y++) memcpy(plane0(r, pl) + (size_t)y * lay.stride(pl), from + (size_t)y * w, w);
        f.rec[pl] = plane0(r, pl);
      }
      emu_expand_frame(p, f);
    }
    for (int pl = 0; pl < 3; pl++) { f.rec[pl] = plane0(n_refs, pl); f.ref[pl] = f.dpb0[pl] = plane0(0, pl); }
    f.dpb_stride = (int64_t)pic_bytes;
    f.mbi = mbi + (size_t)s * n_mb;
    f.dec_aux_b = aux_b ? aux_b + (size_t)s * n_mb : nullptr;
    memset(f.mbi, 0, sizeof(MbInfo) * n_mb);
    for (int y = 0; y < mb_h; y++)
      for (int x = 0; x < mb_w; x++) dec_one_mb(p, f, scratch, x, y, recs[(size_t)s * n_mb + y * mb_w + x], aux[(size_t)s * n_mb + y * mb_w + x]);
    emu_expand_frame(p, f);
    memcpy(planes + (size_t)s * pic_bytes, dpb.data() + (size_t)n_refs * pic_bytes, pic_bytes);
  }
  return 0;
}
