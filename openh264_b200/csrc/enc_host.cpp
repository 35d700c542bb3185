// enc_host.cpp — see enc_host.h.
#include "enc_host.h"

#include <stddef.h>
#include <string.h>

namespace b2h264 {

void StreamCtl::init(int width, int height, int qp, float fps_, int target_bitrate, int entropy_cabac, int profile_idc) {
  memset(&sp, 0, sizeof(sp));
  // WelsEncoderApplyProfile... (encoder_ext.cpp:650-668): CAVLC -> Baseline; CABAC -> High unless the layer asks for Main
  // the reference's resolution of (iEntropyCodingModeFlag, uiProfileIdc) for spatial layer 0: profiles other than Baseline / Main /
  // High count as unspecified (encoder_ext.cpp:126-141), Baseline turns CABAC off, unspecified becomes High with CABAC and
  // Baseline without (encoder_ext.cpp:652-664)
  if (profile_idc != 66 && profile_idc != 77 && profile_idc != 100) profile_idc = 0;
  sp.entropy_cabac = entropy_cabac != 0 && profile_idc != 66;
  sp.profile_idc = profile_idc ? profile_idc : (sp.entropy_cabac ? 100 : 66);
  sp.width = width; sp.height = height;
  sp.mb_w = (width + 15) >> 4; sp.mb_h = (height + 15) >> 4;
  sp.num_ref_frames = 1;
  sp.qp = qp;
  fps = fps_;
  select_level(&sp, fps_, target_bitrate);
  // WelsGetPaddingOffset (au_set.cpp:476): crop offsets in units of 2 luma samples, right/bottom only
  sp.crop = (sp.mb_w * 16 != width) || (sp.mb_h * 16 != height);
  sp.crop_right = (sp.mb_w * 16 - width) / 2;
  sp.crop_bottom = (sp.mb_h * 16 - height) / 2;
  frame_num = 0; idr_pic_id = 0; frames_coded = 0; force_idr = true; parasets_written = 0;
}

EncFrameParams StreamCtl::frame_params(bool idr, bool ref_is_p) const {
  EncFrameParams p;
  memset(&p, 0, sizeof(p));
  p.mb_w = sp.mb_w; p.mb_h = sp.mb_h;
  p.cur_stride_y = sp.mb_w * 16; p.cur_stride_c = sp.mb_w * 8;
  p.rec_stride_y = rec_stride_y(); p.rec_stride_c = rec_stride_c();
  p.qp = sp.qp;
  p.is_idr = idr;
  // GetMvMvdRange (encoder_ext.cpp:1508): min(level vertical MV limit / 4, CAMERA_STARTMV_RANGE = 64)
  p.mv_range = sp.level_idc <= 10 ? 63 : 64;
  p.ref_is_p = ref_is_p;
  p.fast_mode = fast_mode ? 1 : 0;
  p.dbk_idc = sp.dbk_idc; p.dbk_off_a = 2 * sp.dbk_alpha_div2; p.dbk_off_b = 2 * sp.dbk_beta_div2;
  return p;
}

void StreamCtl::write_access_unit(bool idr, const MbOut* mbs, std::vector<uint8_t>* au) {
  const int n = sp.mb_w * sp.mb_h;
  recs_.resize(n);
  for (int i = 0; i < n; i++) recs_[i] = mbs + i;
  write_au(idr, recs_.data(), au);
}

int pack_records_compact(const MbOut* mbs, int n, uint8_t* dst, int32_t* idx) {
  size_t at = 0;
  for (int i = 0; i < n; i++) {
    const MbOut& m = mbs[i];
    if (m.mb_type == MBT_PSKIP) { idx[i] = -1 - (int32_t)m.qp; continue; }
    idx[i] = (int32_t)(at / 32);
    uint8_t* head = dst + at;
    memcpy(head, &m, offsetof(MbOut, luma));
    memcpy(head + offsetof(MbOut, luma), m.chroma_dc, sizeof(m.chroma_dc));
    at += 128;
    unsigned mask = 0;
    for (int b = 0; b < 24; b++) {
      const bool want = m.mb_type == MBT_IPCM ? true
                        : b < 16 ? (m.mb_type == MBT_I16x16 ? (m.cbp & 15) != 0 : ((m.cbp >> (b >> 2)) & 1) != 0) : (m.cbp >> 4) == 2;
      if (!want) continue;
      const int16_t* blk = b < 16 ? m.luma[b] : m.chroma_ac[b - 16];
      bool nz = false;
      for (int q = 0; q < 16; q++) nz |= blk[q] != 0;
      if (!nz) continue;
      mask |= 1u << b;
      memcpy(dst + at, blk, 32);
      at += 32;
    }
    head[5] = (uint8_t)mask; head[6] = (uint8_t)(mask >> 8); head[7] = (uint8_t)(mask >> 16);
  }
  return (int)(at / 32);
}

// compact records (enc_kernels.cu: k_pack_records): idx[mb] = offset in 32-byte units or -1; 128-byte head
// (MbOut bytes [0, 112) + chroma_dc, presence mask of the 24 residual blocks in pad0) + 32 bytes per present block
void StreamCtl::write_access_unit_packed(bool idr, const MbOut* packed, const int32_t* idx, std::vector<uint8_t>* au,
                                         const RefDecision* refs) {
  static const MbOut kSkip = [] { MbOut m; memset(&m, 0, sizeof(m)); m.mb_type = MBT_PSKIP; return m; }();
  const int n = sp.mb_w * sp.mb_h;
  recs_.resize(n);
  int coded = 0;
  for (int i = 0; i < n; i++) coded += idx[i] >= 0;
  expand_.resize(coded);
  last_coded_mbs = coded;
  const uint8_t* base = reinterpret_cast<const uint8_t*>(packed);
  int k = 0;
  for (int i = 0; i < n; i++) {
    if (idx[i] < 0) { recs_[i] = &kSkip; continue; }
    const uint8_t* r = base + (size_t)idx[i] * 32;
    MbOut& m = expand_[k++];
    memcpy(&m, r, offsetof(MbOut, luma));
    memcpy(m.chroma_dc, r + offsetof(MbOut, luma), sizeof(m.chroma_dc));
    const unsigned mask = (unsigned)m.pad0[0] | ((unsigned)m.pad0[1] << 8) | ((unsigned)m.pad0[2] << 16);
    memset(m.pad0, 0, sizeof(m.pad0));
    memset(m.luma, 0, sizeof(m.luma));
    memset(m.chroma_ac, 0, sizeof(m.chroma_ac));
    const uint8_t* blk = r + 128;
    for (int b = 0; b < 24; b++)
      if ((mask >> b) & 1) { memcpy(b < 16 ? m.luma[b] : m.chroma_ac[b - 16], blk, 32); blk += 32; }
    recs_[i] = &m;
  }
  write_au(idr, recs_.data(), au, refs);
}

void StreamCtl::write_au(bool idr, const MbOut* const* mbs, std::vector<uint8_t>* au, const RefDecision* refs) {
  std::vector<uint8_t>& rbsp = rbsp_;             // kept between pictures: its capacity settles at the stream's picture size
  rbsp.clear();
  if (idr) {
    idr_pic_id = refs ? refs->idr_pic_id : (idr_pic_id < 65535 ? idr_pic_id + 1 : 0);
    frame_num = 0;
    if (increasing_ids) { sp.sps_id = parasets_written % 32; sp.pps_id = parasets_written % 57; }
    parasets_written++;
    write_sps(sp, &rbsp); append_nal(au, 3, 7, rbsp); rbsp.clear();
    write_pps(sp, &rbsp); append_nal(au, 3, 8, rbsp); rbsp.clear();
  }
  SliceState ss;
  if (refs) frame_num = refs->frame_num;          // the reference state numbers the pictures it decided (enc_refs.h)
  ss.idr = idr; ss.frame_num = frame_num; ss.idr_pic_id = idr_pic_id; ss.qp = sp.qp;
  if (refs) {
    ss.mod_idc = refs->mod_idc; ss.mod_val = refs->mod_val;
    ss.long_term_reference_flag = refs->long_term_reference_flag;
    ss.n_mmco = refs->n_mmco;
    memcpy(ss.mmco, refs->mmco, sizeof(ss.mmco));
  }
  const int n_slices = slice_first.size() < 2 ? 1 : (int)slice_first.size();
  for (int k = 0; k < n_slices; k++) {            // every slice repeats the header fields, dec_ref_pic_marking included
    ss.first_mb = n_slices > 1 ? slice_first[k] : 0;
    ss.end_mb = k + 1 < n_slices ? slice_first[k + 1] : -1;
    rbsp.clear();
    if (sp.entropy_cabac) write_slice_cabac(sp, ss, mbs, &rbsp);
    else write_slice(sp, ss, mbs, &rbsp, record_mb_bits ? &last_mb_bits : nullptr);
    append_nal(au, 3, idr ? 5 : 1, rbsp);
  }
  frame_num = (frame_num + 1) & 0x7fff;
  frames_coded++;
  force_idr = false;
}

void pad_source(const uint8_t* yuv, int w, int h, int mb_w, int mb_h, uint8_t* y, uint8_t* u, uint8_t* v) {
  const int W = mb_w * 16, H = mb_h * 16, cw = w / 2, ch = h / 2, CW = W / 2, CH = H / 2;
  const uint8_t* sy = yuv;
  const uint8_t* su = yuv + (size_t)w * h;
  const uint8_t* sv = su + (size_t)cw * ch;
  for (int r = 0; r < H; r++) {
    if (r < h) { memcpy(y + (size_t)r * W, sy + (size_t)r * w, w); memset(y + (size_t)r * W + w, 0, W - w); }
    else memset(y + (size_t)r * W, 0, W);
  }
  for (int r = 0; r < CH; r++) {
    if (r < ch) {
      memcpy(u + (size_t)r * CW, su + (size_t)r * cw, cw); memset(u + (size_t)r * CW + cw, 0x80, CW - cw);
      memcpy(v + (size_t)r * CW, sv + (size_t)r * cw, cw); memset(v + (size_t)r * CW + cw, 0x80, CW - cw);
    } else { memset(u + (size_t)r * CW, 0x80, CW); memset(v + (size_t)r * CW, 0x80, CW); }
  }
}

}  // namespace b2h264
