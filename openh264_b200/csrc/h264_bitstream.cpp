// h264_bitstream.cpp — see h264_bitstream.h.
#include "h264_bitstream.h"

#include <stdlib.h>
#include <string.h>

#include "cavlc_tables.h"

namespace b2h264 {

// ---- NAL encapsulation (nal_encap.cpp: start code, header byte, emulation prevention) ------------
void append_nal(std::vector<uint8_t>* dst, int nal_ref_idc, int nal_type, const std::vector<uint8_t>& rbsp) {
  // start code, header, payload with emulation prevention (7.4.1: 00 00 0x -> 00 00 03 0x for x <= 3).  Written through a pointer into
  // space sized for the worst case (every third byte an escape), cut back afterwards
  const size_t base = dst->size(), n = rbsp.size();
  dst->resize(base + 5 + n + n / 2 + 1);
  uint8_t* o = dst->data() + base;
  o[0] = 0; o[1] = 0; o[2] = 0; o[3] = 1;
  o[4] = (uint8_t)((nal_ref_idc << 5) | nal_type);
  o += 5;
  const uint8_t* in = rbsp.data();
  int zeros = 0;
  for (size_t i = 0; i < n; i++) {
    const uint8_t b = in[i];
    if (zeros >= 2 && b <= 3) { *o++ = 3; zeros = 0; }
    *o++ = b;
    zeros = b == 0 ? zeros + 1 : 0;
  }
  dst->resize((size_t)(o - dst->data()));
}

// ---- level selection -------------------------------------------------------------------------------
namespace {
struct LevelLimit { int idc; uint32_t max_mbps, max_fs, max_dpb_mbs, max_br; };
// Rec. H.264 Table A-1 (level 1b carried as idc 9 like the reference's enum)
const LevelLimit kLevels[] = {
    {10, 1485, 99, 396, 64},        {9, 1485, 99, 396, 128},         {11, 3000, 396, 900, 192},
    {12, 6000, 396, 2376, 384},     {13, 11880, 396, 2376, 768},     {20, 11880, 396, 2376, 2000},
    {21, 19800, 792, 4752, 4000},   {22, 20250, 1620, 8100, 4000},   {30, 40500, 1620, 8100, 10000},
    {31, 108000, 3600, 18000, 14000}, {32, 216000, 5120, 20480, 20000}, {40, 245760, 8192, 32768, 20000},
    {41, 245760, 8192, 32768, 50000}, {42, 522240, 8704, 34816, 50000}, {50, 589824, 22080, 110400, 135000},
    {51, 983040, 36864, 184320, 240000}, {52, 2073600, 36864, 184320, 240000}};
}  // namespace

void select_level(StreamParams* sp, float fps, int target_bitrate) {
  const uint32_t w = sp->mb_w, h = sp->mb_h, n = w * h;
  int level = 51;
  for (const LevelLimit& l : kLevels) {
    if (l.max_mbps < (uint32_t)(n * fps)) continue;
    if (l.max_fs < n) continue;
    if ((l.max_fs << 3) < w * w || (l.max_fs << 3) < h * h) continue;
    if (l.max_dpb_mbs < (uint32_t)sp->num_ref_frames * n) continue;
    if (target_bitrate != 0 && (int)l.max_br * 1200 < target_bitrate) continue;
    level = l.idc;
    break;
  }
  sp->constraint_set3 = false;
  if (level == 9) {                     // level 1b: Baseline / Main signal it as level 1.1 + constraint_set3 (au_set.cpp:530-534), High keeps 9
    if (sp->profile_idc == 66 || sp->profile_idc == 77) { level = 11; sp->constraint_set3 = true; }
  }
  sp->level_idc = level;
}

// ---- parameter sets ---------------------------------------------------------------------------------
void write_sps(const StreamParams& sp, std::vector<uint8_t>* rbsp) {
  BitWriter w(rbsp);
  // au_set.cpp:269-300: constraint_set0 for Baseline, set1 up to Main; Main / High add set4 = set5 = 1 (frame macroblocks only, no B slices);
  // High carries chroma_format_idc 1, 8-bit depths, no transform bypass, no scaling matrices
  w.put(8, (uint32_t)sp.profile_idc);
  w.bit(sp.profile_idc == 66); w.bit(sp.profile_idc <= 77); w.bit(0); w.bit(sp.constraint_set3);   // constraint_set0..3
  if (sp.profile_idc == 77 || sp.profile_idc == 100) { w.bit(1); w.bit(1); w.put(2, 0); }
  else w.put(4, 0);
  w.put(8, (uint32_t)sp.level_idc);
  w.ue((uint32_t)sp.sps_id);            // seq_parameter_set_id
  if (sp.profile_idc == 100) { w.ue(1); w.ue(0); w.ue(0); w.bit(0); w.bit(0); }
  w.ue(15 - 4);                         // log2_max_frame_num_minus4
  w.ue(2);                              // pic_order_cnt_type
  w.ue((uint32_t)sp.num_ref_frames);
  w.bit(sp.num_ref_frames != 1);        // gaps_in_frame_num_value_allowed_flag: set unless one layer has one reference (au_set.cpp:540-544)
  w.ue((uint32_t)sp.mb_w - 1);
  w.ue((uint32_t)sp.mb_h - 1);
  w.bit(1);                             // frame_mbs_only_flag
  w.bit(sp.level_idc >= 30);            // direct_8x8_inference_flag
  w.bit(sp.crop);
  if (sp.crop) { w.ue(0); w.ue((uint32_t)sp.crop_right); w.ue(0); w.ue((uint32_t)sp.crop_bottom); }
  w.bit(1);                             // vui_parameters_present_flag
  w.bit(0); w.bit(0); w.bit(0);         // aspect_ratio / overscan / video_signal_type
  w.bit(0); w.bit(0); w.bit(0); w.bit(0); w.bit(0);   // chroma_loc, timing, nal_hrd, vcl_hrd, pic_struct
  w.bit(1);                             // bitstream_restriction_flag
  w.bit(1);                             // motion_vectors_over_pic_boundaries_flag
  w.ue(0); w.ue(0); w.ue(16); w.ue(16);
  w.ue(0);                              // max_num_reorder_frames
  w.ue((uint32_t)sp.num_ref_frames);    // max_dec_frame_buffering
  w.trailing();
}

void write_pps(const StreamParams& sp, std::vector<uint8_t>* rbsp) {
  BitWriter w(rbsp);
  w.ue((uint32_t)sp.pps_id); w.ue((uint32_t)sp.sps_id);   // pps id, sps id
  w.bit(sp.entropy_cabac);              // entropy_coding_mode_flag
  w.bit(0);                             // bottom_field_pic_order_in_frame_present_flag
  w.ue(0);                              // num_slice_groups_minus1
  w.ue(0); w.ue(0);                     // num_ref_idx_l0/l1_default_active_minus1
  w.bit(0); w.put(2, 0);                // weighted_pred_flag, weighted_bipred_idc
  w.se(0); w.se(0);                     // pic_init_qp/qs - 26
  w.se(0);                              // chroma_qp_index_offset
  w.bit(1);                             // deblocking_filter_control_present_flag
  w.bit(0); w.bit(0);                   // constrained_intra_pred, redundant_pic_cnt_present
  w.trailing();
}

// ---- CAVLC residual block (Rec. H.264 9.2; reference WriteBlockResidualCavlc set_mb_syn_cavlc.cpp:109)
namespace {

inline void put_code(BitWriter& w, uint16_t packed) { w.put(packed >> 8, packed & 0xff); }

// levels: scan-ordered coefficients; max_coef = 16 (luma 4x4), 15 (AC), 4 (chroma DC); nc = -1 for chroma DC
// `active` mirrors the reference's iCalRunLevelFlag: a block whose stored non-zero count is 0 is
// written as empty even if stale levels are still in the buffer (svc_set_mb_syn_cavlc.cpp:335,353,398)
void write_block(BitWriter& w, const int16_t* lv, int max_coef, int nc, bool active = true) {
  int16_t level[16];
  uint8_t run[16];
  int total = 0, total_zeros = 0;
  int i = active ? max_coef - 1 : -1;
  while (i >= 0 && lv[i] == 0) i--;
  while (i >= 0) {
    int zeros = 0;
    level[total] = lv[i--];
    while (i >= 0 && lv[i] == 0) { zeros++; i--; }
    total_zeros += zeros;
    run[total++] = (uint8_t)zeros;
  }
  int t1 = 0;
  uint32_t signs = 0;
  for (int k = 0; k < total && k < 3; k++) {
    if (level[k] == 1 || level[k] == -1) { t1++; signs = (signs << 1) | (level[k] < 0); }
    else break;
  }
  const int cls = nc < 0 ? 4 : kNcClass[nc];
  put_code(w, kCoeffToken[cls][total][t1]);
  if (total == 0) return;
  if (t1) w.put(t1, signs);
  int suffix_len = (total > 10 && t1 < 3) ? 1 : 0;
  for (int k = t1; k < total; k++) {
    const int val = level[k];
    int code = val > 0 ? 2 * (val - 1) : -2 * val - 1;       // level_code
    if (k == t1 && t1 < 3) code -= 2;
    int prefix = code >> suffix_len, suffix_size = suffix_len, suffix = code - (prefix << suffix_len);
    if (prefix >= 14 && prefix < 30 && suffix_len == 0) {
      prefix = 14; suffix = code - 14; suffix_size = 4;
    } else if (prefix >= 15) {
      prefix = 15;
      suffix = code - (15 << suffix_len);
      if (suffix_len == 0) suffix -= 15;
      suffix_size = 12;                                    // Baseline escape (levels beyond this are not produced at the supported QPs)
    }
    w.put(prefix, 0);
    w.put(1 + suffix_size, (1u << suffix_size) | (uint32_t)suffix);
    if (suffix_len == 0) suffix_len = 1;
    if (abs(val) > (3 << (suffix_len - 1)) && suffix_len < 6) suffix_len++;
  }
  if (total < max_coef) {
    if (nc >= 0) put_code(w, kTotalZeros[total][total_zeros]);
    else put_code(w, kTotalZerosChromaDc[total][total_zeros]);
  }
  int zeros_left = total_zeros;
  for (int k = 0; k + 1 < total && zeros_left > 0; k++) {
    put_code(w, kRunBefore[zeros_left > 7 ? 7 : zeros_left][run[k]]);
    zeros_left -= run[k];
  }
}

// coded_block_pattern me(v) mapping, Rec. H.264 Table 9-4 (codeNum indexed by cbp), chroma_format_idc 1
const uint8_t kCbpIntra[48] = {3,  29, 30, 17, 31, 18, 37, 8,  32, 38, 19, 9,  20, 10, 11, 2,  16, 33, 34, 21, 35, 22, 39, 4,
                               36, 40, 23, 5,  24, 6,  7,  1,  41, 42, 43, 25, 44, 26, 46, 12, 45, 47, 27, 13, 28, 14, 15, 0};
const uint8_t kCbpInter[48] = {0,  2,  3,  7,  4,  8,  17, 13, 5,  18, 9,  14, 10, 15, 16, 11, 1,  32, 33, 36, 34, 37, 44, 40,
                               35, 45, 38, 41, 39, 42, 43, 19, 6,  24, 25, 20, 26, 21, 46, 28, 27, 47, 22, 29, 23, 30, 31, 12};

inline int nc_of(int a, int b) {          // a/b = neighbour counts or -1 when unavailable
  if (a >= 0 && b >= 0) return (a + b + 1) >> 1;
  if (a >= 0) return a;
  if (b >= 0) return b;
  return 0;
}

}  // namespace

const uint8_t* cbp_me_table(bool intra) { return intra ? kCbpIntra : kCbpInter; }

void write_slice_header(BitWriter& w, const StreamParams& sp, const SliceState& ss) {
  w.ue((uint32_t)ss.first_mb);           // first_mb_in_slice
  w.ue(ss.idr ? 2 : 0);                  // slice_type: I / P
  w.ue((uint32_t)sp.pps_id);             // pic_parameter_set_id
  w.put(15, (uint32_t)ss.frame_num);
  if (ss.idr) w.ue((uint32_t)ss.idr_pic_id);
  if (!ss.idr) {
    w.bit(1); w.ue(0);                   // num_ref_idx_active_override_flag, num_ref_idx_l0_active_minus1
    w.bit(1);                            // ref_pic_list_modification_flag_l0: one command, then 3
    w.ue((uint32_t)ss.mod_idc); w.ue((uint32_t)ss.mod_val); w.ue(3);
    w.bit(ss.n_mmco > 0);                // adaptive_ref_pic_marking_mode_flag
    for (int i = 0; i < ss.n_mmco; i++) {
      const int op = ss.mmco[i][0];
      w.ue((uint32_t)op);
      w.ue((uint32_t)ss.mmco[i][1]);     // difference_of_pic_nums_minus1 (1, 3), long_term_frame_idx (6), max_long_term_frame_idx_plus1 (4)
      if (op == 3) w.ue((uint32_t)ss.mmco[i][2]);   // long_term_frame_idx
    }
    if (ss.n_mmco > 0) w.ue(0);
    if (sp.entropy_cabac) w.ue(0);       // cabac_init_idc (SSlice::iCabacInitIdc stays 0)
  } else {
    w.bit(0); w.bit(ss.long_term_reference_flag);   // no_output_of_prior_pics_flag, long_term_reference_flag
  }
  w.se(ss.qp - 26);                      // slice_qp_delta
  w.ue((uint32_t)sp.dbk_idc);            // disable_deblocking_filter_idc; the offsets only with the filter on (svc_encode_slice.cpp:404-410)
  if (sp.dbk_idc != 1) { w.se(sp.dbk_alpha_div2); w.se(sp.dbk_beta_div2); }
}

void write_slice(const StreamParams& sp, const SliceState& ss, const MbOut* const* recs, std::vector<uint8_t>* rbsp,
                 std::vector<int32_t>* mb_bits) {
  BitWriter w(rbsp);
  write_slice_header(w, sp, ss);

  // ---- slice data ----
  const int mbw = sp.mb_w, n = sp.mb_w * sp.mb_h, first = ss.first_mb, end = ss.end_mb < 0 ? n : ss.end_mb;
  int skip_run = 0;
  int last_qp = ss.qp;
  if (mb_bits) { mb_bits->resize(n); for (int idx = first; idx < end; idx++) (*mb_bits)[idx] = 0; }
  for (int idx = first; idx < end; idx++) {
    const MbOut& m = *recs[idx];
    const int mbx = idx % mbw, mby = idx / mbw;
    if (m.mb_type == MBT_PSKIP) { skip_run++; continue; }
    if (!ss.idr) { w.ue((uint32_t)skip_run); skip_run = 0; }
    const size_t mb_start = w.bit_pos();
    const int off = ss.idr ? 0 : 5;
    const int cbp_l = m.cbp & 15, cbp_c = m.cbp >> 4;
    switch (m.mb_type) {
      case MBT_I4x4:
        w.ue((uint32_t)off);
        for (int k = 0; k < 16; k++) { w.bit(m.prev_i4_flag[k]); if (!m.prev_i4_flag[k]) w.put(3, (uint32_t)m.rem_i4_mode[k]); }
        w.ue(m.chroma_mode);
        break;
      case MBT_I16x16:
        w.ue((uint32_t)(1 + off + m.i16_mode + (cbp_c << 2) + (cbp_l ? 12 : 0)));
        w.ue(m.chroma_mode);
        break;
      case MBT_P16x16: w.ue(0); w.se(m.mvd[0][0]); w.se(m.mvd[0][1]); break;
      case MBT_P16x8:
      case MBT_P8x16:
        w.ue(m.mb_type == MBT_P16x8 ? 1 : 2);
        w.se(m.mvd[0][0]); w.se(m.mvd[0][1]); w.se(m.mvd[1][0]); w.se(m.mvd[1][1]);
        break;
      case MBT_P8x8:
        w.ue(4);                           // P_8x8ref0
        for (int k = 0; k < 4; k++) w.ue(0);   // sub_mb_type: 8x8
        for (int k = 0; k < 4; k++) { w.se(m.mvd[k][0]); w.se(m.mvd[k][1]); }
        break;
      default: break;
    }
    if (m.mb_type == MBT_I4x4) w.ue(kCbpIntra[m.cbp]);
    else if (m.mb_type != MBT_I16x16) w.ue(kCbpInter[m.cbp]);
    if (m.cbp > 0 || m.mb_type == MBT_I16x16) {
      w.se(m.qp - last_qp);
      last_qp = m.qp;
      // neighbour counts
      const int8_t* L = mbx > 0 && idx - 1 >= first ? recs[idx - 1]->nnz : nullptr;
      const int8_t* T = mby > 0 && idx - mbw >= first ? recs[idx - mbw]->nnz : nullptr;
      auto luma_nc = [&](int bx, int by) {
        const int a = bx > 0 ? m.nnz[by * 4 + bx - 1] : (L ? L[by * 4 + 3] : -1);
        const int b = by > 0 ? m.nnz[(by - 1) * 4 + bx] : (T ? T[12 + bx] : -1);
        return nc_of(a, b);
      };
      if (m.mb_type == MBT_I16x16) write_block(w, m.luma_dc, 16, luma_nc(0, 0));
      for (int k = 0; k < 16; k++) {
        if (!(cbp_l & (1 << (k >> 2)))) continue;
        const int bx = (k & 1) | ((k >> 1) & 2), by = ((k >> 1) & 1) | ((k >> 2) & 2);
        const bool act = m.nnz[by * 4 + bx] > 0;
        if (m.mb_type == MBT_I16x16) write_block(w, m.luma[k], 15, luma_nc(bx, by), act);
        else write_block(w, m.luma[k], 16, luma_nc(bx, by), act);
      }
      if (cbp_c) {
        write_block(w, m.chroma_dc[0], 4, -1);
        write_block(w, m.chroma_dc[1], 4, -1);
        if (cbp_c == 2) {
          for (int uv = 0; uv < 2; uv++)
            for (int j = 0; j < 4; j++) {
              const int bx = j & 1, by = j >> 1, base = 16 + 4 * uv;
              const int a = bx > 0 ? m.nnz[base + by * 2] : (L ? L[base + by * 2 + 1] : -1);
              const int b = by > 0 ? m.nnz[base + bx] : (T ? T[base + 2 + bx] : -1);
              write_block(w, m.chroma_ac[4 * uv + j], 15, nc_of(a, b), m.nnz[base + j] > 0);
            }
        }
      }
    }
    if (mb_bits) (*mb_bits)[idx] = (int32_t)(w.bit_pos() - mb_start);
  }
  if (skip_run) w.ue((uint32_t)skip_run);
  w.trailing();
}

}  // namespace b2h264
