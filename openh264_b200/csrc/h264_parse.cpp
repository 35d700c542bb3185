// h264_parse.cpp — see h264_parse.h.  Syntax: Rec. H.264 7.3 (NAL, SPS 7.3.2.1, PPS 7.3.2.2, slice header 7.3.3,
// slice data 7.3.4, macroblock layer 7.3.5, residual CAVLC 7.3.5.3.2 / 9.2).  The reference's counterparts:
// codec/decoder/core/src/au_parser.cpp (ParseSps :~900, ParsePps), decode_slice.cpp (ParseSliceHeaderSyntaxes),
// parse_mb_syn_cavlc.cpp (WelsResidualBlockCavlc :~700, ParseInterInfo, ParseIntra4x4Mode).
#include "h264_parse.h"

#include <stddef.h>
#include <string.h>

#include <algorithm>


#include "cavlc_tables.h"
#include "h264_cabac_dec.h"
#include "h264_motion.h"

namespace b2h264 {

thread_local int g_reject_line = 0;      // source line of the last rejection (diagnostics: why a stream is outside the supported class)

namespace {
#define PARSE_UNSUPPORTED (g_reject_line = __LINE__, b2h264::PARSE_UNSUPPORTED)
#define PARSE_INVALID (g_reject_line = __LINE__, b2h264::PARSE_INVALID)


class BitReader {
 public:
  BitReader(const uint8_t* p, size_t n) : p_(p), nbytes_(n), nbits_(n * 8) {}
  bool ok() const { return !err_; }
  size_t pos() const { return pos_; }
  size_t left() const { return pos_ <= nbits_ ? nbits_ - pos_ : 0; }
  uint32_t peek(int n) const {            // n <= 32; bits beyond the end read as 0
    if (n <= 0) return 0;
    return (uint32_t)(window() >> (64 - n));
  }
  void skip(int n) { pos_ += n; if (pos_ > nbits_) err_ = true; }
  uint32_t get(int n) { const uint32_t v = peek(n); skip(n); return v; }
  int bit() { return (int)get(1); }
  // number of leading zero bits in the next 32 (32 if none is set)
  int leading_zeros() const { const uint32_t v = peek(32); return v ? __builtin_clz(v) : 32; }
  uint32_t ue() {
    const int z = leading_zeros();
    if (z > 31 || (size_t)(2 * z + 1) > left()) { err_ = true; pos_ = nbits_ + 1; return 0; }
    skip(z + 1);
    return z ? ((1u << z) - 1 + get(z)) : 0;
  }
  int32_t se() { const uint32_t k = ue(); return (k & 1) ? (int32_t)((k + 1) >> 1) : -(int32_t)(k >> 1); }
  // 7.2 more_rbsp_data(): anything before the final stop bit?
  bool more_data() const {
    if (left() == 0) return false;
    if (last_one_ == 0) {                   // index after the stop bit, found once (the payload does not change)
      size_t last = nbits_;
      while (last > 0 && !((p_[(last - 1) >> 3] >> (7 - ((last - 1) & 7))) & 1)) last--;
      last_one_ = last + 1;                 // + 1: 0 means "not computed"
    }
    return last_one_ - 1 > pos_ + 1;
  }
 private:
  // the next 64 bits, left aligned (at least 57 of them valid), zero beyond the end
  uint64_t window() const {
    const size_t byte = pos_ >> 3;
    uint64_t v = 0;
    if (byte + 8 <= nbytes_) {
      memcpy(&v, p_ + byte, 8);
      v = __builtin_bswap64(v);
    } else {
      for (size_t i = 0; i < 8; i++) v = (v << 8) | (byte + i < nbytes_ ? p_[byte + i] : 0);
    }
    return v << (pos_ & 7);
  }
  const uint8_t* p_;
  size_t nbytes_, nbits_, pos_ = 0;
  mutable size_t last_one_ = 0;
  bool err_ = false;
};

struct Nal { int ref_idc, type; std::vector<uint8_t> rbsp; };

// splits an Annex-B buffer into NAL units and strips the emulation prevention bytes (7.4.1)
std::vector<Nal> split_nals(const uint8_t* d, size_t n) {
  std::vector<Nal> out;
  size_t i = 0;
  auto start_at = [&](size_t k) { return k + 2 < n && d[k] == 0 && d[k + 1] == 0 && d[k + 2] == 1; };
  while (i + 3 <= n && !start_at(i)) i++;
  while (i + 3 <= n) {
    i += 3;                                                 // past 00 00 01
    size_t e = i;
    while (e + 3 <= n && !start_at(e)) e++;
    size_t end = e + 3 <= n ? e : n;
    if (e + 3 <= n && end > i && d[end - 1] == 0) end--;    // the zero_byte of a 4-byte start code belongs to the next NAL
    if (end > i) {
      Nal u;
      u.ref_idc = (d[i] >> 5) & 3; u.type = d[i] & 31;
      int zeros = 0;
      for (size_t k = i + 1; k < end; k++) {
        if (zeros >= 2 && d[k] == 3) { zeros = 0; continue; }
        u.rbsp.push_back(d[k]);
        zeros = d[k] == 0 ? zeros + 1 : 0;
      }
      out.push_back(std::move(u));
    }
    i = e;
  }
  return out;
}

void activate_sps(ParserState* st, int id) {
  const SpsFields& f = st->sps_tab[id];
  const int pps_id = st->sp.pps_id, qp = st->sp.qp;
  st->sp = f.sp; st->sp.pps_id = pps_id; st->sp.qp = qp;
  st->log2_max_frame_num = f.log2_max_frame_num; st->poc_type = f.poc_type; st->log2_max_poc_lsb = f.log2_max_poc_lsb;
  st->delta_pic_order_always_zero = f.delta_pic_order_always_zero;
  st->n_slots = f.n_slots; st->crop_left = f.crop_left; st->crop_top = f.crop_top;
  st->profile = f.profile; st->direct_8x8_inference = f.direct_8x8_inference;
  st->have_sps = true;
}

int parse_sps(BitReader& r, ParserState* st) {
  const int profile = (int)r.get(8);
  const int flags = (int)r.get(8);            // constraint flags + reserved
  const int level = (int)r.get(8);
  const int sps_id = (int)r.ue();
  if (sps_id < 0 || sps_id > 31) return PARSE_INVALID;
  // Baseline, Main, Extended streams that declare Baseline conformance (constraint_set0_flag), High in its 4:2:0 8-bit form
  // without scaling lists.  Tools outside the supported class (B slices, weighted prediction, interlace, the 8x8 transform, data
  // partitioning) are rejected where they show up: slice type, PPS flags, frame_mbs_only_flag, NAL types 2..4.
  if (!(profile == 66 || profile == 77 || profile == 100 || (profile == 88 && (flags & 0x80)))) return PARSE_UNSUPPORTED;
  if (profile == 100) {
    if (r.ue() != 1) return PARSE_UNSUPPORTED;                // chroma_format_idc
    if (r.ue() != 0 || r.ue() != 0) return PARSE_UNSUPPORTED; // bit_depth_luma_minus8, bit_depth_chroma_minus8
    if (r.bit()) return PARSE_UNSUPPORTED;                    // qpprime_y_zero_transform_bypass_flag
    if (r.bit()) return PARSE_UNSUPPORTED;                    // seq_scaling_matrix_present_flag
  }
  SpsFields f;
  {
    const uint32_t v = r.ue();
    if (v > 12) return PARSE_INVALID;                     // log2_max_frame_num_minus4 in 0..12 (7.4.2.1.1)
    f.log2_max_frame_num = (int)v + 4;
  }
  f.poc_type = (int)r.ue();
  if (f.poc_type == 0) {
    const uint32_t v = r.ue();
    if (v > 12) return PARSE_INVALID;
    f.log2_max_poc_lsb = (int)v + 4;
  } else if (f.poc_type == 1) {
    // picture order count type 1 (7.3.2.1.1): only parsed — pictures leave the decoder in decoding order (no B slices in this
    // stream class, so that is also the output order)
    f.delta_pic_order_always_zero = r.bit() != 0;
    r.se(); r.se();                                       // offset_for_non_ref_pic, offset_for_top_to_bottom_field
    const uint32_t n_cycle = r.ue();
    if (n_cycle > 255) return PARSE_INVALID;
    for (uint32_t i = 0; i < n_cycle; i++) r.se();
  } else if (f.poc_type != 2) return PARSE_INVALID;
  StreamParams sp;
  memset(&sp, 0, sizeof(sp));
  sp.num_ref_frames = (int)r.ue();
  r.bit();                                    // gaps_in_frame_num_value_allowed_flag
  sp.mb_w = (int)r.ue() + 1;
  sp.mb_h = (int)r.ue() + 1;
  if (!r.bit()) return PARSE_UNSUPPORTED;     // frame_mbs_only_flag
  f.direct_8x8_inference = r.bit() != 0;      // direct_8x8_inference_flag
  f.profile = profile;
  sp.crop = r.bit() != 0;
  int cl = 0, ct = 0;
  if (sp.crop) {
    const uint32_t a = r.ue(), b = r.ue(), c = r.ue(), e = r.ue();
    if (a > 4096 || b > 4096 || c > 4096 || e > 4096) return PARSE_INVALID;
    cl = (int)a; sp.crop_right = (int)b; ct = (int)c; sp.crop_bottom = (int)e;
  }
  if (!r.ok()) return PARSE_TRUNCATED;
  if (sp.mb_w < 1 || sp.mb_h < 1 || sp.mb_w > 512 || sp.mb_h > 512 || sp.num_ref_frames > 16) return PARSE_INVALID;
  sp.width = sp.mb_w * 16 - 2 * (cl + sp.crop_right);
  sp.height = sp.mb_h * 16 - 2 * (ct + sp.crop_bottom);
  if (sp.width < 2 || sp.height < 2) return PARSE_INVALID;
  sp.level_idc = level;
  sp.sps_id = sps_id;
  f.sp = sp;
  f.crop_left = cl; f.crop_top = ct;          // the picture is decoded whole; the output skips 2 * crop samples at the left / top
  f.n_slots = sp.num_ref_frames + 1 < 2 ? 2 : sp.num_ref_frames + 1;
  f.valid = true;                             // VUI (if any) is not needed for reconstruction
  st->sps_tab[sps_id] = f;
  if (!st->have_sps || st->sp.sps_id == sps_id) activate_sps(st, sps_id);
  return PARSE_OK;
}

void activate_pps(ParserState* st, int id) {
  const PpsFields& f = st->pps_tab[id];
  st->pic_init_qp = f.pic_init_qp; st->deblocking_control = f.deblocking_control; st->num_ref_idx_default = f.num_ref_idx_default;
  st->constrained_intra_pred = f.constrained_intra_pred;
  st->entropy_cabac = f.entropy_cabac;
  st->num_ref_idx_l1_default = f.num_ref_idx_l1_default; st->weighted_bipred_idc = f.weighted_bipred_idc;
  st->chroma_qp_offset = f.chroma_qp_offset; st->transform_8x8 = f.transform_8x8; st->weighted_pred = f.weighted_pred;
  st->sp.pps_id = id;
  st->have_pps = true;
}

int parse_pps(BitReader& r, ParserState* st) {
  const int pps_id = (int)r.ue();
  const int sps_id = (int)r.ue();
  if (pps_id < 0 || pps_id > 255 || sps_id < 0 || sps_id > 31) return PARSE_INVALID;
  PpsFields f;
  f.sps_id = sps_id;
  f.entropy_cabac = r.bit() != 0;             // entropy_coding_mode_flag
  const int bottom_field_poc = r.bit();
  if (r.ue() != 0) return PARSE_UNSUPPORTED;  // slice groups
  f.num_ref_idx_default = (int)r.ue() + 1;
  f.num_ref_idx_l1_default = (int)r.ue() + 1;
  f.weighted_pred = r.bit() != 0;             // weighted_pred_flag: explicit weights in P slices
  f.weighted_bipred_idc = (int)r.get(2);      // 1: explicit weights in B slices, 2: implicit
  if (f.weighted_bipred_idc == 3) return PARSE_INVALID;
  f.pic_init_qp = 26 + r.se();
  r.se();
  f.chroma_qp_offset = r.se();                // chroma_qp_index_offset
  if (f.chroma_qp_offset < -12 || f.chroma_qp_offset > 12) return PARSE_INVALID;
  f.deblocking_control = r.bit() != 0;
  f.constrained_intra_pred = r.bit() != 0;
  if (r.bit()) return PARSE_UNSUPPORTED;      // redundant_pic_cnt_present_flag
  if (bottom_field_poc) return PARSE_UNSUPPORTED;
  if (!r.ok()) return PARSE_TRUNCATED;
  if (r.more_data()) {                        // High profile tail (7.3.2.2)
    f.transform_8x8 = r.bit() != 0;           // transform_8x8_mode_flag
    if (r.bit()) return PARSE_UNSUPPORTED;    // pic_scaling_matrix_present_flag
    if (r.se() != f.chroma_qp_offset) return PARSE_UNSUPPORTED;   // second_chroma_qp_index_offset: one offset for both chroma planes
    if (!r.ok()) return PARSE_TRUNCATED;
  }
  f.valid = true;
  st->pps_tab[pps_id] = f;
  if (st->sps_tab[sps_id].valid && (!st->have_pps || st->sp.pps_id == pps_id)) { activate_sps(st, sps_id); activate_pps(st, pps_id); }
  return PARSE_OK;
}

// ---- residual block (9.2): the inverse of write_block() ------------------------------------------------------------
// Decoding tables built once from the writer's code tables (cavlc_tables.h; entry = (bits << 8) | codeword), so that a symbol
// costs one look-up instead of a search:
//  * coeff_token: codes of up to 16 bits whose codeword has at most 8 significant bits -> per table class and per count of
//    leading zeros, 128 entries indexed by the 7 bits that follow the first 1 bit;
//  * total_zeros / run_before: short codes (<= 9 / <= 11 bits) -> one table per context indexed by the next 9 / 11 bits.
// entry = (bits << 8) | symbol, 0 = no code.
struct VlcTables {
  uint16_t coeff[3][16][128];
  uint16_t coeff_flc[64], coeff_dc[256];                // nC >= 8 (6-bit fixed length) and chroma DC (<= 8 bits): these two have an all-zero code
  uint16_t tz[16][512];
  uint16_t tz_dc[4][8];
  uint16_t run[8][2048];
  VlcTables() {
    memset(this, 0, sizeof(*this));
    for (int cls = 0; cls < 3; cls++)
      for (int t = 0; t <= 16; t++)
        for (int o = 0; o < 4 && o <= t; o++) {
          const int bits = kCoeffToken[cls][t][o] >> 8, code = kCoeffToken[cls][t][o] & 0xff;
          if (!bits || !code) continue;
          int sig = 0;
          while ((code >> sig) != 0) sig++;               // significant bits of the codeword
          const int z = bits - sig, r = sig - 1;          // leading zeros; bits after the first 1
          const int first = (code & ((1 << r) - 1)) << (7 - r);
          for (int k = 0; k < (1 << (7 - r)); k++) coeff[cls][z][first + k] = (uint16_t)((bits << 8) | (t * 4 + o));
        }
    for (int t = 0; t <= 16; t++)
      for (int o = 0; o < 4 && o <= t; o++)
        for (int cls = 3; cls < 5; cls++) {
          const int bits = kCoeffToken[cls][t][o] >> 8, code = kCoeffToken[cls][t][o] & 0xff, width = cls == 3 ? 6 : 8;
          if (!bits) continue;
          uint16_t* tab = cls == 3 ? coeff_flc : coeff_dc;
          for (int k = 0; k < (1 << (width - bits)); k++) tab[(code << (width - bits)) + k] = (uint16_t)((bits << 8) | (t * 4 + o));
        }
    auto fill = [](uint16_t* tab, int width, const uint16_t* codes, int n) {
      for (int i = 0; i < n; i++) {
        const int bits = codes[i] >> 8, code = codes[i] & 0xff;
        if (!bits) continue;
        const int first = code << (width - bits);
        for (int k = 0; k < (1 << (width - bits)); k++) tab[first + k] = (uint16_t)((bits << 8) | i);
      }
    };
    for (int t = 1; t < 16; t++) fill(tz[t], 9, kTotalZeros[t], 16);
    for (int t = 1; t < 4; t++) fill(tz_dc[t], 3, kTotalZerosChromaDc[t], 4);
    for (int t = 1; t < 8; t++) fill(run[t], 11, kRunBefore[t], 15);
  }
};
const VlcTables& vlc_tables() {
  static const VlcTables t;                              // thread-safe one-time build (streams are parsed on several threads)
  return t;
}

// reads one block into lv[0..max_coef) (scan order); returns total_coeff or a negative ParseError
int read_block(BitReader& r, int16_t* lv, int max_coef, int nc) {
  const VlcTables& V = vlc_tables();
  for (int i = 0; i < max_coef; i++) lv[i] = 0;
  const int cls = nc < 0 ? 4 : kNcClass[nc > 16 ? 16 : nc];
  int total, t1;
  {
    uint16_t e;
    if (cls == 3) e = V.coeff_flc[r.peek(6)];
    else if (cls == 4) e = V.coeff_dc[r.peek(8)];
    else {
      const uint32_t look = r.peek(32);
      const int z = look ? __builtin_clz(look) : 32;
      if (z > 15) return PARSE_INVALID;
      e = V.coeff[cls][z][(uint32_t)(look << (z + 1)) >> 25];
    }
    if (!e) return PARSE_INVALID;
    r.skip(e >> 8);
    total = (e & 0xff) >> 2; t1 = e & 3;
  }
  if (total > max_coef) return PARSE_INVALID;
  if (total == 0) return 0;
  int level[16];
  if (t1) {
    const uint32_t signs = r.get(t1);
    for (int k = 0; k < t1; k++) level[k] = ((signs >> (t1 - 1 - k)) & 1) ? -1 : 1;
  }
  int suffix_len = (total > 10 && t1 < 3) ? 1 : 0;
  for (int k = t1; k < total; k++) {
    const int prefix = r.leading_zeros();
    if (prefix > 31 || (size_t)prefix >= r.left()) return PARSE_INVALID;
    r.skip(prefix + 1);
    int suffix_size = (prefix == 14 && suffix_len == 0) ? 4 : (prefix >= 15 ? prefix - 3 : suffix_len);
    int code = ((prefix < 15 ? prefix : 15) << suffix_len) + (suffix_size ? (int)r.get(suffix_size) : 0);
    if (prefix >= 15 && suffix_len == 0) code += 15;
    if (prefix >= 16) code += (1 << (prefix - 3)) - 4096;
    if (k == t1 && t1 < 3) code += 2;
    level[k] = (code & 1) ? (-code - 1) >> 1 : (code + 2) >> 1;
    if (suffix_len == 0) suffix_len = 1;
    const int a = level[k] < 0 ? -level[k] : level[k];
    if (a > (3 << (suffix_len - 1)) && suffix_len < 6) suffix_len++;
  }
  int zeros_left = 0;
  if (total < max_coef) {
    const uint16_t e = nc >= 0 ? V.tz[total][r.peek(9)] : V.tz_dc[total][r.peek(3)];
    if (!e) return PARSE_INVALID;
    r.skip(e >> 8);
    zeros_left = e & 0xff;
  }
  int run[16];
  for (int k = 0; k < total; k++) run[k] = 0;
  for (int k = 0; k + 1 < total && zeros_left > 0; k++) {
    const uint16_t e = V.run[zeros_left > 7 ? 7 : zeros_left][r.peek(11)];
    if (!e) return PARSE_INVALID;
    r.skip(e >> 8);
    const int rb = e & 0xff;
    if (rb > zeros_left) return PARSE_INVALID;
    run[k] = rb;
    zeros_left -= rb;
  }
  run[total - 1] = zeros_left;
  int pos = -1;
  for (int k = total - 1; k >= 0; k--) {
    pos += run[k] + 1;
    if (pos >= max_coef) return PARSE_INVALID;
    lv[pos] = (int16_t)level[k];
  }
  if (!r.ok()) return PARSE_TRUNCATED;
  return total;
}

inline int nc_of(int a, int b) {
  if (a >= 0 && b >= 0) return (a + b + 1) >> 1;
  if (a >= 0) return a;
  if (b >= 0) return b;
  return 0;
}

// a skipped macroblock: header bytes and chroma DC cleared (levels of such a record are never read), type P_SKIP
static inline void reset_skip_record(MbOut* m) {
  memset(m, 0, offsetof(MbOut, luma));
  memset(m->chroma_dc, 0, sizeof(m->chroma_dc));
  m->mb_type = MBT_PSKIP;
}

// inverse of the me(v) mapping of coded_block_pattern (Table 9-4): built from the writer's table
int cbp_from_code(int code, bool intra) {
  struct Inv { uint8_t t[2][48]; };
  static const Inv inv_s = [] {                      // thread-safe one-time build (streams are parsed on several threads)
    Inv v;
    for (int t = 0; t < 2; t++) {
      const uint8_t* fwd = cbp_me_table(t != 0);
      for (int cbp = 0; cbp < 48; cbp++) v.t[t][fwd[cbp]] = (uint8_t)cbp;
    }
    return v;
  }();
  const uint8_t (*inv)[48] = inv_s.t;
  if (code < 0 || code > 47) return -1;
  return inv[intra ? 1 : 0][code];
}

// One slice: what its header says (7.3.3), and the state its macroblocks are parsed with.
struct SliceCtx {
  ParserState* st = nullptr;
  ParsedPicture* pic = nullptr;
  bool idr = false, is_ref = false, is_p = false, is_b = false, inter = false;
  int first_mb = 0;
  SliceState ss{};               // idr, frame_num, idr_pic_id, slice QP
  int poc = 0, poc_msb = 0, poc_lsb = 0;
  int n_ref[2] = {0, 0};         // num_ref_idx_l0_active, num_ref_idx_l1_active
  RefEntry lists[2][33];         // RefPicList0 / RefPicList1; entries carry the picture SLOT of the construct stage
  WpTable wp;                    // pred_weight_table
  bool adaptive_marking = false, idr_long_term = false;
  std::vector<ParsedPicture::Mmco> mmco;
  int cabac_init_idc = 0;
  int dbk_idc = 0, alpha_off = 0, beta_off = 0;   // disable_deblocking_filter_idc, FilterOffsetA / B
  int slice_no = 0, mbw = 0, n_mb = 0;
  // host-side motion derivation (h264_motion.h): the field of every picture where B slices may occur, B macroblocks resolved here
  bool track = false;
  bool track_fail = false;       // a P macroblock with explicit weights could not be resolved
  MotionCtx M;
  BSliceCtx b;                   // B slices: direct prediction, lists and weights as motion resolution reads them
};

// a picture of the buffer as a list entry; identity PicNum (FrameNumWrap, 8.2.4.1), or LongTermPicNum (= LongTermFrameIdx) + 2^20
RefEntry ref_entry(const ParserState::RefPic& rp, int frame_num, int max_fn) {
  RefEntry e;
  e.slot = rp.slot; e.poc = rp.poc; e.pic_id = rp.pic_id; e.lt = rp.long_term;
  e.key = rp.long_term ? rp.lt_idx + (1 << 20) : (rp.frame_num > frame_num ? rp.frame_num - max_fn : rp.frame_num);
  return e;
}

// initial RefPicList0 / RefPicList1 (8.2.4.2): P slices order the short-term pictures by descending PicNum, B slices by picture
// order count around the current picture; long-term pictures follow by ascending LongTermPicNum
int init_ref_lists(const ParserState* st, SliceCtx& c) {
  RefEntry cand[32];
  int nc = 0;
  for (const ParserState::RefPic& rp : st->refs) {
    if (nc >= 32) break;
    cand[nc++] = ref_entry(rp, c.ss.frame_num, 1 << st->log2_max_frame_num);
  }
  if (nc == 0) return PARSE_INVALID;
  int no[2] = {0, 0};
  auto append_sorted = [&](int l, auto pick, auto before) {   // the candidates `pick` selects, in a stable order by `before`
    const int first = no[l];
    for (int i = 0; i < nc; i++) if (pick(cand[i])) c.lists[l][no[l]++] = cand[i];
    std::stable_sort(c.lists[l] + first, c.lists[l] + no[l], before);
  };
  auto is_lt = [](const RefEntry& e) { return e.lt; };
  auto key_asc = [](const RefEntry& a, const RefEntry& b) { return a.key < b.key; };
  if (c.is_p) {
    append_sorted(0, [](const RefEntry& e) { return !e.lt; }, [](const RefEntry& a, const RefEntry& b) { return a.key > b.key; });
    append_sorted(0, is_lt, key_asc);
  } else {
    const int poc = c.poc;
    auto poc_desc = [](const RefEntry& a, const RefEntry& b) { return a.poc > b.poc; };
    auto poc_asc = [](const RefEntry& a, const RefEntry& b) { return a.poc < b.poc; };
    auto before_cur = [poc](const RefEntry& e) { return !e.lt && e.poc < poc; };
    auto after_cur = [poc](const RefEntry& e) { return !e.lt && e.poc > poc; };
    append_sorted(0, before_cur, poc_desc); append_sorted(0, after_cur, poc_asc); append_sorted(0, is_lt, key_asc);
    append_sorted(1, after_cur, poc_asc); append_sorted(1, before_cur, poc_desc); append_sorted(1, is_lt, key_asc);
    auto same_pic = [](const RefEntry& a, const RefEntry& b) { return a.pic_id == b.pic_id && a.slot == b.slot; };
    if (no[1] > 1 && no[0] == no[1] && std::equal(c.lists[0], c.lists[0] + no[0], c.lists[1], same_pic))
      std::swap(c.lists[1][0], c.lists[1][1]);                // identical lists: the first two entries of list 1 change places
  }
  for (int l = 0; l < (c.is_b ? 2 : 1); l++)
    for (int i = no[l]; i < 33; i++) {
      if (c.is_p && no[l] > 0) { c.lists[l][i] = c.lists[l][no[l] - 1]; c.lists[l][i].key = -0x40000000; }   // entries past the
      else c.lists[l][i] = RefEntry();                                           // available pictures (a conforming stream does not use them)
    }
  return PARSE_OK;
}

// ref_pic_list_modification() of list l (7.3.3.1), each command applied as it is read (8.2.4.3)
int modify_ref_list(BitReader& r, const ParserState* st, SliceCtx& c, int l) {
  if (!r.bit()) return PARSE_OK;                              // ref_pic_list_modification_flag_lX
  const int max_fn = 1 << st->log2_max_frame_num, nref_l = c.n_ref[l];
  RefEntry* L = c.lists[l];
  int pred = c.ss.frame_num, idx = 0;
  for (;;) {
    const uint32_t idc = r.ue();
    if (idc == 3) return PARSE_OK;
    if (idc > 3 || !r.ok()) return PARSE_INVALID;
    const uint32_t v = r.ue();
    if (idx >= nref_l) return PARSE_INVALID;
    int want;
    if (idc == 2) {
      want = (int)v + (1 << 20);                              // long_term_pic_num
    } else {
      if (v >= (uint32_t)max_fn) return PARSE_INVALID;
      int no_wrap = idc == 0 ? pred - ((int)v + 1) : pred + ((int)v + 1);
      if (no_wrap < 0) no_wrap += max_fn;
      if (no_wrap >= max_fn) no_wrap -= max_fn;
      pred = no_wrap;
      want = no_wrap > c.ss.frame_num ? no_wrap - max_fn : no_wrap;
    }
    bool found = false;                                       // the last of the (first 32) pictures of the buffer with that identity
    RefEntry e;
    for (size_t i = 0; i < st->refs.size() && i < 32; i++) {
      const RefEntry x = ref_entry(st->refs[i], c.ss.frame_num, max_fn);
      if (x.key == want) { e = x; found = true; }
    }
    if (!found) return PARSE_UNSUPPORTED;                     // refers to a picture that is not in the buffer (loss): needs concealment
    // insert at idx, shift the rest, drop the later duplicate
    for (int k = nref_l; k > idx; k--) L[k] = L[k - 1];
    L[idx++] = e;
    int nidx = idx;
    for (int k = idx; k <= nref_l; k++)
      if (L[k].key != want) L[nidx++] = L[k];
  }
}

// pred_weight_table() (7.3.3.2)
int read_pred_weight_table(BitReader& r, const ParserState* st, SliceCtx& c) {
  WpTable& wp = c.wp;
  wp.on = true;
  const uint32_t dl = r.ue(), dc = r.ue();
  if (dl > 7 || dc > 7) return PARSE_INVALID;
  wp.log2[0] = (int)dl; wp.log2[1] = (int)dc;
  for (int l = 0; l < (c.is_b ? 2 : 1); l++)
    for (int i = 0; i < c.n_ref[l]; i++) {
      int given = 0;                                          // luma_weight_flag (bit 0), chroma_weight_flag (bit 1)
      for (int pl = 0; pl < 3; pl++) {
        if (pl < 2) given |= r.bit() << pl;
        int w = 1 << wp.log2[pl ? 1 : 0], o = 0;              // absent: the default weight and offset
        if ((given >> (pl ? 1 : 0)) & 1) {
          w = r.se(); o = r.se();
          if (w < -128 || w > 127 || o < -128 || o > 127) return PARSE_INVALID;
        }
        wp.w[l][i][pl][0] = (int16_t)w; wp.w[l][i][pl][1] = (int16_t)o;
      }
      wp.given[l][i] = (uint8_t)given;
    }
  if (!r.ok()) return PARSE_TRUNCATED;
  if (st->profile == 66) return PARSE_INVALID;
  return PARSE_OK;
}

// dec_ref_pic_marking() (7.3.3.3) of a reference picture's slice
int read_dec_ref_pic_marking(BitReader& r, SliceCtx& c) {
  if (c.idr) { r.bit(); c.idr_long_term = r.bit() != 0; return PARSE_OK; }   // no_output_of_prior_pics_flag, long_term_reference_flag
  if (!r.bit()) return PARSE_OK;                              // adaptive_ref_pic_marking_mode_flag 0: sliding window
  c.adaptive_marking = true;
  for (;;) {
    ParsedPicture::Mmco m;
    m.op = (int)r.ue(); m.a = m.b = 0;
    if (m.op == 0) return PARSE_OK;
    if (m.op > 6 || !r.ok()) return PARSE_INVALID;
    if (m.op == 1 || m.op == 3) m.a = (int)r.ue();            // difference_of_pic_nums_minus1
    if (m.op == 2) m.a = (int)r.ue();                         // long_term_pic_num
    if (m.op == 3 || m.op == 6) m.b = (int)r.ue();            // long_term_frame_idx
    if (m.op == 4) m.a = (int)r.ue();                         // max_long_term_frame_idx_plus1
    c.mmco.push_back(m);
    if (c.mmco.size() > 64) return PARSE_INVALID;
  }
}

// slice_header() (7.3.3): activates the slice's parameter sets and builds its reference lists (8.2.4)
int parse_slice_header(BitReader& r, const Nal& nal, ParserState* st, const ParsedPicture* pic, SliceCtx& c) {
  c.idr = nal.type == 5;
  if (!c.idr && !st->have_ref) return PARSE_INVALID;          // a P picture before any IDR: nothing to predict from
  const bool first_slice = pic->n_slices == 0;
  c.first_mb = (int)r.ue();
  if (c.first_mb != pic->next_mb) return PARSE_UNSUPPORTED;   // slices out of raster order / missing slices (ASO, FMO, losses)
  const int slice_type = (int)r.ue() % 5;
  if (slice_type > 2) return PARSE_UNSUPPORTED;               // SP / SI slices
  c.is_p = slice_type == 0; c.is_b = slice_type == 1; c.inter = c.is_p || c.is_b;
  if (c.idr && c.inter) return PARSE_INVALID;
  {                                                           // the slice names its PPS, the PPS its SPS (several of each may be around)
    const uint32_t id = r.ue();
    if (id > 255 || !st->pps_tab[id].valid || !st->sps_tab[st->pps_tab[id].sps_id].valid) return PARSE_NO_PARAMETER_SETS;
    if (!first_slice && (int)id != st->sp.pps_id && st->pps_tab[id].sps_id != st->sp.sps_id) return PARSE_INVALID;
    if (first_slice && (st->sp.sps_id != st->pps_tab[id].sps_id || !st->have_sps)) {
      if (!c.idr && st->have_sps) return PARSE_UNSUPPORTED;   // a new sequence may only start at an IDR picture
      activate_sps(st, st->pps_tab[id].sps_id);
    }
    activate_pps(st, (int)id);
  }
  // B slices: where the profile has them, with picture order count type 0 and direct_8x8_inference (frame macroblocks: the corner
  // blocks of the co-located macroblock stand for its 8x8 blocks)
  if (c.is_b && (st->profile == 66 || st->poc_type != 0 || !st->direct_8x8_inference)) return PARSE_UNSUPPORTED;
  c.ss.idr = c.idr;
  c.ss.frame_num = (int)r.get(st->log2_max_frame_num);
  c.ss.idr_pic_id = c.idr ? (int)r.ue() : 0;
  if (st->poc_type == 0) c.poc_lsb = (int)r.get(st->log2_max_poc_lsb);
  else if (st->poc_type == 1 && !st->delta_pic_order_always_zero) r.se();          // delta_pic_order_cnt[0]
  if (st->poc_type == 0) {                                    // 8.2.1.1
    const int max_lsb = 1 << st->log2_max_poc_lsb;
    const int prev_msb = c.idr ? 0 : st->prev_poc_msb, prev_lsb = c.idr ? 0 : st->prev_poc_lsb;
    if (c.poc_lsb < prev_lsb && prev_lsb - c.poc_lsb >= max_lsb / 2) c.poc_msb = prev_msb + max_lsb;
    else if (c.poc_lsb > prev_lsb && c.poc_lsb - prev_lsb > max_lsb / 2) c.poc_msb = prev_msb - max_lsb;
    else c.poc_msb = prev_msb;
    c.poc = c.poc_msb + c.poc_lsb;
  } else {
    c.poc = 2 * (c.idr ? 0 : st->decode_count);               // types 1 / 2 without B slices: output order is decoding order
  }
  if (c.is_b) c.b.direct_spatial = r.bit() != 0;              // direct_spatial_mv_pred_flag
  int rc;
  if (c.inter) {
    c.n_ref[0] = st->num_ref_idx_default;
    c.n_ref[1] = c.is_b ? st->num_ref_idx_l1_default : 0;
    if (r.bit()) { c.n_ref[0] = (int)r.ue() + 1; if (c.is_b) c.n_ref[1] = (int)r.ue() + 1; }   // num_ref_idx_active_override_flag
    if (c.n_ref[0] < 1 || c.n_ref[0] > 32 || (c.is_b && (c.n_ref[1] < 1 || c.n_ref[1] > 32))) return PARSE_INVALID;
    if ((rc = init_ref_lists(st, c)) != PARSE_OK) return rc;
    for (int l = 0; l < (c.is_b ? 2 : 1); l++)
      if ((rc = modify_ref_list(r, st, c, l)) != PARSE_OK) return rc;
    for (int i = 0; i < c.n_ref[0]; i++) if (c.lists[0][i].slot < 0 && c.is_p) return PARSE_INVALID;
  }
  // explicit weights of a P slice (weighted_pred_flag) or a B slice (weighted_bipred_idc 1)
  if ((c.is_p && st->weighted_pred) || (c.is_b && st->weighted_bipred_idc == 1))
    if ((rc = read_pred_weight_table(r, st, c)) != PARSE_OK) return rc;
  c.is_ref = nal.ref_idc != 0;                                // a non-reference picture is output but never predicted from
  if (c.is_ref && (rc = read_dec_ref_pic_marking(r, c)) != PARSE_OK) return rc;
  if (st->entropy_cabac && c.inter) {
    const uint32_t v = r.ue();
    if (v > 2) return PARSE_INVALID;
    c.cabac_init_idc = (int)v;
  }
  c.ss.qp = st->pic_init_qp + r.se();
  if (st->deblocking_control) {
    c.dbk_idc = (int)r.ue();
    if (c.dbk_idc > 2) return PARSE_INVALID;
    if (c.dbk_idc != 1) {
      c.alpha_off = 2 * r.se(); c.beta_off = 2 * r.se();
      if (c.alpha_off < -12 || c.alpha_off > 12 || c.beta_off < -12 || c.beta_off > 12) return PARSE_INVALID;
    }
  }
  if (!r.ok()) return PARSE_TRUNCATED;
  if (c.ss.qp < 0 || c.ss.qp > 51) return PARSE_INVALID;
  if (c.idr) { if (c.ss.frame_num != 0) return PARSE_INVALID; }
  else if (c.ss.frame_num != ((st->last_frame_num + 1) & ((1 << st->log2_max_frame_num) - 1))) return PARSE_UNSUPPORTED;   // a gap (7.4.3:
                                                            // frame_num follows the last REFERENCE picture): needs error concealment
  return PARSE_OK;
}

// the first slice of a picture sets the picture up
int start_picture(ParserState* st, ParsedPicture* pic, SliceCtx& c) {
  pic->ss = c.ss;
  pic->is_ref = c.is_ref;
  pic->adaptive_marking = c.adaptive_marking;
  pic->mmco = std::move(c.mmco);
  pic->idr_long_term = c.idr_long_term;
  pic->crop_left = 2 * st->crop_left; pic->crop_top = 2 * st->crop_top;
  pic->n_slots = st->n_slots;
  {                                                           // a slot no reference picture occupies
    int slot = 0;
    while (!c.idr && std::any_of(st->refs.begin(), st->refs.end(), [slot](const ParserState::RefPic& rp) { return rp.slot == slot; })) slot++;
    if (slot >= st->n_slots) return PARSE_INVALID;
    pic->cur_slot = slot;
  }
  pic->poc = c.poc; pic->poc_msb = c.poc_msb; pic->poc_lsb = c.poc_lsb;
  pic->pic_id = st->next_pic_id++;
  pic->max_reorder = st->profile == 66 ? 0 : st->sp.num_ref_frames;
  pic->has_b = false;
  pic->has_t8 = st->transform_8x8; pic->chroma_qp_offset = st->chroma_qp_offset;
  const int n = st->sp.mb_w * st->sp.mb_h;
  if (st->profile != 66) {                                    // the stream may hold B slices: keep the motion field of every picture
    if ((int)st->motion.size() < st->n_slots) st->motion.resize(st->n_slots);
    MotionStore& ms = st->motion[pic->cur_slot];
    if ((int)ms.intra.size() != n) ms.size_for(n);
    ms.poc = c.poc; ms.pic_id = pic->pic_id;
  } else {
    st->motion.clear();
  }
  // the records are initialised as the macroblocks are parsed (7.3 MB per 1080p picture are not filled up front: a skipped
  // macroblock resets its 128 header bytes, a coded one its whole record); a picture is only handed out complete (next_mb == n)
  if ((int)pic->mbs.size() != n) pic->mbs.assign(n, MbOut());
  DecMbAux za;
  memset(&za, 0, sizeof(za));
  pic->aux.assign(n, za);
  return PARSE_OK;
}

// the DecMbAux fields every macroblock carries: slice, deblocking control and which neighbours are available (slices come in
// raster order, so a neighbour is in this slice iff it is not before the slice's first macroblock)
DecMbAux& start_aux(const SliceCtx& c, int idx) {
  DecMbAux& ax = c.pic->aux[idx];
  const int w = c.mbw, x = idx % w, y = idx / w;
  auto in_slice = [&](int other) { return other >= c.first_mb; };
  ax.slice = (uint16_t)c.slice_no; ax.dbk_idc = (uint8_t)c.dbk_idc; ax.alpha_off = (int8_t)c.alpha_off; ax.beta_off = (int8_t)c.beta_off;
  ax.avail = (uint8_t)((x > 0 && in_slice(idx - 1) ? 1 : 0) | (y > 0 && in_slice(idx - w) ? 2 : 0) |
                       (x > 0 && y > 0 && in_slice(idx - w - 1) ? 4 : 0) | (y > 0 && x < w - 1 && in_slice(idx - w + 1) ? 8 : 0));
  return ax;
}

// P_Skip (ref_idx 0, vector predicted later) or B_Skip (direct prediction): no residual, QP_Y carried over
int skip_mb(SliceCtx& c, int idx, DecMbAux& ax, int qp) {
  MbOut& m = c.pic->mbs[idx];
  reset_skip_record(&m);
  m.qp = (uint8_t)qp;
  if (!c.is_b) {
    for (int q = 0; q < 4; q++) ax.ref_idx[q] = (int8_t)c.lists[0][0].slot;
    return PARSE_OK;
  }
  m.mb_type = MBT_BSKIP;
  BMbSyntax sx;
  sx.skip = true;
  return derive_b(c.M, idx, ax.avail, sx, c.b, &ax, &c.pic->aux_b[idx]) ? PARSE_OK : PARSE_INVALID;
}

// mb_type of a P or B slice past its inter types is an intra type (Tables 7-13, 7-14): true, t becomes its I-slice number
bool intra_mb_type(const SliceCtx& c, int* t) {
  if (!c.inter) return true;
  const int n_inter = c.is_p ? 5 : 23;
  if (*t < n_inter) return false;
  *t -= n_inter;
  return true;
}

// I_16x16 mb_type t (Table 7-11): the prediction mode into the record; returns the coded_block_pattern it names
int i16x16_record(MbOut& m, int t) {
  m.mb_type = MBT_I16x16;
  const int v = t - 1;
  m.i16_mode = (uint8_t)(v & 3);
  return (((v >> 2) % 3) << 4) | (v >= 12 ? 15 : 0);
}

// the intra prediction modes must have their neighbours (8.3.3, 8.3.4); with constrained intra prediction the construct stage
// knows which count
bool intra_modes_ok(const SliceCtx& c, const MbOut& m, int avail) {
  if (m.chroma_mode > 3) return false;
  if (c.st->constrained_intra_pred) return true;
  const bool L = avail & 1, T = avail & 2;
  if ((m.chroma_mode == 1 && !L) || (m.chroma_mode == 2 && !T) || (m.chroma_mode == 3 && !(L && T))) return false;
  return !(m.mb_type == MBT_I16x16 && ((m.i16_mode == 0 && !T) || (m.i16_mode == 1 && !L) || (m.i16_mode == 3 && !(L && T))));
}

// I_PCM after its samples: every block counts as 16 coefficients for the neighbours' contexts (9.2.1), QP'Y is 0 for the deblocking
// filter; like the reference decoder (decode_slice.cpp:1870: iLastMbQp untouched) the QP predictor of the next macroblock stays
void pcm_record(MbOut& m) {
  m.mb_type = MBT_IPCM;
  for (int i = 0; i < 24; i++) m.nnz[i] = 16;
  m.cbp = 0x2f;
  m.qp = 0;
}

// P macroblock (7.3.5.1 / 7.3.5.2 of P slices): the partitions of mb_type t, their ref_idx_l0 (ri, and as picture slots in ax) and
// their vectors, as the slice's entropy coder reads them.  read_sub() returns -1 for a value out of range; read_ref(q0, qmask) reads
// the ref_idx of the 8x8 blocks in qmask (q0 the first); read_mvd(blk, w4, h4, int16_t v[2]) the vector of the partition whose
// first 4x4 block is blk.
template <class ReadSub, class ReadRef, class ReadMvd>
int read_p_mb(const SliceCtx& c, int t, MbOut& m, DecMbAux& ax, int ri[4], bool* no_sub8, ReadSub read_sub, ReadRef read_ref, ReadMvd read_mvd) {
  static const uint8_t kMask[3][2] = {{15, 0}, {3, 12}, {5, 10}};     // 8x8 blocks of the partitions of P_L0_16x16, _16x8, _8x16
  static const uint8_t kPart[3][2][3] = {{{0, 4, 4}}, {{0, 4, 2}, {8, 4, 2}}, {{0, 2, 4}, {2, 2, 4}}};   // first 4x4 block, w4, h4
  static const uint8_t kN[4] = {1, 2, 2, 4}, kW[4] = {2, 2, 1, 1}, kH[4] = {2, 1, 2, 1};   // per sub_mb_type: partitions, w4, h4
  static const uint8_t kOff[4][4] = {{0}, {0, 4}, {0, 1}, {0, 1, 4, 5}};                  // their first 4x4 blocks in the 8x8
  if (t < 0 || t > 4) return PARSE_INVALID;
  const bool p8x8 = t >= 3;                                   // P_8x8, or P_8x8ref0 (t 4, CAVLC only: every reference index is 0)
  const int np = t == 0 ? 1 : 2;
  m.mb_type = t == 0 ? MBT_P16x16 : t == 1 ? MBT_P16x8 : t == 2 ? MBT_P8x16 : MBT_P8x8;
  bool sub = false;
  for (int k = 0; p8x8 && k < 4; k++) {
    const int v = read_sub();
    if (v < 0) return PARSE_INVALID;
    ax.sub_type[k] = (uint8_t)v;
    sub = sub || v != 0;
  }
  if (!p8x8)
    for (int p = 0; p < np; p++) {
      const int mask = kMask[t][p], v = read_ref(__builtin_ctz(mask), mask);
      for (int q = 0; q < 4; q++) if (mask & (1 << q)) ri[q] = v;
    }
  else if (t == 3) for (int k = 0; k < 4; k++) ri[k] = read_ref(k, 1 << k);
  for (int k = 0; k < 4; k++) {
    if (ri[k] < 0 || ri[k] >= c.n_ref[0]) return PARSE_INVALID;
    ax.ref_idx[k] = (int8_t)c.lists[0][ri[k]].slot;
  }
  if (!p8x8) {
    for (int p = 0; p < np; p++) read_mvd(kPart[t][p][0], kPart[t][p][1], kPart[t][p][2], m.mvd[p]);
    return PARSE_OK;
  }
  for (int k = 0; k < 4; k++) {
    const int st = ax.sub_type[k], b0 = (k & 1) * 2 + (k >> 1) * 8;
    for (int j = 0; j < kN[st]; j++) read_mvd(b0 + kOff[st][j], kW[st], kH[st], ax.mvd[4 * k + j]);
  }
  // with sub-macroblock partitions the vectors stay in ax.mvd; without, the record carries the four 8x8 vectors as the encoder's does
  if (sub) { ax.flags |= DECAUX_SUB; *no_sub8 = false; }
  else for (int k = 0; k < 4; k++) { m.mvd[k][0] = ax.mvd[4 * k][0]; m.mvd[k][1] = ax.mvd[4 * k][1]; }
  return PARSE_OK;
}

// B macroblock (7.3.5.1 / 7.3.5.2 of B slices): sub_mb_type, ref_idx and mvd as the slice's entropy coder reads them, collected for
// derive_b().  read_sub() returns -1 for a value out of range; read_ref(l, unit) and read_mvd(l, unit, int16_t v[2]) read one
// partition's syntax element of list l.
template <class ReadSub, class ReadRef, class ReadMvd>
int read_b_mb(const SliceCtx& c, int t, MbOut& m, BMbSyntax& sx, bool* no_sub8, ReadSub read_sub, ReadRef read_ref, ReadMvd read_mvd) {
  m.mb_type = MBT_B;
  memset(sx.ref, 0, sizeof(sx.ref)); memset(sx.mvd, 0, sizeof(sx.mvd));
  sx.type = t;
  if (t == 22)
    for (int k = 0; k < 4; k++) {
      const int v = read_sub();
      if (v < 0) return PARSE_INVALID;
      sx.sub[k] = v;
      if (v != 0 && b_sub_shape(v) != 0) *no_sub8 = false;
    }
  BUnit ru[4], mu[16];
  const int nru = b_ref_units(sx, ru), nmu = b_mvd_units(sx, mu);
  for (int l = 0; l < 2; l++)
    for (int i = 0; i < nru; i++) {
      if (!(ru[i].lists & (1 << l))) continue;
      const int v = read_ref(l, ru[i]);
      if (v < 0 || v >= c.n_ref[l]) return PARSE_INVALID;
      for (int q = 0; q < 4; q++) if (ru[i].qmask & (1 << q)) sx.ref[l][q] = v;
    }
  for (int l = 0; l < 2; l++)
    for (int i = 0; i < nmu; i++)
      if (mu[i].lists & (1 << l)) read_mvd(l, mu[i], sx.mvd[l][mu[i].slot]);
  return PARSE_OK;
}

// an I or P macroblock is complete: its motion field cells; with explicit weights a P macroblock travels resolved, like a B one
void track_mb(SliceCtx& c, int i, const int ri[4]) {
  if (!c.track) return;
  MbOut& m = c.pic->mbs[i];
  DecMbAux& ax = c.pic->aux[i];
  if (MBT_IS_INTRA(m.mb_type)) c.M.store_intra(i);
  else if (!MBT_IS_B(m.mb_type)) {
    derive_p(c.M, i, ax.avail, m, ax, ri, c.lists[0]);
    if (c.wp.on) {
      if (!emit_resolved_p(c.M, c.lists[0], c.n_ref[0], c.wp, &ax, &c.pic->aux_b[i])) c.track_fail = true;
      m.mb_type = m.mb_type == MBT_PSKIP ? MBT_BSKIP : MBT_B;
    }
  }
}

// ---- slice data, CABAC (7.3.4 with entropy_coding_mode_flag = 1; macroblock layer 7.3.5, context selection 9.3.3.1.1) ----

// transform_size_8x8_flag
int cabac_t8(CabacDecoder& d, const CabacMbInfo* L, const CabacMbInfo* T) {
  return d.decision(399 + (L && L->t8 ? 1 : 0) + (T && T->t8 ? 1 : 0));
}

// ref_idx_lX of the 8x8 blocks in qmask, q0 the first: the context counts the blocks left of and above q0 with ref_idx > 0
int cabac_ref_idx(CabacDecoder& d, const SliceCtx& c, CabacMbInfo& me, const CabacMbInfo* L, const CabacMbInfo* T, int l, int q0, int qmask) {
  if (c.n_ref[l] <= 1) return 0;
  uint8_t& gt = l ? me.ref_gt0_l1 : me.ref_gt0;
  auto bits_of = [l](const CabacMbInfo* nb) { return nb ? (l ? nb->ref_gt0_l1 : nb->ref_gt0) : 0; };
  const int qx = q0 & 1, qy = q0 >> 1;
  const int a = qx ? (gt >> (q0 - 1)) & 1 : (bits_of(L) >> (qy * 2 + 1)) & 1;
  const int b = qy ? (gt >> (q0 - 2)) & 1 : (bits_of(T) >> (2 + qx)) & 1;
  const int v = d.ref_idx(a + 2 * b);
  if (v > 0) gt |= (uint8_t)qmask;
  return v;
}

// mvd_lX of the partition at 4x4 block (bx, by), w4 x h4 blocks: the context sums the neighbours' |mvd|, which it updates
void cabac_mvd(CabacDecoder& d, CabacMbInfo& me, const CabacMbInfo* L, const CabacMbInfo* T, int l, int bx, int by, int w4, int h4, int16_t v[2]) {
  uint8_t (*mine)[2] = l ? me.mvd_l1 : me.mvd;
  int mv[2];
  for (int c = 0; c < 2; c++) {
    const int a = bx > 0 ? mine[by * 4 + bx - 1][c] : (L ? (l ? L->mvd_l1 : L->mvd)[by * 4 + 3][c] : 0);
    const int b = by > 0 ? mine[(by - 1) * 4 + bx][c] : (T ? (l ? T->mvd_l1 : T->mvd)[12 + bx][c] : 0);
    mv[c] = d.mvd(c ? 47 : 40, a + b);
    v[c] = (int16_t)mv[c];
  }
  const uint8_t a0 = (uint8_t)(abs(mv[0]) > 255 ? 255 : abs(mv[0])), a1 = (uint8_t)(abs(mv[1]) > 255 ? 255 : abs(mv[1]));
  for (int y = 0; y < h4; y++)
    for (int x = 0; x < w4; x++) { mine[(by + y) * 4 + bx + x][0] = a0; mine[(by + y) * 4 + bx + x][1] = a1; }
}

// coded_block_flag of a neighbour's block (un: the value for a neighbour that is not available)
inline int cbf_of(const CabacMbInfo* nb, int bit, int un) { return nb ? (int)((nb->cbf >> bit) & 1) : un; }

// the residual of a macroblock with coded_block_pattern cbp (7.3.5.3 with CABAC)
int cabac_residual(CabacDecoder& d, MbOut& m, CabacMbInfo& me, const CabacMbInfo* L, const CabacMbInfo* T, int cbp, bool intra, bool t8) {
  static const int kCbfOff[5] = {0, 4, 8, 12, 16};
  const int cbp_l = cbp & 15, cbp_c = cbp >> 4;
  const int un = intra ? 1 : 0;                               // coded_block_flag of a block in a macroblock that is not available
  if (m.mb_type == MBT_I16x16 && d.decision(85 + kCbfOff[0] + cbf_of(L, 24, un) + 2 * cbf_of(T, 24, un))) {
    if (d.residual_levels(0, m.luma_dc, 16) < 0) return PARSE_INVALID;
    me.cbf |= 1u << 24;
  }
  const int lcat = m.mb_type == MBT_I16x16 ? 1 : 2;
  if (t8) {                                                   // four 8x8 blocks (ctxBlockCat 5: no coded_block_flag, the pattern bit decides)
    for (int q = 0; q < 4; q++) {
      if (!(cbp_l & (1 << q))) continue;
      const int cnt = d.residual_levels8x8(&m.luma[4 * q][0]);
      if (cnt < 0) return PARSE_INVALID;
      const int b0 = (q >> 1) * 8 + (q & 1) * 2;
      m.nnz[b0] = m.nnz[b0 + 1] = m.nnz[b0 + 4] = m.nnz[b0 + 5] = (int8_t)(cnt > 16 ? 16 : cnt);
      me.cbf |= (1u << b0) | (1u << (b0 + 1)) | (1u << (b0 + 4)) | (1u << (b0 + 5));
    }
  }
  for (int k = 0; k < 16 && !t8; k++) {
    if (!(cbp_l & (1 << (k >> 2)))) continue;
    const int bx = (k & 1) | ((k >> 1) & 2), by = ((k >> 1) & 1) | ((k >> 2) & 2);
    const int a = bx > 0 ? (int)((me.cbf >> (by * 4 + bx - 1)) & 1) : cbf_of(L, by * 4 + 3, un);
    const int b = by > 0 ? (int)((me.cbf >> ((by - 1) * 4 + bx)) & 1) : cbf_of(T, 12 + bx, un);
    if (!d.decision(85 + kCbfOff[lcat] + a + 2 * b)) continue;
    const int cnt = d.residual_levels(lcat, m.luma[k], lcat == 1 ? 15 : 16);
    if (cnt < 0) return PARSE_INVALID;
    m.nnz[by * 4 + bx] = (int8_t)cnt;
    me.cbf |= 1u << (by * 4 + bx);
  }
  if (cbp_c) {
    for (int uv = 0; uv < 2; uv++)
      if (d.decision(85 + kCbfOff[3] + cbf_of(L, 25 + uv, un) + 2 * cbf_of(T, 25 + uv, un))) {
        if (d.residual_levels(3, m.chroma_dc[uv], 4) < 0) return PARSE_INVALID;
        me.cbf |= 1u << (25 + uv);
      }
    if (cbp_c == 2)
      for (int uv = 0; uv < 2; uv++)
        for (int j = 0; j < 4; j++) {
          const int bx = j & 1, by = j >> 1, base = 16 + 4 * uv;
          const int a = bx > 0 ? (int)((me.cbf >> (base + by * 2)) & 1) : cbf_of(L, base + by * 2 + 1, un);
          const int b = by > 0 ? (int)((me.cbf >> (base + bx)) & 1) : cbf_of(T, base + 2 + bx, un);
          if (!d.decision(85 + kCbfOff[4] + a + 2 * b)) continue;
          const int cnt = d.residual_levels(4, m.chroma_ac[4 * uv + j], 15);
          if (cnt < 0) return PARSE_INVALID;
          m.nnz[base + j] = (int8_t)cnt;
          me.cbf |= 1u << (base + j);
        }
  }
  return PARSE_OK;
}

int parse_slice_data_cabac(BitReader& r, const Nal& nal, SliceCtx& c) {
  while (r.pos() & 7) if (!r.bit()) return PARSE_INVALID;     // cabac_alignment_one_bit
  if (!r.ok()) return PARSE_TRUNCATED;
  CabacDecoder d(nal.rbsp.data(), nal.rbsp.size());
  d.init_contexts(c.ss.qp, c.inter ? 1 + c.cabac_init_idc : 0);
  d.init_engine(r.pos());
  ParsedPicture* pic = c.pic;
  const int n = c.n_mb, mbw = c.mbw;
  if ((int)pic->cabac_info.size() != n) pic->cabac_info.resize(n);
  CabacMbInfo* info = pic->cabac_info.data();
  int qp = c.ss.qp, idx = c.first_mb, rc;
  bool prev_dqp_nonzero = false;
  for (;;) {
    if (idx >= n) return PARSE_INVALID;                       // the slice goes on beyond the picture
    DecMbAux& ax = start_aux(c, idx);
    const CabacMbInfo* L = (ax.avail & 1) ? &info[idx - 1] : nullptr;
    const CabacMbInfo* T = (ax.avail & 2) ? &info[idx - mbw] : nullptr;
    CabacMbInfo& me = info[idx];
    memset(&me, 0, sizeof(me));
    MbOut& m = pic->mbs[idx];
    int ri[4] = {0, 0, 0, 0};                                 // ref_idx_l0 of the 8x8 blocks of a P macroblock (host-side motion field)
    if (c.inter && d.decision((c.is_b ? 24 : 11) + (L && !L->skip ? 1 : 0) + (T && !T->skip ? 1 : 0))) {      // mb_skip_flag
      if ((rc = skip_mb(c, idx, ax, qp)) != PARSE_OK) return rc;
      me.type = m.mb_type; me.skip = 1; me.direct = c.is_b ? 1 : 0;
      prev_dqp_nonzero = false;
    } else {
      memset(&m, 0, sizeof(m));
      ax.flags = c.st->constrained_intra_pred ? DECAUX_CIP : 0;
      int t = c.is_p ? d.mb_type_p()
            : c.is_b ? d.mb_type_b((L && !L->direct ? 1 : 0) + (T && !T->direct ? 1 : 0))
            : d.mb_type_intra(3 + (L && L->type != MBT_I4x4 ? 1 : 0) + (T && T->type != MBT_I4x4 ? 1 : 0), false);
      const bool intra = intra_mb_type(c, &t);
      me.intra = intra ? 1 : 0;
      int cbp = -1;
      bool no_sub8 = true;                                    // no sub-macroblock partition smaller than 8x8 (7.3.5: gate of transform_size_8x8_flag)
      if (intra && t == 25) {                                 // I_PCM: the arithmetic decoder stopped behind its flush; raw bytes follow
        size_t bp = (d.pos() + 7) & ~(size_t)7;               // pcm_alignment_zero_bit
        const size_t byte0 = bp >> 3;
        if (byte0 + 384 > nal.rbsp.size()) return PARSE_TRUNCATED;
        memcpy(reinterpret_cast<uint8_t*>(m.luma), nal.rbsp.data() + byte0, 256);
        memcpy(reinterpret_cast<uint8_t*>(m.chroma_ac), nal.rbsp.data() + byte0 + 256, 128);
        d.init_engine(bp + 384 * 8);                          // 9.3.1.2: the engine starts over after the samples
        pcm_record(m);
        me.type = MBT_IPCM; me.cbp = 0x2f; me.cbf = 0x7ffffff;
        prev_dqp_nonzero = false;
      } else {
        if (!intra && c.is_b) {                               // the syntax is collected, then resolved on the host (h264_motion.h)
          if (t == 0) me.direct = 1;
          BMbSyntax sx;
          rc = read_b_mb(c, t, m, sx, &no_sub8, [&] { return d.sub_mb_type_b(); },
                         [&](int l, const BUnit& u) { return cabac_ref_idx(d, c, me, L, T, l, u.q0, u.qmask); },
                         [&](int l, const BUnit& u, int16_t* v) { cabac_mvd(d, me, L, T, l, u.bx, u.by, u.w4, u.h4, v); });
          if (rc != PARSE_OK) return rc;
          if (!d.ok()) return PARSE_TRUNCATED;
          if (!derive_b(c.M, idx, ax.avail, sx, c.b, &ax, &c.pic->aux_b[idx])) return PARSE_INVALID;
        } else if (!intra) {
          rc = read_p_mb(c, t, m, ax, ri, &no_sub8, [&] { return d.sub_mb_type_p(); },
                         [&](int q0, int qmask) { return cabac_ref_idx(d, c, me, L, T, 0, q0, qmask); },
                         [&](int blk, int w4, int h4, int16_t* v) { cabac_mvd(d, me, L, T, 0, blk & 3, blk >> 2, w4, h4, v); });
          if (rc != PARSE_OK) return rc;
        } else {
          if (t == 0) {
            m.mb_type = MBT_I4x4;
            const bool t8i = c.st->transform_8x8 && cabac_t8(d, L, T);        // Intra_8x8: four prediction modes instead of sixteen
            if (t8i) { ax.flags |= DECAUX_T8; me.t8 = 1; }
            for (int k = 0; k < (t8i ? 4 : 16); k++) {
              m.prev_i4_flag[k] = (int8_t)d.decision(68);
              if (!m.prev_i4_flag[k]) { int v = d.decision(69); v |= d.decision(69) << 1; v |= d.decision(69) << 2; m.rem_i4_mode[k] = (int8_t)v; }
            }
          } else {
            cbp = i16x16_record(m, t);
          }
          m.chroma_mode = (uint8_t)d.intra_chroma_pred_mode((L && L->chroma_mode != 0 ? 1 : 0) + (T && T->chroma_mode != 0 ? 1 : 0));
          me.chroma_mode = m.chroma_mode;
          if (!intra_modes_ok(c, m, ax.avail)) return PARSE_INVALID;
        }
        me.type = m.mb_type;
        if (cbp < 0) {                                        // coded_block_pattern: prefix (luma, 4 bins) + suffix (chroma)
          const int la[2] = {L ? !((L->cbp >> 1) & 1) : 0, L ? !((L->cbp >> 3) & 1) : 0};
          const int ta[2] = {T ? !((T->cbp >> 2) & 1) : 0, T ? !((T->cbp >> 3) & 1) : 0};
          const int b0 = d.decision(73 + la[0] + 2 * ta[0]);
          const int b1 = d.decision(73 + !b0 + 2 * ta[1]);
          const int b2 = d.decision(73 + la[1] + 2 * !b0);
          const int b3 = d.decision(73 + !b2 + 2 * !b1);
          const int lc = L ? L->cbp >> 4 : 0, tc = T ? T->cbp >> 4 : 0;
          int cc = d.decision(77 + (lc ? 1 : 0) + (tc ? 2 : 0));
          if (cc) cc += d.decision(81 + (lc >> 1) + 2 * (tc >> 1));
          cbp = b0 | (b1 << 1) | (b2 << 2) | (b3 << 3) | (cc << 4);
        }
        m.cbp = (uint8_t)cbp; me.cbp = (uint8_t)cbp;
        if (!intra && (cbp & 15) && c.st->transform_8x8 && no_sub8 && cabac_t8(d, L, T)) { ax.flags |= DECAUX_T8; me.t8 = 1; }
        if (cbp > 0 || m.mb_type == MBT_I16x16) {
          const int dqp = d.mb_qp_delta(prev_dqp_nonzero ? 1 : 0);
          if (dqp < -26 || dqp > 25) return PARSE_INVALID;
          qp = (qp + dqp + 52) % 52;
          prev_dqp_nonzero = dqp != 0;
          if ((rc = cabac_residual(d, m, me, L, T, cbp, intra, (ax.flags & DECAUX_T8) != 0)) != PARSE_OK) return rc;
        } else {
          prev_dqp_nonzero = false;
        }
        m.qp = (uint8_t)qp;
      }
    }
    if (!d.ok()) return PARSE_TRUNCATED;
    track_mb(c, idx, ri);
    idx++;
    if (d.terminate()) break;                                 // end_of_slice_flag
  }
  pic->next_mb = idx;
  return PARSE_OK;
}

// ---- slice data, CAVLC ----

// te(v) of a reference index with range num_ref_idx_active - 1 (9.1): absent for one picture, an inverted bit for two, else ue(v)
inline int read_te(BitReader& r, int n_ref) { return n_ref == 1 ? 0 : n_ref == 2 ? !r.bit() : (int)r.ue(); }

int parse_slice_data_cavlc(BitReader& r, SliceCtx& c) {
  static const int kRiZero[4] = {0, 0, 0, 0};
  ParsedPicture* pic = c.pic;
  const int n = c.n_mb, mbw = c.mbw;
  int qp = c.ss.qp, idx = c.first_mb, rc;
  while (idx < n) {
    if (c.inter) {
      const int run = (int)r.ue();                            // mb_skip_run
      if (!r.ok() || idx + run > n) return PARSE_INVALID;
      for (int k = 0; k < run; k++, idx++) {
        if ((rc = skip_mb(c, idx, start_aux(c, idx), qp)) != PARSE_OK) return rc;
        track_mb(c, idx, kRiZero);
      }
      if (idx == n || !r.more_data()) break;                  // the slice may end with a skip run
    }
    MbOut& m = pic->mbs[idx];
    memset(&m, 0, sizeof(m));
    DecMbAux& ax = start_aux(c, idx);
    ax.flags = c.st->constrained_intra_pred ? DECAUX_CIP : 0;
    int t = (int)r.ue();
    const bool intra = intra_mb_type(c, &t);
    int cbp = -1, ri[4] = {0, 0, 0, 0};
    bool no_sub8 = true;
    if (!intra && c.is_b) {                                   // the syntax is collected, then resolved on the host (h264_motion.h)
      BMbSyntax sx;
      rc = read_b_mb(c, t, m, sx, &no_sub8, [&] { const uint32_t v = r.ue(); return v > 12 ? -1 : (int)v; },
                     [&](int l, const BUnit&) { return read_te(r, c.n_ref[l]); },
                     [&](int, const BUnit&, int16_t* v) { v[0] = (int16_t)r.se(); v[1] = (int16_t)r.se(); });
      if (rc != PARSE_OK) return rc;
      if (!r.ok()) return PARSE_TRUNCATED;
      if (!derive_b(c.M, idx, ax.avail, sx, c.b, &ax, &c.pic->aux_b[idx])) return PARSE_INVALID;
    } else if (!intra) {
      rc = read_p_mb(c, t, m, ax, ri, &no_sub8, [&] { const uint32_t v = r.ue(); return v > 3 ? -1 : (int)v; },
                     [&](int, int) { return read_te(r, c.n_ref[0]); },
                     [&](int, int, int, int16_t* v) { v[0] = (int16_t)r.se(); v[1] = (int16_t)r.se(); });
      if (rc != PARSE_OK) return rc;
    } else {
      if (t == 0) {
        m.mb_type = MBT_I4x4;
        const bool t8i = c.st->transform_8x8 && r.bit();      // transform_size_8x8_flag: Intra_8x8, four prediction modes
        if (t8i) ax.flags |= DECAUX_T8;
        for (int k = 0; k < (t8i ? 4 : 16); k++) { m.prev_i4_flag[k] = (int8_t)r.bit(); m.rem_i4_mode[k] = m.prev_i4_flag[k] ? 0 : (int8_t)r.get(3); }
      } else if (t <= 24) {
        cbp = i16x16_record(m, t);
      } else if (t == 25) {                                   // I_PCM (7.3.5): byte-aligned raw samples
        while (r.pos() & 7) r.skip(1);
        uint8_t* py = reinterpret_cast<uint8_t*>(m.luma);
        uint8_t* pc = reinterpret_cast<uint8_t*>(m.chroma_ac);
        for (int i = 0; i < 256; i++) py[i] = (uint8_t)r.get(8);
        for (int i = 0; i < 128; i++) pc[i] = (uint8_t)r.get(8);
        if (!r.ok()) return PARSE_TRUNCATED;
        pcm_record(m);
        track_mb(c, idx, kRiZero);
        idx++;
        if (!r.more_data()) break;
        continue;
      } else return PARSE_INVALID;
      m.chroma_mode = (uint8_t)r.ue();
      if (!intra_modes_ok(c, m, ax.avail)) return PARSE_INVALID;
    }
    if (cbp < 0) {
      cbp = cbp_from_code((int)r.ue(), m.mb_type == MBT_I4x4);
      if (cbp < 0) return PARSE_INVALID;
    }
    m.cbp = (uint8_t)cbp;
    const int cbp_l = cbp & 15, cbp_c = cbp >> 4;
    if (!intra && cbp_l > 0 && c.st->transform_8x8 && no_sub8 && r.bit()) ax.flags |= DECAUX_T8;   // transform_size_8x8_flag
    const bool t8 = (ax.flags & DECAUX_T8) != 0;
    if (cbp > 0 || m.mb_type == MBT_I16x16) {
      const int dqp = r.se();
      if (dqp < -26 || dqp > 25) return PARSE_INVALID;
      qp = (qp + dqp + 52) % 52;                              // 7.4.5: QP_Y wraps modulo 52
      const int8_t* L = (ax.avail & 1) ? pic->mbs[idx - 1].nnz : nullptr;
      const int8_t* T = (ax.avail & 2) ? pic->mbs[idx - mbw].nnz : nullptr;
      auto luma_nc = [&](int bx, int by) {
        const int a = bx > 0 ? m.nnz[by * 4 + bx - 1] : (L ? L[by * 4 + 3] : -1);
        const int b = by > 0 ? m.nnz[(by - 1) * 4 + bx] : (T ? T[12 + bx] : -1);
        return nc_of(a, b);
      };
      if (m.mb_type == MBT_I16x16 && (rc = read_block(r, m.luma_dc, 16, luma_nc(0, 0))) < 0) return rc;
      for (int k = 0; k < 16; k++) {
        if (!(cbp_l & (1 << (k >> 2)))) continue;
        const int bx = (k & 1) | ((k >> 1) & 2), by = ((k >> 1) & 1) | ((k >> 2) & 2);
        if (t8) {                                             // 8x8 block as four interleaved 4x4 blocks (7.3.5.3.2: level 4 * j + i of the 8x8)
          int16_t tmp[16];
          rc = read_block(r, tmp, 16, luma_nc(bx, by));
          if (rc < 0) return rc;
          int16_t* lv64 = &m.luma[k & ~3][0];
          for (int j = 0; j < 16; j++) lv64[4 * j + (k & 3)] = tmp[j];
        } else {
          rc = read_block(r, m.luma[k], m.mb_type == MBT_I16x16 ? 15 : 16, luma_nc(bx, by));
          if (rc < 0) return rc;
        }
        m.nnz[by * 4 + bx] = (int8_t)rc;
      }
      if (cbp_c) {
        if ((rc = read_block(r, m.chroma_dc[0], 4, -1)) < 0) return rc;
        if ((rc = read_block(r, m.chroma_dc[1], 4, -1)) < 0) return rc;
        if (cbp_c == 2) {
          for (int uv = 0; uv < 2; uv++)
            for (int j = 0; j < 4; j++) {
              const int bx = j & 1, by = j >> 1, base = 16 + 4 * uv;
              const int a = bx > 0 ? m.nnz[base + by * 2] : (L ? L[base + by * 2 + 1] : -1);
              const int b = by > 0 ? m.nnz[base + bx] : (T ? T[base + 2 + bx] : -1);
              rc = read_block(r, m.chroma_ac[4 * uv + j], 15, nc_of(a, b));
              if (rc < 0) return rc;
              m.nnz[base + j] = (int8_t)rc;
            }
        }
      }
    }
    m.qp = (uint8_t)qp;
    if (!r.ok()) return PARSE_TRUNCATED;
    track_mb(c, idx, ri);
    idx++;
    if (!r.more_data()) break;                                // end of this slice
  }
  pic->next_mb = idx;
  return PARSE_OK;
}

int parse_slice(BitReader& r, const Nal& nal, ParserState* st, ParsedPicture* pic) {
  SliceCtx c;
  c.st = st; c.pic = pic;
  int rc = parse_slice_header(r, nal, st, pic, c);
  if (rc != PARSE_OK) return rc;
  if (pic->n_slices == 0) {
    if ((rc = start_picture(st, pic, c)) != PARSE_OK) return rc;
  } else if (c.idr != pic->ss.idr || c.ss.frame_num != pic->ss.frame_num || c.is_ref != pic->is_ref || c.poc != pic->poc) {
    return PARSE_INVALID;                                     // slices of one access unit must agree
  }
  c.mbw = st->sp.mb_w; c.n_mb = st->sp.mb_w * st->sp.mb_h;
  if ((c.is_b || c.wp.on) && !pic->has_b) {                   // B macroblocks, and P macroblocks with explicit weights, travel resolved
    pic->has_b = true;
    DecMbAuxB zb;
    memset(&zb, 0, sizeof(zb));
    pic->aux_b.assign(c.n_mb, zb);
  }
  c.track = !st->motion.empty();
  if (c.track) { c.M.cur = &st->motion[pic->cur_slot]; c.M.mbw = c.mbw; }
  if (c.is_b) {
    BSliceCtx& b = c.b;
    b.cur_poc = c.poc; b.n_ref[0] = c.n_ref[0]; b.n_ref[1] = c.n_ref[1];
    for (int l = 0; l < 2; l++) for (int i = 0; i < 33; i++) b.list[l][i] = c.lists[l][i];
    b.implicit = st->weighted_bipred_idc == 2;
    b.wp = c.wp.on ? &c.wp : nullptr;
    b.cabac = st->entropy_cabac;
    const int cslot = c.lists[1][0].slot;
    b.col = (cslot >= 0 && cslot < (int)st->motion.size()) ? &st->motion[cslot] : nullptr;
    b.col_long_term = c.lists[1][0].lt;
  }
  if (pic->n_slices >= 65535) return PARSE_UNSUPPORTED;
  c.slice_no = pic->n_slices++;
  if (c.dbk_idc != 1) pic->any_deblock = true;
  rc = st->entropy_cabac ? parse_slice_data_cabac(r, nal, c) : parse_slice_data_cavlc(r, c);
  if (rc != PARSE_OK) return rc;
  return c.track_fail ? PARSE_INVALID : PARSE_OK;
}

// decoded reference picture marking (8.2.5) of a complete reference picture: an IDR picture empties the buffer; otherwise the
// memory management commands or the sliding window make room, then the picture joins the references (short-term unless a
// command says otherwise)
void mark_reference_picture(ParserState* st, const ParsedPicture& pic) {
  const int max_fn = 1 << st->log2_max_frame_num, cur = pic.ss.frame_num;
  std::vector<ParserState::RefPic>& refs = st->refs;
  auto pic_num = [&](const ParserState::RefPic& rp) { return rp.frame_num > cur ? rp.frame_num - max_fn : rp.frame_num; };
  auto find = [&](bool lt, int num) -> int {                  // the first short-term picture with PicNum num, or long-term one with
    for (size_t i = 0; i < refs.size(); i++)                  // LongTermFrameIdx num; -1 if none
      if (refs[i].long_term == lt && (lt ? refs[i].lt_idx : pic_num(refs[i])) == num) return (int)i;
    return -1;
  };
  auto drop_long_term = [&](int lt_idx) { const int j = find(true, lt_idx); if (j >= 0) refs.erase(refs.begin() + j); return j; };
  bool cur_long = false, reset = false;
  int cur_lt_idx = 0;
  if (pic.ss.idr) {
    refs.clear();
    cur_long = pic.idr_long_term;
  } else if (pic.adaptive_marking) {
    for (const ParsedPicture::Mmco& m : pic.mmco) {
      if (m.op == 1 || m.op == 3) {                           // a short-term picture: unused, or turned into a long-term one
        int i = find(false, cur - (m.a + 1));
        if (i < 0) continue;
        if (m.op == 1) { refs.erase(refs.begin() + i); continue; }
        if (const int j = drop_long_term(m.b); j >= 0 && j < i) i--;   // the index is taken over
        refs[i].long_term = true; refs[i].lt_idx = m.b;
      } else if (m.op == 2) {
        drop_long_term(m.a);
      } else if (m.op == 4) {
        for (size_t i = 0; i < refs.size();)
          if (refs[i].long_term && refs[i].lt_idx >= m.a) refs.erase(refs.begin() + i); else i++;
      } else if (m.op == 5) {
        refs.clear(); reset = true;
      } else if (m.op == 6) {
        drop_long_term(m.b);
        cur_long = true; cur_lt_idx = m.b;
      }
    }
  }
  const int cap = st->sp.num_ref_frames < 1 ? 1 : st->sp.num_ref_frames;
  while ((int)refs.size() >= cap) {                           // sliding window (8.2.5.3): the short-term picture with the smallest FrameNumWrap goes
    size_t victim = refs.size();
    int best = 0x7fffffff;
    for (size_t i = 0; i < refs.size(); i++)
      if (!refs[i].long_term && pic_num(refs[i]) < best) { best = pic_num(refs[i]); victim = i; }
    if (victim == refs.size()) victim = 0;                    // only long-term pictures left: a non-conforming stream; drop the first
    refs.erase(refs.begin() + victim);
  }
  ParserState::RefPic rp;
  rp.slot = pic.cur_slot; rp.frame_num = reset ? 0 : cur; rp.long_term = cur_long; rp.lt_idx = cur_lt_idx;
  rp.poc = pic.poc; rp.pic_id = pic.pic_id;
  refs.push_back(rp);
  st->have_ref = true; st->last_frame_num = reset ? 0 : cur;
  st->prev_poc_msb = reset ? 0 : pic.poc_msb; st->prev_poc_lsb = reset ? 0 : pic.poc_lsb;
}

}  // namespace

int parse_access_unit(const uint8_t* au, size_t len, ParserState* st, ParsedPicture* pic) {
  if (!au || !st || !pic) return PARSE_INVALID;
  {                                                           // a fresh picture that keeps the storage of the record arrays
    ParsedPicture fresh{};
    fresh.mbs.swap(pic->mbs); fresh.aux.swap(pic->aux); fresh.aux_b.swap(pic->aux_b); fresh.cabac_info.swap(pic->cabac_info);
    *pic = std::move(fresh);
  }
  bool got_slice = false;
  for (const Nal& nal : split_nals(au, len)) {
    BitReader r(nal.rbsp.data(), nal.rbsp.size());
    int rc = PARSE_OK;
    if (nal.type == 7 || nal.type == 8) {
      if (got_slice) return PARSE_UNSUPPORTED;                // parameter sets after the slice of the same unit
      rc = nal.type == 7 ? parse_sps(r, st) : parse_pps(r, st);
    } else if (nal.type == 1 || nal.type == 5) {
      rc = parse_slice(r, nal, st, pic);                      // one of possibly several slices of the picture
      got_slice = true;
    } else if (nal.type == 6 || nal.type == 9 || nal.type == 12) continue;   // SEI, AUD, filler: nothing to reconstruct
    else return PARSE_UNSUPPORTED;
    if (rc != PARSE_OK) return rc;
  }
  if (!got_slice) return PARSE_NO_PICTURE;
  if (pic->next_mb != st->sp.mb_w * st->sp.mb_h) return PARSE_INCOMPLETE;    // macroblocks missing: more slices to come (or lost: needs concealment)
  if (pic->is_ref) mark_reference_picture(st, *pic);
  st->decode_count = pic->ss.idr ? 1 : st->decode_count + 1;
  return PARSE_OK;
}

int probe_access_unit(const uint8_t* au, size_t len, int* width, int* height, int* has_slice) {
  *width = *height = *has_slice = 0;
  for (const Nal& nal : split_nals(au, len)) {
    if (nal.type == 1 || nal.type == 5) *has_slice = 1;
    if (nal.type == 7) {
      BitReader r(nal.rbsp.data(), nal.rbsp.size());
      ParserState tmp;
      const int rc = parse_sps(r, &tmp);
      if (rc != PARSE_OK) return rc;
      *width = tmp.sp.width; *height = tmp.sp.height;
    }
  }
  return PARSE_OK;
}

}  // namespace b2h264

#ifdef B2H264_WP_STATS
// coverage counters of explicit weighted prediction in B slices (WPS_* in wp_formula.h; the host build decodes on one thread)
static long long g_wp_stats[WPS_N];
void b2h264_wp_stat(int which, long long n) { g_wp_stats[which] += n; }
extern "C" int b2h264_dec_wp_stats(long long* out, int n, int reset) {
  for (int i = 0; i < WPS_N; i++) {
    if (out && i < n) out[i] = g_wp_stats[i];
    if (reset) g_wp_stats[i] = 0;
  }
  return WPS_N;
}
#endif
