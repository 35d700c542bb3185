// h264_cabac.cpp — host-side CABAC slice serialisation (entropy_coding_mode_flag = 1), the second entropy coder north_star
// keeps on the CPU.  Consumes the same MbOut records as the CAVLC writer (h264_bitstream.cpp): the device pipeline does not
// know which entropy coder follows (the reference's mode decision does not depend on it: InitCoeffFunc, set_mb_syn_cavlc.cpp:304,
// only swaps the macroblock syntax writer).
// Written from Rec. H.264 7.3.5 / 9.3 (binarisations 9.3.2, context selection 9.3.3.1, arithmetic encoder 9.3.4); what the
// reference emits for the supported configuration (I and P slices, frame macroblocks, one reference picture, partitions >= 8x8,
// no 8x8 transform, no I_PCM) is the normative syntax, so the output is bit-identical to
// codec/encoder/core/src/svc_set_mb_syn_cabac.cpp:56-760 + set_mb_syn_cabac.cpp (checked by tests/test_encoder_emu.py against
// the compiled reference).  Context tables: cabac_tables.h (generated, pinned by tests/test_cavlc_tables.py).
#include "h264_bitstream.h"

#include <stdlib.h>
#include <string.h>

#include "cabac_tables.h"

namespace b2h264 {

namespace {

// ---- arithmetic encoder, Rec. H.264 9.3.4.2 ------------------------------------------------------------------------------
// The Recommendation describes the encoder bit by bit (PutBit with outstanding bits).  This is the same arithmetic with byte-wise
// output: `low_` keeps the 10-bit coding window in its low bits and the bits already shifted out of the window above it; once 8 of
// them (plus the carry position) are complete a byte leaves, a carry runs back into the bytes written before (a run of 0xff bytes
// is held back until it is known whether a carry reaches it).  The first bit PutBit would write is dropped by starting 9 shifts
// short of a byte, as 9.3.4.2 prescribes.  The slice header before the first byte is byte aligned (cabac_alignment_one_bit).
class CabacEncoder {
 public:
  explicit CabacEncoder(std::vector<uint8_t>* out) : out_(out) {}
  void init_contexts(int slice_qp, int table /* 0 = I slice, 1 + cabac_init_idc */) {
    const int qp = slice_qp < 0 ? 0 : slice_qp > 51 ? 51 : slice_qp;
    for (int i = 0; i < 460; i++) {
      int pre = ((kCabacInit[i][table][0] * qp) >> 4) + kCabacInit[i][table][1];
      pre = pre < 1 ? 1 : pre > 126 ? 126 : pre;
      // state in bits 1..6, valMPS in bit 0
      ctx_[i] = pre <= 63 ? (uint8_t)((63 - pre) << 1) : (uint8_t)(((pre - 64) << 1) | 1);
    }
    low_ = 0; range_ = 510; queue_ = -9; outstanding_ = 0;
  }
  void decision(int ctx, int bin) {
    const uint32_t c = ctx_[ctx], st = c >> 1;
    const uint32_t lps = kCabacRangeLps[st][(range_ >> 6) & 3];
    range_ -= lps;
    if ((uint32_t)(bin != 0) != (c & 1)) {
      low_ += range_;
      range_ = lps;
      ctx_[ctx] = (uint8_t)((kCabacNextLps[st] << 1) | ((c & 1) ^ (st == 0)));
    } else {
      ctx_[ctx] = (uint8_t)((kCabacNextMps[st] << 1) | (c & 1));
    }
    renorm();
  }
  void bypass(int bin) {
    low_ <<= 1;
    if (bin) low_ += range_;
    queue_++;
    put_byte();
  }
  void terminate(int bin) {
    range_ -= 2;
    if (!bin) { renorm(); return; }
    // EncodeFlush (9.3.4.5): the window moves 7 places (range 2 -> 256), then its top bit and two more bits leave, the last one
    // forced to 1: the rbsp_stop_one_bit.  What is left of the last byte is rbsp_alignment_zero_bit.
    low_ += range_;
    range_ = 2;
    renorm();
    low_ |= 0x80;
    low_ <<= 3; queue_ += 3;
    put_byte();
    low_ &= ~(uint64_t)0x3ff;                           // the rest of the window is not part of the stream
    if (queue_ > -8) { low_ <<= -queue_; queue_ = 0; put_byte(); }
    for (; outstanding_ > 0; outstanding_--) out_->push_back(0xff);
  }
  // unary-exp-Golomb suffix of order k, bypass coded (9.3.2.3)
  void exp_golomb_bypass(int k, uint32_t v) {
    while (v >= (1u << k)) { bypass(1); v -= 1u << k; k++; }
    bypass(0);
    while (k--) bypass((v >> k) & 1);
  }

 private:
  void renorm() {
    if (range_ >= 256) return;
    const int shift = __builtin_clz(range_) - 23;       // range_ in [2, 255]: up to 7 places
    range_ <<= shift;
    low_ <<= shift;
    queue_ += shift;
    put_byte();
  }
  void put_byte() {
    if (queue_ < 0) return;
    const uint32_t out = (uint32_t)(low_ >> (queue_ + 10));          // 9 bits: a carry on top of the byte
    low_ &= ((uint64_t)0x400 << queue_) - 1;
    queue_ -= 8;
    if ((out & 0xff) == 0xff) { outstanding_++; return; }           // cannot be written before a possible carry is known
    const uint32_t carry = out >> 8;
    if (carry) out_->back() = (uint8_t)(out_->back() + 1);           // the byte before a held-back run is never 0xff
    for (; outstanding_ > 0; outstanding_--) out_->push_back((uint8_t)(carry - 1));   // 0xff without, 0x00 with a carry
    out_->push_back((uint8_t)out);
  }
  std::vector<uint8_t>* out_;
  uint8_t ctx_[460];
  uint64_t low_ = 0;
  uint32_t range_ = 510;
  int queue_ = -9, outstanding_ = 0;
};

// what later macroblocks need to know about a coded macroblock (context selection, 9.3.3.1.1)
struct MbCtxInfo {
  uint8_t type = MBT_PSKIP;
  bool skip = true, intra = false;
  uint8_t cbp = 0, chroma_mode = 0;
  uint32_t cbf = 0;                 // bit 0..15 luma 4x4 (raster), 16..19 Cb AC, 20..23 Cr AC (raster 2x2), 24 luma DC, 25 Cb DC, 26 Cr DC
  int16_t mvd[16][2];               // per 4x4 block (raster)
  MbCtxInfo() { memset(mvd, 0, sizeof(mvd)); }
};

const int kCbfOff[5] = {0, 4, 8, 12, 16}, kSigOff[5] = {0, 15, 29, 44, 47}, kAbsOff[5] = {0, 10, 20, 30, 39};
enum { CAT_LUMA_DC = 0, CAT_LUMA_AC = 1, CAT_LUMA_4x4 = 2, CAT_CHROMA_DC = 3, CAT_CHROMA_AC = 4 };

// residual_block_cabac (7.3.5.3.3): lv = max_coef levels in scan order; coded = coded_block_flag; cbf_inc = its ctxIdxInc
void residual_block(CabacEncoder& e, int cat, const int16_t* lv, int max_coef, bool coded, int cbf_inc) {
  e.decision(85 + kCbfOff[cat] + cbf_inc, coded);
  if (!coded) return;
  int last = max_coef - 1;
  while (last > 0 && lv[last] == 0) last--;
  for (int i = 0; i < max_coef - 1; i++) {
    const int inc = cat == CAT_CHROMA_DC ? (i < 2 ? i : 2) : i;
    const bool sig = lv[i] != 0;
    e.decision(105 + kSigOff[cat] + inc, sig);
    if (sig) {
      e.decision(166 + kSigOff[cat] + inc, i == last);
      if (i == last) break;
    }
  }
  int eq1 = 0, gt1 = 0;
  for (int i = last; i >= 0; i--) {
    if (lv[i] == 0) continue;
    const int a = abs(lv[i]) - 1;
    const int base = 227 + kAbsOff[cat];
    e.decision(base + (gt1 ? 0 : (1 + eq1 < 4 ? 1 + eq1 : 4)), a > 0);
    if (a > 0) {
      const int lim = 4 - (cat == CAT_CHROMA_DC ? 1 : 0);
      const int ctx = base + 5 + (gt1 < lim ? gt1 : lim);
      const int pre = a < 14 ? a : 14;
      for (int k = 1; k < pre; k++) e.decision(ctx, 1);
      if (a < 14) e.decision(ctx, 0);
      else e.exp_golomb_bypass(0, (uint32_t)(a - 14));
      gt1++;
    } else {
      eq1++;
    }
    e.bypass(lv[i] < 0);
  }
}

// mvd_lX component (UEG3, uCoff 9, signed): ctx_base 40 (x) / 47 (y); sum = |mvd| of the left plus the upper neighbouring block
void mvd_comp(CabacEncoder& e, int v, int ctx_base, int sum) {
  const int a = abs(v);
  int inc = sum > 32 ? 2 : sum > 2 ? 1 : 0;
  const int pre = a < 9 ? a : 9;
  for (int k = 0; k < pre; k++) {
    e.decision(ctx_base + inc, 1);
    inc = k == 0 ? 3 : (inc < 6 ? inc + 1 : 6);
  }
  if (a < 9) e.decision(ctx_base + inc, 0);
  else e.exp_golomb_bypass(3, (uint32_t)(a - 9));
  if (a) e.bypass(v < 0);
}

}  // namespace

void write_slice_cabac(const StreamParams& sp, const SliceState& ss, const MbOut* const* recs, std::vector<uint8_t>* rbsp) {
  BitWriter w(rbsp);
  write_slice_header(w, sp, ss);
  while (w.bit_pos() & 7) w.bit(1);      // cabac_alignment_one_bit

  CabacEncoder e(rbsp);                  // the header is byte aligned: the arithmetic coder appends whole bytes
  e.init_contexts(ss.qp, ss.idr ? 0 : 1);

  const int mbw = sp.mb_w, first = ss.first_mb, end = ss.end_mb < 0 ? sp.mb_w * sp.mb_h : ss.end_mb;
  std::vector<MbCtxInfo> info((size_t)(end - first));   // of the slice's macroblocks: a neighbour outside the slice is not available
  int last_qp = ss.qp;
  bool prev_dqp_nonzero = false;          // mb_qp_delta != 0 of the previous macroblock in decoding order (that carried one)
  for (int idx = first; idx < end; idx++) {
    const MbOut& m = *recs[idx];
    const int mbx = idx % mbw, mby = idx / mbw;
    const MbCtxInfo* L = mbx > 0 && idx - 1 >= first ? &info[idx - 1 - first] : nullptr;
    const MbCtxInfo* T = mby > 0 && idx - mbw >= first ? &info[idx - mbw - first] : nullptr;
    MbCtxInfo& me = info[idx - first];
    if (idx > first) e.terminate(0);      // end_of_slice_flag of the previous macroblock

    if (!ss.idr) e.decision(11 + (L && !L->skip ? 1 : 0) + (T && !T->skip ? 1 : 0), m.mb_type == MBT_PSKIP);   // mb_skip_flag
    if (m.mb_type == MBT_PSKIP) { me = MbCtxInfo(); prev_dqp_nonzero = false; continue; }

    me.type = m.mb_type; me.skip = false; me.intra = MBT_IS_INTRA(m.mb_type); me.cbp = m.cbp;
    const int cbp_l = m.cbp & 15, cbp_c = m.cbp >> 4;
    // ---- mb_type (Table 9-36, ctxIdx per Table 9-39) ----
    if (ss.idr) {
      const int ctx = 3 + (L && L->type != MBT_I4x4 ? 1 : 0) + (T && T->type != MBT_I4x4 ? 1 : 0);
      if (m.mb_type == MBT_I4x4) e.decision(ctx, 0);
      else {
        e.decision(ctx, 1);
        e.terminate(0);
        e.decision(6, cbp_l != 0);
        e.decision(7, cbp_c != 0);
        if (cbp_c) e.decision(8, cbp_c >> 1);
        e.decision(9, m.i16_mode >> 1);
        e.decision(10, m.i16_mode & 1);
      }
    } else {
      switch (m.mb_type) {
        case MBT_P16x16: e.decision(14, 0); e.decision(15, 0); e.decision(16, 0); break;
        case MBT_P16x8: e.decision(14, 0); e.decision(15, 1); e.decision(17, 1); break;
        case MBT_P8x16: e.decision(14, 0); e.decision(15, 1); e.decision(17, 0); break;
        case MBT_P8x8: e.decision(14, 0); e.decision(15, 0); e.decision(16, 1); break;
        case MBT_I4x4: e.decision(14, 1); e.decision(17, 0); break;
        default:                           // I16x16: prefix 1, then the I-slice binarisation on ctxIdx 17..20
          e.decision(14, 1);
          e.decision(17, 1);
          e.terminate(0);
          e.decision(18, cbp_l != 0);
          e.decision(19, cbp_c != 0);
          if (cbp_c) e.decision(19, cbp_c >> 1);
          e.decision(20, m.i16_mode >> 1);
          e.decision(20, m.i16_mode & 1);
          break;
      }
    }
    // ---- prediction ----
    if (me.intra) {
      if (m.mb_type == MBT_I4x4)
        for (int k = 0; k < 16; k++) {
          e.decision(68, m.prev_i4_flag[k] != 0);
          if (!m.prev_i4_flag[k]) { e.decision(69, m.rem_i4_mode[k] & 1); e.decision(69, (m.rem_i4_mode[k] >> 1) & 1); e.decision(69, (m.rem_i4_mode[k] >> 2) & 1); }
        }
      me.chroma_mode = m.chroma_mode;
      const int ctx = 64 + (L && L->chroma_mode != 0 ? 1 : 0) + (T && T->chroma_mode != 0 ? 1 : 0);
      e.decision(ctx, m.chroma_mode != 0);
      if (m.chroma_mode != 0) {
        e.decision(67, m.chroma_mode > 1);
        if (m.chroma_mode > 1) e.decision(67, m.chroma_mode > 2);
      }
    } else {
      if (m.mb_type == MBT_P8x8) for (int k = 0; k < 4; k++) e.decision(21, 1);       // sub_mb_type: P_L0_8x8
      // partitions: first 4x4 block (raster), width and height in 4x4 blocks
      int np = 1, first[4] = {0, 0, 0, 0}, pw = 4, ph = 4;
      if (m.mb_type == MBT_P16x8) { np = 2; first[1] = 8; ph = 2; }
      else if (m.mb_type == MBT_P8x16) { np = 2; first[1] = 2; pw = 2; }
      else if (m.mb_type == MBT_P8x8) { np = 4; first[1] = 2; first[2] = 8; first[3] = 10; pw = 2; ph = 2; }
      for (int p = 0; p < np; p++) {
        const int b = first[p], bx = b & 3, by = b >> 2;
        int sum[2];
        for (int c = 0; c < 2; c++) {
          const int a = bx > 0 ? abs(me.mvd[b - 1][c]) : (L ? abs(L->mvd[by * 4 + 3][c]) : 0);
          const int t = by > 0 ? abs(me.mvd[b - 4][c]) : (T ? abs(T->mvd[12 + bx][c]) : 0);
          sum[c] = a + t;
        }
        mvd_comp(e, m.mvd[p][0], 40, sum[0]);
        mvd_comp(e, m.mvd[p][1], 47, sum[1]);
        for (int y = 0; y < ph; y++)
          for (int x = 0; x < pw; x++) { me.mvd[(by + y) * 4 + bx + x][0] = m.mvd[p][0]; me.mvd[(by + y) * 4 + bx + x][1] = m.mvd[p][1]; }
      }
    }
    // ---- coded_block_pattern (not for I16x16: carried by mb_type) ----
    if (m.mb_type != MBT_I16x16) {
      // condTermFlag = neighbouring 8x8 block NOT coded (a macroblock that is not available counts as coded)
      const int la[2] = {L ? !((L->cbp >> 1) & 1) : 0, L ? !((L->cbp >> 3) & 1) : 0};
      const int ta[2] = {T ? !((T->cbp >> 2) & 1) : 0, T ? !((T->cbp >> 3) & 1) : 0};
      const int b0 = cbp_l & 1, b1 = (cbp_l >> 1) & 1, b2 = (cbp_l >> 2) & 1, b3 = (cbp_l >> 3) & 1;
      e.decision(73 + la[0] + 2 * ta[0], b0);
      e.decision(73 + !b0 + 2 * ta[1], b1);
      e.decision(73 + la[1] + 2 * !b0, b2);
      e.decision(73 + !b2 + 2 * !b1, b3);
      const int lc = L ? L->cbp >> 4 : 0, tc = T ? T->cbp >> 4 : 0;
      e.decision(77 + (lc ? 1 : 0) + (tc ? 2 : 0), cbp_c != 0);
      if (cbp_c) e.decision(81 + (lc >> 1) + 2 * (tc >> 1), cbp_c > 1);
    }
    // ---- residual ----
    if (m.cbp > 0 || m.mb_type == MBT_I16x16) {
      // mb_qp_delta (me(v)-like mapping, unary)
      const int dqp = m.qp - last_qp;
      last_qp = m.qp;
      {
        const int ctx0 = 60 + (prev_dqp_nonzero ? 1 : 0);
        if (dqp == 0) e.decision(ctx0, 0);
        else {
          int v = dqp < 0 ? -2 * dqp : 2 * dqp - 1;
          e.decision(ctx0, 1);
          if (v == 1) e.decision(62, 0);
          else { e.decision(62, 1); for (v -= 2; v > 0; v--) e.decision(63, 1); e.decision(63, 0); }
        }
        prev_dqp_nonzero = dqp != 0;
      }
      const int un = me.intra ? 1 : 0;      // coded_block_flag of a block in a macroblock that is not available
      auto cbf_of = [&](const MbCtxInfo* nb, int bit) { return nb ? (int)((nb->cbf >> bit) & 1) : un; };
      auto luma_inc = [&](int bx, int by) {
        const int a = bx > 0 ? (int)((me.cbf >> (by * 4 + bx - 1)) & 1) : cbf_of(L, by * 4 + 3);
        const int b = by > 0 ? (int)((me.cbf >> ((by - 1) * 4 + bx)) & 1) : cbf_of(T, 12 + bx);
        return a + 2 * b;
      };
      if (m.mb_type == MBT_I16x16) {
        bool nz = false;
        for (int i = 0; i < 16; i++) nz |= m.luma_dc[i] != 0;
        residual_block(e, CAT_LUMA_DC, m.luma_dc, 16, nz, cbf_of(L, 24) + 2 * cbf_of(T, 24));
        if (nz) me.cbf |= 1u << 24;
      }
      for (int k = 0; k < 16; k++) {
        if (!(cbp_l & (1 << (k >> 2)))) continue;
        const int bx = (k & 1) | ((k >> 1) & 2), by = ((k >> 1) & 1) | ((k >> 2) & 2);
        const bool act = m.nnz[by * 4 + bx] > 0;           // the stored count decides, as in the CAVLC writer
        if (m.mb_type == MBT_I16x16) residual_block(e, CAT_LUMA_AC, m.luma[k], 15, act, luma_inc(bx, by));
        else residual_block(e, CAT_LUMA_4x4, m.luma[k], 16, act, luma_inc(bx, by));
        if (act) me.cbf |= 1u << (by * 4 + bx);
      }
      if (cbp_c) {
        for (int uv = 0; uv < 2; uv++) {
          bool nz = false;
          for (int i = 0; i < 4; i++) nz |= m.chroma_dc[uv][i] != 0;
          residual_block(e, CAT_CHROMA_DC, m.chroma_dc[uv], 4, nz, cbf_of(L, 25 + uv) + 2 * cbf_of(T, 25 + uv));
          if (nz) me.cbf |= 1u << (25 + uv);
        }
        if (cbp_c == 2)
          for (int uv = 0; uv < 2; uv++)
            for (int j = 0; j < 4; j++) {
              const int bx = j & 1, by = j >> 1, base = 16 + 4 * uv;
              const int a = bx > 0 ? (int)((me.cbf >> (base + by * 2)) & 1) : cbf_of(L, base + by * 2 + 1);
              const int b = by > 0 ? (int)((me.cbf >> (base + bx)) & 1) : cbf_of(T, base + 2 + bx);
              const bool act = m.nnz[base + j] > 0;
              residual_block(e, CAT_CHROMA_AC, m.chroma_ac[4 * uv + j], 15, act, a + 2 * b);
              if (act) me.cbf |= 1u << (base + j);
            }
      }
    } else {
      prev_dqp_nonzero = false;
    }
  }
  e.terminate(1);                          // end_of_slice_flag = 1 + flush: stop bit and alignment included
}

}  // namespace b2h264
