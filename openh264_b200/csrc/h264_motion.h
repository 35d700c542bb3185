// h264_motion.h — host-side motion vector derivation of the parser (Rec. H.264 8.4.1): median / directional prediction
// (8.4.1.3), P_Skip (8.4.1.1), and the direct modes of B slices (spatial 8.4.1.2.2, temporal 8.4.1.2.3) with the co-located
// picture's motion field.  Used by h264_parse.cpp for streams that may hold B slices (every profile but Baseline): there the
// parser keeps the motion field of every decoded picture (MotionStore) and hands B macroblocks to the construct stage with FINAL
// vectors and reference pictures for both lists (DecMbAux / DecMbAuxB), because direct prediction needs the co-located picture's
// vectors, which only the host sees across pictures.  P macroblocks still travel as differences (the device predicts them,
// dec_mb.cuh); the host repeats their prediction only to know the field.
// Reference counterparts: codec/decoder/core/src/mv_pred.cpp (PredMv :706, PredInter16x8Mv :776, PredInter8x16Mv :753,
// PredPSkipMvFromNeighbor :158, PredMvBDirectSpatial :392, PredBDirectTemporal :613, GetColocatedMb :310, FillSpatialDirect8x8Mv :950),
// parse_mb_syn_cavlc.cpp (ParseInterBInfo :1328).
#pragma once
#include <stdint.h>
#include <string.h>

#include "h264_parse.h"
#include "wp_formula.h"

namespace b2h264 {

enum { MREF_NA = -2, MREF_NONE = -1 };           // cell outside the slice / not decoded yet; intra or list not used

// one entry of a slice's reference picture list
struct RefEntry { int slot = -1, key = -0x40000000, poc = 0, pic_id = -1; bool lt = false; };

// explicit weights of a slice (pred_weight_table): [list][ref_idx][plane Y / Cb / Cr][weight, offset]
struct WpTable {
  bool on = false;
  int log2[2] = {0, 0};                          // luma, chroma denominators
  int16_t w[2][32][3][2];
  uint8_t given[2][32];                          // luma_weight_flag (bit 0), chroma_weight_flag (bit 1): 0 = the default weight and offset
};

// what a B slice adds to the slice state
struct BSliceCtx {
  bool direct_spatial = true;
  int cur_poc = 0;
  int n_ref[2] = {0, 0};
  RefEntry list[2][33];
  int implicit = 0;                              // weighted_bipred_idc == 2
  const WpTable* wp = nullptr;                   // weighted_bipred_idc == 1: the slice's pred_weight_table
  const MotionStore* col = nullptr;              // motion field of RefPicList1[0]
  bool col_long_term = false;
  bool cabac = false;                            // entropy coder of the slice: the reference's two parsers treat temporal-direct 8x8s differently
};

// syntax of one B macroblock as read from the stream (both entropy coders fill this, then derive_b() resolves it)
struct BMbSyntax {
  int type = 0;                                  // mb_type 0..22 (Table 7-14); skip: type 0 with skip = true
  bool skip = false;
  int sub[4] = {0, 0, 0, 0};                     // sub_mb_type 0..12 (Table 7-18) when type == 22
  int ref[2][4];                                 // ref_idx per 8x8 and list (only the coded ones are meaningful)
  int16_t mvd[2][16][2];                         // [list][partition slot][c]: 16x16 [0]; 16x8 / 8x16 [0], [1]; 8x8: sub-partition j of 8x8 k at [4k+j]
};

// prediction use of partition p (0 / 1) of mb_type 1..21: bit 0 = list 0, bit 1 = list 1
inline int b_part_lists(int type, int part) {
  if (type <= 3) return type;                                              // 16x16: L0, L1, Bi
  static const uint8_t kPair[9][2] = {{1, 1}, {2, 2}, {1, 2}, {2, 1}, {1, 3}, {2, 3}, {3, 1}, {3, 2}, {3, 3}};
  return kPair[(type - 4) >> 1][part];
}
inline bool b_is_16x8(int type) { return type >= 4 && type <= 21 && !(type & 1); }
inline bool b_is_8x16(int type) { return type >= 4 && type <= 21 && (type & 1); }
// sub_mb_type 1..12: lists used, shape (0 8x8, 1 8x4, 2 4x8, 3 4x4)
inline int b_sub_lists(int sub) { static const uint8_t k[13] = {3, 1, 2, 3, 1, 1, 2, 2, 3, 3, 1, 2, 3}; return k[sub]; }
inline int b_sub_shape(int sub) { static const uint8_t k[13] = {0, 0, 0, 0, 1, 2, 1, 2, 1, 2, 3, 3, 3}; return k[sub]; }

// The syntax units of a B macroblock that is neither skipped nor B_Direct_16x16: who carries a ref_idx (a macroblock partition, or a
// non-direct 8x8 of B_8x8) and who carries a vector difference (a partition / sub-macroblock partition), in syntax order.
struct BUnit { int lists; int bx, by, w4, h4; int qmask; int q0; int slot; };
inline int b_ref_units(const BMbSyntax& sx, BUnit u[4]) {
  int n = 0;
  if (sx.type >= 1 && sx.type <= 3) u[n++] = {b_part_lists(sx.type, 0), 0, 0, 4, 4, 15, 0, 0};
  else if (b_is_16x8(sx.type)) for (int p = 0; p < 2; p++) u[n++] = {b_part_lists(sx.type, p), 0, 2 * p, 4, 2, 3 << (2 * p), 2 * p, p};
  else if (b_is_8x16(sx.type)) for (int p = 0; p < 2; p++) u[n++] = {b_part_lists(sx.type, p), 2 * p, 0, 2, 4, 5 << p, p, p};
  else if (sx.type == 22)
    for (int k = 0; k < 4; k++) if (sx.sub[k] != 0) u[n++] = {b_sub_lists(sx.sub[k]), (k & 1) * 2, (k >> 1) * 2, 2, 2, 1 << k, k, 4 * k};
  return n;
}
inline int b_mvd_units(const BMbSyntax& sx, BUnit u[16]) {
  if (sx.type != 22) return b_ref_units(sx, u);
  int n = 0;
  for (int k = 0; k < 4; k++) {
    if (sx.sub[k] == 0) continue;
    const int st = b_sub_shape(sx.sub[k]), bx = (k & 1) * 2, by = (k >> 1) * 2;
    const int w4 = (st == 0 || st == 1) ? 2 : 1, h4 = (st == 0 || st == 2) ? 2 : 1, np = st == 0 ? 1 : st == 3 ? 4 : 2;
    for (int j = 0; j < np; j++)
      u[n++] = {b_sub_lists(sx.sub[k]), bx + (st == 2 ? j : st == 3 ? (j & 1) : 0), by + (st == 1 ? j : st == 3 ? (j >> 1) : 0), w4, h4, 1 << k, k, 4 * k + j};
  }
  return n;
}

inline int median3(int a, int b, int c) { const int mn = a < b ? a : b, mx = a < b ? b : a; return c < mn ? mn : c > mx ? mx : c; }

class MotionCtx {
 public:
  MotionStore* cur = nullptr;
  int mbw = 0;
  int8_t refc[2][30];
  int16_t mvc[2][30][2];

  static int cell(int bx, int by) { return (by + 1) * 6 + bx + 1; }

  // neighbour cells from the picture's field (avail: NB_LEFT 1 | NB_TOP 2 | NB_TOPLEFT 4 | NB_TOPRIGHT 8, same-slice rule applied by
  // the caller); the macroblock's own cells start as "not decoded yet" and are filled in decoding order
  void load(int idx, int avail) {
    for (int l = 0; l < 2; l++) {
      for (int i = 0; i < 30; i++) { refc[l][i] = MREF_NA; mvc[l][i][0] = mvc[l][i][1] = 0; }
      auto take = [&](int c, int mb, int blk) {
        refc[l][c] = cur->ref[l][(size_t)mb * 16 + blk];
        mvc[l][c][0] = cur->mv[l][((size_t)mb * 16 + blk) * 2]; mvc[l][c][1] = cur->mv[l][((size_t)mb * 16 + blk) * 2 + 1];
      };
      if (avail & 4) take(0, idx - mbw - 1, 15);
      if (avail & 2) for (int x = 0; x < 4; x++) take(1 + x, idx - mbw, 12 + x);
      if (avail & 8) take(5, idx - mbw + 1, 12);
      if (avail & 1) for (int y = 0; y < 4; y++) take(6 + 6 * y, idx - 1, 3 + 4 * y);
    }
  }
  void set(int l, int bx, int by, int w4, int h4, int ref, int mvx, int mvy) {
    for (int y = 0; y < h4; y++)
      for (int x = 0; x < w4; x++) { const int c = cell(bx + x, by + y); refc[l][c] = (int8_t)ref; mvc[l][c][0] = (int16_t)mvx; mvc[l][c][1] = (int16_t)mvy; }
  }
  // 8.4.1.3 for the partition whose first 4x4 block is (bx, by), w4 blocks wide
  void pred(int l, int bx, int by, int w4, int ref, int* px, int* py) const {
    const int c = cell(bx, by), A = c - 1, B = c - 6, D = B - 1;
    int C = B + w4;
    const int rA = refc[l][A], rB = refc[l][B];
    int rC = refc[l][C];
    if (rC == MREF_NA) { C = D; rC = refc[l][D]; }
    if (rB == MREF_NA && rC == MREF_NA && rA != MREF_NA) { *px = mvc[l][A][0]; *py = mvc[l][A][1]; return; }
    const int match = (rA == ref) + (rB == ref) + (rC == ref);
    if (match == 1) {
      const int k = rA == ref ? A : rB == ref ? B : C;
      *px = mvc[l][k][0]; *py = mvc[l][k][1];
    } else {
      *px = median3(mvc[l][A][0], mvc[l][B][0], mvc[l][C][0]);
      *py = median3(mvc[l][A][1], mvc[l][B][1], mvc[l][C][1]);
    }
  }
  void pred_16x8(int l, int part, int ref, int* px, int* py) const {
    if (part == 0) { const int B = cell(0, 0) - 6; if (refc[l][B] == ref) { *px = mvc[l][B][0]; *py = mvc[l][B][1]; return; } pred(l, 0, 0, 4, ref, px, py); }
    else { const int A = cell(0, 2) - 1; if (refc[l][A] == ref) { *px = mvc[l][A][0]; *py = mvc[l][A][1]; return; } pred(l, 0, 2, 4, ref, px, py); }
  }
  void pred_8x16(int l, int part, int ref, int* px, int* py) const {
    if (part == 0) { const int A = cell(0, 0) - 1; if (refc[l][A] == ref) { *px = mvc[l][A][0]; *py = mvc[l][A][1]; return; } pred(l, 0, 0, 2, ref, px, py); }
    else {
      int C = 5;
      if (refc[l][C] == MREF_NA) C = 2;
      if (refc[l][C] == ref) { *px = mvc[l][C][0]; *py = mvc[l][C][1]; return; }
      pred(l, 2, 0, 2, ref, px, py);
    }
  }
  void pred_pskip(int* px, int* py) const {
    *px = *py = 0;
    if (refc[0][6] == MREF_NA || refc[0][1] == MREF_NA) return;
    if ((refc[0][6] == 0 && mvc[0][6][0] == 0 && mvc[0][6][1] == 0) || (refc[0][1] == 0 && mvc[0][1][0] == 0 && mvc[0][1][1] == 0)) return;
    pred(0, 0, 0, 4, 0, px, py);
  }
  // the macroblock's cells -> the picture's field; ref_id through the slice's lists
  void store(int idx, const RefEntry* l0, const RefEntry* l1) {
    for (int l = 0; l < 2; l++) {
      const RefEntry* L = l ? l1 : l0;
      for (int b = 0; b < 16; b++) {
        const int c = cell(b & 3, b >> 2);
        const int r = refc[l][c];
        const size_t o = (size_t)idx * 16 + b;
        cur->ref[l][o] = (int8_t)(r < 0 ? -1 : r);
        cur->ref_id[l][o] = (r >= 0 && L) ? L[r].pic_id : -1;
        cur->mv[l][o * 2] = r < 0 ? 0 : mvc[l][c][0]; cur->mv[l][o * 2 + 1] = r < 0 ? 0 : mvc[l][c][1];
      }
    }
    cur->intra[idx] = 0;
  }
  void store_intra(int idx) {
    for (int l = 0; l < 2; l++)
      for (int b = 0; b < 16; b++) {
        const size_t o = (size_t)idx * 16 + b;
        cur->ref[l][o] = -1; cur->ref_id[l][o] = -1; cur->mv[l][o * 2] = cur->mv[l][o * 2 + 1] = 0;
      }
    cur->intra[idx] = 1;
  }
};

// motion of a P macroblock from its record (type, differences) and the reference indices `ri` of its 8x8 blocks
inline void derive_p(MotionCtx& M, int idx, int avail, const MbOut& m, const DecMbAux& ax, const int ri[4], const RefEntry* l0) {
  M.load(idx, avail);
  int px, py;
  switch (m.mb_type) {
    case MBT_PSKIP: M.pred_pskip(&px, &py); M.set(0, 0, 0, 4, 4, 0, px, py); break;
    case MBT_P16x16: M.pred(0, 0, 0, 4, ri[0], &px, &py); M.set(0, 0, 0, 4, 4, ri[0], px + m.mvd[0][0], py + m.mvd[0][1]); break;
    case MBT_P16x8:
      for (int p = 0; p < 2; p++) { M.pred_16x8(0, p, ri[2 * p], &px, &py); M.set(0, 0, 2 * p, 4, 2, ri[2 * p], px + m.mvd[p][0], py + m.mvd[p][1]); }
      break;
    case MBT_P8x16:
      for (int p = 0; p < 2; p++) { M.pred_8x16(0, p, ri[p], &px, &py); M.set(0, 2 * p, 0, 2, 4, ri[p], px + m.mvd[p][0], py + m.mvd[p][1]); }
      break;
    default:                                                       // P_8x8
      for (int k = 0; k < 4; k++) {
        const int bx = (k & 1) * 2, by = (k >> 1) * 2;
        const int st = (ax.flags & DECAUX_SUB) ? ax.sub_type[k] : 0;
        const int w4 = (st == 0 || st == 1) ? 2 : 1, h4 = (st == 0 || st == 2) ? 2 : 1, np = st == 0 ? 1 : st == 3 ? 4 : 2;
        for (int j = 0; j < np; j++) {
          const int sx = bx + (st == 2 ? j : st == 3 ? (j & 1) : 0), sy = by + (st == 1 ? j : st == 3 ? (j >> 1) : 0);
          const int16_t* d = (ax.flags & DECAUX_SUB) ? ax.mvd[4 * k + j] : m.mvd[k];
          M.pred(0, sx, sy, w4, ri[k], &px, &py);
          M.set(0, sx, sy, w4, h4, ri[k], px + d[0], py + d[1]);
        }
      }
      break;
  }
  for (int b = 0; b < 16; b++) M.refc[1][MotionCtx::cell(b & 3, b >> 2)] = MREF_NONE;
  M.store(idx, l0, nullptr);
}

inline int clip3i(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }
// DistScaleFactor of 8.4.1.2.3 / 8.4.2.3.1; false: no scaling (long-term picture or equal counts)
inline bool dist_scale(int cur_poc, int poc0, int poc1, bool lt, int* dsf) {
  const int tb = clip3i(cur_poc - poc0, -128, 127), td = clip3i(poc1 - poc0, -128, 127);
  if (lt || td == 0) return false;
  const int tx = (16384 + (td < 0 ? -td : td) / 2) / td;
  *dsf = clip3i((tb * tx + 32) >> 6, -1024, 1023);
  return true;
}

inline bool emit_resolved(const MotionCtx& M, const BMbSyntax& sx, const BSliceCtx& S, const WpTable* wp, DecMbAux* ax, DecMbAuxB* axb);

// Resolves a B macroblock: final vectors and reference pictures of both lists into ax (list 0) / axb (list 1), the field, and
// returns false if the stream refers to a picture that is not there.
inline bool derive_b(MotionCtx& M, int idx, int avail, const BMbSyntax& sx, const BSliceCtx& S, DecMbAux* ax, DecMbAuxB* axb) {
  M.load(idx, avail);
  const bool any_direct = sx.skip || sx.type == 0 || (sx.type == 22 && (sx.sub[0] == 0 || sx.sub[1] == 0 || sx.sub[2] == 0 || sx.sub[3] == 0));
  int dref[2][4], dmv[2][4][2];                                    // direct prediction per 8x8
  if (any_direct) {
    const MotionStore* col = S.col;
    if (!col || col->intra.empty()) return false;
    static const int kCorner[4] = {0, 3, 12, 15};
    if (S.direct_spatial) {
      int ref[2], mvp[2][2];
      for (int l = 0; l < 2; l++) {
        const int rA = M.refc[l][6], rB = M.refc[l][1];
        int C = 5, rC = M.refc[l][5];
        if (rC == MREF_NA) { C = 0; rC = M.refc[l][0]; }
        auto minpos = [](int a, int b) { return (a >= 0 && b >= 0) ? (a < b ? a : b) : (a > b ? a : b); };
        int r = minpos(rA, minpos(rB, rC));
        if (r >= 0) {
          const int match = (rA == r) + (rB == r) + (rC == r);
          if (match == 1) { const int k = rA == r ? 6 : rB == r ? 1 : C; mvp[l][0] = M.mvc[l][k][0]; mvp[l][1] = M.mvc[l][k][1]; }
          else { mvp[l][0] = median3(M.mvc[l][6][0], M.mvc[l][1][0], M.mvc[l][C][0]); mvp[l][1] = median3(M.mvc[l][6][1], M.mvc[l][1][1], M.mvc[l][C][1]); }
        } else { r = -1; mvp[l][0] = mvp[l][1] = 0; }
        ref[l] = r;
      }
      if (ref[0] < 0 && ref[1] < 0) ref[0] = ref[1] = 0;
      for (int k = 0; k < 4; k++) {
        bool col_zero = false;
        if (!S.col_long_term && !col->intra[idx]) {
          const size_t o = (size_t)idx * 16 + kCorner[k];
          const int rc0 = col->ref[0][o], rc1 = col->ref[1][o];
          const int16_t* mvcol = nullptr;
          if (rc0 == 0) mvcol = &col->mv[0][o * 2];
          else if (rc0 < 0 && rc1 == 0) mvcol = &col->mv[1][o * 2];
          if (mvcol && mvcol[0] >= -1 && mvcol[0] <= 1 && mvcol[1] >= -1 && mvcol[1] <= 1) col_zero = true;
        }
        for (int l = 0; l < 2; l++) {
          dref[l][k] = ref[l];
          const bool zero = ref[l] < 0 || (ref[l] == 0 && col_zero);
          dmv[l][k][0] = zero ? 0 : mvp[l][0]; dmv[l][k][1] = zero ? 0 : mvp[l][1];
        }
      }
    } else {
      for (int k = 0; k < 4; k++) {
        dref[0][k] = dref[1][k] = 0;
        dmv[0][k][0] = dmv[0][k][1] = dmv[1][k][0] = dmv[1][k][1] = 0;
        if (col->intra[idx]) continue;
        const size_t o = (size_t)idx * 16 + kCorner[k];
        const int l_col = col->ref[0][o] >= 0 ? 0 : 1;
        const int16_t* mvcol = &col->mv[l_col][o * 2];
        const int id = col->ref_id[l_col][o];
        int r0 = 0;
        for (int i = 0; i < S.n_ref[0]; i++) if (S.list[0][i].pic_id == id) { r0 = i; break; }
        dref[0][k] = r0;
        int dsf;
        if (dist_scale(S.cur_poc, S.list[0][r0].poc, S.list[1][0].poc, S.list[0][r0].lt, &dsf)) {
          dmv[0][k][0] = (dsf * mvcol[0] + 128) >> 8; dmv[0][k][1] = (dsf * mvcol[1] + 128) >> 8;
          dmv[1][k][0] = dmv[0][k][0] - mvcol[0]; dmv[1][k][1] = dmv[0][k][1] - mvcol[1];
        } else {
          dmv[0][k][0] = mvcol[0]; dmv[0][k][1] = mvcol[1];
        }
      }
    }
  }
  if (sx.skip || sx.type == 0) {
    for (int l = 0; l < 2; l++)
      for (int k = 0; k < 4; k++) M.set(l, (k & 1) * 2, (k >> 1) * 2, 2, 2, dref[l][k], dmv[l][k][0], dmv[l][k][1]);
  } else if (sx.type <= 21) {
    const bool h = b_is_16x8(sx.type), v = b_is_8x16(sx.type);
    const int np = (h || v) ? 2 : 1;
    for (int l = 0; l < 2; l++)
      for (int p = 0; p < np; p++) {
        const int bx = v ? 2 * p : 0, by = h ? 2 * p : 0, w4 = v ? 2 : 4, h4 = h ? 2 : 4;
        if (!(b_part_lists(sx.type, p) & (1 << l))) { M.set(l, bx, by, w4, h4, MREF_NONE, 0, 0); continue; }
        const int ref = sx.ref[l][h ? 2 * p : p];
        int px, py;
        if (h) M.pred_16x8(l, p, ref, &px, &py);
        else if (v) M.pred_8x16(l, p, ref, &px, &py);
        else M.pred(l, 0, 0, 4, ref, &px, &py);
        M.set(l, bx, by, w4, h4, ref, px + sx.mvd[l][p][0], py + sx.mvd[l][p][1]);
      }
  } else {
    // temporal-direct 8x8s inside B_8x8, as the reference's two parsers have them while the OTHER 8x8s predict their vectors (its
    // output is the oracle): the CABAC parser (ParseInterBMotionInfoCabac, parse_mb_syn_cabac.cpp:943-970) enters their reference
    // indices into the cache BEFORE any vector is predicted — so even an earlier 8x8 sees them as neighbour C — whereas the CAVLC
    // parser (ParseInterBInfo, parse_mb_syn_cavlc.cpp:1618-1624) leaves their cache cells at "not in list".  Spatial direct follows
    // the decoding order in both.  The picture's arrays get the real indices either way (corrected below).
    const bool early = !S.direct_spatial && S.cabac;
    if (early)
      for (int l = 0; l < 2; l++)
        for (int k = 0; k < 4; k++)
          if (sx.sub[k] == 0) M.set(l, (k & 1) * 2, (k >> 1) * 2, 2, 2, dref[l][k], dmv[l][k][0], dmv[l][k][1]);
    for (int l = 0; l < 2; l++)
      for (int k = 0; k < 4; k++) {
        const int bx = (k & 1) * 2, by = (k >> 1) * 2;
        if (sx.sub[k] == 0 && early) continue;
        if (sx.sub[k] == 0) {
          // the reference leaves the reference-index CACHE of a temporal-direct 8x8 at "not in list" while the other 8x8s of the
          // macroblock predict their vectors (ParseInterBInfo, parse_mb_syn_cavlc.cpp:1618-1624: ref_idx_list is only filled for
          // spatial direct); the picture's arrays get the real index.  Its output is the oracle: the cells are corrected below
          M.set(l, bx, by, 2, 2, S.direct_spatial ? dref[l][k] : MREF_NONE, dmv[l][k][0], dmv[l][k][1]);
          continue;
        }
        if (!(b_sub_lists(sx.sub[k]) & (1 << l))) { M.set(l, bx, by, 2, 2, MREF_NONE, 0, 0); continue; }
        const int st = b_sub_shape(sx.sub[k]), ref = sx.ref[l][k];
        const int w4 = (st == 0 || st == 1) ? 2 : 1, h4 = (st == 0 || st == 2) ? 2 : 1, np = st == 0 ? 1 : st == 3 ? 4 : 2;
        // the reference index of the whole 8x8 is known before its vectors (ParseInterBInfo: the four cells are set first)
        for (int j = 0; j < np; j++) {
          const int sxx = bx + (st == 2 ? j : st == 3 ? (j & 1) : 0), syy = by + (st == 1 ? j : st == 3 ? (j >> 1) : 0);
          int px, py;
          M.pred(l, sxx, syy, w4, ref, &px, &py);
          M.set(l, sxx, syy, w4, h4, ref, px + sx.mvd[l][4 * k + j][0], py + sx.mvd[l][4 * k + j][1]);
        }
      }
  }
  if (sx.type == 22 && !sx.skip && !S.direct_spatial)
    for (int l = 0; l < 2; l++)
      for (int k = 0; k < 4; k++)
        if (sx.sub[k] == 0) M.set(l, (k & 1) * 2, (k >> 1) * 2, 2, 2, dref[l][k], dmv[l][k][0], dmv[l][k][1]);
  if (!emit_resolved(M, sx, S, S.wp, ax, axb)) return false;
  M.store(idx, S.list[0], S.list[1]);
  return true;
}

// the macroblock's cells -> hand-over records: picture slots per 8x8, final vectors in coding order, and how each 8x8 forms its sample
// prediction (DecMbAuxB: the lists that are motion compensated, the weighting formula and its weights).  `wp`: explicit weights of the
// slice (pred_weight_table of a P slice with weighted_pred_flag or a B slice with weighted_bipred_idc 1), else NULL.
inline bool emit_resolved(const MotionCtx& M, const BMbSyntax& sx, const BSliceCtx& S, const WpTable* wp, DecMbAux* ax, DecMbAuxB* axb) {
  const bool ex = wp && wp->on;
  const int ld[2] = {ex ? wp->log2[0] : S.implicit ? 5 : 0, ex ? wp->log2[1] : S.implicit ? 5 : 0};
  ax->wp_log2 = (uint8_t)(ld[0] | ld[1] << 4);
  const bool explicit_b = ex && S.n_ref[1] > 0;
  if (explicit_b) ax->flags |= DECAUX_EXPLICIT_B;
  for (int k = 0; k < 4; k++) {
    const int c0 = MotionCtx::cell((k & 1) * 2, (k >> 1) * 2);
    int r[2];
    for (int l = 0; l < 2; l++) {
      r[l] = M.refc[l][c0];
      if (r[l] >= S.n_ref[l]) return false;
      const int slot = r[l] < 0 ? -1 : S.list[l][r[l]].slot;
      if (r[l] >= 0 && slot < 0) return false;
      if (l == 0) ax->ref_idx[k] = (int8_t)slot; else axb->ref_idx[k] = (int8_t)slot;
      for (int j = 0; j < 4; j++) {
        const int c = MotionCtx::cell((k & 1) * 2 + (j & 1), (k >> 1) * 2 + (j >> 1));
        int16_t* d = l == 0 ? ax->mvd[4 * k + j] : axb->mv[4 * k + j];
        d[0] = r[l] < 0 ? 0 : M.mvc[l][c][0]; d[1] = r[l] < 0 ? 0 : M.mvc[l][c][1];
      }
    }
    const int lists = (r[0] >= 0 ? 1 : 0) | (r[1] >= 0 ? 2 : 0);
    // The reference's GetInterBPred (rec_mb.cpp:737-827) motion compensates both lists of a two-list 16x8 / 8x16 partition into the
    // same destination before it combines that destination with the list-1 prediction of the second buffer, and advances the
    // destination of the second partition twice.  So the FIRST partition is the two-list formula on its list-1 prediction twice
    // (weights of refIdxL0 and refIdxL1: with default or implicit weights, or any w0 + w1 = 2^(ld + 1) and no offsets, that is the
    // list-1 prediction itself), and the SECOND is its list-0 prediction, unweighted: the combined samples land outside the macroblock
    // and the one-list weighting only runs for one-list partitions.  The vectors and reference indices stay as coded (neighbours'
    // prediction, direct modes, the filter).
    int quirk = 0;                                                 // 1 / 2: first / second such partition
    if (!sx.skip && sx.type >= 4 && sx.type <= 21) {
      const int part = b_is_16x8(sx.type) ? (k >> 1) : (k & 1);
      if (b_part_lists(sx.type, part) == 3) quirk = part + 1;
    }
    // A one-list 8x4 / 4x8 sub-macroblock of B_8x8: the reference weights its second half only (WeightPrediction runs once, after the
    // destination was advanced to the second sub-macroblock partition, rec_mb.cpp:934-944, :977-987).
    const bool direct = sx.skip || sx.type == 0 || (sx.type == 22 && sx.sub[k] == 0);
    const int shape = (sx.type == 22 && !direct && b_sub_lists(sx.sub[k]) != 3) ? b_sub_shape(sx.sub[k]) : 0;
    int pred = quirk == 1 ? (ex ? DECB_L1 | DECB_BI : DECB_L1) : quirk == 2 ? DECB_L0 : lists;
    if (lists == 3 && !quirk) pred |= DECB_BI;
    if (ex && lists != 3) pred |= DECB_WEIGHT | (shape == 1 ? DECB_LOWER : shape == 2 ? DECB_RIGHT : 0);
    axb->pred[k] = (uint8_t)pred;
    for (int pl = 0; pl < 3; pl++) {
      int w0 = 0, w1 = 0, o = 0;
      if ((pred & DECB_BI) && ex) {                                // explicit weights (8.4.2.3.2)
        w0 = wp->w[0][r[0]][pl][0]; w1 = wp->w[1][r[1]][pl][0];
        o = wp_bi_offset(wp->w[0][r[0]][pl][1], wp->w[1][r[1]][pl][1]);
      } else if (pred & DECB_BI) {                                 // implicit weights (8.4.2.3.1), else the plain average
        w1 = S.implicit ? 32 : 1;
        const RefEntry& e0 = S.list[0][r[0]];
        const RefEntry& e1 = S.list[1][r[1]];
        int dsf;
        if (S.implicit && dist_scale(S.cur_poc, e0.poc, e1.poc, e0.lt || e1.lt, &dsf) && (dsf >> 2) >= -64 && (dsf >> 2) <= 128) w1 = dsf >> 2;
        w0 = S.implicit ? 64 - w1 : 1;
      } else if (pred & DECB_WEIGHT) {
        const int l = (pred & DECB_L0) ? 0 : 1;
        w0 = wp->w[l][r[l]][pl][0]; o = wp->w[l][r[l]][pl][1];
      }
      axb->w0[4 * pl + k] = (int16_t)w0; axb->w1[4 * pl + k] = (int16_t)w1; axb->o[4 * pl + k] = (int8_t)o;
    }
#ifdef B2H264_WP_STATS
    if (explicit_b) {                                              // coverage counters (host build only, wp_formula.h)
      if (quirk) {
        const int sum = wp->w[0][r[0]][0][0] + wp->w[1][r[1]][0][0];
        if (sum != 1 << (ld[0] + 1) && (wp->w[0][r[0]][0][1] | wp->w[1][r[1]][0][1])) b2h264_wp_stat(quirk == 1 ? WPS_QUIRK_FIRST : WPS_QUIRK_SECOND, 1);
      }
      if (lists != 3) b2h264_wp_stat(lists == 1 ? WPS_SINGLE_L0 : WPS_SINGLE_L1, 1);
      else if (!direct) b2h264_wp_stat(sx.type == 3 ? WPS_BI_16x16 : b_is_16x8(sx.type) ? WPS_BI_16x8 : b_is_8x16(sx.type) ? WPS_BI_8x16 : WPS_BI_SUB, 1);
      if (direct) b2h264_wp_stat(S.direct_spatial ? WPS_SPATIAL_DIRECT : WPS_TEMPORAL_DIRECT, 1);
      if (sx.skip) b2h264_wp_stat(WPS_B_SKIP, 1);
      if (shape == 1 || shape == 2) b2h264_wp_stat(WPS_HALF, 1);
      if (quirk != 2) {                                            // the table entries whose values enter the samples
        for (int l = 0; l < 2; l++) {
          if (r[l] < 0) continue;
          if (r[l] > 0) b2h264_wp_stat(l ? WPS_REF_L1_GT0 : WPS_REF_L0_GT0, 1);
          if (wp->given[l][r[l]] != 3) b2h264_wp_stat(WPS_DEFAULTED, 1);
          for (int pl = 0; pl < 3; pl++) {
            const int w = wp->w[l][r[l]][pl][0], o = wp->w[l][r[l]][pl][1];
            if (w == -128) b2h264_wp_stat(WPS_WEIGHT_MIN, 1);
            if (w == 127) b2h264_wp_stat(WPS_WEIGHT_MAX, 1);
            if (o == -128) b2h264_wp_stat(WPS_OFFSET_MIN, 1);
            if (o == 127) b2h264_wp_stat(WPS_OFFSET_MAX, 1);
          }
        }
        if (ld[0] == 0) b2h264_wp_stat(WPS_DENOM_Y0, 1);
        if (ld[0] == 7) b2h264_wp_stat(WPS_DENOM_Y7, 1);
        if (ld[1] == 0) b2h264_wp_stat(WPS_DENOM_C0, 1);
        if (ld[1] == 7) b2h264_wp_stat(WPS_DENOM_C7, 1);
      }
    }
#endif
  }
  return true;
}

// a P macroblock of a slice with explicit weights travels RESOLVED like a B macroblock (list 0 only): its prediction is weighted per
// reference index, which the device — it knows picture slots, not indices — cannot look up.  Call after derive_p().
inline bool emit_resolved_p(const MotionCtx& M, const RefEntry* l0, int n_ref, const WpTable& wp, DecMbAux* ax, DecMbAuxB* axb) {
  BSliceCtx S;
  S.n_ref[0] = n_ref; S.n_ref[1] = 0;
  for (int i = 0; i < 33; i++) S.list[0][i] = l0[i];
  BMbSyntax sx;
  sx.skip = true;                                                  // no partition quirk applies (one list)
  return emit_resolved(M, sx, S, &wp, ax, axb);
}

}  // namespace b2h264
