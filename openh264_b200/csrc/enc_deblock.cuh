// enc_deblock.cuh — in-loop deblocking of one macroblock by one warp, one pixel line per lane (H.264 8.7).
// Restates DeblockingMbAvcbase / DeblockingBSCalc_c / DeblockingInterMb / DeblockingIntraMb
// (codec/encoder/core/src/deblocking.cpp:357-655) on top of the edge filters of mbk_deblock.cuh.
// Order inside an MB: luma vertical edges 0..3, luma horizontal edges 0..3 (chroma: edges 0 and 2); MBs in
// raster order (the device runs them as a wavefront with the same left / top / top-right dependencies).
#pragma once
#include <string.h>
#include "enc_types.h"
#include "mbk_deblock.cuh"

namespace mbk {

#ifdef __CUDACC__
extern __constant__ uint8_t c_alpha[52];
extern __constant__ uint8_t c_beta[52];
extern __constant__ uint8_t c_tc0[52][3];
#endif
extern uint8_t h_alpha[52];
extern uint8_t h_beta[52];
extern uint8_t h_tc0[52][3];
MBK_HD int tbl_alpha(int i) { return MBK_TBL(c_alpha, h_alpha)[i]; }
MBK_HD int tbl_beta(int i) { return MBK_TBL(c_beta, h_beta)[i]; }
MBK_HD int tbl_tc0(int i, int bs) { return bs == 0 ? -1 : MBK_TBL(c_tc0, h_tc0)[i][bs - 1]; }

// boundary strength of the 4 segments of one edge; dir 0 = vertical edge (left neighbour), 1 = horizontal
// motion of 4x4 block `blk` (raster) of a decoded macroblock for the filter: reference picture (slot, -1: list not used) and
// vector per list.  List 0 lives in MbInfo (dec_mb.cuh), list 1 of a B macroblock in its DecMbAuxB record (vectors in coding order).
MBK_HD void dbk_block_motion(const MbInfo* m, const DecMbAuxB* b, int blk, int r[2], int mv[2][2]) {
  r[0] = m->i4_mode[blk];
  mv[0][0] = r[0] < 0 ? 0 : m->mv[blk][0]; mv[0][1] = r[0] < 0 ? 0 : m->mv[blk][1];
  r[1] = -1; mv[1][0] = mv[1][1] = 0;
  if (b) {
    const int bx = blk & 3, by = blk >> 2, z = ((by >> 1) * 2 + (bx >> 1)) * 4 + (by & 1) * 2 + (bx & 1);
    r[1] = b->ref_idx[z >> 2];
    if (r[1] >= 0) { mv[1][0] = b->mv[z][0]; mv[1][1] = b->mv[z][1]; }
  }
}
MBK_HD bool dbk_mv_far(const int a[2], const int b[2]) { return iabs(a[0] - b[0]) >= 4 || iabs(a[1] - b[1]) >= 4; }

// boundary strength of segment `seg` (4 samples) of edge `edge`; dir 0 = vertical edge (left neighbour), 1 = horizontal.
// nb = the other macroblock for edge 0, else == cur.
template <bool BSL = true>
MBK_HD int dbk_bs(const MbInfo* cur, const MbInfo* nb, int dir, int edge, int seg,
                  bool ref_ids = false /* decoder: i4_mode holds the reference picture of every 4x4 block */,
                  const DecMbAuxB* cur_b = nullptr, const DecMbAuxB* nb_b = nullptr /* list 1 of a B macroblock, else NULL */) {
  const bool mb_edge = edge == 0;
  // q block in cur, p block in nb (raster 4x4 indices)
  const int q = dir == 0 ? seg * 4 + edge : edge * 4 + seg;
  const int p = dir == 0 ? (mb_edge ? seg * 4 + 3 : q - 1) : (mb_edge ? 12 + seg : q - 4);
  if (MBT_IS_INTRA(cur->mb_type) || MBT_IS_INTRA(nb->mb_type)) return mb_edge ? 4 : 3;
  if (!mb_edge && (cur->mb_type == MBT_PSKIP || (BSL && cur->mb_type == MBT_BSKIP))) return 0;
  if (cur->nnz[q] | nb->nnz[p]) return 2;
  if (BSL && (cur_b || nb_b)) {
    // a B macroblock on either side (DeblockingBSliceBsMarginalMBAvcbase / IN_SMB_EDGE_MV, deblocking.cpp:544, :95): strength 1
    // unless both blocks use the same set of reference pictures and their vectors — matched by picture — are close
    int rq[2], rp[2], mq[2][2], mp[2][2];
    dbk_block_motion(cur, cur_b, q, rq, mq);
    dbk_block_motion(nb, nb_b, p, rp, mp);
    int v = 1;
    if ((rq[0] == rp[0] && rq[1] == rp[1]) || (rq[0] == rp[1] && rq[1] == rp[0])) {
      if (rq[0] != rq[1]) v = rq[0] == rp[0] ? (dbk_mv_far(mq[0], mp[0]) || dbk_mv_far(mq[1], mp[1])) : (dbk_mv_far(mq[0], mp[1]) || dbk_mv_far(mq[1], mp[0]));
      else v = (dbk_mv_far(mq[0], mp[0]) || dbk_mv_far(mq[1], mp[1])) && (dbk_mv_far(mq[0], mp[1]) || dbk_mv_far(mq[1], mp[0]));
    }
    return v;
  }
  if (ref_ids && cur->i4_mode[q] != nb->i4_mode[p]) return 1;      // different reference pictures
  const int dx = cur->mv[q][0] - nb->mv[p][0], dy = cur->mv[q][1] - nb->mv[p][1];
  return (iabs(dx) >= 4 || iabs(dy) >= 4) ? 1 : 0;
}

// Working set of one macroblock's deblocking (shared memory on the device): the macroblock's samples plus the 4
// columns / rows of the left / top macroblock its edge-0 filters read and modify, the three MbInfo records and the 32
// boundary strengths.  The macroblock's own samples sit on 16-byte (luma) / 8-byte (chroma) boundaries so that they can
// be copied asynchronously.
enum { DBK_PY = 32, DBK_PC = 16, DBK_OY = 4 * DBK_PY + 16, DBK_OC = 4 * DBK_PC + 8 };
struct alignas(16) DbkTile {
  uint8_t y[20 * DBK_PY];          // rows -4..15: cols -4..-1 at bytes 12..15, cols 0..15 at bytes 16..31 (sample (0,0) at y[DBK_OY])
  uint8_t c[2][12 * DBK_PC];       // rows -4..7: cols -4..-1 at bytes 4..7, cols 0..7 at bytes 8..15 (sample (0,0) at c[pl][DBK_OC])
  MbInfo m[3];                     // cur, left, top
  uint8_t bs[2][4][4];             // boundary strength per direction, edge and 4-sample segment
};
struct alignas(16) DbkTileB : DbkTile {
  DecMbAuxB b[3];                  // decoder, pictures with B slices: list 1 of those of the three that are B macroblocks
};
static_assert(sizeof(MbInfo) % 8 == 0, "MbInfo is copied in 8-byte pieces");

// global -> shared copies of 16 / 8 bytes: asynchronous on the device (cp.async, waited for by dbk_cp_wait_prev), plain
// copies on the host
MBK_HD void dbk_cp16(void* s, const void* g) {
#ifdef __CUDA_ARCH__
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(s)), "l"(g) : "memory");
#else
  memcpy(s, g, 16);
#endif
}
MBK_HD void dbk_cp8(void* s, const void* g) {
#ifdef __CUDA_ARCH__
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(s)), "l"(g) : "memory");
#else
  memcpy(s, g, 8);
#endif
}
MBK_HD void dbk_cp_commit() {
#ifdef __CUDA_ARCH__
  asm volatile("cp.async.commit_group;" ::: "memory");
#endif
}
// every copy group but the one committed last has landed (in this lane: a warp_sync makes them visible to the warp)
MBK_HD void dbk_cp_wait_prev() {
#ifdef __CUDA_ARCH__
  asm volatile("cp.async.wait_group 1;" ::: "memory");
#endif
}
MBK_HD uint32_t& dbk_w32(uint8_t* p) { return *reinterpret_cast<uint32_t*>(p); }
MBK_HD uint32_t dbk_w32(const uint8_t* p) { return *reinterpret_cast<const uint32_t*>(p); }

// What the macroblock's filtering reads and depends on no other macroblock of the picture: its own samples, its MbInfo
// and the top neighbour's.  Issued one macroblock ahead on the device.
template <typename Tile>
MBK_HD void dbk_fetch_own(const EncFrameParams& p, const EncFramePtrs& f, int mbx, int mby, Tile& t) {
  const uint8_t* y = f.rec[0] + (size_t)(mby * 16) * p.rec_stride_y + mbx * 16;
  const size_t oc = (size_t)(mby * 8) * p.rec_stride_c + mbx * 8;
  for (int i = lane_id(); i < 32; i += MBK_WS) {
    if (i < 16) {
      dbk_cp16(t.y + DBK_OY + i * DBK_PY, y + (ptrdiff_t)i * p.rec_stride_y);
    } else {
      const int pl = (i - 16) >> 3, r = i & 7;
      dbk_cp8(t.c[pl] + DBK_OC + r * DBK_PC, f.rec[1 + pl] + oc + (ptrdiff_t)r * p.rec_stride_c);
    }
  }
  constexpr int kW = (int)(sizeof(MbInfo) / 8);
  const uint8_t* mi = reinterpret_cast<const uint8_t*>(f.mbi + mby * p.mb_w + mbx);
  for (int i = lane_id(); i < (mby > 0 ? 2 * kW : kW); i += MBK_WS) {
    const int k = i >= kW ? 1 : 0, w = i - k * kW;
    dbk_cp8(reinterpret_cast<uint8_t*>(&t.m[2 * k]) + 8 * w, mi - (ptrdiff_t)k * p.mb_w * (ptrdiff_t)sizeof(MbInfo) + 8 * w);
  }
}
// The left neighbour's 4 right columns and MbInfo: the tile `s` of the previous macroblock of the row holds them as they are
// after its filtering, which is what this macroblock's vertical edge 0 reads.  (s may be t: the host reuses one tile.)
template <typename Tile>
MBK_HD void dbk_carry_left(const Tile& s, Tile& t) {
  constexpr int kW = (int)(sizeof(MbInfo) / 4);
  for (int i = lane_id(); i < 32 + kW; i += MBK_WS) {
    if (i < 16) {
      dbk_w32(t.y + (4 + i) * DBK_PY + 12) = dbk_w32(s.y + (4 + i) * DBK_PY + 28);
    } else if (i < 32) {
      const int pl = (i - 16) >> 3, r = i & 7;
      dbk_w32(t.c[pl] + (4 + r) * DBK_PC + 4) = dbk_w32(s.c[pl] + (4 + r) * DBK_PC + 12);
    } else {
      reinterpret_cast<uint32_t*>(&t.m[1])[i - 32] = reinterpret_cast<const uint32_t*>(&s.m[0])[i - 32];
    }
  }
}
// The 4 bottom rows of the top neighbour: final once the row above has filtered the macroblock above-right.
template <typename Tile>
MBK_HD void dbk_fetch_top(const EncFrameParams& p, const EncFramePtrs& f, int mbx, int mby, Tile& t) {
  if (mby == 0) return;
  const uint8_t* y = f.rec[0] + (size_t)(mby * 16) * p.rec_stride_y + mbx * 16;
  const size_t oc = (size_t)(mby * 8) * p.rec_stride_c + mbx * 8;
  for (int i = lane_id(); i < 12; i += MBK_WS) {
    if (i < 4) {
      *reinterpret_cast<uint4*>(t.y + i * DBK_PY + 16) = *reinterpret_cast<const uint4*>(y + (ptrdiff_t)(i - 4) * p.rec_stride_y);
    } else {
      const int pl = (i - 4) >> 2, r = i & 3;
      *reinterpret_cast<uint2*>(t.c[pl] + r * DBK_PC + 8) = *reinterpret_cast<const uint2*>(f.rec[1 + pl] + oc + (ptrdiff_t)(r - 4) * p.rec_stride_c);
    }
  }
}

// One direction of the macroblock's edges, one LINE PER LANE: lanes 0..15 the 16 luma lines, lanes 16..31 the 8 + 8 chroma
// lines (device; the host runs the same loop).  A lane runs edges 0..3 of its line in order.  Exact because H.264 8.7
// filters every vertical edge of a macroblock before any horizontal edge and the lines across edges of one direction are
// independent.  α / β / tc0 are looked up once per lane for edge 0 (mean QP with the neighbour) and once for the inner edges.
template <typename Tile>
MBK_HD void dbk_filter_dir(Tile& t, int dir, int off_a, int off_b) {
  const MbInfo* cur = &t.m[0];
  const MbInfo* nb = &t.m[1 + dir];
  for (int l = lane_id(); l < 32; l += MBK_WS) {
    const bool luma = l < 16;
    const int k = l - 16, ln = luma ? l : (k & 7);
    const int qp_in = luma ? cur->qp : cur->qp_c, qp_e0 = (qp_in + (luma ? nb->qp : nb->qp_c) + 1) >> 1;
    const int ia0 = clip3(qp_e0 + off_a, 0, 51), ia1 = clip3(qp_in + off_a, 0, 51);
    const int a0 = tbl_alpha(ia0), b0 = tbl_beta(clip3(qp_e0 + off_b, 0, 51)), tc0 = tbl_tc0(ia0, 1) | tbl_tc0(ia0, 2) << 8 | tbl_tc0(ia0, 3) << 16;
    const int a1 = tbl_alpha(ia1), b1 = tbl_beta(clip3(qp_in + off_b, 0, 51)), tc1 = tbl_tc0(ia1, 1) | tbl_tc0(ia1, 2) << 8 | tbl_tc0(ia1, 3) << 16;
    const uint8_t* bs = &t.bs[dir][0][luma ? (l >> 2) : (ln >> 1)];
    if (luma) {
      const int sx = dir == 0 ? 1 : DBK_PY;
      uint8_t* line = t.y + DBK_OY + (dir == 0 ? l * DBK_PY : l);
      for (int e = 0; e < 4; e++) {
        const int s = bs[4 * e], a = e ? a1 : a0, b = e ? b1 : b0;
        if (s == 0) continue;
        if (s == 4) deblock_luma_eq4_line(line + 4 * e * sx, sx, a, b);
        else deblock_luma_lt4_line(line + 4 * e * sx, sx, a, b, ((e ? tc1 : tc0) >> (8 * (s - 1))) & 255);
      }
    } else {                                                   // chroma: edges 0 and 2 only
      const int sx = dir == 0 ? 1 : DBK_PC;
      uint8_t* line = t.c[k >> 3] + DBK_OC + (dir == 0 ? ln * DBK_PC : ln);
      for (int e = 0; e < 4; e += 2) {
        const int s = bs[4 * e], a = e ? a1 : a0, b = e ? b1 : b0;
        if (s == 0) continue;
        if (s == 4) deblock_chroma_eq4_line(line + 2 * e * sx, sx, a, b);
        else deblock_chroma_lt4_line(line + 2 * e * sx, sx, a, b, (((e ? tc1 : tc0) >> (8 * (s - 1))) & 255) + 1);
      }
    }
  }
}

// Filters the staged macroblock and writes back what changed: the macroblock, the 4 columns to its left (if any), the 3
// luma rows / 1 chroma row above (if any).  Nothing is written when every boundary strength is 0.
// BSL: the picture may hold B macroblocks or macroblocks with the 8x8 transform (decoder only: Main / High tools).  The
// encoder and B-free decoder pictures run the BSL = false instantiation, whose code and shared-memory footprint are those of
// the single-list filter.
template <bool BSL, typename Tile>
MBK_HD void dbk_filter_store(const EncFrameParams& p, const EncFramePtrs& f, int mbx, int mby, Tile& t) {
  const MbInfo* cur = &t.m[0];
  // decoder: per-slice control travels in MbInfo::p16x16_mv (dec_mb.cuh): disable_deblocking_filter_idc, FilterOffsetA / B and the
  // slice number (idc 2: edges between slices stay unfiltered).  The encoder's control is per picture, and its slices are raster
  // runs: a neighbour is in another slice when its address is below the first of the macroblock's slice (EncFramePtrs::slice_first,
  // present whenever the encoder codes idc 2; bLeftBsValid / bTopBsValid, deblocking.cpp:367-368)
  int idc = p.dbk_idc, off_a = p.dbk_off_a, off_b = p.dbk_off_b;
  if (p.dec_mode) {
    const int v = (uint16_t)cur->p16x16_mv[1];
    idc = v & 3; off_a = ((v >> 2) & 31) - 16; off_b = ((v >> 7) & 31) - 16;
  }
  if (idc == 1) return;
  // idc 2: edges between slices stay unfiltered
  bool cut_left = false, cut_top = false;
  if (idc == 2) {
    if (p.dec_mode) { cut_left = t.m[1].p16x16_mv[0] != cur->p16x16_mv[0]; cut_top = t.m[2].p16x16_mv[0] != cur->p16x16_mv[0]; }
    else {
      const int idx = mby * p.mb_w + mbx, first = f.slice_first[idx];
      cut_left = idx - 1 < first; cut_top = idx - p.mb_w < first;
    }
  }
  const bool have_left = mbx > 0 && !cut_left;
  const bool have_top = mby > 0 && !cut_top;
  [[maybe_unused]] const DecMbAuxB* lb[3] = {nullptr, nullptr, nullptr};
  if constexpr (BSL) if (f.dec_aux_b) {                                         // a picture with B slices: list 1 of the B macroblocks among the three
    constexpr int kWb = (int)(sizeof(DecMbAuxB) / 4);
    const int idx = mby * p.mb_w + mbx, nidx[3] = {idx, idx - 1, idx - p.mb_w};
    for (int k = 0; k < 3; k++) {
      if ((k == 1 && mbx == 0) || (k == 2 && mby == 0) || !MBT_IS_B(t.m[k].mb_type)) continue;
      for (int i = lane_id(); i < kWb; i += MBK_WS)
        reinterpret_cast<uint32_t*>(&t.b[k])[i] = reinterpret_cast<const uint32_t*>(f.dec_aux_b + nidx[k])[i];
      lb[k] = &t.b[k];
    }
    warp_sync();
  }
  // all 32 boundary strengths at once, one per lane: direction, edge, segment
  int any = 0;
  for (int i = lane_id(); i < 32; i += MBK_WS) {
    const int dir = i >> 4, edge = (i >> 2) & 3, seg = i & 3;
    bool on = edge != 0 || (dir ? have_top : have_left);
    if constexpr (BSL) on = on && !(cur->t8x8 && (edge & 1));  // 8x8 transform: the inner 4x4 edges are no transform edges (chroma has none there)
    int v = 0;
    if (on) {
      const MbInfo* other = edge == 0 ? (dir ? &t.m[2] : &t.m[1]) : cur;
      if constexpr (BSL) v = dbk_bs<true>(cur, other, dir, edge, seg, p.dec_mode != 0, lb[0], edge == 0 ? (dir ? lb[2] : lb[1]) : lb[0]);
      else v = dbk_bs<false>(cur, other, dir, edge, seg, p.dec_mode != 0);
    }
    t.bs[dir][edge][seg] = (uint8_t)v;
    any |= v;
  }
#ifdef __CUDA_ARCH__
  any = __any_sync(MBK_FULL, any);
#endif
  if (!any) return;
  warp_sync();
  dbk_filter_dir(t, 0, off_a, off_b);
  warp_sync();
  dbk_filter_dir(t, 1, off_a, off_b);
  warp_sync();
  uint8_t* y = f.rec[0] + (size_t)(mby * 16) * p.rec_stride_y + mbx * 16;
  const size_t oc = (size_t)(mby * 8) * p.rec_stride_c + mbx * 8;
  for (int i = lane_id(); i < 32; i += MBK_WS) {
    if (i < 16) {
      uint8_t* g = y + (ptrdiff_t)i * p.rec_stride_y;
      const uint8_t* r = t.y + (4 + i) * DBK_PY;
      *reinterpret_cast<uint4*>(g) = *reinterpret_cast<const uint4*>(r + 16);
      if (mbx > 0) dbk_w32(g - 4) = dbk_w32(r + 12);
    } else {
      const int pl = (i - 16) >> 3, rr = i & 7;
      uint8_t* g = f.rec[1 + pl] + oc + (ptrdiff_t)rr * p.rec_stride_c;
      const uint8_t* r = t.c[pl] + (4 + rr) * DBK_PC;
      *reinterpret_cast<uint2*>(g) = *reinterpret_cast<const uint2*>(r + 8);
      if (mbx > 0) dbk_w32(g - 4) = dbk_w32(r + 4);
    }
  }
  if (mby > 0) {
    for (int i = lane_id(); i < 5; i += MBK_WS) {
      if (i < 3) *reinterpret_cast<uint4*>(y + (ptrdiff_t)(i - 3) * p.rec_stride_y) = *reinterpret_cast<const uint4*>(t.y + (i + 1) * DBK_PY + 16);
      else *reinterpret_cast<uint2*>(f.rec[i - 2] + oc - p.rec_stride_c) = *reinterpret_cast<const uint2*>(t.c[i - 3] + 3 * DBK_PC + 8);
    }
  }
}

// One macroblock row, left to right, with the two tiles t[0], t[1] of the calling warp.  The next macroblock's own samples
// are fetched before this one is filtered; only the 4 rows above wait for the row above: wait_above(n) returns once that row
// has finished its first n macroblocks.  done(x) publishes that macroblock x is finished.
template <bool BSL, typename Tile, typename WaitAbove, typename Done>
MBK_HD void deblock_row_t(const EncFrameParams& p, const EncFramePtrs& f, int mby, Tile* t, WaitAbove wait_above, Done done) {
  const int mb_w = p.mb_w;
  dbk_fetch_own(p, f, 0, mby, t[0]);
  dbk_cp_commit();
  for (int x = 0; x < mb_w; x++) {
    Tile& c = t[x & 1];
    if (x > 0) dbk_carry_left(t[(x - 1) & 1], c);
    warp_sync();                                       // the tile of x - 1 is read: it takes the samples of x + 1
    if (x + 1 < mb_w) dbk_fetch_own(p, f, x + 1, mby, t[(x + 1) & 1]);
    dbk_cp_commit();
    if (mby > 0) wait_above(x + 2 < mb_w ? x + 2 : mb_w);
    dbk_fetch_top(p, f, x, mby, c);
    dbk_cp_wait_prev();
    warp_sync();
    dbk_filter_store<BSL>(p, f, x, mby, c);
    done(x);
  }
}

// Host build: the macroblocks of a picture in raster order, all with the same tile (which still holds the previous macroblock
// of the row, so the left columns are carried over as on the device).
template <bool BSL, typename Tile>
MBK_HD void deblock_one_mb_t(const EncFrameParams& p, const EncFramePtrs& f, int mbx, int mby, Tile& t) {
  if (mbx > 0) dbk_carry_left(t, t);
  warp_sync();
  dbk_fetch_own(p, f, mbx, mby, t);
  dbk_cp_commit();
  dbk_fetch_top(p, f, mbx, mby, t);
  dbk_cp_commit();
  dbk_cp_wait_prev();
  warp_sync();
  dbk_filter_store<BSL>(p, f, mbx, mby, t);
  warp_sync();
}
MBK_HD void deblock_one_mb(const EncFrameParams& p, const EncFramePtrs& f, int mbx, int mby, DbkTile& t) { deblock_one_mb_t<false>(p, f, mbx, mby, t); }
MBK_HD void deblock_one_mb_b(const EncFrameParams& p, const EncFramePtrs& f, int mbx, int mby, DbkTileB& t) { deblock_one_mb_t<true>(p, f, mbx, mby, t); }

}  // namespace mbk
