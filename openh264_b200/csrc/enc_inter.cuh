// enc_inter.cuh — P-slice macroblock mode decision and coding for one macroblock owned by one warp.
// Restates the decision order of
//   WelsMdInterMb / WelsMdInterJudgePskip / WelsMdPSkipEnc / WelsMdP16x16 / WelsMdP16x8 / WelsMdP8x16 /
//   WelsMdP8x8 / WelsMdInterFinePartition / WelsMdInterMbRefinement / WelsMdFirstIntraMode /
//   WelsMdInterEncode / WelsMdInterDoubleCheckPskip      codec/encoder/core/src/svc_base_layer_md.cpp:978-2021
//   MeRefineFracPixel, PredictSad, PredictSadSkip, FillNeighborCacheInterWithoutBGD  .../src/md.cpp:132-250,575-790,826-910
//   PredMv, PredInter16x8Mv, PredInter8x16Mv, PredSkipMv and the cache updates        .../src/mv_pred.cpp
//   WelsEncInterY, WelsTryPYskip, WelsTryPUVskip                                      .../src/svc_encode_mb.cpp:180-383
// for CAMERA_VIDEO_REAL_TIME, complexity MEDIUM/HIGH (SATD costs, all partitions), no BGD/AQ/scene detect.
#pragma once
#include "enc_mb.cuh"
#include "mbk_mc.cuh"
#include "mbk_me.cuh"
#include "mbk_pix8.cuh"

namespace mbk {

// motion cache: 6 columns x 5 rows, index = row*6 + col; the MB's 4x4 blocks sit at rows 1..4, cols 1..4
// (g_kuiCache30ScanIdx, common_tables.cpp): cache index of 4x4 block k (coding order)
MBK_HD int cache30(int k) { return 7 + blk_y(k) * 6 + blk_x(k); }


MBK_HD int median3(int a, int b, int c) {
  const int mn = a < b ? a : b, mx = a < b ? b : a;
  return c < mn ? mn : (c > mx ? mx : c);
}

// ---- neighbour caches (FillNeighborCacheInterWithoutBGD, md.cpp:132) ----------------------------------
// ref_ids: the decoder keeps, per 4x4 block of an inter macroblock, the picture slot of its reference in MbInfo::i4_mode
// (unused for inter macroblocks otherwise); the encoder has one reference picture (index 0 everywhere)
// availability bit of neighbour slot k (0 TL, 1 T, 2 TR, 3 L) without a lane-indexed table (that would live in local memory)
MBK_HD int nb_slot_bit(int k) {
  return (int)((((uint32_t)NB_TOPLEFT) | ((uint32_t)NB_TOP << 8) | ((uint32_t)NB_TOPRIGHT << 16) | ((uint32_t)NB_LEFT << 24)) >> (8 * k)) & 0xff;
}
MBK_FN void fill_inter_cache(const MbCtx& c, MbScratch& s, bool ref_ids = false) {
  // one lane per cache cell: cells 0..5 = top-left, top x4, top-right; cells 6,12,18,24 = left column
  for (int ci = lane_id(); ci < 30; ci += MBK_WS) {
    int k = -1, blk = 0;                       // neighbour slot (0 TL, 1 T, 2 TR, 3 L) and its 4x4 block (raster)
    if (ci == 0) { k = 0; blk = 15; }
    else if (ci <= 4) { k = 1; blk = 12 + ci - 1; }
    else if (ci == 5) { k = 2; blk = 12; }
    else if (ci % 6 == 0) { k = 3; blk = 4 * (ci / 6 - 1) + 3; }
    int16_t mx = 0, my = 0;
    int8_t ref = 0;
    if (k >= 0) {
      const bool avail = (c.nb & nb_slot_bit(k)) != 0;
      const MbInfo* n = &s.nbi[k];
      if (avail && MBT_IS_INTER(n->mb_type)) { mx = n->mv[blk][0]; my = n->mv[blk][1]; if (ref_ids) ref = n->i4_mode[blk]; }
      else ref = avail ? REF_NOT_IN_LIST : REF_NOT_AVAIL;
    } else if (ci == 9 || ci == 11 || ci == 17 || ci == 21 || ci == 23) {
      ref = REF_NOT_AVAIL;                     // blocks whose top-right neighbour is never available
    }
    s.mvc[ci][0] = mx; s.mvc[ci][1] = my; s.refc[ci] = ref;
  }
  for (int k = lane_id(); k < 4; k += MBK_WS) {
    const bool avail = (c.nb & nb_slot_bit(k)) != 0;
    const MbInfo* n = &s.nbi[k];
    const bool inter = avail && MBT_IS_INTER(n->mb_type);
    const bool skip = inter && n->mb_type == MBT_PSKIP;
    s.sadc[k] = inter ? s.nb_sad[k] : 0;
    s.skip_flag[k] = skip;
    s.sad_skip[k] = skip ? s.nb_skip_sad[k] : 0;
  }
  warp_sync();
}

// ---- motion vector prediction (mv_pred.cpp:45-150) ----------------------------------------------------
MBK_FN void pred_mv(const MbScratch& s, int blk /*coding idx*/, int part_w, int ref, int* px, int* py) {
  const int left = cache30(blk) - 1, top = cache30(blk) - 6;
  const int lr = s.refc[left], tr = s.refc[top], rtr = s.refc[top + part_w];
  int dr, dmx, dmy;
  if (rtr == REF_NOT_AVAIL) { dr = s.refc[top - 1]; dmx = s.mvc[top - 1][0]; dmy = s.mvc[top - 1][1]; }
  else { dr = rtr; dmx = s.mvc[top + part_w][0]; dmy = s.mvc[top + part_w][1]; }
  if (tr == REF_NOT_AVAIL && dr == REF_NOT_AVAIL && lr != REF_NOT_AVAIL) { *px = s.mvc[left][0]; *py = s.mvc[left][1]; return; }
  const int match = (ref == lr ? 1 : 0) | (ref == tr ? 2 : 0) | (ref == dr ? 4 : 0);
  if (match == 1) { *px = s.mvc[left][0]; *py = s.mvc[left][1]; }
  else if (match == 2) { *px = s.mvc[top][0]; *py = s.mvc[top][1]; }
  else if (match == 4) { *px = dmx; *py = dmy; }
  else { *px = median3(s.mvc[left][0], s.mvc[top][0], dmx); *py = median3(s.mvc[left][1], s.mvc[top][1], dmy); }
}
MBK_HD void pred_16x8_mv(const MbScratch& s, int blk, int ref, int* px, int* py) {
  if (blk == 0) { if (ref == s.refc[1]) { *px = s.mvc[1][0]; *py = s.mvc[1][1]; return; } }
  else { if (ref == s.refc[18]) { *px = s.mvc[18][0]; *py = s.mvc[18][1]; return; } }
  pred_mv(s, blk, 4, ref, px, py);
}
MBK_HD void pred_8x16_mv(const MbScratch& s, int blk, int ref, int* px, int* py) {
  if (blk == 0) { if (ref == s.refc[6]) { *px = s.mvc[6][0]; *py = s.mvc[6][1]; return; } }
  else {
    int di = 5;
    if (s.refc[5] == REF_NOT_AVAIL) di = 2;
    if (ref == s.refc[di]) { *px = s.mvc[di][0]; *py = s.mvc[di][1]; return; }
  }
  pred_mv(s, blk, 2, ref, px, py);
}
MBK_HD void pred_skip_mv(const MbScratch& s, int* px, int* py, int ref0 = 0 /* id of reference index 0 */) {
  const int lr = s.refc[6], tr = s.refc[1];
  if (lr == REF_NOT_AVAIL || tr == REF_NOT_AVAIL || (lr == ref0 && s.mvc[6][0] == 0 && s.mvc[6][1] == 0) ||
      (tr == ref0 && s.mvc[1][0] == 0 && s.mvc[1][1] == 0)) { *px = 0; *py = 0; return; }
  pred_mv(s, 0, 4, ref0, px, py);
}
// writes (ref 0, mv) into a w4 x h4 rectangle of cache cells starting at block `blk`
MBK_HD void cache_set(MbScratch& s, int blk, int w4, int h4, int mvx, int mvy, int ref = 0) {
  if (lane_id() == 0) {
    const int c0 = cache30(blk);
    for (int y = 0; y < h4; y++)
      for (int x = 0; x < w4; x++) { s.mvc[c0 + 6 * y + x][0] = (int16_t)mvx; s.mvc[c0 + 6 * y + x][1] = (int16_t)mvy; s.refc[c0 + 6 * y + x] = (int8_t)ref; }
  }
  warp_sync();
}
MBK_HD void mb_mv_set(MbScratch& s, int blk, int w4, int h4, int mvx, int mvy) {
  if (lane_id() == 0) {
    const int x0 = blk_x(blk), y0 = blk_y(blk);
    for (int y = 0; y < h4; y++)
      for (int x = 0; x < w4; x++) { s.info.mv[(y0 + y) * 4 + x0 + x][0] = (int16_t)mvx; s.info.mv[(y0 + y) * 4 + x0 + x][1] = (int16_t)mvy; }
  }
  warp_sync();
}

// ---- SAD predictors (md.cpp:826-910) ---------------------------------------------------------------------
MBK_HD int predict_sad(const MbScratch& s) {
  const int rb = s.refc[1], ra = s.refc[6];
  int rc = s.refc[5], sc = s.sadc[2];
  const int sb = s.sadc[1], sa = s.sadc[3];
  if (rc == REF_NOT_AVAIL) { rc = s.refc[0]; sc = s.sadc[0]; }
  int pred;
  if (rb == REF_NOT_AVAIL && rc == REF_NOT_AVAIL && ra != REF_NOT_AVAIL) pred = sa;
  else {
    const int m = (0 == ra ? 1 : 0) | (0 == rb ? 2 : 0) | (0 == rc ? 4 : 0);
    pred = m == 1 ? sa : m == 2 ? sb : m == 4 ? sc : median3(sa, sb, sc);
  }
  const int t = pred << 6;
  return ((t - (t >> 3) + (t >> 5)) + 32) >> 6;
}
MBK_HD int predict_sad_skip(const MbScratch& s) {
  const int rb = s.refc[1], ra = s.refc[6];
  int rc = s.refc[5];
  const int sb = s.skip_flag[1] ? s.sad_skip[1] : 0, sa = s.skip_flag[3] ? s.sad_skip[3] : 0;
  int sc = s.skip_flag[2] ? s.sad_skip[2] : 0, rskip = s.skip_flag[2];
  if (rc == REF_NOT_AVAIL) { rc = s.refc[0]; sc = s.skip_flag[0] ? s.sad_skip[0] : 0; rskip = s.skip_flag[0]; }
  if (rb == REF_NOT_AVAIL && rc == REF_NOT_AVAIL && ra != REF_NOT_AVAIL) return sa;
  const int m = ((0 == ra && s.skip_flag[3]) ? 1 : 0) | ((0 == rb && s.skip_flag[1]) ? 2 : 0) | ((0 == rc && rskip) ? 4 : 0);
  return m == 1 ? sa : m == 2 ? sb : m == 4 ? sc : median3(sa, sb, sc);
}

// ---- reference plane access ------------------------------------------------------------------------------
MBK_HD const uint8_t* ref_luma(const MbCtx& c, int px, int py) {
  return c.f.ref[0] + (ptrdiff_t)(c.mby * 16 + py) * c.p.rec_stride_y + c.mbx * 16 + px;
}
MBK_HD const uint8_t* ref_chroma(const MbCtx& c, int pl, int px, int py) {
  return c.f.ref[pl] + (ptrdiff_t)(c.mby * 8 + py) * c.p.rec_stride_c + c.mbx * 8 + px;
}

// chroma prediction of a (w x h luma) partition at luma offset (ox, oy) with quarter-pel luma mv
MBK_STAGE void mc_chroma_part(const MbCtx& c, uint8_t* dst /*Cb, Cr at +64, stride 8*/, int ox, int oy, int w, int h, int mvx, int mvy) {
  const int cx = ox >> 1, cy = oy >> 1;
  warp_mc_chroma_pair(ref_chroma(c, 1, cx + (mvx >> 3), cy + (mvy >> 3)), ref_chroma(c, 2, cx + (mvx >> 3), cy + (mvy >> 3)),
                      c.p.rec_stride_c, dst + cy * 8 + cx, 8, mvx, mvy, w >> 1, h >> 1);
  warp_sync();
}

enum { QP_STRIDE = 32 };                  // row pitch of the staged windows and half-sample planes

// ---- P-skip test (WelsMdPSkipEnc :1423, WelsTryPYskip / WelsTryPUVskip svc_encode_mb.cpp:325,352) -----------
struct SkipResult { bool ok; int cost_luma; int cost_skip; int mvx, mvy; };

// Outcomes of the skip test, in the order the reference decides them.  The host build counts them (and the prediction
// phases the test ran with) so that tests can show which branches their clips reach.
enum { SKIP_RANGE = 0, SKIP_SAD_OK, SKIP_Y_LEVEL, SKIP_Y_CTR, SKIP_UV_DC, SKIP_UV_LEVEL, SKIP_CB_CTR, SKIP_CR_CTR, SKIP_DCT_OK,
       SKIP_OUTCOMES };
inline uint64_t g_skip_outcome[SKIP_OUTCOMES];
inline uint64_t g_skip_phase_luma, g_skip_phase_chroma;      // bit (mvx & 3) + 4 (mvy & 3) / (mvx & 7) + 8 (mvy & 7)
#ifndef __CUDA_ARCH__
#define SKIP_COUNT(i) (g_skip_outcome[i]++)
#else
#define SKIP_COUNT(i) ((void)0)
#endif

// One 4x4 block of the residual tests: b = 0..15 the luma blocks (coding order), 16..19 Cb and 20..23 Cr (raster); the
// residual is the source minus s.skip_pred.  mx / ctr: largest quantised level and JVT-O079 score (WelsTryPYskip /
// WelsTryPUVskip: the chroma AC blocks are quantised WITH their DC still in place, their scan skips it), dc = the
// unquantised DC (chroma 2x2 test), satd = SATD of the luma block.
struct SkipBlk { int mx, ctr, dc, satd; };
MBK_HD SkipBlk skip_block(const MbCtx& c, const MbScratch& s, int b, bool tests, bool satd) {
  SkipBlk r = {0, 0, 0, 0};
  const bool luma = b < 16;
  const int t = b & 3, st = luma ? 16 : 8;
  const int o = luma ? blk_y(b) * 64 + blk_x(b) * 4 : 64 * ((b - 16) >> 2) + (t >> 1) * 32 + (t & 1) * 4;
  const uint8_t* cur = (luma ? s.cur_y : s.cur_c) + o;
  const uint8_t* pr = s.skip_pred + (luma ? 0 : 256) + o;
  uint32_t a[4], p[4];
#pragma unroll
  for (int y = 0; y < 4; y++) {
    a[y] = *reinterpret_cast<const uint32_t*>(cur + y * st);
    p[y] = *reinterpret_cast<const uint32_t*>(pr + y * st);
  }
  if (satd && luma) r.satd = satd4x4_words(a, p);
  if (tests) {
    int16_t d[16], l[16];
    dct4x4_rows(d, a, p);
    r.dc = d[0];
    const int q = luma ? c.qp : c.qp_c;
    r.mx = (uint16_t)quant4x4_max(d, tbl_quant_ff(q), tbl_quant_mf(q));
    if (r.mx == 1) {
      if (luma) scan4x4_dcac(l, d);
      else scan4x4_ac(l, d);
      r.ctr = single_ctr4x4(l);
    }
  }
  return r;
}
// 2x2 chroma DC test of WelsTryPUVskip from the four DCs of a plane (raster)
MBK_HD bool skip_dc_fails(const MbCtx& c, const int16_t dc[4]) {
  const int16_t* ff = tbl_quant_ff(c.qp_c);
  const int16_t* mf = tbl_quant_mf(c.qp_c);
  return hadamard_quant2x2_skip(dc, (int16_t)(ff[0] << 1), (int16_t)(mf[0] >> 1)) != 0;
}
// A block's share of its plane's score: the reference walks the blocks serially and returns at the first failing test, and
// every term of its running score is >= 0, so a plane passes iff no block has a level > 1 (nor, chroma, the DC test fails)
// AND the summed score stays below the threshold — order independent.  A failing block adds the threshold itself, a
// block's score is capped there: each plane's sum fits 8 bits, and the three planes are summed in one reduction.
MBK_HD int skip_share(const SkipBlk& b, bool fail, int thr) { return (fail || b.mx > 1) ? thr : (b.ctr < thr ? b.ctr : thr); }
MBK_HD bool skip_sum_ok(int sum) { return (sum & 0xff) < 6 && ((sum >> 8) & 0xff) < 7 && (sum >> 16) < 7; }

struct SkipPass { bool ok; int satd; };
// the residual tests (tests) and the luma SATD (satd) of the skip prediction in one warp pass: lanes 0..15 take the luma
// blocks, 16..23 the chroma blocks; the chroma DC test exchanges the DCs of a plane among its four lanes
MBK_STAGE SkipPass skip_residual_pass(const MbCtx& c, const MbScratch& s, bool tests, bool satd) {
  SkipPass r;
#ifdef __CUDA_ARCH__
  const int l = lane_id();
  SkipBlk b = {0, 0, 0, 0};
  if (l < 24) b = skip_block(c, s, l, tests, satd);
  r.ok = true;
  if (tests) {
    int16_t dc[4];
#pragma unroll
    for (int t = 0; t < 4; t++) dc[t] = (int16_t)__shfl_sync(MBK_FULL, b.dc, (l & ~3) + t);
    int v = 0;
    if (l < 16) v = skip_share(b, false, 6);
    else if (l < 24) v = skip_share(b, (l & 3) == 0 && skip_dc_fails(c, dc), 7) << (l < 20 ? 8 : 16);
    r.ok = skip_sum_ok(warp_sum(v));
  }
  r.satd = satd ? warp_sum(b.satd) : 0;
#else
  SkipBlk b[24];
  for (int k = 0; k < 24; k++) b[k] = skip_block(c, s, k, tests, satd);
  r.ok = true;
  r.satd = 0;
  for (int k = 0; k < 16; k++) r.satd += b[k].satd;
  if (tests) {
    bool dcf[2];
    int sum = 0;
    for (int k = 0; k < 16; k++) sum += skip_share(b[k], false, 6);
    for (int uv = 0; uv < 2; uv++) {
      const int16_t dc[4] = {(int16_t)b[16 + 4 * uv].dc, (int16_t)b[17 + 4 * uv].dc, (int16_t)b[18 + 4 * uv].dc, (int16_t)b[19 + 4 * uv].dc};
      dcf[uv] = skip_dc_fails(c, dc);
      for (int t = 0; t < 4; t++) sum += skip_share(b[16 + 4 * uv + t], t == 0 && dcf[uv], 7) << (8 + 8 * uv);
    }
    r.ok = skip_sum_ok(sum);
    // which test the reference's serial walk stops at: block by block, the first level > 1 or the first block that takes
    // the running score to the threshold (a level > 1 in a LATER block does not count)
    int ctr = 0, why = SKIP_DCT_OK;
    for (int k = 0; k < 16 && why == SKIP_DCT_OK; k++) {
      if (b[k].mx > 1) why = SKIP_Y_LEVEL;
      else if ((ctr += b[k].ctr) >= 6) why = SKIP_Y_CTR;
    }
    for (int uv = 0; uv < 2 && why == SKIP_DCT_OK; uv++) {
      ctr = 0;
      if (dcf[uv]) why = SKIP_UV_DC;
      for (int t = 0; t < 4 && why == SKIP_DCT_OK; t++) {
        if (b[16 + 4 * uv + t].mx > 1) why = SKIP_UV_LEVEL;
        else if ((ctr += b[16 + 4 * uv + t].ctr) >= 7) why = uv ? SKIP_CR_CTR : SKIP_CB_CTR;
      }
    }
    SKIP_COUNT(why);
  }
#endif
  return r;
}

#ifdef __CUDA_ARCH__
// The skip prediction for quarter-sample vector (mvx, mvy) into s.skip_pred in ONE memory round trip: every lane issues all
// of its reference loads before it uses any.  Luma with an integer vector: rows l / 4 and 8 + l / 4, four samples each (word
// loads).  Fractional luma: the 21 x 21 window from (-2, -2) as the aligned words that hold it (6 per row), staged in the
// refinement planes (stage A does not use them) and filtered eight samples per lane (mbk_pix8.cuh).  Chroma: one lane per
// plane, row and four samples (chroma4), at the INTEGER luma vector's chroma position (ix >> 1, iy >> 1) with the full
// eighth-sample phase, as the reference does.  Returns the lane's SADs against the source: luma | chroma << 16.
__device__ __forceinline__ uint32_t skip_predict(const MbCtx& c, MbScratch& s, int mvx, int mvy) {
  const int l = lane_id(), ix = mvx >> 2, iy = mvy >> 2, fx = mvx & 3, fy = mvy & 3;
  const int rs = c.p.rec_stride_y;
  const bool frac = (fx | fy) != 0;
  const uint8_t* ry = ref_luma(c, ix, iy);
  // ---- issue ----
  const uint8_t* wsrc = ry - 2 * rs - 2;
  const uint32_t wsh = (uint32_t)(reinterpret_cast<uintptr_t>(wsrc) & 3);
  const uint32_t* wa = reinterpret_cast<const uint32_t*>(reinterpret_cast<uintptr_t>(wsrc) & ~uintptr_t(3));
  uint32_t v[4];
  if (!frac) {
    v[0] = ld4u(ry + (l >> 2) * rs + ((l & 3) << 2));
    v[1] = ld4u(ry + (8 + (l >> 2)) * rs + ((l & 3) << 2));
    v[2] = v[3] = 0u;
  } else {
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int i = l + 32 * k, r = i / 6;
      v[k] = i < 21 * 6 ? wa[r * (rs >> 2) + i - 6 * r] : 0u;
    }
  }
  const int pl = l >> 4, cr = (l >> 1) & 7, cx = (l & 1) << 2;
  const uint8_t* pc = ref_chroma(c, 1 + pl, ix >> 1, iy >> 1) + cr * c.p.rec_stride_c + cx;
  uint32_t cw[4];
  chroma4_load(pc, c.p.rec_stride_c, cw);
  // ---- use ----
  uint32_t y0, y1;
  int yo;                                  // offset of y0 in the 16x16 block; y1 follows at yo + dy1
  int dy1;
  if (!frac) {
    y0 = v[0]; y1 = v[1]; yo = (l >> 2) * 16 + ((l & 3) << 2); dy1 = 128;
  } else {
    static_assert(sizeof(s.qplane) >= 21 * QP_STRIDE, "skip window in the refinement planes");
    const uint32_t sw = (uint32_t)__cvta_generic_to_shared(s.qplane[0]);
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const int i = l + 32 * k, r = i / 6;
      if (i < 21 * 6) asm volatile("st.shared.u32 [%0], %1;" ::"r"(sw + r * QP_STRIDE + 4 * (i - 6 * r)), "r"(v[k]) : "memory");
    }
    warp_sync();
    // lane: row y, samples x .. x+7; integer sample (x, y) at o.  The prediction is the rounded average of two of the
    // integer (G), half-sample H / V and centre (C) samples around it, as qpel_pair picks them
    const int y = l >> 1, x = (l & 1) << 3;
    const uint32_t o = sw + wsh + (y + 2) * QP_STRIDE + x + 2;
    const uint32_t x3 = fx == 3 ? 1 : 0, y3 = fy == 3 ? QP_STRIDE : 0;
    int ka, kb;                            // 0 G, 1 H, 2 V, 3 C
    uint32_t oa = 0, ob = 0;
    if (fy == 0) { ka = 1; kb = fx == 2 ? 1 : 0; ob = fx == 2 ? 0 : x3; }
    else if (fx == 0) { ka = 2; kb = fy == 2 ? 2 : 0; ob = fy == 2 ? 0 : y3; }
    else if (fx == 2 && fy == 2) { ka = 3; kb = 3; }
    else if (fx == 2) { ka = 1; oa = y3; kb = 3; }
    else if (fy == 2) { ka = 2; oa = x3; kb = 3; }
    else { ka = 1; oa = y3; kb = 2; ob = x3; }
    uint2 pa = make_uint2(0, 0), pb = make_uint2(0, 0);
    MBK_NO_UNROLL
    for (int j = 0; j < 2; j++) {
      const int k = j ? kb : ka;
      const uint32_t p = o + (j ? ob : oa);
      uint2 q;
      if (k == 0) { uint32_t g[2]; seg_words<2>(p, g); q = make_uint2(g[0], g[1]); }
      else if (k == 1) q = h8(p);
      else if (k == 2) q = v8(p, QP_STRIDE);
      else q = c8(p, QP_STRIDE);
      if (j) pb = q; else pa = q;
    }
    y0 = vavgu4(pa.x, pb.x); y1 = vavgu4(pa.y, pb.y); yo = y * 16 + x; dy1 = 4;
  }
  const uint32_t cv = chroma4(cw, (uint32_t)(reinterpret_cast<uintptr_t>(pc) & 3), mvx & 7, mvy & 7);
  const int co = 64 * pl + cr * 8 + cx;
  *reinterpret_cast<uint32_t*>(s.skip_pred + yo) = y0;
  *reinterpret_cast<uint32_t*>(s.skip_pred + yo + dy1) = y1;
  *reinterpret_cast<uint32_t*>(s.skip_pred + 256 + co) = cv;
  return vsadu4(y0, *reinterpret_cast<const uint32_t*>(s.cur_y + yo)) + vsadu4(y1, *reinterpret_cast<const uint32_t*>(s.cur_y + yo + dy1)) +
         (vsadu4(cv, *reinterpret_cast<const uint32_t*>(s.cur_c + co)) << 16);
}
#endif

MBK_STAGE SkipResult pskip_enc(const MbCtx& c, MbScratch& s, int sad_pred_skip) {
  SkipResult r;
  r.ok = false; r.cost_luma = 0; r.cost_skip = 0;
  int mvx, mvy;
  pred_skip_mv(s, &mvx, &mvy);
  r.mvx = mvx; r.mvy = mvy;
  const int ix = mvx >> 2, iy = mvy >> 2;
  int n = c.mbx * 16 + ix;
  if (n < -29 || n > c.p.mb_w * 16 + 12) { SKIP_COUNT(SKIP_RANGE); return r; }
  n = c.mby * 16 + iy;
  if (n < -29 || n > c.p.mb_h * 16 + 12) { SKIP_COUNT(SKIP_RANGE); return r; }
  phase_mark(s, 12);
#ifdef __CUDA_ARCH__
  const int sads = warp_sum((int)skip_predict(c, s, mvx, mvy));
  const int sad_y = sads & 0xffff, sad_c = sads >> 16;      // at most 256 * 255 and 128 * 255
  warp_sync();
#else
  g_skip_phase_luma |= 1ull << ((mvx & 3) + 4 * (mvy & 3));
  g_skip_phase_chroma |= 1ull << ((mvx & 7) + 8 * (mvy & 7));
  warp_mc_luma(ref_luma(c, ix, iy), c.p.rec_stride_y, s.skip_pred, 16, mvx, mvy, 16, 16);
  warp_mc_chroma_pair(ref_chroma(c, 1, ix >> 1, iy >> 1), ref_chroma(c, 2, ix >> 1, iy >> 1), c.p.rec_stride_c, s.skip_pred + 256, 8,
                      mvx, mvy, 8, 8);
  const int sad_y = warp_sad(s.cur_y, 16, s.skip_pred, 16, 4, 4);
  const int sad_c = warp_sad(s.cur_c, 8, s.skip_pred + 256, 8, 3, 3) + warp_sad(s.cur_c + 64, 8, s.skip_pred + 320, 8, 3, 3);
#endif
  const int sad_mb = sad_y + sad_c;
  phase_mark(s, 13);
  bool ok = sad_mb == 0 || sad_mb < sad_pred_skip || (c.p.ref_is_p && s.col.mb_type == MBT_PSKIP && sad_mb < s.col.skip_sad);
  if (ok) SKIP_COUNT(SKIP_SAD_OK);
  // HIGH complexity costs an accepted skip by its luma SATD: taken in the same pass as the residual tests
  int satd = 0;
  if (!ok || !c.p.fast_mode) {
    const SkipPass p = skip_residual_pass(c, s, !ok, !c.p.fast_mode);
    ok = ok || p.ok;
    satd = p.satd;
  }
  phase_mark(s, 15);
  if (ok) {
    r.ok = true;
    if (c.p.fast_mode) {                   // bMdUsingSad (:1493,:1524): the luma SAD is the cost AND goes into pSadCost[0]
      r.cost_luma = sad_y;
      if (lane_id() == 0) c.f.sad_cost[c.mby * c.p.mb_w + c.mbx] = sad_y;
    } else {
      r.cost_luma = satd;
    }
    phase_mark(s, 16);
    r.cost_skip = sad_mb;
  }
  return r;
}

// ---- search window of the macroblock (device: one bulk tensor copy into shared memory) -----------------------------
// (sx, sy) = integer start point of the 16x16 search relative to the macroblock; the window covers
// [sx-16, sx+32) x [sy-16, sy+32).  win_issue starts the copy (one lane), win_wait makes it visible to the warp.
MBK_HD void win_issue(const MbCtx& c, MbScratch& s, int sx, int sy) {
#ifdef __CUDA_ARCH__
  warp_sync();
  if (c.tmap_ref == nullptr) { if (lane_id() == 0) s.win_ok = 0; warp_sync(); return; }
  // plane coordinates (from the padded origin) of the window; X rounded down to a 16-byte boundary (bulk tensor copies need
  // an aligned start; the padded stride is a multiple of 16, so the alignment is the same in every row)
  const int X = (32 + c.mbx * 16 + sx - 16) & ~15, Y = 32 + c.mby * 16 + sy - 16, Z = c.p.ref_plane;
  const int wx0 = X - 32 - c.mbx * 16;                  // window origin relative to the macroblock
  if (lane_id() == 0) {
    s.win_x0 = wx0; s.win_y0 = sy - 16; s.win_ok = 1;
    const uint32_t dst = (uint32_t)__cvta_generic_to_shared(scratch_win(s));
    const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&c.wbar->bar);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // earlier generic accesses to the window bytes
    asm volatile("{ .reg .b64 st; mbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1; }" ::"r"(bar), "r"(WIN_W * WIN_H) : "memory");
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 ::"r"(dst), "l"(c.tmap_ref), "r"(X), "r"(Y), "r"(Z), "r"(bar) : "memory");
  }
  warp_sync();
#else
  (void)c; (void)sx; (void)sy;
  s.win_ok = 0;
#endif
}
MBK_HD void win_wait(const MbCtx& c, MbScratch& s) {
#ifdef __CUDA_ARCH__
  if (s.win_ok) {
    const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&c.wbar->bar);
    const uint32_t ph = c.wbar->phase;
    uint32_t ok = 0;
    while (!ok)
      asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                   : "=r"(ok) : "r"(bar), "r"(ph) : "memory");
    warp_sync();
    if (lane_id() == 0) c.wbar->phase = ph ^ 1;
    warp_sync();
  }
#else
  (void)c; (void)s;
#endif
}

// ---- integer search of one partition ------------------------------------------------------------------------
MBK_STAGE void me_partition(const MbCtx& c, MbScratch& s, int blk_size, int ox, int oy, int mvp_x, int mvp_y, uint32_t sad_pred,
                         int n_mvc, const int16_t* mvc, MeState* st) {
  MeIn in;
  in.enc = s.cur_y + oy * 16 + ox; in.enc_stride = 16;
  in.ref = ref_luma(c, ox, oy); in.ref_stride = c.p.rec_stride_y;
  in.blk = blk_size;
  in.mvp_x = mvp_x; in.mvp_y = mvp_y;
  // SetMvWithinIntegerMvRange (svc_motion_estimate.h:345): one window per MB, shared by its partitions
  const int r = c.p.mv_range;
  const int lo_x = -((c.mbx + 1) << 4) + 3, lo_y = -((c.mby + 1) << 4) + 3;
  const int hi_x = ((c.p.mb_w - c.mbx) << 4) - 3, hi_y = ((c.p.mb_h - c.mby) << 4) - 3;
  in.min_x = lo_x > -r ? lo_x : -r; in.min_y = lo_y > -r ? lo_y : -r;
  in.max_x = hi_x < r ? hi_x : r; in.max_y = hi_y < r ? hi_y : r;
  in.n_mvc = n_mvc; in.mvc = mvc;
  in.sad_pred = sad_pred;
  in.lambda = c.lambda;
  in.calc_satd = !c.p.fast_mode;            // NotCalculateSatdCost in LOW_COMPLEXITY (encoder_ext.cpp:2687)
  in.win = s.win_ok ? scratch_win(s) : nullptr;
  in.win_w = WIN_W; in.win_h = WIN_H;
  in.win_dx = s.win_x0 - ox; in.win_dy = s.win_y0 - oy;
  MeOut o;
  warp_me_search(in, o);
  if (lane_id() == 0) {                    // st lives in the scratch: one writer
    st->mv_x = o.mv_x; st->mv_y = o.mv_y; st->mvp_x = mvp_x; st->mvp_y = mvp_y;
    st->sad_cost = o.sad_cost; st->satd_cost = o.satd_cost;
    st->satd = (int)o.satd_cost - mvd_cost(c.lambda, o.mv_x - mvp_x, o.mv_y - mvp_y);
    st->ref = o.ref_best;
  }
  warp_sync();
}
// the same integer-pel range clip as me_partition: start point of a search with predictor (mvp_x, mvp_y), relative to the MB
MBK_HD void me_start_point(const MbCtx& c, int mvp_x, int mvp_y, int* sx, int* sy) {
  const int r = c.p.mv_range;
  const int lo_x = -((c.mbx + 1) << 4) + 3, lo_y = -((c.mby + 1) << 4) + 3;
  const int hi_x = ((c.p.mb_w - c.mbx) << 4) - 3, hi_y = ((c.p.mb_h - c.mby) << 4) - 3;
  *sx = clip3((2 + mvp_x) >> 2, lo_x > -r ? lo_x : -r, hi_x < r ? hi_x : r);
  *sy = clip3((2 + mvp_y) >> 2, lo_y > -r ? lo_y : -r, hi_y < r ? hi_y : r);
}

// ---- fractional refinement (MeRefineFracPixel, md.cpp:575) ------------------------------------------------------
// candidate cost = SATD(enc, prediction(mv)) + mvd cost, visited in the reference's order with strict '<'; the
// winning prediction is left in dst (stride 16).
// Like the reference, the half-sample planes of the partition are filtered ONCE: the (w+6) x (h+6) integer window
// around the matched block is staged in shared memory, H / V (and C, only if a half-sample point won) are computed
// from it, and every quarter-sample prediction is the rounded average of two plane samples (H.264 8.4.2.2.1; equal
// to McLuma_c for every phase: tests/test_gpu_motion_search.py checks every refinement, its vector, cost and prediction,
// against orc_me_refine, which predicts each candidate with McLuma on its own).  Plane coordinates are relative to
// the integer-sample position of the block: G covers [-3, w+3) x [-3, h+3), H/V/C start at (-1, -1); stride 32.
struct QpelPlanes { const uint8_t* g; const uint8_t* hh; const uint8_t* vv; const uint8_t* cc; };
// the two plane samples whose average is the prediction at quarter-sample offset (dx, dy) in [-3, 3]^2
MBK_HD void qpel_pair(const QpelPlanes& q, int dx, int dy, const uint8_t** pa, const uint8_t** pb) {
  const int ix = dx < 0 ? -1 : 0, iy = dy < 0 ? -1 : 0, fx = dx & 3, fy = dy & 3;
  const uint8_t* G = q.g + (iy + 3) * QP_STRIDE + (ix + 3);       // integer sample (ix, iy)
  const uint8_t* H = q.hh + (iy + 1) * QP_STRIDE + (ix + 1);
  const uint8_t* V = q.vv + (iy + 1) * QP_STRIDE + (ix + 1);
  const uint8_t* C = q.cc + (iy + 1) * QP_STRIDE + (ix + 1);
  const int x3 = fx == 3 ? 1 : 0, y3 = fy == 3 ? QP_STRIDE : 0;
  if ((fx | fy) == 0) { *pa = G; *pb = G; }
  else if (fy == 0) { *pa = H; *pb = fx == 2 ? H : G + x3; }
  else if (fx == 0) { *pa = V; *pb = fy == 2 ? V : G + y3; }
  else if (fx == 2 && fy == 2) { *pa = C; *pb = C; }
  else if (fx == 2) { *pa = H + y3; *pb = C; }
  else if (fy == 2) { *pa = V + x3; *pb = C; }
  else { *pa = H + y3; *pb = V + x3; }
}

// one half-sample plane of the refinement (0 = H, 1 = V, 2 = C): nx x ny samples, sample (x, y) from the staged window
// at win + (y + 2) * QP_STRIDE + x + 2.  The device computes eight samples of a row per lane from 32-bit shared addresses
// (mbk_pix8.cuh); the columns up to the next multiple of 8 come from bytes the window did not stage and are never read.
MBK_FN void refine_halfpel(int which, const uint8_t* win, uint8_t* dst, int nx, int ny) {
#ifdef __CUDA_ARCH__
  const uint32_t sw = (uint32_t)__cvta_generic_to_shared(win), sd = (uint32_t)__cvta_generic_to_shared(dst);
  const int gx = (nx + 7) >> 3;                      // 2 or 3 groups of 8 per row
  for (int i = lane_id(); i < gx * ny; i += 32) {
    const int r = gx == 2 ? i >> 1 : (i * 0xAAAB) >> 17, x = (i - r * gx) << 3;
    const uint32_t p = sw + r * QP_STRIDE + x + 2 * QP_STRIDE + 2;
    const uint2 v = which == 0 ? h8(p) : which == 1 ? v8(p, QP_STRIDE) : c8(p, QP_STRIDE);
    asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(sd + r * QP_STRIDE + x), "r"(v.x), "r"(v.y) : "memory");
  }
#else
  for (int i = 0; i < nx * ny; i++) {
    const int r = i / nx, x = i - r * nx;
    const uint8_t* p = win + (r + 2) * QP_STRIDE + (x + 2);
    dst[r * QP_STRIDE + x] = (uint8_t)(which == 0 ? half_h(p) : which == 1 ? half_v(p, QP_STRIDE) : half_c(p, QP_STRIDE));
  }
#endif
}

MBK_HD QpelPlanes refine_planes(MbScratch& s) {
  QpelPlanes q;
  q.g = reinterpret_cast<const uint8_t*>(s.coef); q.hh = s.qplane[0]; q.vv = s.qplane[1]; q.cc = s.qplane[2];
  return q;
}
// one round of the refinement: the four points (fx, fy) + step * (up, down, left, right), all four SATDs in one warp pass,
// then taken in that order with strict '<' as the reference visits them (mvd cost of offset (dx, dy): (mdx + dx, mdy + dy)).
// Returns (new best cost) * 8 + (winning direction + 1), direction -1 if no point beat `best`.
MBK_FN int refine_round(MbScratch& s, const uint8_t* enc, int lw, int lh, int lambda, int fx, int fy, int step, int mdx, int mdy, int best) {
  const QpelPlanes q = refine_planes(s);
  const uint8_t* base = reinterpret_cast<const uint8_t*>(&s);
  uint4 oa, ob;
  MBK_NO_UNROLL
  for (int k = 0; k < 4; k++) {
    const uint8_t *a, *b;
    qpel_pair(q, fx + (k == 2 ? -step : k == 3 ? step : 0), fy + (k == 0 ? -step : k == 1 ? step : 0), &a, &b);
    const uint32_t da = (uint32_t)(a - base), db = (uint32_t)(b - base);
    if (k == 0) { oa.x = da; ob.x = db; } else if (k == 1) { oa.y = da; ob.y = db; } else if (k == 2) { oa.z = da; ob.z = db; } else { oa.w = da; ob.w = db; }
  }
  const int4 sv = warp_satd_cands(enc, 16, base, oa, ob, QP_STRIDE, lw, lh);
  int bi = -1;
  MBK_NO_UNROLL
  for (int k = 0; k < 4; k++) {
    const int dx = fx + (k == 2 ? -step : k == 3 ? step : 0), dy = fy + (k == 0 ? -step : k == 1 ? step : 0);
    const int cst = (k == 0 ? sv.x : k == 1 ? sv.y : k == 2 ? sv.z : sv.w) + mvd_cost(lambda, mdx + dx, mdy + dy);
    if (cst < best) { best = cst; bi = k; }
  }
  return best * 8 + bi + 1;
}

MBK_STAGE void me_refine(const MbCtx& c, MbScratch& s, MeState* st, int ox, int oy, int w, int h, uint8_t* dst) {
  const int lw = w == 16 ? 4 : 3, lh = h == 16 ? 4 : 3;
  const uint8_t* enc = s.cur_y + oy * 16 + ox;
  const int rs = c.p.rec_stride_y;
  const int px = st->mvp_x, py = st->mvp_y;
  const int mv0x = st->mv_x, mv0y = st->mv_y;
  const uint8_t* ref0 = st->ref;
  // bSatdInMdFlag (md.cpp:601-606): with SATD mode costs the search already holds the SATD at the integer position;
  // in LOW_COMPLEXITY (SAD mode costs) it is computed here — pfMeCost stays SATD either way
  int best = (c.p.fast_mode ? warp_satd(enc, 16, ref0, rs, lw, lh) : st->satd) + mvd_cost(c.lambda, mv0x - px, mv0y - py);
  // ---- stage the integer window (the coefficient buffer is free until the residual is coded) ----
  uint8_t* win = reinterpret_cast<uint8_t*>(s.coef);
  static_assert(sizeof(s.coef) >= 22 * QP_STRIDE, "window aliases the coefficient buffer");
  const int ww = w + 6, wh = h + 6, wq = (ww + 3) >> 2;            // words per row (the padded reference allows the overshoot)
  // source: the search window of the macroblock while it is still intact and covers the region, else the plane
  const uint8_t* src = ref0 - (ptrdiff_t)3 * rs - 3;
  int srs = rs;
  if (s.win_ok) {
    const int x0 = ox + (mv0x >> 2) - 3 - s.win_x0, y0 = oy + (mv0y >> 2) - 3 - s.win_y0;
    if (x0 >= 0 && y0 >= 0 && x0 + 4 * wq <= WIN_W && y0 + wh <= WIN_H) { src = scratch_win(s) + y0 * WIN_W + x0; srs = WIN_W; }
  }
#ifdef __CUDA_ARCH__
  {
    // the window's last rows share their bytes with the coefficient buffer this copy writes to: read everything into registers
    // (at most 6 x 22 = 132 words: 5 per lane), then store
    uint32_t v[5];
#pragma unroll
    for (int k = 0; k < 5; k++) {
      const int i = lane_id() + 32 * k;
      const int r = i / wq, q4 = (i - r * wq) << 2;
      v[k] = i < wq * wh ? ld4u(src + (ptrdiff_t)r * srs + q4) : 0u;
    }
    warp_sync();
#pragma unroll
    for (int k = 0; k < 5; k++) {
      const int i = lane_id() + 32 * k;
      if (i < wq * wh) {
        const int r = i / wq, q4 = (i - r * wq) << 2;
        uint8_t* d = win + r * QP_STRIDE + q4;
        d[0] = (uint8_t)v[k]; d[1] = (uint8_t)(v[k] >> 8); d[2] = (uint8_t)(v[k] >> 16); d[3] = (uint8_t)(v[k] >> 24);
      }
    }
  }
#else
  for (int i = lane_id(); i < wq * wh; i += MBK_WS) {
    const int r = i / wq, q4 = (i - r * wq) << 2;
    const uint32_t v = ld4u(src + (ptrdiff_t)r * srs + q4);
    uint8_t* d = win + r * QP_STRIDE + q4;
    d[0] = (uint8_t)v; d[1] = (uint8_t)(v >> 8); d[2] = (uint8_t)(v >> 16); d[3] = (uint8_t)(v >> 24);
  }
#endif
  warp_sync();
  if (lane_id() == 0) s.win_ok = 0;          // the planes below overwrite the window bytes
  warp_sync();
  uint8_t* ph = s.qplane[0];
  uint8_t* pv = s.qplane[1];
  uint8_t* pc = s.qplane[2];
  // H(X, Y): X in [-1, w-1], Y in [-1, h];  V(X, Y): X in [-1, w], Y in [-1, h-1]
  refine_halfpel(0, win, ph, w + 1, h + 2);
  refine_halfpel(1, win, pv, w + 2, h + 1);
  warp_sync();
  int fx = 0, fy = 0;                    // offsets from the integer vector
  MBK_NO_UNROLL
  for (int step = 2; step >= 1; step--) {
    if (step == 1 && (fx | fy)) {        // quarter positions around a half-sample point need the centre plane
      refine_halfpel(2, win, pc, w + 1, h + 1);
      warp_sync();
    }
    const int r = refine_round(s, enc, lw, lh, c.lambda, fx, fy, step, mv0x - px, mv0y - py, best);
    const int bi = (r & 7) - 1;
    best = r >> 3;
    if (bi >= 0) { fx += bi == 2 ? -step : bi == 3 ? step : 0; fy += bi == 0 ? -step : bi == 1 ? step : 0; }
  }
  // final prediction
  {
    const uint8_t *a, *b;
    qpel_pair(refine_planes(s), fx, fy, &a, &b);
    const int gsh = lw - 2;
    for (int g = lane_id(); g < (w * h) >> 2; g += MBK_WS) {
      const int y = g >> gsh, x = (g & ((1 << gsh) - 1)) << 2;
      const uint32_t v = vavgu4(ld4u(a + y * QP_STRIDE + x), ld4u(b + y * QP_STRIDE + x));
      uint8_t* d = dst + y * 16 + x;
      d[0] = (uint8_t)v; d[1] = (uint8_t)(v >> 8); d[2] = (uint8_t)(v >> 16); d[3] = (uint8_t)(v >> 24);
    }
    warp_sync();
  }
  if (lane_id() == 0) { st->mv_x = mv0x + fx; st->mv_y = mv0y + fy; st->satd_cost = (uint32_t)best; }
  warp_sync();
}

// ---- residual of an inter MB: luma (WelsEncInterY, svc_encode_mb.cpp:180) and chroma (WelsEncRecUV, :244) -----------------
// The host build codes it serially through s.coef (these functions are the specification of inter_residual_pass); it also
// counts what the JVT-O079 decisions did, so that tests can show which outcomes their clips reach.
//   RES_LUMA_ZEROED  luma levels present, all dropped by the macroblock score (ctr_mb < 6)
//   RES_MIXED_8x8    one 8x8 kept and another one with levels dropped (ctr8 < 4) in the same macroblock
//   RES_CBP_C0..C2   chroma part of the cbp
//   RES_P16x16..     the partition shape stage B coded (P16x16, P16x8, P8x16, P8x8), or a 16x16 without residual that
//   RES_PSKIP_CODED  became P_SKIP after coding (step 8)
enum { RES_LUMA_ZEROED = 0, RES_MIXED_8x8, RES_CBP_C0, RES_CBP_C1, RES_CBP_C2, RES_P16x16, RES_P16x8, RES_P8x16, RES_P8x8,
       RES_PSKIP_CODED, RES_OUTCOMES };
inline uint64_t g_res_outcome[RES_OUTCOMES];
#ifndef __CUDA_ARCH__
MBK_FN void dct_luma_mb(MbScratch& s, const uint8_t* pred /*stride 16*/) {
  for (int k = lane_id(); k < 16; k += MBK_WS) {
    int16_t d[16];
    const int o = blk_y(k) * 4 * 16 + blk_x(k) * 4;
    dct4x4(d, s.cur_y + o, 16, pred + o, 16);
    for (int i = 0; i < 16; i++) s.coef[16 * k + i] = d[i];
  }
  warp_sync();
}
MBK_STAGE void enc_inter_y(const MbCtx& c, MbScratch& s) {
  const int16_t* ff = tbl_quant_ff(c.qp);
  const int16_t* mf = tbl_quant_mf(c.qp);
  // per-block quantisation / scan in parallel; the JVT-O079 accumulation is order dependent -> serial scalar part
  for (int k = lane_id(); k < 16; k += MBK_WS) {
    int16_t d[16], l[16];
    for (int i = 0; i < 16; i++) d[i] = s.coef[16 * k + i];
    const int16_t mx = quant4x4_max(d, ff, mf);
    if (mx == 0) { for (int i = 0; i < 16; i++) l[i] = 0; }
    else scan4x4_dcac(l, d);
    for (int i = 0; i < 16; i++) { s.coef[16 * k + i] = d[i]; s.out.luma[k][i] = l[i]; }
    s.red[k] = mx;
    s.red[16 + k] = mx == 0 ? 0 : single_ctr4x4(l);
  }
  warp_sync();
  int ctr8[4], ctr_mb = 0;
  for (int i = 0; i < 4; i++) {
    ctr8[i] = 0;
    for (int j = 0; j < 4; j++) {
      const int mx = s.red[4 * i + j];
      if (mx == 0) continue;
      if (mx > 1) ctr8[i] += 9;
      else if (ctr8[i] < 6) ctr8[i] += s.red[16 + 4 * i + j];
    }
    ctr_mb += ctr8[i];
  }
  {
    int lev = 0, kept = 0, dropped = 0;                  // 8x8s with levels
    for (int i = 0; i < 4; i++) {
      const int has = s.red[4 * i] | s.red[4 * i + 1] | s.red[4 * i + 2] | s.red[4 * i + 3];
      lev |= has; kept |= ctr8[i] >= 4; dropped |= has && ctr8[i] < 4;
    }
    if (lev && ctr_mb < 6) g_res_outcome[RES_LUMA_ZEROED]++;
    if (ctr_mb >= 6 && kept && dropped) g_res_outcome[RES_MIXED_8x8]++;
  }
  for (int i = lane_id(); i < 16; i += MBK_WS) s.info.nnz[i] = 0;
  warp_sync();
  if (ctr_mb < 6) {
    for (int i = lane_id(); i < 256; i += MBK_WS) s.coef[i] = 0;
  } else {
    for (int k = lane_id(); k < 16; k += MBK_WS) {
      if (ctr8[k >> 2] >= 4) {
        s.info.nnz[blk_raster(k)] = (int8_t)nonzero_count(s.out.luma[k]);
        int16_t d[16];
        for (int i = 0; i < 16; i++) d[i] = s.coef[16 * k + i];
        dequant4x4(d, tbl_dequant(c.qp));
        for (int i = 0; i < 16; i++) s.coef[16 * k + i] = d[i];
      } else {
        for (int i = 0; i < 16; i++) s.coef[16 * k + i] = 0;
      }
    }
    if (lane_id() == 0)
      for (int i = 0; i < 4; i++) if (ctr8[i] >= 4) s.info.cbp |= (uint8_t)(1 << i);
  }
  warp_sync();
}
#endif

// luma reconstruction of an inter MB: pred + IDCT(coef) for all 16 blocks (OutputPMbWithoutConstructCsRsNoCopy; the decoder's too)
MBK_FN void rec_luma_inter(MbScratch& s, const uint8_t* pred) {
  for (int k = lane_id(); k < 16; k += MBK_WS) {
    int16_t d[16];
    for (int i = 0; i < 16; i++) d[i] = s.coef[16 * k + i];
    const int oy = blk_y(k) * 4, ox = blk_x(k) * 4;
    idct4x4_rec(tile_y(s.tile, ox, oy), TY_PITCH, pred + oy * 16 + ox, 16, d);
  }
  warp_sync();
}

// The luma and chroma residual of an inter macroblock against the prediction pl (stride 16) / pc (Cb, Cr at +64, stride 8),
// its coding decisions and its reconstruction (step 7 of stage B); with `intra`, the chroma residual of an intra macroblock
// whose luma is coded already (the intra tail: pl is unused, s.info.cbp's luma bits are kept).  Writes s.out.luma (inter) /
// chroma_dc / chroma_ac (the levels of every block, kept or dropped), s.info.nnz, s.info.cbp and the tile.
// Device: ONE warp pass from registers.  Lane l < 16 takes luma block l (coding order; idle for intra), lanes 16..19 / 20..23
// the Cb / Cr blocks (raster).  The serial JVT-O079 walks (four blocks of an 8x8 in coding order, the four blocks of a chroma
// plane in raster order) run on every lane of an aligned group of four over the group's shuffled scores; the 2x2 chroma DC
// goes through the same shuffles.  Intra chroma rounds with ff(qp_c + 6) and keeps a plane's AC whenever it has a level
// (WelsEncRecUV: ctr = INT_MAX).  No coefficients are written: nothing after the pass reads them.
MBK_STAGE void residual_pass(const MbCtx& c, MbScratch& s, const uint8_t* pl, const uint8_t* pc, bool intra) {
#ifdef __CUDA_ARCH__
  const int l = lane_id(), t = l & 3, g0 = l & ~3;
  const bool luma = !intra && l < 16, chroma = l >= 16 && l < 24;
  const int uv = (l >> 2) & 1;                           // chroma lanes: plane
  const int bx = luma ? blk_x(l) : t & 1, by = luma ? blk_y(l) : t >> 1;
  const int st = luma ? 16 : 8, o = luma ? by * 64 + bx * 4 : 64 * uv + by * 32 + bx * 4;   // lanes 24..31 read Cb / Cr too
  const uint8_t* cur = (luma ? s.cur_y : s.cur_c) + o;
  const uint8_t* pr = (luma ? pl : pc) + o;
  uint32_t a[4], p[4];
#pragma unroll
  for (int y = 0; y < 4; y++) {
    a[y] = *reinterpret_cast<const uint32_t*>(cur + y * st);
    p[y] = *reinterpret_cast<const uint32_t*>(pr + y * st);
  }
  int16_t d[16], lv[16];
  dct4x4_rows(d, a, p);
  const int q = luma ? c.qp : c.qp_c;
  const int16_t dc = d[0];
  if (!luma) d[0] = 0;                                   // chroma AC: the DC position is quantised as 0
  const int mx = quant4x4_max(d, tbl_quant_ff(q + (intra ? 6 : 0)), tbl_quant_mf(q));
#pragma unroll
  for (int i = 0; i < 16; i++) lv[i] = luma ? d[zigzag_pos(i)] : i < 15 ? d[zigzag_pos(i + 1)] : (int16_t)0;
  const int nz = nonzero_count(lv);
  // the block's term in the serial walk: 0x100 = a level > 1 (adds 9; intra: any level), else its single-coefficient score
  // (0 without levels)
  const int v = intra ? (mx != 0 ? 0x100 : 0) : mx > 1 ? 0x100 : single_ctr4x4(lv);
  const int thr = luma ? 6 : 7;
  int grp = 0;                                           // ctr8 of the lane's 8x8 / the AC score of its chroma plane
  int16_t dcin[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int vj = __shfl_sync(MBK_FULL, v, g0 + j);
    if (vj & 0x100) grp += 9;
    else if (grp < thr) grp += vj;
    dcin[j] = (int16_t)__shfl_sync(MBK_FULL, (int)dc, g0 + j);
  }
  const int ctr_mb = __shfl_sync(MBK_FULL, grp, 0) + __shfl_sync(MBK_FULL, grp, 4) + __shfl_sync(MBK_FULL, grp, 8) +
                     __shfl_sync(MBK_FULL, grp, 12);
  const bool keep = luma ? ctr_mb >= 6 && grp >= 4 : chroma && grp >= 7;
  // chroma DC 2x2 of the lane's plane (every lane of the group computes it; luma lanes ignore it)
  const int16_t* ffc = tbl_quant_ff(c.qp_c + (intra ? 6 : 0));
  const int16_t* mfc = tbl_quant_mf(c.qp_c);
  int16_t dq[4];
  const int nz_dc = hadamard_quant2x2(dcin, (int16_t)(ffc[0] << 1), (int16_t)(mfc[0] >> 1), dq);
  const int16_t dcl = t == 0 ? dq[0] : t == 1 ? dq[1] : t == 2 ? dq[2] : dq[3];
  if (nz_dc > 0) dequant_ihadamard2x2_dc(dq, tbl_dequant(c.qp_c)[0]);
  const int16_t dcr = t == 0 ? dq[0] : t == 1 ? dq[1] : t == 2 ? dq[2] : dq[3];
  // cbp: luma bit i = 8x8 i kept; chroma 2 = some plane keeps its AC, else 1 = some plane has a DC level
  const uint32_t bk = __ballot_sync(MBK_FULL, keep), bdc = __ballot_sync(MBK_FULL, chroma && nz_dc > 0);
  const int cbp = (intra ? s.info.cbp & 15 : (int)((bk & 1) | ((bk >> 3) & 2) | ((bk >> 6) & 4) | ((bk >> 9) & 8))) |
                  ((bk & 0x00ff0000u) ? 0x20 : bdc ? 0x10 : 0);
  if (luma || chroma) {
    uint32_t w[8];
#pragma unroll
    for (int i = 0; i < 8; i++) w[i] = (uint32_t)(uint16_t)lv[2 * i] | ((uint32_t)(uint16_t)lv[2 * i + 1] << 16);
    uint4* ol = reinterpret_cast<uint4*>(luma ? s.out.luma[l] : s.out.chroma_ac[l - 16]);
    ol[0] = make_uint4(w[0], w[1], w[2], w[3]);
    ol[1] = make_uint4(w[4], w[5], w[6], w[7]);
    if (!luma) s.out.chroma_dc[uv][t] = dcl;
    s.info.nnz[luma ? blk_raster(l) : l] = (int8_t)(keep ? nz : 0);
    // reconstruction: the kept blocks dequantised, the chroma DC put back, inverse transform onto the prediction
    if (keep) dequant4x4(d, tbl_dequant(q));
    else {
#pragma unroll
      for (int i = 0; i < 16; i++) d[i] = 0;
    }
    if (!luma && nz_dc > 0) d[0] = dcr;
    idct4x4_rec_rows(luma ? tile_y(s.tile, 4 * bx, 4 * by) : tile_c(uv ? s.tile.v : s.tile.u, 4 * bx, 4 * by), luma ? TY_PITCH : TC_PITCH, p, d);
  }
  if (l == 0) s.info.cbp = (uint8_t)cbp;
  warp_sync();
#else
  if (!intra) {
    s.info.cbp = 0;
    dct_luma_mb(s, pl);
    enc_inter_y(c, s);
  }
  dct_chroma(s, pc);
  enc_rec_uv(c, s, 0, !intra);
  enc_rec_uv(c, s, 1, !intra);
  if (!intra) rec_luma_inter(s, pl);
  rec_chroma(s, pc);
  if (!intra) g_res_outcome[RES_CBP_C0 + (s.info.cbp >> 4)]++;
#endif
}
MBK_STAGE void inter_residual_pass(const MbCtx& c, MbScratch& s, const uint8_t* pl, const uint8_t* pc) { residual_pass(c, s, pl, pc, false); }

// ---- an intra macroblock after its I16x16 decision (WelsMdIntraMb :956 / WelsMdFirstIntraMode :1829 +
// WelsMdIntraSecondaryModesEnc :2023) -------------------------------------------------------------------------------
// cost16 / bb: the I16x16 cost and prediction buffer (md_i16x16).  Tries I4x4 against it, codes the luma of the winner and
// the chroma; an intra macroblock has no reference and no SAD cost (pSadCost[0] = 0, :2038).  Stage I (every macroblock of
// an IDR picture) and stage C (the intra branch of a P macroblock) end here.  Returns the I4x4 cost (INT_MAX when I4x4 was
// not tried).
MBK_FN int intra_mb_finish(const MbCtx& c, MbScratch& s, int cost16, int bb) {
  bool use_i4 = false;                       // warp-uniform; the staged record is written by lane 0 only
  int cost4 = 0x7fffffff;
  phase_mark(s, 17);
  if (lane_id() == 0) { s.info.mb_type = MBT_I16x16; s.info.cbp = 0; }
  warp_sync();
  fill_i4_cache(c, s);
  if (intra_try_i4x4(c, s)) {
    cost4 = md_enc_i4x4(c, s, cost16);                 // pfIntraFineMd = WelsMdIntraFinePartition[Vaa] (:932, :942)
    if (cost4 < cost16) { use_i4 = true; if (lane_id() == 0) s.info.mb_type = MBT_I4x4; warp_sync(); }
  }
#ifndef __CUDA_ARCH__
  if (use_i4) g_i4_end[I4_END_WON]++;
#endif
  phase_mark(s, 18);
  if (!use_i4) {
    if (lane_id() == 0) s.info.cbp = 0;        // the I4x4 attempt may have set bits
    warp_sync();
    enc_rec_i16x16(c, s, s.pred_y[bb]);
  }
  phase_mark(s, 19);
  int cb;
  md_chroma(c, s, &cb);
  phase_mark(s, 20);
  residual_pass(c, s, nullptr, s.pred_c[cb], true);
  phase_mark(s, 21);
  if (lane_id() == 0) { c.f.sad_cost[c.mby * c.p.mb_w + c.mbx] = 0; s.info.ref_idx = REF_NOT_IN_LIST; }
  warp_sync();
  return cost4;
}

// ---- decided skip (WelsMdInterDecidedPskip :1954 + WelsRecPskip svc_encode_mb.cpp:315) ------------------------------
// the reconstruction of a P_SKIP macroblock stays in s.skip_pred (mb_store_recon_skip writes it to the picture)
MBK_HD void decided_pskip(const MbCtx& c, MbScratch& s) {
  (void)c;
  if (lane_id() == 0) {
    s.info.mb_type = MBT_PSKIP;
    s.info.cbp = 0;
  }
  for (int i = lane_id(); i < 24; i += MBK_WS) s.info.nnz[i] = 0;
  warp_sync();
}

// ---- the P-slice macroblock (WelsMdInterMb :1858 + WelsMdInterSecondaryModesEnc :1997) --------------------------------
// The macroblock is coded in up to three STAGES; the device scheduler runs each stage of many macroblocks as a
// lock-step batch (enc_kernels.cu) and parks the scratch between stages, the host build runs them back to back.
//   A  skip test; a skip candidate also takes the intra-16x16 check here and ends as P_SKIP or goes on to C
//      (WelsMdInterMb decides it in one pass too: skip judgement, then WelsMdFirstIntraMode)
//   B  16x16 search, intra-16x16 check, sub-partitions, refinement, residual
//   C  the intra branch of a P macroblock (taken from A or B when intra 16x16 beats the inter cost)
// Values that cross a stage boundary live in s.st (warp-uniform; written by lane 0).
// Stage ids (each stage has a ready list, enc_kernels.cu: enc_list).  Id 3 is not a stage: the host build reports the intra
// check of a skip candidate, which stage A runs, as a step of its own with that id (mb_run_stage), so that the paths it
// records (bit id = the step ran: tests/emu, tools/sched_sim.py, tools/sim_data) keep the numbering of the time that check
// was a stage (Bs).
enum { MBS_DONE = 0, MBS_A = 1, MBS_I = 2, MBP_SKIPCAND_INTRA = 3, MBS_B = 4, MBS_C = 5, MBS_COUNT = 6 };
// host build: stage A ran the skip candidate's intra check (set by inter_stage_a), and the stage that follows it
inline bool g_skipcand_intra;
inline int g_skipcand_next;

// bookkeeping for the neighbours and the next frame
MBK_FN void inter_tail(const MbCtx& c, MbScratch& s) {
  const int idx = c.mby * c.p.mb_w + c.mbx;
  const int final_type = s.st.final_type, p16_mvx = s.st.p16_mvx, p16_mvy = s.st.p16_mvy, cost_skip_mb = s.st.cost_skip_mb;
  if (lane_id() == 0) {
    s.info.mb_type = (uint8_t)final_type;
    s.info.p16x16_mv[0] = (int16_t)p16_mvx; s.info.p16x16_mv[1] = (int16_t)p16_mvy;
    if (MBT_IS_INTER(final_type)) s.info.ref_idx = 0;
    RefMbInfo ri;
    ri.mv16[0] = (int16_t)p16_mvx; ri.mv16[1] = (int16_t)p16_mvy;
    ri.skip_sad = final_type == MBT_PSKIP ? cost_skip_mb : 0;      // WelsMdInterSaveSadAndRefMbType (:1987)
    ri.mb_type = (uint8_t)final_type;
    ri.pad[0] = ri.pad[1] = ri.pad[2] = 0;
    c.f.rec_info[idx] = ri;
  }
  warp_sync();
}

MBK_HD void st_save(MbScratch& s, int is_skip, int cost_luma, int cost_skip_mb, int p16_mvx, int p16_mvy, int final_type) {
  warp_sync();
  if (lane_id() == 0) {
    s.st.is_skip = is_skip; s.st.cost_luma = cost_luma; s.st.cost_skip_mb = cost_skip_mb;
    s.st.p16_mvx = p16_mvx; s.st.p16_mvy = p16_mvy; s.st.final_type = final_type;
  }
  warp_sync();
}

MBK_STAGE int inter_stage_a(const MbCtx& c, MbScratch& s) {
  fill_inter_cache(c, s);
  phase_mark(s, 1);
  int p16_mvx = 0, p16_mvy = 0;                       // sP16x16Mv / sMvList (WelsMdInterInit :352-353)
  const bool sk_l = (c.nb & NB_LEFT) && s.nbi[3].mb_type == MBT_PSKIP;
  const bool sk_t = (c.nb & NB_TOP) && s.nbi[1].mb_type == MBT_PSKIP;
  const bool sk_tl = (c.nb & NB_TOPLEFT) && s.nbi[0].mb_type == MBT_PSKIP;
  const bool sk_tr = (c.nb & NB_TOPRIGHT) && s.nbi[2].mb_type == MBT_PSKIP;
  const bool try_skip = sk_l || sk_t || sk_tl || sk_tr;
  const bool keep_skip = sk_l && sk_t && sk_tr;
  int cost_luma = 0, cost_skip_mb = 0;
  bool is_skip = false;
  // step 1: SKIP (WelsMdInterJudgePskip :1906)
  if ((c.p.ref_is_p && s.col.mb_type == MBT_PSKIP) || try_skip) {
    const SkipResult r = pskip_enc(c, s, predict_sad_skip(s));
    if (r.ok) {
      is_skip = true;
      cost_luma = r.cost_luma; cost_skip_mb = r.cost_skip;
      p16_mvx = r.mvx; p16_mvy = r.mvy;
      mb_mv_set(s, 0, 4, 4, r.mvx, r.mvy);
    }
  }
  phase_mark(s, 2);
  if (is_skip && !keep_skip) {
    // intra check of a skip candidate (WelsMdFirstIntraMode :1829): the skip test wrote skip_pred and the refinement planes
    // only, so the tile borders and cur_y are still those mb_load_all staged
#ifndef __CUDA_ARCH__
    g_skipcand_intra = true;
#endif
    int bb;
    const int cost16 = md_i16x16_inl(c, s, &bb);
    phase_mark(s, 4);
    if (cost16 < cost_luma) {
      st_save(s, 1, cost_luma, cost_skip_mb, p16_mvx, p16_mvy, MBT_P16x16);
      if (lane_id() == 0) { s.st.cost16 = cost16; s.st.bb = bb; }
      warp_sync();
      return MBS_C;
    }
  }
  if (is_skip) {
    decided_pskip(c, s);
    st_save(s, 1, cost_luma, cost_skip_mb, p16_mvx, p16_mvy, MBT_PSKIP);
    inter_tail(c, s);
    return MBS_DONE;
  }
  st_save(s, 0, cost_luma, cost_skip_mb, p16_mvx, p16_mvy, MBT_P16x16);
  return MBS_B;
}

MBK_STAGE int inter_stage_b(const MbCtx& c, MbScratch& s) {
  const int mbw = c.p.mb_w, idx = c.mby * mbw + c.mbx;
  int cost_luma = s.st.cost_luma, cost_skip_mb = s.st.cost_skip_mb, p16_mvx = s.st.p16_mvx, p16_mvy = s.st.p16_mvy;
  MeState& me16 = s.me[0];
  MeState* me16x8 = &s.me[1];
  MeState* me8x16 = &s.me[3];
  MeState* me8x8 = &s.me[5];
  int final_type = MBT_P16x16;
  int sad_pred_mb = 0;
  if (lane_id() == 0) s.win_ok = 0;
  warp_sync();
  // Every integer search of the macroblock goes through ONE call site (me_partition is inlined there: no callee-saved
  // register traffic, the search state stays in registers): round t = -1 is the 16x16 search (WelsMdP16x16 :978), rounds
  // t >= 0 are the sub-partition shapes of `plan` (WelsMdInterFinePartition :1238 / WelsMdInterFinePartitionVaa :1270).
  int16_t (*mvc)[2] = s.mvcand;
  int px16 = 0, py16 = 0, n16 = 1;
  pred_mv(s, 0, 4, 0, &px16, &py16);
  {                                        // the window copy flies while the candidate list is put together
    int sx, sy;
    me_start_point(c, px16, py16, &sx, &sy);
    win_issue(c, s, sx, sy);
  }
  sad_pred_mb = predict_sad(s);
  n16 += (c.nb & NB_LEFT) ? 1 : 0;                                        // [0] = sMvBase (0,0)
  n16 += (c.nb & NB_TOP) ? 1 : 0;
  if (c.p.ref_is_p) { n16 += c.mbx < mbw - 1 ? 1 : 0; n16 += c.mby < c.p.mb_h - 1 ? 1 : 0; }
  if (lane_id() == 0) {
    int k = 0;
    mvc[k][0] = 0; mvc[k][1] = 0; k++;
    if (c.nb & NB_LEFT) { mvc[k][0] = s.nbi[3].p16x16_mv[0]; mvc[k][1] = s.nbi[3].p16x16_mv[1]; k++; }
    if (c.nb & NB_TOP) { mvc[k][0] = s.nbi[1].p16x16_mv[0]; mvc[k][1] = s.nbi[1].p16x16_mv[1]; k++; }
    if (c.p.ref_is_p) {
      if (c.mbx < mbw - 1) { mvc[k][0] = c.f.ref_info[idx + 1].mv16[0]; mvc[k][1] = c.f.ref_info[idx + 1].mv16[1]; k++; }
      if (c.mby < c.p.mb_h - 1) { mvc[k][0] = c.f.ref_info[idx + mbw].mv16[0]; mvc[k][1] = c.f.ref_info[idx + mbw].mv16[1]; k++; }
    }
  }
  warp_sync();
  win_wait(c, s);
  int plan[3] = {0, 0, 0}, n_plan = 0, cost = 0;       // shapes: 0 = 16x16, 1 = 16x8, 2 = 8x16, 3 = 8x8
  MBK_NO_UNROLL
  for (int t = -1; t < n_plan; t++) {
    const int shape = t < 0 ? 0 : plan[t];
    int cst = 0;
    const int np = shape == 0 ? 1 : shape == 3 ? 4 : 2;
    MeState* arr = shape == 0 ? &me16 : shape == 1 ? me16x8 : shape == 2 ? me8x16 : me8x8;
    MBK_NO_UNROLL
    for (int i = 0; i < np; i++) {
      int px = px16, py = py16, ox = 0, oy = 0, blk = BLK_16x16, ci = 0, cw = 4, ch = 4, ncand = n16;
      uint32_t sp = (uint32_t)sad_pred_mb;
      if (shape == 1) { pred_16x8_mv(s, 8 * i, 0, &px, &py); oy = 8 * i; blk = BLK_16x8; ci = 8 * i; ch = 2; sp = (uint32_t)(sad_pred_mb >> 1); ncand = 1; }
      else if (shape == 2) { pred_8x16_mv(s, 4 * i, 0, &px, &py); ox = 8 * i; blk = BLK_8x16; ci = 4 * i; cw = 2; sp = (uint32_t)(sad_pred_mb >> 1); ncand = 1; }
      else if (shape == 3) { pred_mv(s, 4 * i, 2, 0, &px, &py); ox = (i & 1) * 8; oy = (i >> 1) * 8; blk = BLK_8x8; ci = 4 * i; cw = 2; ch = 2; sp = (uint32_t)(sad_pred_mb >> 2); ncand = 1; }
      me_partition(c, s, blk, ox, oy, px, py, sp, ncand, &mvc[0][0], &arr[i]);       // sub-partitions: candidate [0] = (0, 0) only
      if (shape != 0) cache_set(s, ci, cw, ch, arr[i].mv_x, arr[i].mv_y);
      cst += (int)arr[i].satd_cost;
    }
    if (t >= 0) {
      // the first shape of the plan has to beat 16x16, a later one only the best so far (<=: md.cpp keeps the later shape on a tie)
      if (t == 0) { if (cst < cost_luma) { cost = cst; final_type = shape == 3 ? MBT_P8x8 : shape == 1 ? MBT_P16x8 : MBT_P8x16; } else break; }
      else if (cst <= cost) { cost = cst; final_type = shape == 1 ? MBT_P16x8 : MBT_P8x16; }
      continue;
    }
    // ---- after the 16x16 round ----
    p16_mvx = me16.mv_x; p16_mvy = me16.mv_y; cost_luma = cst;
    mbk_batch_sync(2, c.batch_n);                                          // list B: together again after the 16x16 search
    phase_mark(s, 3);
    {
      // intra check (WelsMdFirstIntraMode :1829)
      int bb;
      const int cost16 = md_i16x16_inl(c, s, &bb);
      phase_mark(s, 4);
      if (cost16 < cost_luma) {
        st_save(s, 0, cost_luma, cost_skip_mb, p16_mvx, p16_mvy, final_type);
        if (lane_id() == 0) { s.st.cost16 = cost16; s.st.bb = bb; }
        warp_sync();
        mbk_batch_leave(3, c.batch_n); mbk_batch_leave(4, c.batch_n);
        return MBS_C;
      }
    }
    // LOW_COMPLEXITY: the four 8x8 SADs of the macroblock against the previous source picture say which partition shapes
    // are worth a search (MdInterAnalysisVaaInfo_c md.cpp:389): 15 = homogeneous, none; 3/12 -> 16x8; 5/10 -> 8x16;
    // 6/9 -> 8x8; anything else -> the full sequence of the other complexity modes (8x8, then 16x8 and 8x16 if 8x8 won)
    int vaa_sign = 0;
    if (c.p.fast_mode) {
      const int32_t* v = c.f.vaa_sad8x8 + 4 * idx;
      const int b0 = v[0], b1 = v[1], b2 = v[2], b3 = v[3], avg = (b0 + b1 + b2 + b3) >> 2;
      const int d0 = (b0 >> 6) - (avg >> 6), d1 = (b1 >> 6) - (avg >> 6), d2 = (b2 >> 6) - (avg >> 6), d3 = (b3 >> 6) - (avg >> 6);
      if (d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3 < 20) vaa_sign = 15;               // INTER_VARIANCE_SAD_THRESHOLD
      else vaa_sign = (b0 > avg ? 8 : 0) | (b1 > avg ? 4 : 0) | (b2 > avg ? 2 : 0) | (b3 > avg ? 1 : 0);
    }
    if (c.p.fast_mode && vaa_sign == 15) n_plan = 0;
    else if (c.p.fast_mode && (vaa_sign == 3 || vaa_sign == 12)) { plan[0] = 1; n_plan = 1; }
    else if (c.p.fast_mode && (vaa_sign == 5 || vaa_sign == 10)) { plan[0] = 2; n_plan = 1; }
    else if (c.p.fast_mode && (vaa_sign == 6 || vaa_sign == 9)) { plan[0] = 3; n_plan = 1; }
    else { plan[0] = 3; plan[1] = 1; plan[2] = 2; n_plan = 3; }
  }
  {
    mbk_batch_sync(3, c.batch_n);                                            // ... after the sub-partition searches
    phase_mark(s, 6);
    // refinement (WelsMdInterMbRefinement :1573)
    uint8_t* pl = s.pred_y[0];
    uint8_t* pc = s.pred_c[0];
    int best_sad = 0;
    {
      // one loop over the partitions of the chosen shape: me_refine and mc_chroma_part have ONE call site (inlined there)
      const int shape = final_type == MBT_P16x16 ? 0 : final_type == MBT_P16x8 ? 1 : final_type == MBT_P8x16 ? 2 : 3;
      const int np = shape == 0 ? 1 : shape == 3 ? 4 : 2;
      MeState* arr = shape == 0 ? &me16 : shape == 1 ? me16x8 : shape == 2 ? me8x16 : me8x8;
      if (shape == 3) {
        if (lane_id() == 0) { s.refc[9] = s.refc[21] = REF_NOT_AVAIL; }
        warp_sync();
      }
      MBK_NO_UNROLL
      for (int i = 0; i < np; i++) {
        int ox = 0, oy = 0, w = 16, h = 16, ci = 0, cw = 4, ch = 4;
        if (shape != 0) {                      // the predictor is taken again with the neighbours' final vectors
          int qx, qy;
          if (shape == 1) { pred_16x8_mv(s, 8 * i, 0, &qx, &qy); oy = 8 * i; h = 8; ci = 8 * i; ch = 2; }
          else if (shape == 2) { pred_8x16_mv(s, 4 * i, 0, &qx, &qy); ox = 8 * i; w = 8; ci = 4 * i; cw = 2; }
          else { pred_mv(s, 4 * i, 2, 0, &qx, &qy); ox = (i & 1) * 8; oy = (i >> 1) * 8; w = 8; h = 8; ci = 4 * i; cw = 2; ch = 2; }
          if (lane_id() == 0) { arr[i].mvp_x = qx; arr[i].mvp_y = qy; }
          warp_sync();
        }
        me_refine(c, s, &arr[i], ox, oy, w, h, pl + oy * 16 + ox);
        cache_set(s, ci, cw, ch, arr[i].mv_x, arr[i].mv_y);
        mb_mv_set(s, ci, cw, ch, arr[i].mv_x, arr[i].mv_y);
        if (lane_id() == 0) { s.out.mvd[i][0] = (int16_t)(arr[i].mv_x - arr[i].mvp_x); s.out.mvd[i][1] = (int16_t)(arr[i].mv_y - arr[i].mvp_y); }
        best_sad += (int)arr[i].sad_cost;
        mc_chroma_part(c, pc, ox, oy, w, h, arr[i].mv_x, arr[i].mv_y);
      }
      if (shape == 0)
        cost_skip_mb = warp_sad(s.cur_y, 16, pl, 16, 4, 4) + warp_sad(s.cur_c, 8, pc, 8, 3, 3) + warp_sad(s.cur_c + 64, 8, pc + 64, 8, 3, 3);
    }
    if (lane_id() == 0) c.f.sad_cost[idx] = best_sad;          // pCurMb->pSadCost[0]
    mbk_batch_sync(4, c.batch_n);                                            // ... and after the refinement
    phase_mark(s, 7);
    // step 7: residual coding (WelsMdInterEncode :1964)
    inter_residual_pass(c, s, pl, pc);
    // step 8: a 16x16 MB without residual whose vector equals the skip predictor becomes P_SKIP (:1937)
    if (final_type == MBT_P16x16 && s.info.cbp == 0) {
      // PredSkipMv reads the cache, whose in-MB cells now hold this MB's vector; it only looks at cells 6, 1, 5/0
      int sx, sy;
      pred_skip_mv(s, &sx, &sy);
      if (sx == me16.mv_x && sy == me16.mv_y) final_type = MBT_PSKIP;
    }
#ifndef __CUDA_ARCH__
    g_res_outcome[final_type == MBT_PSKIP ? RES_PSKIP_CODED : RES_P16x16 + final_type - MBT_P16x16]++;
#endif
    if (lane_id() == 0) s.info.mb_type = (uint8_t)final_type;
    warp_sync();
  }
  phase_mark(s, 8);
  st_save(s, 0, cost_luma, cost_skip_mb, p16_mvx, p16_mvy, final_type);
  inter_tail(c, s);
  return MBS_DONE;
}

// the intra branch of a P macroblock (WelsMdFirstIntraMode :1829 after the 16x16 cost won)
MBK_STAGE int inter_stage_c(const MbCtx& c, MbScratch& s) {
  intra_mb_finish(c, s, s.st.cost16, s.st.bb);
  phase_mark(s, 5);
  if (lane_id() == 0) s.st.final_type = s.info.mb_type;
  warp_sync();
  inter_tail(c, s);
  return MBS_DONE;
}

}  // namespace mbk
