// stage_hooks.cuh — the per-macroblock stage test hooks, written once for the device hooks b2h264_debug_* (enc_kernels.cu)
// and their host-build twins emu_* (tests/emu/*_hooks.cu): the record sizes, the argument check each hook applies before it
// runs anything, and the case body that unpacks one case record, runs the stage calls in the stage's order and packs the
// output record.  A case body is run by one warp on the device and by the 1-lane host build (mbk_common.cuh), on a scratch the
// caller has zeroed.  The record layouts are described at the device hooks.
#pragma once
#include <string.h>

#include "enc_frame.cuh"

namespace mbk {

constexpr int kInterResOut = (int)sizeof(MbOut) + 32 + 384;
constexpr int kIntraTailIn = (int)sizeof(RecTile) + 384 + 32;
constexpr int kIntraTailOut = (int)(sizeof(MbOut) + sizeof(MbInfo)) + 16 + (int)sizeof(RecTile);
constexpr int kMeJobIn = 80 * 4 + 256;
constexpr int kMeJobOut = 64 * 4 + 256 + 128;
constexpr int kSkipJobIn = 32 * 4 + 384;
constexpr int kSkipJobOut = 8 * 4 + 384;
constexpr int32_t kSkipSadUnset = 0x5a5a5a5a;     // the skip hook's sad_cost slot before the test runs

// ---- argument checks (host) ----------------------------------------------------------------------------------------------
inline bool inter_residual_args_ok(int n, const uint8_t* src_pred, const int* qp, const uint8_t* out) {
  if (n < 1 || !src_pred || !qp || !out) return false;
  for (int i = 0; i < n; i++)
    if (qp[i] < 0 || qp[i] > 51) return false;
  return true;
}

inline bool intra_tail_args_ok(int n, const uint8_t* in, const uint8_t* out) {
  if (n < 1 || !in || !out) return false;
  for (int i = 0; i < n; i++) {
    const int32_t* prm = reinterpret_cast<const int32_t*>(in + (size_t)kIntraTailIn * i + sizeof(RecTile) + 384);
    if (prm[0] < 0 || prm[0] > 51 || prm[1] < 0 || prm[1] > 15) return false;
  }
  return true;
}

// true when strides sy / sc hold a padded row of mb_w macroblocks and the three padded planes of mb_h rows fit in set_bytes
inline bool padded_set_ok(int mb_w, int mb_h, int sy, int sc, long long set_bytes) {
  return mb_w >= 1 && mb_h >= 1 && sy >= 16 * mb_w + 64 && sc >= 8 * mb_w + 32 &&
         (long long)sy * (16 * mb_h + 64) + 2LL * sc * (8 * mb_h + 32) <= set_bytes;
}

// a negative mv_range is refused: the clip window of the search would no longer keep every block inside the padding
inline bool me_partitions_args_ok(int n, const uint8_t* planes, long long set_bytes, const uint8_t* jobs, const uint8_t* out) {
  if (n < 1 || !planes || !jobs || !out) return false;
  for (int i = 0; i < n; i++) {
    const int32_t* J = reinterpret_cast<const int32_t*>(jobs + (size_t)kMeJobIn * i);
    if (!padded_set_ok(J[0], J[1], J[2], J[3], set_bytes)) return false;
    if (J[4] < 0 || J[5] < 0 || J[5] >= J[0] || J[6] < 0 || J[6] >= J[1] || J[7] < 0 || J[7] > 51 || J[11] < 0 || J[11] > 3) return false;
    for (int q = 0; q < 4; q++)
      if (J[12 + 16 * q + 2] < 0 || J[12 + 16 * q + 2] > 5) return false;
  }
  return true;
}

inline bool skip_test_args_ok(int n, const uint8_t* planes, long long set_bytes, const uint8_t* jobs, const uint8_t* out) {
  if (n < 1 || !planes || !jobs || !out) return false;
  for (int i = 0; i < n; i++) {
    const int32_t* J = reinterpret_cast<const int32_t*>(jobs + (size_t)kSkipJobIn * i);
    if (!padded_set_ok(J[0], J[1], J[2], J[3], set_bytes)) return false;
    if (J[4] < 0 || J[4] >= J[0] || J[5] < 0 || J[5] >= J[1] || J[6] < 0 || J[6] > 51 || J[8] < 0 || J[8] > 15) return false;
    if (J[10] < 0 || J[10] > MBT_PSKIP) return false;
    for (int k = 0; k < 4; k++)
      if (J[12 + 5 * k] < 0 || J[12 + 5 * k] > MBT_PSKIP) return false;
  }
  return true;
}

// ---- case bodies ---------------------------------------------------------------------------------------------------------
// the reference planes of a padded set (Y, then Cb and Cr) at their sample (0, 0)
MBK_HD void set_planes(EncFramePtrs& f, const uint8_t* set, const EncFrameParams& p) {
  const size_t cb = (size_t)p.rec_stride_y * (16 * p.mb_h + 64), cr = cb + (size_t)p.rec_stride_c * (8 * p.mb_h + 32);
  f.ref[0] = set + (size_t)32 * p.rec_stride_y + 32;
  f.ref[1] = set + cb + (size_t)16 * p.rec_stride_c + 16;
  f.ref[2] = set + cr + (size_t)16 * p.rec_stride_c + 16;
}

// stage B's residual step: src = source then prediction (768 bytes), o = the kInterResOut record
MBK_HD void inter_residual_case(const uint8_t* src, int qp, uint8_t* o, MbScratch& s) {
  for (int k = lane_id(); k < 256; k += MBK_WS) { s.cur_y[k] = src[k]; s.pred_y[0][k] = src[384 + k]; }
  for (int k = lane_id(); k < 128; k += MBK_WS) { s.cur_c[k] = src[256 + k]; s.pred_c[0][k] = src[640 + k]; }
  MbCtx c;
  memset(&c, 0, sizeof(c));
  c.qp = qp; c.qp_c = tbl_chroma_qp(c.qp);
  warp_sync();
  inter_residual_pass(c, s, s.pred_y[0], s.pred_c[0]);
  warp_sync();
  for (int k = lane_id(); k < (int)sizeof(MbOut); k += MBK_WS) o[k] = reinterpret_cast<const uint8_t*>(&s.out)[k];
  o += sizeof(MbOut);
  for (int k = lane_id(); k < 32; k += MBK_WS) o[k] = k < 24 ? (uint8_t)s.info.nnz[k] : k == 24 ? s.info.cbp : 0;
  o += 32;
  for (int k = lane_id(); k < 384; k += MBK_WS)
    o[k] = k < 256 ? *tile_y(s.tile, k & 15, k >> 4) : *tile_c(k < 320 ? s.tile.u : s.tile.v, k & 7, (k >> 3) & 7);
}

// stage I's intra tail (md_i16x16, then intra_mb_finish): src = the kIntraTailIn record, o = the kIntraTailOut record;
// sad_slot is the macroblock's sad_cost word
MBK_HD void intra_tail_case(const uint8_t* src, int32_t* sad_slot, uint8_t* o, MbScratch& s) {
  for (int k = lane_id(); k < (int)sizeof(RecTile); k += MBK_WS) reinterpret_cast<uint8_t*>(&s.tile)[k] = src[k];
  src += sizeof(RecTile);
  for (int k = lane_id(); k < 256; k += MBK_WS) s.cur_y[k] = src[k];
  for (int k = lane_id(); k < 128; k += MBK_WS) s.cur_c[k] = src[256 + k];
  const int32_t* prm = reinterpret_cast<const int32_t*>(src + 384);
  const int8_t* nm = reinterpret_cast<const int8_t*>(src + 400);
  if (lane_id() == 0)
    for (int j = 0; j < 8; j++) {
      MbInfo& m = s.nbi[j < 4 ? 3 : 1];
      m.mb_type = nm[j & 4] >= 0 ? MBT_I4x4 : MBT_I16x16;
      m.i4_mode[j < 4 ? 4 * j + 3 : 8 + j] = nm[j];
    }
  MbCtx c;
  memset(&c, 0, sizeof(c));
  c.qp = prm[0]; c.qp_c = tbl_chroma_qp(c.qp); c.lambda = tbl_lambda(c.qp); c.nb = prm[1];
  c.p.fast_mode = prm[2]; c.p.mb_w = 1; c.f.sad_cost = sad_slot;
  warp_sync();
  int bb;
  const int cost16 = md_i16x16(c, s, &bb);
  const int limit = prm[3] < 0 ? cost16 : prm[3];
  const int cost4 = intra_mb_finish(c, s, limit, bb);
  warp_sync();
  for (int k = lane_id(); k < (int)sizeof(MbOut); k += MBK_WS) o[k] = reinterpret_cast<const uint8_t*>(&s.out)[k];
  o += sizeof(MbOut);
  for (int k = lane_id(); k < (int)sizeof(MbInfo); k += MBK_WS) o[k] = reinterpret_cast<const uint8_t*>(&s.info)[k];
  o += sizeof(MbInfo);
  for (int k = lane_id(); k < 4; k += MBK_WS) reinterpret_cast<int32_t*>(o)[k] = k == 0 ? limit : k == 1 ? cost4 : k == 2 ? c.lambda : 0;
  o += 16;
  for (int k = lane_id(); k < (int)sizeof(RecTile); k += MBK_WS) o[k] = reinterpret_cast<const uint8_t*>(&s.tile)[k];
}

// stage B's motion search of one partition shape: job i's kMeJobIn record, its padded plane set, o = its kMeJobOut record.
// tmap_ref / wbar: the search window's tensor map (z = job) and barrier, or NULL (the searches read the planes).
MBK_HD void me_partitions_case(int i, const uint8_t* set, const uint8_t* job, uint8_t* out, MbScratch& s, const void* tmap_ref,
                               WinBar* wbar) {
  const int32_t* J = reinterpret_cast<const int32_t*>(job);
  int32_t* o = reinterpret_cast<int32_t*>(out);
  for (int k = lane_id(); k < kMeJobOut / 4; k += MBK_WS) o[k] = 0;
  for (int k = lane_id(); k < 256; k += MBK_WS) s.cur_y[k] = job[320 + k];
  EncFrameParams p;
  EncFramePtrs f;
  memset(&p, 0, sizeof(p));
  memset(&f, 0, sizeof(f));
  p.mb_w = J[0]; p.mb_h = J[1]; p.rec_stride_y = J[2]; p.rec_stride_c = J[3]; p.mv_range = J[4]; p.qp = J[7]; p.fast_mode = J[8];
  p.ref_plane = i;
  set_planes(f, set, p);
  mb_ctx(s.ctx, p, f, J[5], J[6]);
  if (lane_id() == 0) { s.ctx.tmap_ref = tmap_ref; s.ctx.wbar = wbar; }
  warp_sync();
  const MbCtx& c = s.ctx;
  {
    int sx, sy;
    me_start_point(c, J[9], J[10], &sx, &sy);
    win_issue(c, s, sx, sy);
    win_wait(c, s);
  }
  if (lane_id() == 0) { o[48] = s.win_x0; o[49] = s.win_y0; o[50] = s.win_ok; }
  const int shape = J[11], np = shape == 0 ? 1 : shape == 3 ? 4 : 2;
  const int blk = shape == 0 ? BLK_16x16 : shape == 1 ? BLK_16x8 : shape == 2 ? BLK_8x16 : BLK_8x8;
  const int w = shape == 0 || shape == 1 ? 16 : 8, h = shape == 0 || shape == 2 ? 16 : 8;
  for (int q = 0; q < np; q++) {
    const int32_t* P = J + 12 + 16 * q;
    const int ox = shape == 2 ? 8 * q : shape == 3 ? (q & 1) * 8 : 0, oy = shape == 1 ? 8 * q : shape == 3 ? (q >> 1) * 8 : 0;
    for (int k = lane_id(); k < 10; k += MBK_WS) s.mvcand[k >> 1][k & 1] = (int16_t)P[4 + k];
    warp_sync();
    me_partition(c, s, blk, ox, oy, P[0], P[1], (uint32_t)P[3], P[2], &s.mvcand[0][0], &s.me[q]);
    const MeState& m = s.me[q];
    if (lane_id() == 0) {
      int32_t* r = o + 12 * q;
      r[0] = m.mv_x; r[1] = m.mv_y; r[2] = m.mvp_x; r[3] = m.mvp_y; r[4] = (int32_t)m.sad_cost; r[5] = (int32_t)m.satd_cost;
      r[6] = m.satd; r[7] = (int32_t)(m.ref - c.f.ref[0]);
    }
    warp_sync();
  }
  for (int q = 0; q < np; q++) {
    const int32_t* P = J + 12 + 16 * q;
    const int ox = shape == 2 ? 8 * q : shape == 3 ? (q & 1) * 8 : 0, oy = shape == 1 ? 8 * q : shape == 3 ? (q >> 1) * 8 : 0;
    if (lane_id() == 0) { s.me[q].mvp_x = P[14]; s.me[q].mvp_y = P[15]; }
    warp_sync();
    me_refine(c, s, &s.me[q], ox, oy, w, h, s.pred_y[0] + oy * 16 + ox);
    mc_chroma_part(c, s.pred_c[0], ox, oy, w, h, s.me[q].mv_x, s.me[q].mv_y);
    if (lane_id() == 0) { int32_t* r = o + 12 * q; r[8] = s.me[q].mv_x; r[9] = s.me[q].mv_y; r[10] = (int32_t)s.me[q].satd_cost; }
    warp_sync();
  }
  uint8_t* ob = out + 256;
  for (int k = lane_id(); k < 256; k += MBK_WS) ob[k] = s.pred_y[0][k];
  for (int k = lane_id(); k < 128; k += MBK_WS) ob[256 + k] = s.pred_c[0][k];
}

// stage A's P-skip test: the kSkipJobIn record, the one plane set every job reads, o = the kSkipJobOut record; sad_slot is
// the macroblock's sad_cost word, holding kSkipSadUnset
MBK_HD void skip_test_case(const uint8_t* job, const uint8_t* planes, int32_t* sad_slot, uint8_t* out, MbScratch& s) {
  const int32_t* J = reinterpret_cast<const int32_t*>(job);
  for (int k = lane_id(); k < 256; k += MBK_WS) s.cur_y[k] = job[128 + k];
  for (int k = lane_id(); k < 128; k += MBK_WS) s.cur_c[k] = job[384 + k];
  for (int k = lane_id(); k < 4; k += MBK_WS) {
    const int32_t* N = J + 12 + 5 * k;
    s.nbi[k].mb_type = (uint8_t)N[0];
    for (int b = 0; b < 16; b++) { s.nbi[k].mv[b][0] = (int16_t)N[1]; s.nbi[k].mv[b][1] = (int16_t)N[2]; }
    s.nb_sad[k] = N[3];
    s.nb_skip_sad[k] = N[4];
  }
  if (lane_id() == 0) { s.col.mb_type = (uint8_t)J[10]; s.col.skip_sad = J[11]; }
  EncFrameParams p;
  EncFramePtrs f;
  memset(&p, 0, sizeof(p));
  memset(&f, 0, sizeof(f));
  p.mb_w = J[0]; p.mb_h = J[1]; p.rec_stride_y = J[2]; p.rec_stride_c = J[3]; p.qp = J[6]; p.fast_mode = J[7]; p.ref_is_p = J[9];
  set_planes(f, planes, p);
  f.sad_cost = sad_slot - (J[5] * p.mb_w + J[4]);      // the macroblock's own slot is the one word
  mb_ctx(s.ctx, p, f, J[4], J[5]);
  if (lane_id() == 0) s.ctx.nb = J[8];
  warp_sync();
  const MbCtx& c = s.ctx;
  fill_inter_cache(c, s);
  const int sad_pred = predict_sad_skip(s);
  const SkipResult r = pskip_enc(c, s, sad_pred);
  warp_sync();
  int32_t* o = reinterpret_cast<int32_t*>(out);
  if (lane_id() == 0) { o[0] = r.ok; o[1] = r.mvx; o[2] = r.mvy; o[3] = sad_pred; o[4] = r.cost_luma; o[5] = r.cost_skip; o[6] = *sad_slot; o[7] = 0; }
  for (int k = lane_id(); k < 384; k += MBK_WS) out[32 + k] = s.skip_pred[k];
}

}  // namespace mbk
