// dec_mb.cuh — decoder CONSTRUCT stage of one macroblock by one warp: prediction (intra / motion compensated) +
// dequantisation + inverse transform + reconstruction from a parsed MbOut record (h264_parse.h).  It is the mirror
// image of the encoder's reconstruction path and is built from the same pieces (mbk_mc / mbk_xform / enc_intra /
// the MV-prediction cache of enc_inter.cuh), so what the encoder reconstructs and what this stage reconstructs from
// the encoder's own bitstream are the same samples by construction — and both are checked against the reference
// decoder (tests/test_decoder_emu.py runs the host build of this file against ISVCDecoder::DecodeFrameNoDelay).
// Reference counterparts: codec/decoder/core/src/rec_mb.cpp (BaseMC :244, GetInterPred :462, RecI4x4Mb / RecI16x16Mb
// :64-215), decode_mb_aux.cpp (IdctResAddPred_c :42), mv_pred.cpp (PredMv, PredPSkipMvFromNeighbor), parse side
// ParseIntra4x4Mode (parse_mb_syn_cavlc.cpp).
// Runs on the device as k_decode_mbs (enc_kernels.cu) and, compiled for the host, as the debugging build of tests/emu.
#pragma once
#include "enc_inter.cuh"
#include "dec_t8x8.cuh"
#include "wp_formula.h"

namespace mbk {

MBK_HD void unscan16(int16_t d[16], const int16_t lv[16]) {
  for (int i = 0; i < 16; i++) d[zigzag_pos(i)] = lv[i];
}
MBK_HD void unscan15(int16_t d[16], const int16_t lv[16]) {     // AC levels: scan positions 1..15
  d[0] = 0;
  for (int i = 1; i < 16; i++) d[zigzag_pos(i)] = lv[i - 1];
}

// neighbour records only (the encoder's loader also fetches SAD history the decoder does not have)
MBK_HD void dec_load_neighbors(const MbCtx& c, MbScratch& s) {
  const int mbw = c.p.mb_w, idx = c.mby * mbw + c.mbx;
  const int offs[4] = {-mbw - 1, -mbw, -mbw + 1, -1};
  const int bits[4] = {NB_TOPLEFT, NB_TOP, NB_TOPRIGHT, NB_LEFT};
  constexpr int kW = (int)(sizeof(MbInfo) / 4);
  for (int i = lane_id(); i < 4 * kW; i += MBK_WS) {
    const int k = i / kW, w = i - k * kW;
    reinterpret_cast<uint32_t*>(&s.nbi[k])[w] =
        (c.nb & bits[k]) ? ld_cg_u32(reinterpret_cast<const uint32_t*>(c.f.mbi + idx + offs[k]) + w) : 0u;
  }
  for (int k = lane_id(); k < 4; k += MBK_WS) { s.nb_sad[k] = 0; s.nb_skip_sad[k] = 0; }
  warp_sync();
}

// luma residual of the 16 blocks into s.coef (dequantised, raster within a block), zero where nothing is coded
MBK_HD void dec_luma_coef(MbScratch& s, const MbOut& m, int qp, bool i16, const int16_t* dcq) {
  for (int k = lane_id(); k < 16; k += MBK_WS) {
    int16_t d[16];
    for (int i = 0; i < 16; i++) d[i] = 0;
    if (m.cbp & (1 << (k >> 2))) {
      if (i16) unscan15(d, m.luma[k]);
      else unscan16(d, m.luma[k]);
      dequant4x4(d, tbl_dequant(qp));
    }
    if (i16) d[0] = dcq[blk_raster(k)];
    for (int i = 0; i < 16; i++) s.coef[16 * k + i] = d[i];
  }
  warp_sync();
}

MBK_HD void dec_chroma_coef(MbScratch& s, const MbOut& m, int qp_c) {
  const int cbp_c = m.cbp >> 4;
  for (int t = lane_id(); t < 8; t += MBK_WS) {
    const int uv = t >> 2, j = t & 3;
    int16_t d[16];
    for (int i = 0; i < 16; i++) d[i] = 0;
    if (cbp_c == 2) { unscan15(d, m.chroma_ac[t]); dequant4x4(d, tbl_dequant(qp_c)); }
    if (cbp_c) {
      int16_t dc[4] = {m.chroma_dc[uv][0], m.chroma_dc[uv][1], m.chroma_dc[uv][2], m.chroma_dc[uv][3]};
      if (dc[0] | dc[1] | dc[2] | dc[3]) { dequant_ihadamard2x2_dc(dc, tbl_dequant(qp_c)[0]); d[0] = dc[j]; }
    }
    for (int i = 0; i < 16; i++) s.coef[256 + 64 * uv + 16 * j + i] = d[i];
  }
  warp_sync();
}

// picture slot -> plane pointers (pixel (0,0)); REF_NOT_AVAIL cells of the motion cache sit below the slot numbers (0..16)
MBK_HD const uint8_t* dec_ref_plane(const MbCtx& c, int pl, int slot) { return c.f.dpb0[pl] + (ptrdiff_t)slot * c.f.dpb_stride; }
// motion compensation of one partition from picture `slot` into the prediction buffers (BaseMC, rec_mb.cpp:244)
MBK_HD void dec_mc_part(const MbCtx& c, uint8_t* pl, uint8_t* pc, int slot, int blk, int w4, int h4, int mvx, int mvy) {
  const int ox = blk_x(blk) * 4, oy = blk_y(blk) * 4, w = w4 * 4, h = h4 * 4;
  // absolute quarter-sample position, clipped like BaseMC (rec_mb.cpp:248-253: the padded reference is 32 wide);
  // luma and chroma both derive from the clipped position
  int fx = ((c.mbx * 16 + ox) << 2) + mvx, fy = ((c.mby * 16 + oy) << 2) + mvy;
  fx = clip3(fx, (-32 + 2) * 4, (c.p.mb_w * 16 + 32 - 19) * 4);
  fy = clip3(fy, (-32 + 2) * 4, (c.p.mb_h * 16 + 32 - 19) * 4);
  warp_mc_luma(dec_ref_plane(c, 0, slot) + (ptrdiff_t)(fy >> 2) * c.p.rec_stride_y + (fx >> 2), c.p.rec_stride_y, pl + oy * 16 + ox, 16, fx, fy, w, h);
  for (int cpl = 0; cpl < 2; cpl++)
    warp_mc_chroma(dec_ref_plane(c, 1 + cpl, slot) + (ptrdiff_t)(fy >> 3) * c.p.rec_stride_c + (fx >> 3), c.p.rec_stride_c,
                   pc + 64 * cpl + (oy >> 1) * 8 + (ox >> 1), 8, fx, fy, w >> 1, h >> 1);
  warp_sync();
}
// reference slot of the 8x8 quadrant that holds 4x4 block `blk` (coding order)
MBK_HD int dec_ref_of(const DecMbAux& aux, int blk) { return aux.ref_idx[blk >> 2]; }

// luma of an inter macroblock with the 8x8 transform: lane k reconstructs 8x8 block k (prediction + inverse transform of its 64 levels)
// (real functions, not inlined: their 64-entry arrays live on the stack, and only High-profile macroblocks pay for that frame)
MBK_FN void rec_luma_inter8(MbScratch& s, const MbOut& m, int qp, const uint8_t* pl) {
  for (int k = lane_id(); k < 4; k += MBK_WS) {
    const int ox = (k & 1) * 8, oy = (k >> 1) * 8;
    uint8_t* org = tile_y(s.tile, ox, oy);
    if (m.cbp & (1 << k)) {
      int16_t d[64];
      unscan_dequant8x8(d, &m.luma[4 * k][0], qp);
      idct8x8_rec(org, TY_PITCH, pl + oy * 16 + ox, 16, d);
    } else {
      for (int y = 0; y < 8; y++) for (int x = 0; x < 8; x++) org[y * TY_PITCH + x] = pl[(oy + y) * 16 + ox + x];
    }
  }
  warp_sync();
}

// the four Intra_8x8 blocks of a macroblock on lane 0, each predicting from what was just reconstructed (mode cache s.i4m prepared)
MBK_FN void dec_i8x8_blocks(MbScratch& s, const MbOut& m, int nb_i, int qp) {
  if (lane_id() == 0) {
    for (int k = 0; k < 4; k++) {
      const int bx = (k & 1) * 2, by = (k >> 1) * 2;
      uint8_t* org = tile_y(s.tile, bx * 4, by * 4);
      const int lm = s.i4m[(by + 1) * 5 + bx], tm = s.i4m[by * 5 + bx + 1];
      const int pm = (lm == -1 || tm == -1) ? 2 : (lm < tm ? lm : tm);
      const int coded = m.prev_i4_flag[k] ? pm : (m.rem_i4_mode[k] < pm ? m.rem_i4_mode[k] : m.rem_i4_mode[k] + 1);
      // neighbouring samples of the 8x8 block (6.4.11): left / top from the neighbouring macroblock or from inside, top-right of
      // block 1 from the top-right macroblock, of block 2 from block 1, of block 3 never
      const bool aL = (k & 1) ? true : (nb_i & NB_LEFT) != 0, aT = (k >> 1) ? true : (nb_i & NB_TOP) != 0;
      const bool aTL = k == 0 ? (nb_i & NB_TOPLEFT) != 0 : k == 1 ? (nb_i & NB_TOP) != 0 : k == 2 ? (nb_i & NB_LEFT) != 0 : true;
      const bool aTR = k == 0 ? (nb_i & NB_TOP) != 0 : k == 1 ? (nb_i & NB_TOPRIGHT) != 0 : k == 2;
      for (int y = 0; y < 2; y++) for (int x = 0; x < 2; x++) {
        s.i4m[(by + y + 1) * 5 + bx + x + 1] = (int8_t)coded;
        s.info.i4_mode[(by + y) * 4 + bx + x] = (int8_t)coded;
      }
      uint8_t pr[64];
      pred_i8x8(pr, org, TY_PITCH, coded, (aL ? 1 : 0) | (aT ? 2 : 0) | (aTL ? 4 : 0) | (aTR ? 8 : 0));
      if (m.cbp & (1 << k)) {
        int16_t d[64];
        unscan_dequant8x8(d, &m.luma[4 * k][0], qp);
        idct8x8_rec(org, TY_PITCH, pr, 8, d);
      } else {
        for (int y = 0; y < 8; y++) for (int x = 0; x < 8; x++) org[y * TY_PITCH + x] = pr[8 * y + x];
      }
    }
  }
}

// A B macroblock (or a P macroblock that travels resolved: explicit weights).  A real function: the Baseline path of dec_one_mb keeps
// its registers and stack frame.
MBK_FN void dec_b_mb(const MbCtx& c, const EncFrameParams& p, MbScratch& s, const MbOut& m, const DecMbAux& aux, int mbx, int mby,
                     uint8_t* pl, uint8_t* pc, int qp) {
  // B macroblock (GetInterBPred, rec_mb.cpp:666 ff.): the parser resolved both lists (h264_motion.h) — per 8x8 a picture slot and
  // FINAL vectors per 4x4 block for list 0 (aux) and list 1 (dec_aux_b).  Each list is motion compensated like a P partition (one
  // 8x8 where the four blocks move together, else 4x4 by 4x4), then the 8x8 goes through the weighting formula its record names
  // (DecMbAuxB: one list, two lists, or none; default, implicit and explicit weights are all values of the same two formulas).
  const DecMbAuxB& ab = c.f.dec_aux_b[mby * p.mb_w + mbx];
  uint8_t* pl1 = s.pred_y[1];
  uint8_t* pc1 = s.pred_c[1];
  for (int k = 0; k < 4; k++) {
    const int pred = ab.pred[k];
    const int r0 = (pred & DECB_L0) ? aux.ref_idx[k] : -1, r1 = (pred & DECB_L1) ? ab.ref_idx[k] : -1;
    bool whole = true;
    for (int j = 1; j < 4; j++)
      whole = whole && aux.mvd[4 * k + j][0] == aux.mvd[4 * k][0] && aux.mvd[4 * k + j][1] == aux.mvd[4 * k][1] &&
              ab.mv[4 * k + j][0] == ab.mv[4 * k][0] && ab.mv[4 * k + j][1] == ab.mv[4 * k][1];
    for (int l = 0; l < 2; l++) {
      const int slot = l ? r1 : r0;
      if (slot < 0) continue;
      uint8_t* dl = (l && r0 >= 0) ? pl1 : pl;                   // list 1 alone predicts straight into the first buffer
      uint8_t* dc = (l && r0 >= 0) ? pc1 : pc;
      if (whole) {
        const int mvx = l ? ab.mv[4 * k][0] : aux.mvd[4 * k][0], mvy = l ? ab.mv[4 * k][1] : aux.mvd[4 * k][1];
        dec_mc_part(c, dl, dc, slot, 4 * k, 2, 2, mvx, mvy);
      } else {
        for (int j = 0; j < 4; j++) {
          const int mvx = l ? ab.mv[4 * k + j][0] : aux.mvd[4 * k + j][0], mvy = l ? ab.mv[4 * k + j][1] : aux.mvd[4 * k + j][1];
          dec_mc_part(c, dl, dc, slot, 4 * k + j, 1, 1, mvx, mvy);
        }
      }
    }
    if (pred & (DECB_WEIGHT | DECB_BI)) {
      // the 8x8's samples, luma then Cb / Cr: first input from buffer 0, second from buffer 1 where both lists were motion compensated,
      // else from buffer 0 as well; the one-list formula may cover the lower 8x4 / right 4x8 only (DECB_LOWER / DECB_RIGHT)
      const bool bi = (pred & DECB_BI) != 0, two = r0 >= 0 && r1 >= 0;
      const int qx = (k & 1) * 8, qy = (k >> 1) * 8, x0 = (pred & DECB_RIGHT) ? 4 : 0, y0 = (pred & DECB_LOWER) ? 4 : 0;
      for (int i = lane_id(); i < 64 + 32; i += MBK_WS) {
        int pos, plane, x, y;
        uint8_t *a, *b;
        if (i < 64) { x = i & 7; y = i >> 3; pos = (qy + y) * 16 + qx + x; a = pl; b = two ? pl1 : pl; plane = 0; }
        else {
          const int t = i - 64, cpl = t >> 4;
          x = 2 * (t & 3); y = 2 * ((t & 15) >> 2);                 // chroma sample in luma units of the 8x8, for the region test
          pos = 64 * cpl + ((qy + y) >> 1) * 8 + ((qx + x) >> 1); a = pc; b = two ? pc1 : pc; plane = 1 + cpl;
        }
        if (x < x0 || y < y0) continue;
        const int e = 4 * plane + k, ld = (aux.wp_log2 >> (plane ? 4 : 0)) & 15;
        const int v = bi ? wp_bi(a[pos], b[pos], ab.w0[e], ab.w1[e], ab.o[e], ld) : wp_single(a[pos], ab.w0[e], ab.o[e], ld);
#ifdef B2H264_WP_STATS
        if ((aux.flags & DECAUX_EXPLICIT_B) && (v < 0 || v > 255)) b2h264_wp_stat(v < 0 ? WPS_CLIP_LOW : WPS_CLIP_HIGH, 1);
#endif
        a[pos] = (uint8_t)clip255(v);
      }
      warp_sync();
    }
  }
  if (lane_id() == 0)
    for (int b = 0; b < 16; b++) {
      const int bx = b & 3, by = b >> 2, z = ((by >> 1) * 2 + (bx >> 1)) * 4 + (by & 1) * 2 + (bx & 1);
      const bool used = aux.ref_idx[z >> 2] >= 0;
      s.info.mv[b][0] = used ? aux.mvd[z][0] : 0; s.info.mv[b][1] = used ? aux.mvd[z][1] : 0;
    }
  warp_sync();
  if (aux.flags & DECAUX_T8) rec_luma_inter8(s, m, qp, pl);
  else { dec_luma_coef(s, m, qp, false, nullptr); rec_luma_inter(s, pl); }
}

// One macroblock.  f.rec = picture being reconstructed, f.ref = reference picture (padded), f.mbi = MbInfo array of
// the picture (neighbour lookups + what deblocking reads).  Raster / wavefront order like the encoder.
MBK_HD void dec_one_mb(const EncFrameParams& p, const EncFramePtrs& f, MbScratch& s, int mbx, int mby, const MbOut& m, const DecMbAux& aux) {
  mb_ctx(s.ctx, p, f, mbx, mby);
  // neighbour availability comes from the parser: macroblocks of other slices do not count (6.4.x)
  if (lane_id() == 0) { s.ctx.qp = m.qp; s.ctx.qp_c = tbl_chroma_qp(clip3(m.qp + p.dec_cqp_off, 0, 51)); s.ctx.nb = aux.avail; }
  warp_sync();
  const MbCtx& c = s.ctx;
  {
    uint32_t* a = reinterpret_cast<uint32_t*>(&s.info);
    for (int i = lane_id(); i < (int)(sizeof(MbInfo) / 4); i += MBK_WS) a[i] = 0;
  }
  warp_sync();
  dec_load_neighbors(c, s);
  mb_load_borders(c, s);
  const int type = m.mb_type, qp = m.qp, qp_c = c.qp_c;
  if (lane_id() == 0) {
    s.info.mb_type = (uint8_t)type; s.info.cbp = m.cbp;
    for (int i = 0; i < 24; i++) s.info.nnz[i] = m.nnz[i];
    s.info.ref_idx = MBT_IS_INTER(type) ? 0 : REF_NOT_IN_LIST;
  }
  warp_sync();
  uint8_t* pl = s.pred_y[0];
  uint8_t* pc = s.pred_c[0];
  // constrained intra prediction: inter-coded neighbours do not count for INTRA prediction (8.3.1.2, 8.3.3, 8.3.4)
  int nb_i = c.nb;
  if (aux.flags & DECAUX_CIP) {
    if ((nb_i & NB_TOPLEFT) && MBT_IS_INTER(s.nbi[0].mb_type)) nb_i &= ~NB_TOPLEFT;
    if ((nb_i & NB_TOP) && MBT_IS_INTER(s.nbi[1].mb_type)) nb_i &= ~NB_TOP;
    if ((nb_i & NB_TOPRIGHT) && MBT_IS_INTER(s.nbi[2].mb_type)) nb_i &= ~NB_TOPRIGHT;
    if ((nb_i & NB_LEFT) && MBT_IS_INTER(s.nbi[3].mb_type)) nb_i &= ~NB_LEFT;
  }
  const bool L = (nb_i & NB_LEFT) != 0, T = (nb_i & NB_TOP) != 0;
  if (type == MBT_IPCM) {                       // raw samples: straight into the tile; nothing to predict or transform
    const uint8_t* py = reinterpret_cast<const uint8_t*>(m.luma);
    const uint8_t* pcs = reinterpret_cast<const uint8_t*>(m.chroma_ac);
    for (int i = lane_id(); i < 256; i += MBK_WS) *tile_y(s.tile, i & 15, i >> 4) = py[i];
    for (int i = lane_id(); i < 64; i += MBK_WS) {
      *tile_c(s.tile.u, i & 7, i >> 3) = pcs[i];
      *tile_c(s.tile.v, i & 7, i >> 3) = pcs[64 + i];
    }
    warp_sync();
    mb_store_recon(c, s);
    if (lane_id() == 0) {
      s.info.qp = 0; s.info.qp_c = (uint8_t)tbl_chroma_qp(clip3(p.dec_cqp_off, 0, 51));
      s.info.p16x16_mv[0] = (int16_t)aux.slice;
      s.info.p16x16_mv[1] = (int16_t)(aux.dbk_idc | ((aux.alpha_off + 16) << 2) | ((aux.beta_off + 16) << 7));
    }
    warp_sync();
    const uint32_t* si0 = reinterpret_cast<const uint32_t*>(&s.info);
    uint32_t* di0 = reinterpret_cast<uint32_t*>(c.f.mbi + (mby * p.mb_w + mbx));
    for (int i = lane_id(); i < (int)(sizeof(MbInfo) / 4); i += MBK_WS) di0[i] = si0[i];
    warp_sync();
    return;
  }
  if (MBT_IS_B(type)) {
    dec_b_mb(c, p, s, m, aux, mbx, mby, pl, pc, qp);
  } else if (type == MBT_P8x8 && (aux.flags & DECAUX_SUB)) {
    // sub-macroblock partitions (8x4, 4x8, 4x4): every partition predicts its vector from the cells decoded so far —
    // the in-macroblock cells start as "not available" and are filled in decoding order (8.4.1.3.2: a partition that
    // comes later in decoding order is not available as neighbour C, the top-left neighbour D steps in)
    fill_inter_cache(c, s, true);
    if (lane_id() == 0)
      for (int r = 1; r < 5; r++) for (int q = 1; q < 5; q++) s.refc[r * 6 + q] = REF_NOT_AVAIL;
    warp_sync();
    for (int k = 0; k < 4; k++) {
      const int st = aux.sub_type[k];
      const int w4 = (st == 0 || st == 1) ? 2 : 1, h4 = (st == 0 || st == 2) ? 2 : 1, np = st == 0 ? 1 : st == 3 ? 4 : 2;
      for (int j = 0; j < np; j++) {
        const int blk = 4 * k + (st == 1 ? 2 * j : j);           // 8x4: rows of the 8x8; 4x8 / 4x4: blocks in coding order
        int px, py;
        const int ref = aux.ref_idx[k];
        pred_mv(s, blk, w4, ref, &px, &py);
        const int mvx = px + aux.mvd[4 * k + j][0], mvy = py + aux.mvd[4 * k + j][1];
        cache_set(s, blk, w4, h4, mvx, mvy, ref);
        mb_mv_set(s, blk, w4, h4, mvx, mvy);
        dec_mc_part(c, pl, pc, ref, blk, w4, h4, mvx, mvy);
      }
    }
    dec_luma_coef(s, m, qp, false, nullptr);
    rec_luma_inter(s, pl);
  } else if (MBT_IS_INTER(type)) {
    fill_inter_cache(c, s, true);
    const int nparts = type == MBT_P8x8 ? 4 : (type == MBT_P16x8 || type == MBT_P8x16) ? 2 : 1;
    if (type == MBT_P8x8) { if (lane_id() == 0) { s.refc[9] = s.refc[21] = REF_NOT_AVAIL; } warp_sync(); }
    for (int i = 0; i < nparts; i++) {
      int blk = 0, w4 = 4, h4 = 4, px = 0, py = 0;
      if (type == MBT_P16x8) { blk = 8 * i; h4 = 2; }
      else if (type == MBT_P8x16) { blk = 4 * i; w4 = 2; }
      else if (type == MBT_P8x8) { blk = 4 * i; w4 = 2; h4 = 2; }
      const int ref = dec_ref_of(aux, blk);                       // picture slot of this partition's reference
      if (type == MBT_PSKIP) pred_skip_mv(s, &px, &py, ref);
      else if (type == MBT_P16x16) pred_mv(s, 0, 4, ref, &px, &py);
      else if (type == MBT_P16x8) pred_16x8_mv(s, blk, ref, &px, &py);
      else if (type == MBT_P8x16) pred_8x16_mv(s, blk, ref, &px, &py);
      else pred_mv(s, blk, 2, ref, &px, &py);
      const int mvx = px + (type == MBT_PSKIP ? 0 : m.mvd[i][0]), mvy = py + (type == MBT_PSKIP ? 0 : m.mvd[i][1]);
      cache_set(s, blk, w4, h4, mvx, mvy, ref);
      mb_mv_set(s, blk, w4, h4, mvx, mvy);
      dec_mc_part(c, pl, pc, ref, blk, w4, h4, mvx, mvy);
    }
    warp_sync();
    if (aux.flags & DECAUX_T8) rec_luma_inter8(s, m, qp, pl);
    else { dec_luma_coef(s, m, qp, false, nullptr); rec_luma_inter(s, pl); }
  } else if (type == MBT_I16x16) {
    const int mode = m.i16_mode == 2 ? (L && T ? I16_DC : L ? I16_DC_L : T ? I16_DC_T : I16_DC_128) : m.i16_mode;
    pred_i16(pl, tile_y(s.tile, 0, 0), TY_PITCH, mode);
    warp_sync();
    int16_t dcq[16];
    unscan16(dcq, m.luma_dc);
    bool any = false;
    for (int i = 0; i < 16; i++) any = any || dcq[i] != 0;
    if (any) {
      if (qp < 12) { ihadamard4x4(dcq); dequant_luma_dc4x4(dcq, qp); }
      else dequant_ihadamard4x4(dcq, (uint16_t)(tbl_dequant(qp)[0] >> 2));
    }
    dec_luma_coef(s, m, qp, true, dcq);
    rec_luma_inter(s, pl);                       // inverse transform + prediction for all 16 blocks
  } else if (aux.flags & DECAUX_T8) {            // Intra_8x8: four blocks, each predicts from what was just reconstructed
    fill_i4_cache(c, s);                         // mode cache at 4x4 granularity: an Intra_8x8 block's mode stands in its four cells
    if (aux.flags & DECAUX_CIP) {
      if (lane_id() == 0) {
        if ((c.nb & NB_LEFT) && MBT_IS_INTER(s.nbi[3].mb_type)) for (int y = 0; y < 4; y++) s.i4m[(y + 1) * 5] = -1;
        if ((c.nb & NB_TOP) && MBT_IS_INTER(s.nbi[1].mb_type)) for (int x = 0; x < 4; x++) s.i4m[x + 1] = -1;
      }
      warp_sync();
    }
    dec_i8x8_blocks(s, m, nb_i, qp);
    warp_sync();
  } else {                                       // I4x4: block by block, each predicts from what was just reconstructed
    fill_i4_cache(c, s);
    if (aux.flags & DECAUX_CIP) {              // 8.3.1.1: an Inter neighbour under constrained_intra_pred forces the DC prediction of the
      if (lane_id() == 0) {                    // mode (dcPredModePredictedFlag), exactly like a missing neighbour — not "mode 2 in the min"
        if ((c.nb & NB_LEFT) && MBT_IS_INTER(s.nbi[3].mb_type)) for (int y = 0; y < 4; y++) s.i4m[(y + 1) * 5] = -1;
        if ((c.nb & NB_TOP) && MBT_IS_INTER(s.nbi[1].mb_type)) for (int x = 0; x < 4; x++) s.i4m[x + 1] = -1;
      }
      warp_sync();
    }
    for (int k = 0; k < 16; k++) {
      const int bx = blk_x(k), by = blk_y(k);
      uint8_t* org = tile_y(s.tile, bx * 4, by * 4);
      const int lm = s.i4m[(by + 1) * 5 + bx], tm = s.i4m[by * 5 + bx + 1];
      const int pm = (lm == -1 || tm == -1) ? 2 : (lm < tm ? lm : tm);
      const int coded = m.prev_i4_flag[k] ? pm : (m.rem_i4_mode[k] < pm ? m.rem_i4_mode[k] : m.rem_i4_mode[k] + 1);
      const int av = i4_avail(nb_i, k);
      const int mode = coded == 2 ? ((av & 1) && (av & 2) ? I4_DC : (av & 1) ? I4_DC_L : (av & 2) ? I4_DC_T : I4_DC_128) : coded;
      if (lane_id() == 0) {
        s.i4m[(by + 1) * 5 + bx + 1] = (int8_t)coded;
        s.info.i4_mode[by * 4 + bx] = (int8_t)coded;
        // 8.3.1.2: when the top-right 4 samples are not available they are replaced by the last top sample.  (The
        // encoder never selects DDL / VL in that situation, a decoder has to cope; the tile cells written here belong
        // to a block that is decoded later or to nobody.)
        if ((mode == I4_DDL || mode == I4_VL) && !(av & 8))
          for (int i = 4; i < 8; i++) org[-TY_PITCH + i] = org[-TY_PITCH + 3];
        uint8_t pr[16];
        int16_t d[16];
        for (int i = 0; i < 16; i++) d[i] = 0;
        pred_i4(pr, org, TY_PITCH, mode);
        if (m.cbp & (1 << (k >> 2))) { unscan16(d, m.luma[k]); dequant4x4(d, tbl_dequant(qp)); }
        idct4x4_rec(org, TY_PITCH, pr, 4, d);
      }
      warp_sync();
    }
  }
  if (MBT_IS_INTRA(type)) {
    const int cm = m.chroma_mode == 0 ? (L && T ? C_DC : L ? C_DC_L : T ? C_DC_T : C_DC_128) : m.chroma_mode;
    pred_chroma(pc, tile_c(s.tile.u, 0, 0), TC_PITCH, cm);
    pred_chroma(pc + 64, tile_c(s.tile.v, 0, 0), TC_PITCH, cm);
    warp_sync();
  }
  dec_chroma_coef(s, m, qp_c);
  rec_chroma(s, pc);
  mb_store_recon(c, s);
  // what the neighbours and the deblocking filter read
  if (lane_id() == 0) {
    s.info.qp = (uint8_t)qp; s.info.qp_c = (uint8_t)qp_c;
    if (aux.flags & DECAUX_T8) {                // the filter asks whether the 8x8 TRANSFORM block holds coefficients (8.7.2.1)
      s.info.t8x8 = 1;
      for (int k = 0; k < 4; k++) {
        const int b0 = (k >> 1) * 8 + (k & 1) * 2;
        const int tot = s.info.nnz[b0] + s.info.nnz[b0 + 1] + s.info.nnz[b0 + 4] + s.info.nnz[b0 + 5];
        s.info.nnz[b0] = s.info.nnz[b0 + 1] = s.info.nnz[b0 + 4] = s.info.nnz[b0 + 5] = (int8_t)(tot > 64 ? 64 : tot);
      }
    }
    if (MBT_IS_INTER(type))                     // reference picture slot of every 4x4 block (raster): MV prediction of the neighbours, bS
      for (int b = 0; b < 16; b++) s.info.i4_mode[b] = aux.ref_idx[(b >> 3) * 2 + ((b >> 1) & 1)];
    // the decoder has no use for sP16x16Mv: the field carries what the deblocking pass needs to know about the slice
    s.info.p16x16_mv[0] = (int16_t)aux.slice;
    s.info.p16x16_mv[1] = (int16_t)(aux.dbk_idc | ((aux.alpha_off + 16) << 2) | ((aux.beta_off + 16) << 7));
  }
  warp_sync();
  const uint32_t* si = reinterpret_cast<const uint32_t*>(&s.info);
  uint32_t* di = reinterpret_cast<uint32_t*>(c.f.mbi + (mby * p.mb_w + mbx));
  for (int i = lane_id(); i < (int)(sizeof(MbInfo) / 4); i += MBK_WS) di[i] = si[i];
  warp_sync();
}

}  // namespace mbk
