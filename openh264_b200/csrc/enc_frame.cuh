// enc_frame.cuh — macroblock entry point shared by the CUDA wavefront kernel (enc_kernels.cu) and the
// host emulation build (tests/emu).  One call = one macroblock = one warp.
#pragma once
#include "enc_mb.cuh"
#include "enc_cavlc_bits.cuh"
#include "enc_inter.cuh"

namespace mbk {

// fills the context kept in the scratch (s.ctx); the warp copies the frame descriptor word by word
MBK_HD void mb_ctx(MbCtx& c, const EncFrameParams& p, const EncFramePtrs& f, int mbx, int mby) {
  static_assert(sizeof(EncFrameParams) % 4 == 0 && sizeof(EncFramePtrs) % 4 == 0, "copied as words");
  warp_sync();
  const uint32_t* sp = reinterpret_cast<const uint32_t*>(&p);
  const uint32_t* sfp = reinterpret_cast<const uint32_t*>(&f);
  uint32_t* dp = reinterpret_cast<uint32_t*>(&c.p);
  uint32_t* df = reinterpret_cast<uint32_t*>(&c.f);
  for (int i = lane_id(); i < (int)(sizeof(EncFrameParams) / 4); i += MBK_WS) dp[i] = sp[i];
  for (int i = lane_id(); i < (int)(sizeof(EncFramePtrs) / 4); i += MBK_WS) df[i] = sfp[i];
  if (lane_id() == 0) {
    c.mbx = mbx; c.mby = mby;
    // a neighbour is available when it lies in the picture and in the macroblock's slice: slices are raster runs, so when its
    // address is not below the slice's first (with one slice every neighbour in the picture qualifies)
    const int idx = mby * p.mb_w + mbx, first = f.slice_first ? f.slice_first[idx] : 0, top = idx - p.mb_w;
    c.nb = (mbx > 0 && idx - 1 >= first ? NB_LEFT : 0) | (mby > 0 && top >= first ? NB_TOP : 0) |
           (mbx > 0 && mby > 0 && top - 1 >= first ? NB_TOPLEFT : 0) | (mby > 0 && mbx < p.mb_w - 1 && top + 1 >= first ? NB_TOPRIGHT : 0);
    c.qp = p.qp;
    c.qp_c = tbl_chroma_qp(p.qp);          // chroma_qp_index_offset = 0
    c.lambda = tbl_lambda(p.qp);
    c.tmap_ref = nullptr; c.wbar = nullptr;       // the device encode kernel fills these in after mb_ctx
  }
  warp_sync();
}

// Runs ONE stage of a macroblock (see enc_inter.cuh) and returns the stage to run next (MBS_DONE: the
// reconstruction and the records are stored and published).  MBS_A / MBS_I are the entry stages of a P / an IDR
// picture's macroblock: they start from an empty scratch; the others continue on the scratch the previous stage left.
// Host build: after a stage A that ran the skip candidate's intra check it returns MBP_SKIPCAND_INTRA, and called with that
// id it returns the stage that really follows (enc_inter.cuh: the paths keep their numbering).
MBK_HD int mb_run_stage(const MbCtx& c, MbScratch& s, int stage) {
#ifndef __CUDA_ARCH__
  if (stage == MBP_SKIPCAND_INTRA) return g_skipcand_next;
  g_skipcand_intra = false;
#endif
  int next = MBS_DONE;
  if (stage == MBS_A || stage == MBS_I) {
    phase_mark(s, 31);
    // clear the staged records (levels need no clearing: every block that gets written to the bitstream is
    // produced by this MB's own coding path; only the header part must be deterministic)
    uint32_t* a = reinterpret_cast<uint32_t*>(&s.info);
    for (int i = lane_id(); i < (int)(sizeof(MbInfo) / 4); i += MBK_WS) a[i] = 0;
    uint32_t* b = reinterpret_cast<uint32_t*>(&s.out);
    for (int i = lane_id(); i < MBOUT_HEADER_WORDS; i += MBK_WS) b[i] = 0;
    mb_load_all(c, s);
    phase_mark(s, 0);
  } else {
    mb_load_cur(c, s);                     // not parked: the source picture is read-only
  }
  if (stage == MBS_I) {
    int bb;
    const int cost16 = md_i16x16(c, s, &bb);
    intra_mb_finish(c, s, cost16, bb);
  }
  else if (stage == MBS_A) next = inter_stage_a(c, s);
  else if (stage == MBS_B) next = inter_stage_b(c, s);
  else if (stage == MBS_C) next = inter_stage_c(c, s);
  warp_sync();
  if (next == MBS_DONE) {
    phase_mark(s, 10);
    // a DECIDED skip (decided_pskip: st.is_skip) keeps its reconstruction in skip_pred; a 16x16 macroblock that turned out to be
    // codable as P_SKIP (no residual, vector == skip vector) has it in the tile like every other coded macroblock
    if (s.info.mb_type == MBT_PSKIP && s.st.is_skip != 0) mb_store_recon_skip(c, s);
    else mb_store_recon(c, s);
    mb_publish(c, s);
    if (c.f.mb_bits != nullptr) {          // exact entropy-coded size of this macroblock, without emitting a bit
      const int b = mb_cavlc_bits(c, s);
      if (lane_id() == 0) c.f.mb_bits[c.mby * c.p.mb_w + c.mbx] = b;
    }
    phase_mark(s, 11);
  }
#ifndef __CUDA_ARCH__
  if (g_skipcand_intra) { g_skipcand_next = next; return MBP_SKIPCAND_INTRA; }
#endif
  return next;
}

}  // namespace mbk
