/*
 * oracle/ref_shim.cpp — plain-C entry points onto the UNMODIFIED reference (cisco/openh264).
 *
 * TEST INFRASTRUCTURE ONLY.  Compiled (only where /root/reference exists) against the reference's
 * own headers and linked to oracle/_ref/libopenh264_ref.so; output oracle/_ref/librefshim.so.
 * Every ref_* function has exactly the signature of the oracle's orc_* twin (h264_oracle.h) and
 * forwards to the reference function through the reference's own function-pointer tables
 * initialised with uiCpuFlag = 0 (the *_c path), so tests can diff oracle vs reference call by
 * call.  Nothing here re-implements any arithmetic.
 */
#include <limits.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "wels_func_ptr_def.h"
#include "svc_motion_estimate.h"
#include "sample.h"
#include "encode_mb_aux.h"
#include "decode_mb_aux.h"
#include "md.h"
#include "mc.h"
#include "sad_common.h"
#include "deblocking_common.h"
#include "expand_pic.h"
#include "slice.h"
#include "svc_enc_frame.h"
#include "picture.h"
#include "encoder_context.h"
#include "mv_pred.h"
#include "svc_base_layer_md.h"
#include "get_intra_predictor.h"
#include "svc_encode_mb.h"
#include "svc_encode_slice.h"
#include "encoder.h"

#include "../oracle/h264_oracle.h"

using namespace WelsEnc;

namespace WelsDec {
void IdctResAddPred_c (uint8_t* pPred, const int32_t kiStride, int16_t* pRs);
void IdctResAddPred8x8_c (uint8_t* pPred, const int32_t kiStride, int16_t* pRs);
}
namespace WelsEnc {
extern const int32_t g_kiQpCostTable[52];
}
/* non-static but undeclared in deblocking_common.h (deblocking_common.cpp:5,39,93,135) */
void DeblockLumaLt4_c (uint8_t* pPix, int32_t iStrideX, int32_t iStrideY, int32_t iAlpha, int32_t iBeta, int8_t* pTc);
void DeblockLumaEq4_c (uint8_t* pPix, int32_t iStrideX, int32_t iStrideY, int32_t iAlpha, int32_t iBeta);
void DeblockChromaLt4_c (uint8_t* pPixCb, uint8_t* pPixCr, int32_t iStrideX, int32_t iStrideY, int32_t iAlpha,
                         int32_t iBeta, int8_t* pTc);
void DeblockChromaEq4_c (uint8_t* pPixCb, uint8_t* pPixCr, int32_t iStrideX, int32_t iStrideY, int32_t iAlpha,
                         int32_t iBeta);

static SWelsFuncPtrList* Funcs() {
  static SWelsFuncPtrList* p = NULL;
  if (!p) {
    p = (SWelsFuncPtrList*) calloc (1, sizeof (SWelsFuncPtrList));
    WelsInitSampleSadFunc (p, 0);
    WelsInitEncodingFuncs (p, 0);
    WelsInitReconstructionFuncs (p, 0);
    WelsCommon::InitMcFunc (&p->sMcFuncs, 0);
    WelsInitMeFunc (p, 0, false);
    InitExpandPictureFunc (&p->sExpandPicFunc, 0);
  }
  return p;
}

extern "C" {

const int16_t* ref_quant_ff (int q) { return g_kiQuantInterFF[q]; }
const int16_t* ref_quant_mf (int q) { return g_kiQuantMF[q]; }
const uint16_t* ref_dequant_coeff (int q) { return WelsCommon::g_kuiDequantCoeff[q]; }
int ref_qp_lambda (int q) { return g_kiQpCostTable[q]; }
int ref_chroma_qp (int q) { return WelsCommon::g_kuiChromaQpTable[q]; }
/* full reference table for all 52 qps, stride = 2*sz+1 (md.cpp:797) */
void ref_mvd_cost_init_all (uint16_t* table, int mvd_sz) { MvdCostInit (table, mvd_sz); }

int32_t ref_sad (int blk, const uint8_t* a, int sa, const uint8_t* b, int sb) {
  return Funcs()->sSampleDealingFuncs.pfSampleSad[blk] ((uint8_t*)a, sa, (uint8_t*)b, sb);
}
void ref_sad_four (int blk, const uint8_t* a, int sa, const uint8_t* b, int sb, int32_t out[4]) {
  Funcs()->sSampleDealingFuncs.pfSample4Sad[blk] ((uint8_t*)a, sa, (uint8_t*)b, sb, out);
}
int32_t ref_satd (int blk, const uint8_t* a, int sa, const uint8_t* b, int sb) {
  return Funcs()->sSampleDealingFuncs.pfSampleSatd[blk] ((uint8_t*)a, sa, (uint8_t*)b, sb);
}
void ref_mc_luma (const uint8_t* src, int ss, uint8_t* dst, int ds, int mvx, int mvy, int w, int h) {
  Funcs()->sMcFuncs.pMcLumaFunc (src, ss, dst, ds, (int16_t)mvx, (int16_t)mvy, w, h);
}
void ref_mc_chroma (const uint8_t* src, int ss, uint8_t* dst, int ds, int mvx, int mvy, int w, int h) {
  Funcs()->sMcFuncs.pMcChromaFunc (src, ss, dst, ds, (int16_t)mvx, (int16_t)mvy, w, h);
}
void ref_pixel_avg (uint8_t* dst, int ds, const uint8_t* a, int sa, const uint8_t* b, int sb, int w, int h) {
  Funcs()->sMcFuncs.pfSampleAveraging (dst, ds, a, sa, b, sb, w, h);
}
/* the three half-sample plane producers used by MeRefineFracPixel (mc.h:46-49) */
void ref_halfpel (int which, const uint8_t* src, int ss, uint8_t* dst, int ds, int w, int h) {
  SMcFunc* m = &Funcs()->sMcFuncs;
  (which == 0 ? m->pfLumaHalfpelHor : which == 1 ? m->pfLumaHalfpelVer : m->pfLumaHalfpelCen) (src, ss, dst, ds, w, h);
}

void ref_dct4x4 (int16_t* d, const uint8_t* p1, int s1, const uint8_t* p2, int s2) {
  Funcs()->pfDctT4 (d, (uint8_t*)p1, s1, (uint8_t*)p2, s2);
}
void ref_dct_four4x4 (int16_t* d, const uint8_t* p1, int s1, const uint8_t* p2, int s2) {
  Funcs()->pfDctFourT4 (d, (uint8_t*)p1, s1, (uint8_t*)p2, s2);
}
void ref_quant4x4 (int16_t* d, const int16_t* ff, const int16_t* mf) { Funcs()->pfQuantization4x4 (d, ff, mf); }
void ref_quant4x4_dc (int16_t* d, int16_t ff, int16_t mf) { Funcs()->pfQuantizationDc4x4 (d, ff, mf); }
void ref_quant_four4x4 (int16_t* d, const int16_t* ff, const int16_t* mf) { Funcs()->pfQuantizationFour4x4 (d, ff, mf); }
void ref_quant_four4x4_max (int16_t* d, const int16_t* ff, const int16_t* mf, int16_t* mx) {
  Funcs()->pfQuantizationFour4x4Max (d, ff, mf, mx);
}
int32_t ref_hadamard_quant2x2_skip (const int16_t* rs, int16_t ff, int16_t mf) {
  return Funcs()->pfQuantizationHadamard2x2Skip ((int16_t*)rs, ff, mf);
}
int32_t ref_hadamard_quant2x2 (int16_t* rs, int16_t ff, int16_t mf, int16_t* dct, int16_t* block) {
  return Funcs()->pfQuantizationHadamard2x2 (rs, ff, mf, dct, block);
}
void ref_hadamard_t4_dc (int16_t* dc, const int16_t* dct) { Funcs()->pfTransformHadamard4x4Dc (dc, (int16_t*)dct); }
void ref_scan4x4_dcac (int16_t* level, const int16_t* dct) { Funcs()->pfScan4x4 (level, (int16_t*)dct); }
void ref_scan4x4_ac (int16_t* level, const int16_t* dct) { Funcs()->pfScan4x4Ac (level, (int16_t*)dct); }
int32_t ref_single_ctr4x4 (const int16_t* d) { return Funcs()->pfCalculateSingleCtr4x4 ((int16_t*)d); }
int32_t ref_nonzero_count (const int16_t* l) { return Funcs()->pfGetNoneZeroCount ((int16_t*)l); }

void ref_ihadamard4x4_dc (int16_t* r) { WelsIHadamard4x4Dc (r); }
void ref_dequant_luma_dc4x4 (int16_t* r, int qp) { WelsDequantLumaDc4x4 (r, qp); }
void ref_dequant_ihadamard4x4 (int16_t* r, uint16_t mf) { Funcs()->pfDequantizationIHadamard4x4 (r, mf); }
void ref_dequant_ihadamard2x2_dc (int16_t* r, uint16_t mf) { WelsDequantIHadamard2x2Dc (r, mf); }
void ref_dequant4x4 (int16_t* r, const uint16_t* mf) { Funcs()->pfDequantization4x4 (r, mf); }
void ref_dequant_four4x4 (int16_t* r, const uint16_t* mf) { Funcs()->pfDequantizationFour4x4 (r, mf); }
void ref_idct4x4_rec (uint8_t* rec, int rs, const uint8_t* pred, int ps, const int16_t* dct) {
  Funcs()->pfIDctT4 (rec, rs, (uint8_t*)pred, ps, (int16_t*)dct);
}
void ref_idct_four4x4_rec (uint8_t* rec, int rs, const uint8_t* pred, int ps, const int16_t* dct) {
  Funcs()->pfIDctFourT4 (rec, rs, (uint8_t*)pred, ps, (int16_t*)dct);
}
void ref_idct_rec_i16x16_dc (uint8_t* rec, int rs, const uint8_t* pred, int ps, const int16_t* dc) {
  Funcs()->pfIDctI16x16Dc (rec, rs, (uint8_t*)pred, ps, (int16_t*)dc);
}
void ref_idct_res_add_pred (uint8_t* pred, int stride, const int16_t* rs) { WelsDec::IdctResAddPred_c (pred, stride, (int16_t*)rs); }
void ref_idct_res_add_pred8x8 (uint8_t* pred, int stride, const int16_t* rs) { WelsDec::IdctResAddPred8x8_c (pred, stride, (int16_t*)rs); }

void ref_deblock_luma_lt4 (uint8_t* pix, int sx, int sy, int alpha, int beta, const int8_t tc[4]) {
  DeblockLumaLt4_c (pix, sx, sy, alpha, beta, (int8_t*)tc);
}
void ref_deblock_luma_eq4 (uint8_t* pix, int sx, int sy, int alpha, int beta) { DeblockLumaEq4_c (pix, sx, sy, alpha, beta); }
void ref_deblock_chroma_lt4 (uint8_t* cb, uint8_t* cr, int sx, int sy, int alpha, int beta, const int8_t tc[4]) {
  DeblockChromaLt4_c (cb, cr, sx, sy, alpha, beta, (int8_t*)tc);
}
void ref_deblock_chroma_eq4 (uint8_t* cb, uint8_t* cr, int sx, int sy, int alpha, int beta) {
  DeblockChromaEq4_c (cb, cr, sx, sy, alpha, beta);
}
/* pad = 32 -> luma expander, pad = 16 -> chroma expander (expand_pic.h:49-50) */
void ref_expand_plane (uint8_t* pic, int stride, int w, int h, int pad) {
  if (pad == 32) Funcs()->sExpandPicFunc.pfExpandLumaPicture (pic, stride, w, h);
  else Funcs()->sExpandPicFunc.pfExpandChromaPicture[0] (pic, stride, w, h);
}

/* WelsMotionEstimateSearch (svc_motion_estimate.cpp:170) driven with the reference's own structs */
void ref_me_search (const uint8_t* cur, int cs, const uint8_t* ref, int rs, const orc_me_job* j, orc_me_result* out) {
  static uint16_t* cost = NULL;
  const int kSz = 1100, kStride = 2 * kSz + 1;
  if (!cost) { cost = (uint16_t*) malloc (sizeof (uint16_t) * 52 * kStride); MvdCostInit (cost, kStride); }
  SWelsFuncPtrList* f = Funcs();
  static SDqLayer* layer = NULL; static SPicture* pic = NULL; static SSlice* slice = NULL;
  if (!layer) {
    layer = (SDqLayer*) calloc (1, sizeof (SDqLayer));
    pic = (SPicture*) calloc (1, sizeof (SPicture));
    slice = (SSlice*) calloc (1, sizeof (SSlice));
    layer->pRefPic = pic;
  }
  layer->iEncStride[0] = cs;
  pic->iLineSize[0] = rs;
  slice->uiMvcNum = j->n_mvc;
  for (int i = 0; i < j->n_mvc; i++) { slice->sMvc[i].iMvX = j->mvc[i][0]; slice->sMvc[i].iMvY = j->mvc[i][1]; }
  slice->sMvStartMin.iMvX = j->mv_min_x; slice->sMvStartMin.iMvY = j->mv_min_y;
  slice->sMvStartMax.iMvX = j->mv_max_x; slice->sMvStartMax.iMvY = j->mv_max_y;
  for (int b = 0; b < BLOCK_SIZE_ALL; b++) f->pfSearchMethod[b] = WelsDiamondSearch;
  f->pfCalculateSatd = j->calc_satd ? CalculateSatdCost : NotCalculateSatdCost;

  SWelsME me;
  memset (&me, 0, sizeof (me));
  me.pMvdCost = cost + j->qp * kStride + kSz;
  me.uSadPredISatd.uiSadPred = j->sad_pred;
  me.uiBlockSize = (uint8_t) j->blk;
  me.pEncMb = (uint8_t*) cur + j->cur_off;
  me.pRefMb = me.pColoRefMb = (uint8_t*) ref + j->ref_off;
  me.sMvp.iMvX = j->mvp_x; me.sMvp.iMvY = j->mvp_y;
  WelsMotionEstimateSearch (f, layer, &me, slice);
  out->mv_x = me.sMv.iMvX; out->mv_y = me.sMv.iMvY;
  out->sad_cost = me.uiSadCost; out->satd_cost = me.uiSatdCost;
  out->ref_off = (int32_t) (me.pRefMb - ref);
}

/* MeRefineFracPixel (md.cpp:575) driven with a minimal encoder context and the refinement buffers of InitMeRefinePointer,
 * as WelsMdInterMbRefinement (svc_base_layer_md.cpp:1573) sets them up for each partition shape */
void ref_me_refine (const uint8_t* cur, int cs, const uint8_t* ref, int rs, const orc_refine_job* j, orc_refine_result* out,
                    uint8_t* pred) {
  static uint16_t* cost = NULL;
  const int kSz = 1100, kStride = 2 * kSz + 1;
  if (!cost) { cost = (uint16_t*) malloc (sizeof (uint16_t) * 52 * kStride); MvdCostInit (cost, kStride); }
  SWelsFuncPtrList* f = Funcs();
  f->sSampleDealingFuncs.pfMeCost = f->sSampleDealingFuncs.pfSampleSatd;     /* CAMERA_VIDEO_REAL_TIME (encoder_ext.cpp:2686) */
  static sWelsEncCtx* ctx = NULL; static SDqLayer* layer = NULL; static SPicture* pic = NULL; static SMbCache* cache = NULL;
  if (!ctx) {
    ctx = (sWelsEncCtx*) calloc (1, sizeof (sWelsEncCtx));
    layer = (SDqLayer*) calloc (1, sizeof (SDqLayer));
    pic = (SPicture*) calloc (1, sizeof (SPicture));
    cache = (SMbCache*) calloc (1, sizeof (SMbCache));
    cache->pBufferInterPredMe = (uint8_t*) calloc (4 * 640, 1);         /* svc_encode_slice.cpp:782 */
    layer->pRefPic = pic;
    ctx->pCurDqLayer = layer;
  }
  ctx->pFuncList = f;
  layer->iEncStride[0] = cs;
  pic->iLineSize[0] = rs;
  layer->bSatdInMdFlag = j->satd_in_md != 0;
  SMeRefinePointer mr;
  memset (&mr, 0, sizeof (mr));
  InitMeRefinePointer (&mr, cache, 0);
  const int blk = j->w == 16 ? (j->h == 16 ? BLOCK_16x16 : BLOCK_16x8) : (j->h == 16 ? BLOCK_8x16 : BLOCK_8x8);
  mr.pfCopyBlockByMode = blk == BLOCK_16x16 ? f->pfCopy16x16NotAligned : blk == BLOCK_16x8 ? f->pfCopy16x8NotAligned :
                         blk == BLOCK_8x16 ? f->pfCopy8x16Aligned : f->pfCopy8x8Aligned;
  SWelsME me;
  memset (&me, 0, sizeof (me));
  me.pMvdCost = cost + j->qp * kStride + kSz;
  me.uSadPredISatd.uiSatd = j->satd;
  me.uiBlockSize = (uint8_t) blk;
  me.pEncMb = (uint8_t*) cur + j->cur_off;
  me.pRefMb = me.pColoRefMb = (uint8_t*) ref + j->ref_off;
  me.sMv.iMvX = j->mv_x; me.sMv.iMvY = j->mv_y;
  me.sMvp.iMvX = j->mvp_x; me.sMvp.iMvY = j->mvp_y;
  MeRefineFracPixel (ctx, pred, &me, &mr, j->w, j->h);
  out->mv_x = me.sMv.iMvX; out->mv_y = me.sMv.iMvY;
  out->cost = me.uiSatdCost;
}

/* PredictSadSkip (md.cpp:870) and WelsMdPSkipEnc (svc_base_layer_md.cpp:1423) driven with a minimal encoder context, layer,
 * macroblock and cache, as WelsMdInterJudgePskip (:1906) calls them.  The reference reports neither its SADs, nor which test
 * decided, nor its scores: those fields are -1 here; the vector comes from PredSkipMv (mv_pred.cpp:132) itself. */
void ref_pskip (const uint8_t* cur, int cs, int csc, const uint8_t* ref, int rs, int rsc, const orc_pskip_job* j,
                orc_pskip_result* out, uint8_t* pred) {
  SWelsFuncPtrList* f = Funcs();
  InitIntraAnalysisVaaInfo (f, 0);                                             /* pfUpdateMbMv */
  static int32_t stride_tab[24 * 4];
  static SStrideTables tabs;
  static SWelsPPS pps;
  static SPicture ref_pic, dec_pic;
  static SDqLayer layer;
  static sWelsEncCtx ctx;
  static SDCTCoeff dct;
  alignas (16) static int16_t coef[384];
  alignas (16) static uint8_t skip_mb[384];
  tabs.pStrideEncBlockOffset[0] = stride_tab;                                  /* chroma blocks 16 / 20 at their plane's origin */
  layer.sLayerInfo.pPpsP = &pps;
  layer.pRefPic = &ref_pic;
  layer.pDecPic = &dec_pic;
  layer.iEncStride[0] = cs; layer.iEncStride[1] = layer.iEncStride[2] = csc;
  layer.iMbWidth = (int16_t) j->mb_w; layer.iMbHeight = (int16_t) j->mb_h;
  ref_pic.iLineSize[0] = rs; ref_pic.iLineSize[1] = ref_pic.iLineSize[2] = rsc;
  ref_pic.iPictureType = j->ref_is_p ? P_SLICE : I_SLICE;
  int32_t* skip_sad = (int32_t*) calloc (j->mb_w * j->mb_h, sizeof (int32_t));
  SMVUnitXY* mv_list = (SMVUnitXY*) calloc (j->mb_w * j->mb_h, sizeof (SMVUnitXY));
  const int xy = j->mb_y * j->mb_w + j->mb_x;
  skip_sad[xy] = j->col_skip_sad;
  ref_pic.pMbSkipSad = skip_sad;
  dec_pic.sMvList = mv_list;
  ctx.pCurDqLayer = &layer;
  ctx.pFuncList = f;
  ctx.pStrideTab = &tabs;
  ctx.uiDependencyId = 0;
  SMbCache cache;
  memset (&cache, 0, sizeof (cache));
  cache.pCoeffLevel = coef;
  cache.pSkipMb = skip_mb;
  cache.pDct = &dct;
  static const int kCell[4] = {6, 1, 5, 0};                                    /* A, B, C, D */
  for (int k = 0; k < 4; k++) {
    cache.sMvComponents.iRefIndexCache[kCell[k]] = (int8_t) j->ref[k];
    cache.sMvComponents.sMotionVectorCache[kCell[k]].iMvX = (int16_t) j->mv[k][0];
    cache.sMvComponents.sMotionVectorCache[kCell[k]].iMvY = (int16_t) j->mv[k][1];
    cache.bMbTypeSkip[k] = j->skip[k] != 0;
    cache.iSadCostSkip[k] = j->skip_sad[k];
  }
  cache.uiRefMbType = j->col_type == ORC_MB_PSKIP ? MB_TYPE_SKIP : MB_TYPE_16x16;
  for (int p = 0; p < 3; p++) {
    cache.SPicData.pEncMb[p] = (uint8_t*) cur + j->cur_off[p];
    cache.SPicData.pRefMb[p] = (uint8_t*) ref + j->ref_off[p];
  }
  SMVUnitXY mv[16];
  int8_t ref_idx[4];
  int32_t sad_cost = -1;
  SMB mb;
  memset (&mb, 0, sizeof (mb));
  mb.iMbX = (int16_t) j->mb_x; mb.iMbY = (int16_t) j->mb_y; mb.iMbXY = xy;
  mb.uiLumaQp = (uint8_t) j->qp;
  mb.sMv = mv; mb.pRefIndex = ref_idx; mb.pSadCost = &sad_cost;
  SWelsMD md;
  memset (&md, 0, sizeof (md));
  md.bMdUsingSad = j->md_using_sad != 0;
  memset (skip_mb, 0, sizeof (skip_mb));
  PredictSadSkip (cache.sMvComponents.iRefIndexCache, cache.bMbTypeSkip, cache.iSadCostSkip, 0, &md.iSadPredSkip);
  const bool ok = WelsMdPSkipEnc (&ctx, &md, &mb, &cache);
  SMVUnitXY smv;
  PredSkipMv (&cache, &smv);
  memset (out, -1, sizeof (*out));
  out->ok = ok;
  out->mv_x = smv.iMvX; out->mv_y = smv.iMvY;
  out->sad_pred_skip = md.iSadPredSkip;
  out->cost_luma = md.iCostLuma; out->cost_skip = md.iCostSkipMb;
  out->sad_cost = sad_cost;
  memcpy (pred, skip_mb, 384);
  free (skip_sad);
  free (mv_list);
}

/* WelsMotionCrossSearch (svc_motion_estimate.cpp:620) with the reference's own structs; io = SWelsME::sMv (integer pels) / uiSadCost / pRefMb */
void ref_me_cross_search (const uint8_t* cur, int cs, const uint8_t* ref, int rs, const orc_cross_job* j, orc_me_result* io) {
  static uint16_t* cost = NULL;
  const int kSz = 1100, kStride = 2 * kSz + 1;
  if (!cost) { cost = (uint16_t*) malloc (sizeof (uint16_t) * 52 * kStride); MvdCostInit (cost, kStride); }
  SWelsFuncPtrList* f = Funcs();
  f->pfVerticalFullSearch = LineFullSearch_c;
  f->pfHorizontalFullSearch = LineFullSearch_c;
  static SSlice* slice = NULL;
  if (!slice) slice = (SSlice*) calloc (1, sizeof (SSlice));
  slice->sMvStartMin.iMvX = j->mv_min_x; slice->sMvStartMin.iMvY = j->mv_min_y;
  slice->sMvStartMax.iMvX = j->mv_max_x; slice->sMvStartMax.iMvY = j->mv_max_y;
  SWelsME me;
  memset (&me, 0, sizeof (me));
  me.pMvdCost = cost + j->qp * kStride + kSz;
  me.uiBlockSize = (uint8_t) j->blk;
  me.pEncMb = (uint8_t*) cur + j->cur_off;
  me.pColoRefMb = (uint8_t*) ref + j->ref_off;
  me.pRefMb = (uint8_t*) ref + io->ref_off;
  me.sMvp.iMvX = j->mvp_x; me.sMvp.iMvY = j->mvp_y;
  me.sMv.iMvX = io->mv_x; me.sMv.iMvY = io->mv_y;
  me.uiSadCost = io->sad_cost;
  me.uiSadCostThreshold = j->sad_cost_threshold;
  me.iCurMeBlockPixX = 64; me.iCurMeBlockPixY = 64;          /* only differences of positions enter the result */
  WelsMotionCrossSearch (f, &me, slice, cs, rs);
  io->mv_x = me.sMv.iMvX; io->mv_y = me.sMv.iMvY;
  io->sad_cost = me.uiSadCost;
  io->ref_off = (int32_t) (me.pRefMb - ref);
}

} // extern "C"

/* The intra path of one macroblock as WelsMdIntraMb (svc_base_layer_md.cpp:956) runs it for stage I, and as
 * WelsMdFirstIntraMode (:1829) runs it for stage C once I16x16 has beaten the inter cost: WelsMdI16x16, then
 * WelsMdIntraSecondaryModesEnc (:2023) = pfIntraFineMd (WelsMdI4x4, or the texture gate MdIntraAnalysisVaaInfo plus
 * WelsMdI4x4Fast in LOW complexity), WelsEncRecI16x16Y when I16x16 stays, WelsMdIntraChroma and WelsIMbChromaEncode.
 * Driven with a minimal encoder context in the style of ref_pskip and the C function table (the C-only build leaves
 * pfIntra16x16Combined3 / pfIntra8x8Combined3 / pfIntra4x4Combined3 unset, so the mode loops run).
 *
 * in / out: the case and result records of b2h264_debug_intra_tail (openh264_b200/csrc/enc_kernels.cu), n of each.  The
 * macroblock sits at (1, 1) of a 3 x 2 macroblock reconstructed picture; the case's neighbour samples go where their
 * neighbour is available and every other sample of that picture, including the macroblock itself, gets pseudo-random bytes, so
 * a predictor that reads a neighbour it must not use changes the result.  The neighbours' I4x4 modes reach the mode cache
 * through FillNeighborCacheIntra (md.cpp:51).  The output record holds what the reference computed in the product's layouts
 * (MbOut: modes, prev / rem flags, levels; MbInfo: nnz, i4_mode, mb_type, cbp; the tail: cost limit used, I4x4 cost or
 * INT_MAX when the try did not run, lambda, 0; the reconstruction tile).  Fields the reference leaves stale (rem flags of
 * predicted modes, AC entry 15, the I16x16 DC of an I4x4 macroblock) are copied as the reference has them.
 * costs[3 i]: I16x16 cost, I4x4 cost (INT_MAX: not tried), chroma cost.  Returns -1 for a bad argument. */
namespace {
enum { kTyPitch = 32, kTcPitch = 16, kTile = 17 * 32 + 2 * 9 * 16, kIn = kTile + 384 + 32, kOutMbOut = 896, kOutInfo = 120,
       kOut = kOutMbOut + kOutInfo + 16 + kTile };
int32_t g_cost4;
int32_t FineMdRecordingCost (sWelsEncCtx* ctx, SWelsMD* md, SMB* mb, SMbCache* cache) {
  /* WelsMdIntraFinePartition[Vaa] (:932, :942), keeping the I4x4 cost that they fold into iCostLuma */
  const bool fast = ctx->pFuncList->sSampleDealingFuncs.pfMdCost == ctx->pFuncList->sSampleDealingFuncs.pfSampleSad;
  g_cost4 = INT_MAX;
  if (!fast) g_cost4 = WelsMdI4x4 (ctx, md, mb, cache);
  else if (MdIntraAnalysisVaaInfo (ctx, cache->SPicData.pEncMb[0])) g_cost4 = WelsMdI4x4Fast (ctx, md, mb, cache);
  if (g_cost4 < md->iCostLuma) {
    mb->uiMbType = MB_TYPE_INTRA4x4;
    md->iCostLuma = g_cost4;
  }
  return md->iCostLuma;
}
}  // namespace

extern "C" int ref_intra_mb (int n, const uint8_t* in, uint8_t* out, int32_t* costs) {
  if (n < 1 || !in || !out) return -1;
  SWelsFuncPtrList* f = Funcs();
  WelsInitIntraPredFuncs (f, 0);
  InitIntraAnalysisVaaInfo (f, 0);
  f->pfSetMemZeroSize8 = f->pfSetMemZeroSize64 = WelsSetMemZero_c;   /* InitFunctionPointers (encoder.cpp:157) */
  f->pfIntraFineMd = FineMdRecordingCost;
  static int32_t enc_offs[24], dec_offs[24];
  static SStrideTables tabs;
  static SDqLayer layer;
  static sWelsEncCtx ctx;
  static SDCTCoeff dct;
  const int ys = 64, cs = 32;                                       /* reconstructed picture: 48 x 32 luma at stride 64 */
  alignas (16) static uint8_t rec[32 * 64 + 2 * 16 * 32];
  alignas (16) static uint8_t src[16 * 16 + 2 * 8 * 8];
  alignas (16) static int16_t coef[384];
  alignas (16) static uint8_t pred_mb[2 * 256], pred_blk4[2 * 16];
  static bool prev_flag[16];
  static int8_t rem_flag[16];
  WelsGetEncBlockStrideOffset (enc_offs, 16, 8);
  WelsGetEncBlockStrideOffset (dec_offs, ys, cs);
  tabs.pStrideEncBlockOffset[0] = enc_offs;
  tabs.pStrideDecBlockOffset[0][1] = dec_offs;                      /* [did][temporal id == 0] */
  layer.iEncStride[0] = 16; layer.iEncStride[1] = layer.iEncStride[2] = 8;
  layer.iCsStride[0] = ys; layer.iCsStride[1] = layer.iCsStride[2] = cs;
  layer.iMbWidth = 2;
  ctx.pCurDqLayer = &layer;
  ctx.pFuncList = f;
  ctx.pStrideTab = &tabs;
  ctx.uiDependencyId = 0; ctx.uiTemporalId = 0;
  uint32_t seed = 0x9e3779b9u;
  for (int i = 0; i < n; i++) {
    const uint8_t* c = in + (size_t) kIn * i;
    const int32_t* prm = (const int32_t*) (c + kTile + 384);
    const int8_t* nm = (const int8_t*) (c + kTile + 400);
    const int qp = prm[0], nb = prm[1], fast = prm[2], limit = prm[3];
    if (qp < 0 || qp > 51 || nb < 0 || nb > 15) return -1;
    const uint8_t* ty = c;
    const uint8_t* tc[2] = {c + 17 * kTyPitch, c + 17 * kTyPitch + 9 * kTcPitch};
    for (size_t k = 0; k < sizeof (rec); k++) { seed = seed * 1664525u + 1013904223u; rec[k] = (uint8_t) (seed >> 24); }
    uint8_t* py = rec + 16 * ys + 16;                                /* the macroblock at (1, 1) */
    uint8_t* pc[2] = {rec + 32 * ys + 8 * cs + 8, rec + 32 * ys + 16 * cs + 8 * cs + 8};
    if (nb & 4) py[-ys - 1] = ty[0];
    for (int x = 0; x < 16; x++) if (nb & 2) py[-ys + x] = ty[1 + x];
    for (int x = 16; x < 24; x++) if (nb & 8) py[-ys + x] = ty[1 + x];
    for (int y = 0; y < 16; y++) if (nb & 1) py[y * ys - 1] = ty[(y + 1) * kTyPitch];
    for (int p = 0; p < 2; p++) {
      if (nb & 4) pc[p][-cs - 1] = tc[p][0];
      for (int x = 0; x < 8; x++) if (nb & 2) pc[p][-cs + x] = tc[p][1 + x];
      for (int y = 0; y < 8; y++) if (nb & 1) pc[p][y * cs - 1] = tc[p][(y + 1) * kTcPitch];
    }
    memcpy (src, c + kTile, 384);
    /* macroblocks 0 top-left, 1 top, 2 left, 3 current of a 2-wide array (the current one's top-right neighbour is only a bit) */
    SMB mbs[4];
    int8_t modes[4 * INTRA_4x4_MODE_NUM], nnz[4 * MB_LUMA_CHROMA_BLOCK4x4_NUM];
    int32_t sad[4];
    memset (mbs, 0, sizeof (mbs));
    memset (modes, 0, sizeof (modes));
    memset (nnz, 0, sizeof (nnz));
    for (int k = 0; k < 4; k++) {
      mbs[k].pIntra4x4PredMode = modes + INTRA_4x4_MODE_NUM * k;
      mbs[k].pNonZeroCount = nnz + MB_LUMA_CHROMA_BLOCK4x4_NUM * k;
      mbs[k].pSadCost = sad + k;
      mbs[k].uiMbType = MB_TYPE_INTRA16x16;
    }
    if (nm[0] >= 0) {                                                /* left: right column, rows 0..3 (pIntra4x4PredMode[4, 5, 6, 3]) */
      mbs[2].uiMbType = MB_TYPE_INTRA4x4;
      mbs[2].pIntra4x4PredMode[4] = nm[0]; mbs[2].pIntra4x4PredMode[5] = nm[1];
      mbs[2].pIntra4x4PredMode[6] = nm[2]; mbs[2].pIntra4x4PredMode[3] = nm[3];
    }
    if (nm[4] >= 0) {                                                /* top: bottom row (pIntra4x4PredMode[0..3]) */
      mbs[1].uiMbType = MB_TYPE_INTRA4x4;
      for (int x = 0; x < 4; x++) mbs[1].pIntra4x4PredMode[x] = nm[4 + x];
    }
    SMB* mb = &mbs[3];
    mb->iMbX = 1; mb->iMbY = 1; mb->iMbXY = 3;
    mb->uiLumaQp = (uint8_t) qp;
    mb->uiChromaQp = WelsCommon::g_kuiChromaQpTable[qp];
    mb->uiNeighborAvail = (uint8_t) ((nb & 3) | ((nb & 4) ? TOPLEFT_MB_POS : 0) | ((nb & 8) ? TOPRIGHT_MB_POS : 0));
    SMbCache cache;
    memset (&cache, 0, sizeof (cache));
    memset (&dct, 0, sizeof (dct));
    memset (coef, 0, sizeof (coef));
    memset (prev_flag, 0, sizeof (prev_flag));
    memset (rem_flag, 0, sizeof (rem_flag));
    cache.pCoeffLevel = coef;
    cache.pDct = &dct;
    cache.pMemPredMb = pred_mb;
    cache.pMemPredBlk4 = pred_blk4;
    cache.pPrevIntra4x4PredModeFlag = prev_flag;
    cache.pRemIntra4x4PredModeFlag = rem_flag;
    cache.SPicData.pEncMb[0] = src; cache.SPicData.pEncMb[1] = src + 256; cache.SPicData.pEncMb[2] = src + 320;
    cache.SPicData.pCsMb[0] = py; cache.SPicData.pCsMb[1] = pc[0]; cache.SPicData.pCsMb[2] = pc[1];
    /* WelsMdIntraInit (:259) */
    mb->uiCbp = 0;
    FillNeighborCacheIntra (&cache, mb, layer.iMbWidth);
    cache.pMemPredLuma = cache.pMemPredMb;
    cache.pMemPredChroma = cache.pMemPredMb + 256;
    f->sSampleDealingFuncs.pfMdCost = fast ? f->sSampleDealingFuncs.pfSampleSad : f->sSampleDealingFuncs.pfSampleSatd;
    SWelsMD md;
    memset (&md, 0, sizeof (md));
    md.iLambda = g_kiQpCostTable[qp];
    const int32_t cost16 = WelsMdI16x16 (f, &layer, &cache, md.iLambda);
    md.iCostLuma = limit < 0 ? cost16 : limit;
    mb->uiMbType = MB_TYPE_INTRA16x16;
    WelsMdIntraSecondaryModesEnc (&ctx, &md, mb, &cache);
    /* ---- the result in the product's layouts ---- */
    uint8_t* o = out + (size_t) kOut * i;
    memset (o, 0, kOut);
    const bool i4 = IS_INTRA4x4 (mb->uiMbType);
    o[3] = (uint8_t) g_kiMapModeI16x16[cache.uiLumaI16x16Mode];
    o[4] = (uint8_t) g_kiMapModeIntraChroma[cache.uiChmaI8x8Mode];
    for (int k = 0; k < 16; k++) { o[8 + k] = (uint8_t) prev_flag[k]; o[24 + k] = (uint8_t) rem_flag[k]; }
    memcpy (o + 80, dct.iLumaI16x16Dc, 32);
    memcpy (o + 112, dct.iLumaBlock, 512);
    memcpy (o + 624, dct.iChromaDc, 16);
    memcpy (o + 640, dct.iChromaBlock, 256);
    uint8_t* info = o + kOutMbOut;
    int8_t* inz = (int8_t*) info + 64;
    for (int k = 0; k < 16; k++) inz[k] = mb->pNonZeroCount[k];                          /* luma: raster in both */
    for (int j = 0; j < 8; j++) inz[16 + j] = mb->pNonZeroCount[g_kuiMbCountScan4Idx[16 + j]];   /* chroma: 2 x 2 raster per plane */
    for (int k = 0; k < 16; k++) ((int8_t*) info)[88 + k] = cache.iIntraPredMode[9 + (k & 3) + 8 * (k >> 2)];
    info[112] = i4 ? 0 : 1;                                                               /* MBT_I4x4 / MBT_I16x16 */
    info[113] = mb->uiCbp;
    const int32_t tail[4] = {limit < 0 ? cost16 : limit, g_cost4, md.iLambda, 0};
    memcpy (o + kOutMbOut + kOutInfo, tail, 16);
    uint8_t* t = o + kOutMbOut + kOutInfo + 16;
    memcpy (t, c, kTile);
    for (int y = 0; y < 16; y++) memcpy (t + (y + 1) * kTyPitch + 1, py + y * ys, 16);
    for (int p = 0; p < 2; p++)
      for (int y = 0; y < 8; y++) memcpy (t + 17 * kTyPitch + 9 * kTcPitch * p + (y + 1) * kTcPitch + 1, pc[p] + y * cs, 8);
    if (costs) { costs[3 * i] = cost16; costs[3 * i + 1] = g_cost4; costs[3 * i + 2] = md.iCostChroma; }
  }
  return 0;
}

/* ------------------------------------------------------------------------------------------------
 * Frame-level drivers through the reference's own PUBLIC API (codec_api.h): used as the end-to-end
 * oracle (bitstream / YUV parity) and as the CPU baseline ("kind": "reference").
 * ---------------------------------------------------------------------------------------------- */
#include "codec_api.h"
#include <time.h>

static double now_s() { struct timespec t; clock_gettime (CLOCK_MONOTONIC, &t); return t.tv_sec + 1e-9 * t.tv_nsec; }

extern "C" {

/* Encode n I420 frames (tightly packed w*h*3/2 each) at constant QP, camera mode, single layer, CAVLC,
 * deblock on, no denoise/BGD/AQ/scene-change/LTR, IDR only at frame 0 — the configuration of
 * BASELINE.md configs 2/3.  complexity: 0 low, 1 medium, 2 high.  threads = iMultipleThreadIdc
 * (1 = single thread, single slice; >1 = that many fixed slices + threads: a speed reference only,
 * it changes the bitstream).  Returns total bytes written to out (or <0 on error); seconds spent in
 * EncodeFrame in *enc_seconds; per-frame byte counts in frame_bytes[n]. */
/* entropy coder / profile of the following ref_encode calls (0 / 66 = CAVLC Baseline, the default; 1 / 0 = CABAC with the profile the
 * reference picks itself, i.e. High; 1 / 77 = CABAC Main) */
static int g_entropy_cabac = 0, g_profile_idc = 66, g_intra_period = 0;
void ref_set_entropy (int cabac, int profile_idc) { g_entropy_cabac = cabac; g_profile_idc = profile_idc; }
static int g_dbk_idc = 0, g_dbk_alpha = 0, g_dbk_beta = 0;
void ref_set_loop_filter (int idc, int alpha, int beta) { g_dbk_idc = idc; g_dbk_alpha = alpha; g_dbk_beta = beta; }   /* iLoopFilterDisableIdc / offsets */
void ref_set_intra_period (int n) { g_intra_period = n; }      /* uiIntraPeriod of the following ref_encode calls (0: the default) */

long ref_encode (const uint8_t* yuv, int w, int h, int n, int qp, int complexity, int threads, float fps,
                 uint8_t* out, long out_cap, int32_t* frame_bytes, double* enc_seconds) {
  ISVCEncoder* enc = NULL;
  if (WelsCreateSVCEncoder (&enc) || !enc) return -1;
  SEncParamExt p;
  enc->GetDefaultParams (&p);
  p.iUsageType = CAMERA_VIDEO_REAL_TIME;
  p.iPicWidth = w; p.iPicHeight = h;
  p.iTargetBitrate = 5000000;
  p.iRCMode = RC_OFF_MODE;
  p.fMaxFrameRate = fps;
  p.iTemporalLayerNum = 1;
  p.iSpatialLayerNum = 1;
  p.iComplexityMode = (ECOMPLEXITY_MODE) complexity;
  p.uiIntraPeriod = (unsigned int) g_intra_period;
  p.iNumRefFrame = 1;
  p.iEntropyCodingModeFlag = g_entropy_cabac;
  p.bEnableFrameSkip = false;
  p.bEnableLongTermReference = false;
  p.iMultipleThreadIdc = (unsigned short) threads;
  p.iLoopFilterDisableIdc = g_dbk_idc;
  p.iLoopFilterAlphaC0Offset = g_dbk_alpha;
  p.iLoopFilterBetaOffset = g_dbk_beta;
  p.bEnableDenoise = false;
  p.bEnableBackgroundDetection = false;
  p.bEnableAdaptiveQuant = false;
  p.bEnableFrameCroppingFlag = true;
  p.bEnableSceneChangeDetect = false;
  p.sSpatialLayers[0].iVideoWidth = w;
  p.sSpatialLayers[0].iVideoHeight = h;
  p.sSpatialLayers[0].fFrameRate = fps;
  p.sSpatialLayers[0].iSpatialBitrate = 5000000;
  p.sSpatialLayers[0].iDLayerQp = qp;
  p.sSpatialLayers[0].uiProfileIdc = (EProfileIdc) g_profile_idc;
  if (threads > 1) {
    p.sSpatialLayers[0].sSliceArgument.uiSliceMode = SM_FIXEDSLCNUM_SLICE;
    p.sSpatialLayers[0].sSliceArgument.uiSliceNum = threads;
  } else {
    p.sSpatialLayers[0].sSliceArgument.uiSliceMode = SM_SINGLE_SLICE;
  }
  if (enc->InitializeExt (&p)) { WelsDestroySVCEncoder (enc); return -2; }
  int lvl = WELS_LOG_QUIET;
  enc->SetOption (ENCODER_OPTION_TRACE_LEVEL, &lvl);
  long total = 0;
  double secs = 0;
  const size_t fsz = (size_t) w * h * 3 / 2;
  for (int i = 0; i < n; i++) {
    SSourcePicture pic;
    memset (&pic, 0, sizeof (pic));
    pic.iColorFormat = videoFormatI420;
    pic.iPicWidth = w; pic.iPicHeight = h;
    pic.iStride[0] = w; pic.iStride[1] = pic.iStride[2] = w / 2;
    pic.pData[0] = (uint8_t*) yuv + i * fsz;
    pic.pData[1] = pic.pData[0] + (size_t) w * h;
    pic.pData[2] = pic.pData[1] + (size_t) w * h / 4;
    pic.uiTimeStamp = (long long) (i * 1000.0 / fps);
    SFrameBSInfo info;
    memset (&info, 0, sizeof (info));
    const double t0 = now_s();
    const int rc = enc->EncodeFrame (&pic, &info);
    secs += now_s() - t0;
    if (rc) { WelsDestroySVCEncoder (enc); return -3; }
    int fb = 0;
    if (info.eFrameType != videoFrameTypeSkip) {
      for (int l = 0; l < info.iLayerNum; l++) {
        int sz = 0;
        for (int k = 0; k < info.sLayerInfo[l].iNalCount; k++) sz += info.sLayerInfo[l].pNalLengthInByte[k];
        if (total + sz > out_cap) { WelsDestroySVCEncoder (enc); return -4; }
        memcpy (out + total, info.sLayerInfo[l].pBsBuf, sz);
        total += sz; fb += sz;
      }
    }
    if (frame_bytes) frame_bytes[i] = fb;
  }
  if (enc_seconds) *enc_seconds = secs;
  enc->Uninitialize();
  WelsDestroySVCEncoder (enc);
  return total;
}

/* Decode an Annex-B stream; writes cropped I420 frames back to back into out. Returns frame count
 * (or <0); *w,*h = picture size; seconds in the decode calls in *dec_seconds. */
int ref_decode (const uint8_t* bs, long len, uint8_t* out, long out_cap, int* w, int* h, double* dec_seconds) {
  ISVCDecoder* dec = NULL;
  if (WelsCreateDecoder (&dec) || !dec) return -1;
  SDecodingParam dp;
  memset (&dp, 0, sizeof (dp));
  dp.sVideoProperty.eVideoBsType = VIDEO_BITSTREAM_AVC;
  dp.eEcActiveIdc = ERROR_CON_DISABLE;
  if (dec->Initialize (&dp)) { WelsDestroyDecoder (dec); return -2; }
  int lvl = WELS_LOG_QUIET;
  dec->SetOption (DECODER_OPTION_TRACE_LEVEL, &lvl);
  long pos = 0, outpos = 0;
  int frames = 0;
  double secs = 0;
  auto emit = [&] (uint8_t** d, SBufferInfo& bi) {
    if (bi.iBufferStatus != 1) return;
    const int W = bi.UsrData.sSystemBuffer.iWidth, H = bi.UsrData.sSystemBuffer.iHeight;
    *w = W; *h = H;
    if (outpos + (long) W * H * 3 / 2 > out_cap) return;
    for (int pl = 0; pl < 3; pl++) {
      const int pw = pl ? W / 2 : W, ph = pl ? H / 2 : H, st = bi.UsrData.sSystemBuffer.iStride[pl ? 1 : 0];
      for (int y = 0; y < ph; y++) { memcpy (out + outpos, d[pl] + (size_t) y * st, pw); outpos += pw; }
    }
    frames++;
  };
  while (pos < len) {
    /* next access-unit chunk: up to the next start code that follows at least one slice NAL */
    long end = pos + 4;
    while (end + 4 <= len && ! (bs[end] == 0 && bs[end + 1] == 0 && bs[end + 2] == 0 && bs[end + 3] == 1)) end++;
    if (end + 4 > len) end = len;
    uint8_t* d[3] = {0, 0, 0};
    SBufferInfo bi;
    memset (&bi, 0, sizeof (bi));
    const double t0 = now_s();
    dec->DecodeFrameNoDelay (bs + pos, (int) (end - pos), d, &bi);
    secs += now_s() - t0;
    emit (d, bi);
    pos = end;
  }
  for (;;) {
    int32_t remain = 0;
    dec->GetOption (DECODER_OPTION_NUM_OF_FRAMES_REMAINING_IN_BUFFER, &remain);
    if (remain <= 0) break;
    uint8_t* d[3] = {0, 0, 0};
    SBufferInfo bi;
    memset (&bi, 0, sizeof (bi));
    dec->FlushFrame (d, &bi);
    if (bi.iBufferStatus != 1) break;
    emit (d, bi);
  }
  if (dec_seconds) *dec_seconds = secs;
  dec->Uninitialize();
  WelsDestroyDecoder (dec);
  return frames;
}

}  // extern "C"

/* persistent-instance variant of ref_encode for throughput runs (bench.py --impl reference / cpu_baseline):
 * one encoder per stream lives across calls so that only the first picture is an IDR */
extern "C" {
void* ref_enc_open (int w, int h, int qp, int complexity, int threads, float fps) {
  ISVCEncoder* enc = NULL;
  if (WelsCreateSVCEncoder (&enc) || !enc) return NULL;
  SEncParamExt p;
  enc->GetDefaultParams (&p);
  p.iUsageType = CAMERA_VIDEO_REAL_TIME;
  p.iPicWidth = w; p.iPicHeight = h; p.iTargetBitrate = 5000000; p.iRCMode = RC_OFF_MODE; p.fMaxFrameRate = fps;
  p.iTemporalLayerNum = 1; p.iSpatialLayerNum = 1; p.iComplexityMode = (ECOMPLEXITY_MODE) complexity;
  p.uiIntraPeriod = 0; p.iNumRefFrame = 1; p.iEntropyCodingModeFlag = 0; p.bEnableFrameSkip = false;
  p.bEnableLongTermReference = false; p.iMultipleThreadIdc = (unsigned short) threads; p.iLoopFilterDisableIdc = 0;
  p.bEnableDenoise = false; p.bEnableBackgroundDetection = false; p.bEnableAdaptiveQuant = false;
  p.bEnableFrameCroppingFlag = true; p.bEnableSceneChangeDetect = false;
  p.sSpatialLayers[0].iVideoWidth = w; p.sSpatialLayers[0].iVideoHeight = h; p.sSpatialLayers[0].fFrameRate = fps;
  p.sSpatialLayers[0].iSpatialBitrate = 5000000; p.sSpatialLayers[0].iDLayerQp = qp;
  p.sSpatialLayers[0].uiProfileIdc = PRO_BASELINE;
  p.sSpatialLayers[0].sSliceArgument.uiSliceMode = threads > 1 ? SM_FIXEDSLCNUM_SLICE : SM_SINGLE_SLICE;
  if (threads > 1) p.sSpatialLayers[0].sSliceArgument.uiSliceNum = threads;
  if (enc->InitializeExt (&p)) { WelsDestroySVCEncoder (enc); return NULL; }
  int lvl = WELS_LOG_QUIET;
  enc->SetOption (ENCODER_OPTION_TRACE_LEVEL, &lvl);
  return enc;
}
/* encodes n pictures (tightly packed I420); returns bytes produced (discarded) or <0 */
long ref_enc_frames (void* h, const uint8_t* yuv, int w, int h_, int n, long long* ts_ms) {
  ISVCEncoder* enc = (ISVCEncoder*) h;
  long total = 0;
  const size_t fsz = (size_t) w * h_ * 3 / 2;
  for (int i = 0; i < n; i++) {
    SSourcePicture pic;
    memset (&pic, 0, sizeof (pic));
    pic.iColorFormat = videoFormatI420; pic.iPicWidth = w; pic.iPicHeight = h_;
    pic.iStride[0] = w; pic.iStride[1] = pic.iStride[2] = w / 2;
    pic.pData[0] = (uint8_t*) yuv + i * fsz; pic.pData[1] = pic.pData[0] + (size_t) w * h_; pic.pData[2] = pic.pData[1] + (size_t) w * h_ / 4;
    pic.uiTimeStamp = (*ts_ms) += 33;
    SFrameBSInfo info;
    memset (&info, 0, sizeof (info));
    if (enc->EncodeFrame (&pic, &info)) return -1;
    for (int l = 0; l < info.iLayerNum; l++)
      for (int k = 0; k < info.sLayerInfo[l].iNalCount; k++) total += info.sLayerInfo[l].pNalLengthInByte[k];
  }
  return total;
}
void ref_enc_close (void* h) { ISVCEncoder* enc = (ISVCEncoder*) h; enc->Uninitialize(); WelsDestroySVCEncoder (enc); }
}
