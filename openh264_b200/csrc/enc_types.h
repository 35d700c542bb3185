// enc_types.h — plain-data structures shared by the device macroblock pipeline, the host entropy
// coder and the frame-level C-ABI (include/b2h264_codec.h).  No CUDA or C++ types in here.
#pragma once
#include <stdint.h>

// macroblock types (own numbering)
enum {
  MBT_I4x4 = 0, MBT_I16x16 = 1, MBT_P16x16 = 2, MBT_P16x8 = 3, MBT_P8x16 = 4, MBT_P8x8 = 5, MBT_PSKIP = 6,
  MBT_IPCM = 7,              // decoder only: raw samples (luma in MbOut::luma as 256 bytes, Cb / Cr in MbOut::chroma_ac as 2 x 64 bytes)
  MBT_B = 8, MBT_BSKIP = 9   // decoder only: a macroblock of a B slice; the parser resolved its vectors and reference pictures for both
                             // lists (DecMbAux: list 0, DecMbAuxB: list 1).  B_Skip is kept apart because the reference's filter gives its
                             // inner edges strength 0 (deblocking.cpp:1186 IS_SKIP covers B_Skip)
};
#define MBT_IS_INTRA(t) ((t) <= MBT_I16x16 || (t) == MBT_IPCM)
#define MBT_IS_B(t) ((t) == MBT_B || (t) == MBT_BSKIP)
#define MBT_IS_INTER(t) (((t) >= MBT_P16x16 && (t) <= MBT_PSKIP) || MBT_IS_B(t))

// Per-macroblock state kept in HBM for the frame being coded: read by the neighbours' mode decision,
// by the deblocking pass and (through MbOut) by the host entropy coder.
// Mirrors the parts of the reference's SMB (codec/encoder/core/inc/svc_enc_macroblock.h:49-77)
// this path needs.
typedef struct {
  int16_t mv[16][2];        // per 4x4 block, RASTER order (row*4+col), quarter-pel
  int8_t  nnz[24];          // non-zero counts: luma raster 0..15, Cb 16..19, Cr 20..23 (raster 2x2)
  int8_t  i4_mode[16];      // intra4x4 pred modes (0..8), raster order; valid when mb_type == MBT_I4x4
  int16_t p16x16_mv[2];     // sP16x16Mv: 16x16 search result, candidate for the neighbours' search
  int32_t sad_cost;         // pSadCost[0] (0 for intra) -> neighbours' SAD predictor
  uint8_t mb_type;
  uint8_t cbp;
  uint8_t qp, qp_c;
  int8_t  ref_idx;          // 0 for inter, -2 for intra (REF_NOT_IN_LIST)
  uint8_t t8x8;             // decoder: transform_size_8x8_flag (the filter leaves the inner 4x4 edges of such a macroblock alone)
  uint8_t pad[2];
} MbInfo;                   // 64+24+16+4+4+8 = 120 bytes

// Per-macroblock info a coded picture carries for the NEXT frame's decisions
// (SPicture::uiRefMbType / pMbSkipSad / sMvList, codec/encoder/core/inc/picture.h).
typedef struct {
  int16_t mv16[2];          // sMvList
  int32_t skip_sad;         // pMbSkipSad
  uint8_t mb_type;          // uiRefMbType
  uint8_t pad[3];
} RefMbInfo;                // 12 bytes

// What the device hands to the host entropy coder for one macroblock (pinned-async copy-back).
// Levels are already zig-zag scanned (SDCTCoeff, codec/encoder/core/inc/mb_cache.h:63-72).
typedef struct {
  uint8_t mb_type, cbp, qp, i16_mode;     // i16_mode: 0..3 as coded
  uint8_t chroma_mode;                    // 0..3 as coded
  uint8_t pad0[3];
  int8_t  prev_i4_flag[16];               // prev_intra4x4_pred_mode_flag, coding (z) order
  int8_t  rem_i4_mode[16];                // rem_intra4x4_pred_mode
  int16_t mvd[4][2];                      // mv - mvp per partition in coding order
  int8_t  nnz[24];                        // same layout as MbInfo::nnz
  int16_t luma_dc[16];                    // I16x16 DC levels (scan order)
  int16_t luma[16][16];                   // per 4x4 block in CODING (z) order; I16x16: AC in [0..14]
  int16_t chroma_dc[2][4];
  int16_t chroma_ac[8][16];               // Cb 0..3, Cr 4..7
} MbOut;                                  // 8+32+16+24+32+512+16+256 = 896 bytes
/* Decoder only: what the parser knows about a macroblock beyond MbOut (slices, sub-macroblock partitions, deblocking control).
 * One record per macroblock next to the MbOut array (h264_parse.h -> dec_mb.cuh / enc_deblock.cuh). */
typedef struct {
  uint8_t avail;                          // NB_LEFT | NB_TOP | NB_TOPLEFT | NB_TOPRIGHT: neighbours in the SAME slice (6.4.x availability)
  uint8_t flags;                          // DECAUX_* below
  uint8_t dbk_idc;                        // disable_deblocking_filter_idc of the macroblock's slice
  int8_t  alpha_off, beta_off;            // FilterOffsetA / FilterOffsetB (already x2)
  uint8_t wp_log2;                        // macroblocks with a DecMbAuxB record: ld of its weighting formula, luma bits 0-3, chroma 4-7
  uint16_t slice;                        // slice number inside the picture
  uint8_t sub_type[4];                    // per 8x8: 0 8x8, 1 8x4, 2 4x8, 3 4x4
  int8_t  ref_idx[4];                     // per 8x8: PICTURE SLOT of its reference picture (the parser resolves RefPicList0)
  int16_t mvd[16][2];                     // sub-macroblock partition j of 8x8 k at [4 * k + j]
} DecMbAux;                               // 16 + 64 = 80 bytes
/* Decoder: list 1 and the sample weighting of a macroblock that travels resolved (a B macroblock, or a P macroblock of a slice with
 * explicit weights); one record per macroblock, uploaded only for pictures that hold such macroblocks.  For these DecMbAux::ref_idx /
 * mvd hold list 0 the same way: picture slot per 8x8 (-1: list not used) and the FINAL vector of 4x4 block j of 8x8 k at [4 * k + j]
 * (coding order), not a difference.
 * The sample prediction of 8x8 k is its motion-compensated lists (pred[k] bits 0 / 1) put through one of the two formulas of
 * wp_formula.h with w0 / w1 / o at [4 * plane + k] (plane Y, Cb, Cr) and ld from DecMbAux::wp_log2: the one-list formula
 * (DECB_WEIGHT: w0, o), the two-list formula (DECB_BI: w0, w1, o), or neither (the prediction as it is).  Default averaging is ld 0
 * with weights 1 / 1, implicit weights ld 5 with w0 = 64 - w1, explicit weights the table's values (two lists: o = (o0 + o1 + 1) >> 1).
 * ref_idx and mv sit where the deblocking filter reads them (enc_deblock.cuh). */
typedef struct {
  int8_t  ref_idx[4];                     // per 8x8: picture slot of the list-1 reference, -1: list 1 not used
  int8_t  o[12];                          // offset of the weighting formula, plane p / 8x8 k at [4 * p + k]
  int16_t mv[16][2];                      // final list-1 vector of 4x4 block j of 8x8 k at [4 * k + j]
  int16_t w0[12], w1[12];                 // weights of the formula's first / second input, [4 * p + k]
  uint8_t pred[4];                        // per 8x8: DECB_* below
} DecMbAuxB;                              // 4 + 12 + 64 + 48 + 4 = 132 bytes
#define DECB_L0 1                         /* list 0 is motion compensated into prediction buffer 0 */
#define DECB_L1 2                         /* list 1 is motion compensated: into buffer 1 next to list 0, else into buffer 0 */
#define DECB_WEIGHT 4                     /* one-list formula on buffer 0 */
#define DECB_BI 8                         /* two-list formula on buffers 0 and 1, on buffer 0 twice when one list is motion compensated */
#define DECB_LOWER 16                     /* DECB_WEIGHT covers the lower 8x4 of the 8x8 only (see emit_resolved, h264_motion.h) */
#define DECB_RIGHT 32                     /* DECB_WEIGHT covers the right 4x8 of the 8x8 only */
#define DECAUX_SUB 1
#define DECAUX_CIP 2
#define DECAUX_T8 4                       /* transform_size_8x8_flag: the luma levels are four 8x8 blocks (MbOut::luma[4k .. 4k+3] = 64 levels in
                                             8x8 zig-zag order); an MBT_I4x4 record with this flag is an Intra_8x8 macroblock (prev / rem flags [0..3]) */
#define DECAUX_EXPLICIT_B 8               /* a macroblock of a B slice with explicit weights (weighted_bipred_idc 1) */

#define MBOUT_HEADER_WORDS 20             /* mb_type .. nnz: all a P_SKIP macroblock needs to hand over */

typedef struct {
  int32_t mb_w, mb_h;
  int32_t cur_stride_y, cur_stride_c;     // source picture (MB-aligned, unpadded)
  int32_t rec_stride_y, rec_stride_c;     // reconstructed / reference pictures (padded 32 / 16)
  int32_t qp;                             // constant luma QP (RC_OFF_MODE)
  int32_t is_idr;                         // 1: I slice, 0: P slice
  int32_t mv_range;                       // iMvRange (integer pel)
  int32_t ref_is_p;                       // reference picture was coded as P (temporal candidates valid)
  int32_t ref_plane;                      // z coordinate of the stream's reference picture in the encoder's luma tensor map
  int32_t dec_mode;                       // 1: decoder construct path (MbInfo::p16x16_mv carries slice / deblocking control)
  int32_t fast_mode;                      // iComplexityMode == LOW_COMPLEXITY: SAD mode costs, VAA-driven partition choice
                                          // (SetFastCodingFunc / WelsMdInterFinePartitionVaa, encoder_ext.cpp:2616,2688)
  int32_t dbk_idc, dbk_off_a, dbk_off_b;  // encoder: disable_deblocking_filter_idc (0 / 1, 2 with several slices), FilterOffsetA / B (2 x the slice header's div2 values)
  int32_t dec_cqp_off;                    // decoder: chroma_qp_index_offset of the picture's PPS (both chroma planes)
} EncFrameParams;

typedef struct {
  const uint8_t* cur[3];                  // source Y,U,V (pixel (0,0))
  uint8_t* rec[3];                        // picture being reconstructed (pixel (0,0) inside padding)
  const uint8_t* ref[3];                  // reference picture (padded, expanded)
  MbInfo* mbi;                            // mb_w*mb_h, frame being coded
  RefMbInfo* rec_info;                    // written for the next frame
  const RefMbInfo* ref_info;              // of the reference picture
  MbOut* out;                             // mb_w*mb_h
  int32_t* sad_cost;                      // mb_w*mb_h, PERSISTS across frames like the reference's pSadCostMb
                                          // (encoder_ext.cpp:1675): a decided-skip MB keeps its older value
  const int32_t* vaa_sad8x8;              // fast mode: SAD of the four 8x8 blocks of every macroblock against the PREVIOUS
                                          // SOURCE picture (VAACalcSad_c), indexed like the reference: [iMbXY * 4 + k]
  const uint8_t* dpb0[3];                 // decoder: planes (pixel (0,0)) of picture slot 0; slot k lies dpb_stride bytes further
  int64_t dpb_stride;
  const DecMbAux* dec_aux;                // decoder: per-macroblock side records (NULL in the encoder)
  const DecMbAuxB* dec_aux_b;             // decoder: list-1 records of the picture's macroblocks (NULL unless the picture holds B slices)
  const uint8_t* prev_luma;               // fast mode: luma of the previous SOURCE picture (same layout as cur[0])
  int32_t* mb_bits;                       // optional (NULL = off): exact CAVLC bits of every macroblock (enc_cavlc_bits.cuh)
  const int32_t* slice_first;             // encoder, several slices per picture: per macroblock, the address of its slice's first
                                          // macroblock (enc_slices.h); NULL: one slice
} EncFramePtrs;
