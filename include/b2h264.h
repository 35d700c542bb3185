/*
 * include/b2h264.h — C-ABI of libopenh264_b200.so, layer 1: the macroblock-kernel boundary.
 *
 * This is the GPU-side shim SURVEY.md §8(b) calls for: it plays the role of the reference's
 * internal operator table SWelsFuncPtrList (codec/encoder/core/inc/wels_func_ptr_def.h:198-296)
 * and the decoder's function pointers (codec/decoder/core/src/decoder.cpp:981-1001), but BATCHED:
 * every entry point runs n independent jobs of one reference function in one launch, one warp (or
 * one thread for the 4x4 transforms) per job.  The frame-level entry points that compose these
 * (layer 2) and the ISVCEncoder/ISVCDecoder objects (layer 3) are declared in b2h264_codec.h.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless named h_*; no torch / C++ types cross this boundary;
 *   - `stream` is a cudaStream_t passed as void* (NULL = default stream); calls are asynchronous;
 *   - return value: 0 on success, otherwise the cudaError_t of the failing call (never a CPU
 *     fallback: without a CUDA device every entry point fails with a non-zero code);
 *   - block-size ids: 0=16x16 1=16x8 2=8x16 3=8x8 4=4x4 5=8x4 6=4x8 (wels_const.h:139-148);
 *   - *_off arrays are byte offsets of each job's block inside the given plane.
 *   - pixel planes must have >= 4 readable bytes after the last byte any job touches.
 */
#ifndef B2H264_H
#define B2H264_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B2H264_ABI_VERSION 1

/* ---- runtime -------------------------------------------------------------------------------- */
int  b2h264_init (int device);                 /* selects the device, uploads the quantiser tables */
int  b2h264_abi_version (void);
int  b2h264_dev_malloc (void** dptr, size_t bytes);
int  b2h264_dev_free (void* dptr);
int  b2h264_h2d (void* dptr, const void* h_src, size_t bytes, void* stream);
int  b2h264_d2h (void* h_dst, const void* dptr, size_t bytes, void* stream);
int  b2h264_sync (void* stream);
const char* b2h264_error_string (int code);
/* number of kernels this library has launched since load (bench.py's gpu_launches) */
unsigned long long b2h264_launch_count (void);

/* host-side views of the constant tables the kernels use (for tests that pin them to the reference) */
const int16_t*  b2h264_table_quant_ff (int qp_plus);   /* g_kiQuantInterFF row, 0..57 */
const int16_t*  b2h264_table_quant_mf (int qp);        /* g_kiQuantMF row */
const uint16_t* b2h264_table_dequant (int qp);         /* g_kuiDequantCoeff row */
int             b2h264_table_lambda (int qp);          /* g_kiQpCostTable */
int             b2h264_table_chroma_qp (int qp);       /* g_kuiChromaQpTable */

/* ---- SAD / SATD: pfSampleSad[], pfSample4Sad[], pfSampleSatd[]  (sample.cpp:336-372) -------- */
/* any of sad / satd / sad4 may be NULL; sad4 holds 4 values per job (up, down, left, right)     */
int b2h264_k_sad (const uint8_t* a, int sa, const int32_t* a_off, const uint8_t* b, int sb, const int32_t* b_off,
                  int blk, int n, int32_t* sad, int32_t* satd, int32_t* sad4, void* stream);

/* ---- motion compensation: SMcFunc (mc.h:46-54, mc.cpp:335,369,4528) ------------------------- */
/* dst: n tiles of 16x16 bytes (stride 16) for luma, 8x8 (stride 8) for chroma; mv = (x,y) pairs */
int b2h264_k_mc_luma (const uint8_t* src, int ss, const int32_t* src_off, const int16_t* mv, int w, int h, int n,
                      uint8_t* dst, void* stream);
int b2h264_k_mc_chroma (const uint8_t* src, int ss, const int32_t* src_off, const int16_t* mv, int w, int h, int n,
                        uint8_t* dst, void* stream);
/* which: 0 = pfLumaHalfpelHor, 1 = pfLumaHalfpelVer, 2 = pfLumaHalfpelCen; w,h <= 17; dst tiles 17x17 stride 17 */
int b2h264_k_halfpel (int which, const uint8_t* src, int ss, const int32_t* src_off, int w, int h, int n, uint8_t* dst,
                      void* stream);
/* pfSampleAveraging: dst tiles 16x16 stride 16 */
int b2h264_k_pixel_avg (const uint8_t* a, int sa, const int32_t* a_off, const uint8_t* b, int sb, const int32_t* b_off,
                        int w, int h, int n, uint8_t* dst, void* stream);

/* ---- forward transform / quant (encode_mb_aux.cpp:464) -------------------------------------- */
/* pfDctFourT4: dct = n x 64 int16 (four 4x4 blocks, z order) */
int b2h264_k_dct_four4x4 (const uint8_t* p1, int s1, const int32_t* p1_off, const uint8_t* p2, int s2,
                          const int32_t* p2_off, int n, int16_t* dct, void* stream);
/* pfQuantizationFour4x4(Max): in place on n x 64; ff row = qp (+6 when intra); max4 (n x 4) may be NULL */
int b2h264_k_quant_four4x4 (int16_t* dct, int qp, int intra, int n, int16_t* max4, void* stream);
/* pfQuantizationDc4x4: in place on n x 16 */
int b2h264_k_quant4x4_dc (int16_t* dct, int ff, int mf, int n, void* stream);
/* pfQuantizationHadamard2x2(+Skip): rs n x 64 (DCs at 0,16,32,48 are consumed and zeroed);
 * dct n x 4, nz n, skip n (skip computed BEFORE the DCs are zeroed) */
int b2h264_k_hadamard_quant2x2 (int16_t* rs, int ff, int mf, int n, int16_t* dct, int32_t* nz, int32_t* skip,
                                void* stream);
/* pfTransformHadamard4x4Dc: dct n x 256 -> dc n x 16 */
int b2h264_k_hadamard_t4_dc (const int16_t* dct, int n, int16_t* dc, void* stream);
/* pfScan4x4 / pfScan4x4Ac / pfCalculateSingleCtr4x4 / pfGetNoneZeroCount on n x 16;
 * ctr_nzc: n x 2 = (single-ctr of the DC+AC scan, non-zero count of the DC+AC scan) */
int b2h264_k_scan4x4 (const int16_t* dct, int n, int16_t* level_dcac, int16_t* level_ac, int32_t* ctr_nzc, void* stream);

/* ---- dequant / reconstruction (encoder decode_mb_aux.cpp:251, decoder decode_mb_aux.cpp) ----- */
int b2h264_k_dequant_four4x4 (int16_t* res, int qp, int n, void* stream);                /* n x 64 */
int b2h264_k_dequant_ihadamard4x4 (int16_t* res, int mf, int n, void* stream);           /* n x 16, qp >= 12 path */
int b2h264_k_dequant_luma_dc (int16_t* res, int qp, int n, void* stream);                /* n x 16, qp < 12: WelsIHadamard4x4Dc + WelsDequantLumaDc4x4 */
int b2h264_k_dequant_ihadamard2x2 (int16_t* res, int mf, int n, void* stream);           /* n x 4 */
/* pfIDctFourT4: rec tiles 8x8 stride 8 */
int b2h264_k_idct_four4x4_rec (const uint8_t* pred, int ps, const int32_t* pred_off, const int16_t* dct, int n,
                               uint8_t* rec, void* stream);
/* pfIDctI16x16Dc: rec tiles 16x16 stride 16, dc n x 16 */
int b2h264_k_idct_rec_i16x16_dc (const uint8_t* pred, int ps, const int32_t* pred_off, const int16_t* dc, int n,
                                 uint8_t* rec, void* stream);
/* decoder IdctResAddPred_c (size 4, rs n x 16) / IdctResAddPred8x8_c (size 8, rs n x 64): in place on pic */
int b2h264_k_idct_res_add_pred (uint8_t* pic, int stride, const int32_t* off, const int16_t* rs, int size, int n,
                                void* stream);

/* ---- deblocking edge filters (deblocking_common.cpp) ---------------------------------------- */
typedef struct {
  int32_t off;        /* byte offset of q0 of the first line (luma) / in both chroma planes */
  int32_t sx, sy;     /* step across / along the edge */
  int16_t alpha, beta;
  int8_t  tc[4];      /* bS<4: tc0 per group of lines; ignored when strong */
  int32_t strong;     /* 1 = bS==4 filter */
} b2h264_edge_job;
int b2h264_k_deblock_luma (uint8_t* pic, const b2h264_edge_job* jobs, int n, void* stream);
int b2h264_k_deblock_chroma (uint8_t* cb, uint8_t* cr, const b2h264_edge_job* jobs, int n, void* stream);

/* ---- ExpandReferencingPicture (expand_pic.cpp:388): pad = 32 (luma) or 16 (chroma) ----------- */
int b2h264_k_expand_plane (uint8_t* pic, int stride, int w, int h, int pad, void* stream);

/* VPP bilinear down-sampler (codec/processing/src/downsample/downsamplefuncs.cpp): mode 0 = DyadicBilinearDownsampler_c :47,
 * 1 = ...QuarterDownsampler_c :73, 2 = ...OneThirdDownsampler_c :99, 3 = GeneralBilinearFastDownsampler_c :118 (luma),
 * 4 = GeneralBilinearAccurateDownsampler_c :189 (chroma).  n_planes planes of identical geometry, plane p at
 * dst + p * dst_plane_bytes / src + p * src_plane_bytes (the same plane of n streams in one launch). */
int b2h264_k_downsample (int mode, uint8_t* dst, int dst_stride, int dst_w, int dst_h, const uint8_t* src, int src_stride,
                         int src_w, int src_h, int n_planes, size_t dst_plane_bytes, size_t src_plane_bytes, void* stream);
/* the function CDownsampling::Process (downsample.cpp:143-215) picks for a plane: 0..2 dyadic forms, else 3 (luma) / 4 (chroma) */
int b2h264_downsample_mode (int src_w, int src_h, int dst_w, int dst_h, int is_chroma);

/* One destination plane of a down-sampling ladder.  mode: b2h264_downsample_mode; sx / sy: the general ratio's fixed-point steps
 * (modes 3 and 4: WELS_ROUND(src / dst * 2^16) horizontally for luma, 2^15 otherwise; 0 for modes 0-2); src_offset /
 * dst_offset: the plane's first byte inside one picture; row0: the plane's first row in the launch (0 for the first descriptor,
 * then the previous descriptor's row0 + dst_h). */
typedef struct {
  int32_t  mode, sx, sy;
  int32_t  src_w, src_h, src_stride;
  int32_t  dst_w, dst_h, dst_stride;
  int32_t  row0;
  uint64_t src_offset, dst_offset;
} b2h264_ds_plane;
#define B2H264_LADDER_MAX_PLANES 24      /* 8 rungs x 3 planes */

/* Every plane of every rung for the pictures of streams [lo, lo + cnt) in one launch: picture s is read at src + s * src_pitch
 * and written at dst + s * dst_pitch, plane k at its offsets.  h_planes is a HOST array of n_planes (1..24) descriptors;
 * descriptors with an invalid mode, an empty size or a row0 that is not the running sum of dst_h are refused (cudaErrorInvalidValue). */
int b2h264_k_downsample_ladder (const b2h264_ds_plane* h_planes, int n_planes, uint8_t* dst, size_t dst_pitch, const uint8_t* src,
                                size_t src_pitch, int lo, int cnt, void* stream);

/* ---- WelsMotionEstimateSearch (svc_motion_estimate.cpp:170) --------------------------------- */
typedef struct {
  int32_t blk;
  int32_t cur_off, ref_off;
  int16_t mvp_x, mvp_y;
  int16_t mv_min_x, mv_min_y, mv_max_x, mv_max_y;
  int32_t n_mvc;
  int16_t mvc[5][2];
  uint32_t sad_pred;
  int32_t qp;
  int32_t calc_satd;
} b2h264_me_job;
typedef struct {
  int16_t mv_x, mv_y;
  uint32_t sad_cost, satd_cost;
  int32_t ref_off;
} b2h264_me_result;
int b2h264_k_me_search (const uint8_t* cur, int cs, const uint8_t* ref, int rs, const b2h264_me_job* jobs, int n,
                        b2h264_me_result* out, void* stream);

/* ---- WelsMotionCrossSearch (svc_motion_estimate.cpp:620-643): LineFullSearch_c (:568-618) along the vertical line through the
 * co-located block, then — while the cost is still >= sad_cost_threshold — along the horizontal line.  The screen-content refinement
 * after the diamond search (WelsDiamondCrossSearch :388).  mv_min / mv_max = SSlice::sMvStartMin / sMvStartMax (integer pels, the
 * maximum is exclusive).  `io` carries SWelsME::sMv (INTEGER pels, as inside the search), uiSadCost and pRefMb in and out. */
typedef struct {
  int32_t blk;
  int32_t cur_off, ref_off;            /* pEncMb; pColoRefMb */
  int16_t mvp_x, mvp_y;                /* quarter-pel predictor */
  int16_t mv_min_x, mv_min_y, mv_max_x, mv_max_y;
  int32_t qp;
  uint32_t sad_cost_threshold;
} b2h264_cross_job;
int b2h264_k_me_cross_search (const uint8_t* cur, int cs, const uint8_t* ref, int rs, const b2h264_cross_job* jobs, int n,
                              b2h264_me_result* io, void* stream);

/* ---- decoder inter prediction beyond plain MC (rec_mb.cpp): WeightPrediction :298 (explicit weights of one list), BiWeightPrediction :366
 * (explicit, or implicit with w1 + w2 = 64 and log2_denom 5), BiPrediction :425 (rounded average).  n blocks of w x h samples of ONE
 * plane, in place on dst + dst_off[i]; the second prediction at tmp + tmp_off[i] with the same stride.  mode 0 weight, 1 bi-weight, 2 average. */
typedef struct {
  int32_t log2_denom;
  int32_t w1, o1, w2, o2;              /* mode 0 uses w1 / o1 only */
} b2h264_weight_job;
int b2h264_k_weighted_pred (int mode, uint8_t* dst, const uint8_t* tmp, int stride, const int32_t* dst_off, const int32_t* tmp_off,
                            const b2h264_weight_job* jobs, int w, int h, int n, void* stream);

/* ---- MC + SAD (the roofline-graded unit, SURVEY.md §8d) --------------------------------------
 * For every macroblock m of an (mb_w x mb_h) frame: interpolate the 16x16 luma prediction at each of
 * the k quarter-pel motion vectors mv[m][0..k) (McLuma_c) and return SAD16x16 against the current
 * macroblock (WelsSampleSad16x16_c).  ref is a padded plane (pad >= 32 on all sides, ref points at
 * pixel (0,0)); |mv| must keep the 21x21 footprint inside the padding.  cost: m*k int32. */
int b2h264_k_mc_sad (const uint8_t* cur, int cs, const uint8_t* ref, int rs, int mb_w, int mb_h, const int16_t* mv,
                     int k, int32_t* cost, void* stream);

#ifdef __cplusplus
}
#endif
#endif
