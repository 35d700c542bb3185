/*
 * include/b2h264_codec.h — C-ABI of libopenh264_b200.so, layers 2 and 3: frame-level encoding.
 *
 * Layer 2 — batched frame encoder (b2h264_enc_*): N independent streams of identical geometry are coded
 * together, one picture per stream per call.  This is the GPU-shaped entry point: the macroblock loop
 * of the reference (WelsCodeOneSlice -> WelsISliceMdEnc / WelsMdInterMbLoop,
 * codec/encoder/core/src/svc_encode_slice.cpp:534,1642,1807) plus PerformDeblockingFilter
 * (deblocking.cpp:744) and ExpandReferencingPicture (expand_pic.cpp:388) run on the GPU as a wavefront
 * over macroblock rows x streams; CAVLC or CABAC / NAL serialisation (svc_set_mb_syn_cavlc.cpp,
 * svc_set_mb_syn_cabac.cpp, nal_encap.cpp) runs on host threads from the pinned copy-back of the per-macroblock records.
 *
 * Layer 3 — the reference's own public API (codec/api/wels/codec_api.h:272-339,545-586):
 * WelsCreateSVCEncoder() returns an object whose vtable layout is that of ISVCEncoder, so a caller
 * built against the reference's header can link this library instead (see INTEGRATION.md).  It wraps a
 * 1-stream layer-2 encoder.
 *
 * Supported configuration (everything else is rejected with an error, never silently approximated):
 * CAMERA_VIDEO_REAL_TIME, 1 spatial / 1 temporal layer, RC_OFF_MODE (constant QP), SM_SINGLE_SLICE, SM_FIXEDSLCNUM_SLICE or SM_RASTER_SLICE,
 * CAVLC or CABAC (Baseline / Main / High parameter sets, no 8x8 transform), any iComplexityMode (LOW / MEDIUM / HIGH), 1 reference frame, any loop filter idc / offsets, IDR at the first frame, every uiIntraPeriod frames and on
 * ForceIntraFrame, no denoise / background detection / scene-change / LTR.  (Adaptive quantisation: the reference switches it off
 * for every configuration, encoder_ext.cpp:300-301, so its output with the flag set is this constant-QP output.)
 * For that configuration the bitstream is bit-identical to the reference's.
 */
#ifndef B2H264_CODEC_H
#define B2H264_CODEC_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct b2h264_enc b2h264_enc;

typedef struct {
  int32_t width, height;        /* luma samples, multiples of 2 (width % 4 == 0) */
  int32_t qp;                   /* constant QP 0..51 (SSpatialLayerConfig::iDLayerQp) */
  float   fps;                  /* fMaxFrameRate: only used for level selection */
  int32_t target_bitrate;       /* iTargetBitrate in bps: only used for level selection (0 = unspecified) */
  int32_t n_streams;            /* independent streams coded per call */
  int32_t entropy_threads;      /* host threads for CAVLC (0 = min(n_streams, hardware threads)) */
  int32_t device;               /* CUDA device ordinal */
  int32_t sps_pps_id_strategy;  /* eSpsPpsIdStrategy: 0 CONSTANT_ID, 1 INCREASING_ID (the reference's default) */
  int32_t complexity_low;       /* 1: iComplexityMode = LOW_COMPLEXITY (the reference's default: SAD mode costs, VAA-driven
                                 * partition choice, pruned I4x4 search); 0: MEDIUM / HIGH (identical bitstreams for this class) */
  int32_t entropy_cabac;        /* SEncParamExt::iEntropyCodingModeFlag: 0 CAVLC, 1 CABAC (the host slice writer changes, the
                                 * macroblock kernel and its records do not) */
  int32_t profile_idc;          /* SSpatialLayerConfig::uiProfileIdc: 0 unspecified (Baseline, High with CABAC), 66, 77 or 100; resolved
                                 * as the reference does (encoder_ext.cpp:126-141,652-664): Baseline turns CABAC off, other values
                                 * count as unspecified.  No High-profile tool is used (no 8x8 transform): only the SPS / PPS change */
  int32_t intra_period;         /* SEncParamExt::uiIntraPeriod: 0 = only the first picture (and forced ones) is IDR; N: a stream codes an
                                 * IDR picture once N - 1 P pictures followed the last one (wels_preprocess.cpp:369-371) */
  int32_t loop_filter_idc;      /* iLoopFilterDisableIdc: 0 on, 1 off, 2 on except at slice edges (= 0 with one slice per picture) */
  int32_t loop_filter_alpha_c0_offset, loop_filter_beta_offset;   /* iLoopFilterAlphaC0Offset / iLoopFilterBetaOffset, -6..6 */
} b2h264_enc_config;

/* returns 0 or a negative b2h264 error / positive cudaError_t */
int  b2h264_enc_create (const b2h264_enc_config* cfg, b2h264_enc** out);
void b2h264_enc_destroy (b2h264_enc* e);

/* Submits one picture per stream.  src[i] = I420 picture of stream i (w*h*3/2 bytes, tightly packed), or NULL: stream
 * i sits this batch out (its state is untouched; collect reports 0 bytes / frame type 0 for it) — this is how
 * ISVCEncoder objects that call EncodeFrame at their own pace share one batched encoder (layer 3's broker).
 * src_on_device = 0: host pointers.  Pageable pictures are copied into the encoder's pinned ring inside this
 * call (the caller may reuse them on return).  PAGE-LOCKED pictures (cudaHostAlloc / cudaHostRegister) are DMA'd
 * straight from the caller's memory by the asynchronous pipeline: they must stay untouched until the matching
 * b2h264_enc_collect returns.  src_on_device = 1: device pointers (already in HBM), same lifetime rule.
 * At most 2 submissions may be in flight before b2h264_enc_collect is called (-3 otherwise; -5: every src NULL). */
int  b2h264_enc_submit (b2h264_enc* e, const uint8_t* const* src, int src_on_device);

/* Waits for the oldest submitted batch, entropy-codes it, and returns per-stream Annex-B access units.
 * bs[i] / bs_bytes[i]: encoder-owned buffer of stream i, valid until the next collect on this encoder
 * (like SFrameBSInfo::pBsBuf, codec_app_def.h:647-654).  frame_type[i]: 1 = IDR, 2 = P, 0 = the stream sat
 * the call out, -1 = its picture was not coded (bs[i] NULL: a recovery request found no confirmed long-term picture, and the
 * stream's next picture is an IDR; the reference's EncodeFrame fails the same way) (may be NULL). */
int  b2h264_enc_collect (b2h264_enc* e, const uint8_t** bs, int32_t* bs_bytes, int32_t* frame_type);

/* next picture of stream i (or all streams when i < 0) is coded as IDR (ISVCEncoder::ForceIntraFrame) */
int  b2h264_enc_force_idr (b2h264_enc* e, int stream);

/* Reference pictures, before the first submit (-3 after it; -2 for a value out of range).  num_ref_frames is
 * SEncParamExt::iNumRefFrame: -1 (AUTO_REF_PIC_COUNT) or 1..10; with ltr_enable (bEnableLongTermReference) the encoder keeps
 * two long-term pictures and marks a new one every ltr_mark_period (iLtrMarkPeriod) P pictures once the last is confirmed.
 * Resolved as the reference resolves them: max_num_ref_frames of the SPS is the larger of num_ref_frames and what LTR needs
 * (1, or 3 with LTR).  Each stream keeps 2 pictures on the device without LTR and 4 with it.  Defaults: 1, 0, 30.
 * b2h264_enc_get_references: out4 = iNumRefFrame and max_num_ref_frames as resolved, iLTRRefNum, pictures kept per stream. */
int  b2h264_enc_set_references (b2h264_enc* e, int num_ref_frames, int ltr_enable, int ltr_mark_period);
int  b2h264_enc_get_references (b2h264_enc* e, int32_t* out4);

/* Slices, before the first submit (-3 after it; -2 for a request that is refused).  mode, num and mb_num are SSliceArgument's
 * uiSliceMode, uiSliceNum and uiSliceMbNum (35 entries, or NULL for zeros), resolved as the reference resolves them
 * (encoder_ext.cpp:173-250,540-612): SM_SINGLE_SLICE (0); SM_FIXEDSLCNUM_SLICE (1): num slices of floor(macroblocks / num)
 * macroblocks, the last one taking the remainder, num clamped to 35; SM_RASTER_SLICE (2): mb_num[0] == 0 codes one slice per
 * macroblock row (refused with more than 35 rows), otherwise the runs of mb_num, the last one cut or a remainder added.  A
 * picture of at most 48 macroblocks, or a request for one slice, falls back to SM_SINGLE_SLICE.  Refused: SM_SIZELIMITED_SLICE,
 * and SM_FIXEDSLCNUM_SLICE with num 0 (the reference takes the CPU core count).  All streams of the encoder share the
 * partition.  Each slice is one NAL unit; with several slices loop_filter_idc 2 leaves the edges between slices unfiltered.
 * b2h264_enc_get_slices: the resolved mode, slice count and run lengths (any pointer may be NULL). */
int  b2h264_enc_set_slices (b2h264_enc* e, int mode, int num, const uint32_t* mb_num);
int  b2h264_enc_get_slices (b2h264_enc* e, int32_t* mode, int32_t* num, uint32_t* mb_num);

/* Loss-recovery feedback of stream i (SLTRRecoverRequest / SLTRMarkingFeedback of ENCODER_LTR_RECOVERY_REQUEST /
 * ENCODER_LTR_MARKING_FEEDBACK; feedback_type 1 = LTR_RECOVERY_REQUEST, 4 / 5 = LTR_MARKING_SUCCESS / _FAILED).  It takes
 * effect on the stream's next submitted picture: a valid recovery request makes it predict from the newest confirmed
 * long-term picture, a request with last_correct_frame_num -1 (or any request while LTR is off) makes it an IDR; a valid request while no long-term
 * picture is confirmed drops the next picture (b2h264_enc_collect: frame type -1) and makes the one after it an IDR.  Feedback
 * whose idr_pic_id is not that of the stream's last IDR is ignored.  b2h264_enc_ltr_mark_period changes the marking period
 * of one stream (ENCODER_LTR_MARKING_PERIOD). */
int  b2h264_enc_ltr_recovery_request (b2h264_enc* e, int stream, int feedback_type, int idr_pic_id, int cur_frame_num,
                                      int last_correct_frame_num);
int  b2h264_enc_ltr_marking_feedback (b2h264_enc* e, int stream, int feedback_type, int idr_pic_id, int ltr_frame_num);
int  b2h264_enc_ltr_mark_period (b2h264_enc* e, int stream, int period);

/* stream i starts over as a fresh encoder would (next picture IDR, parameter-set ids, frame_num, SAD / reference
 * history and long-term state cleared); only while nothing is in flight.  Used when an ISVCEncoder slot of a shared encoder is re-used. */
int  b2h264_enc_reset_stream (b2h264_enc* e, int stream);

/* Exact CAVLC bit count on the device (the reference's rate control reads it from the bitstream position per macroblock:
 * ratectl.cpp:1239-1278, svc_set_mb_syn_cavlc.cpp:260).  set_mb_bits(on): every following picture also yields, per
 * macroblock, the number of bits its macroblock_layer() takes (0 for P_SKIP; mb_skip_run excluded), computed by the
 * macroblock kernel without emitting a bit.  get_mb_bits: device_bits[n_mb] = that array for the last COLLECTED picture
 * of a stream, host_bits[n_mb] = what the host CAVLC writer actually spent (either may be NULL): they are equal. */
int  b2h264_enc_set_mb_bits (b2h264_enc* e, int on);
int  b2h264_enc_get_mb_bits (b2h264_enc* e, int stream, int32_t* device_bits, int32_t* host_bits);

/* copies the picture of stream i reconstructed (and deblocked) last into dst
 * (cropped I420, w*h*3/2 bytes, host memory): for parity tests */
int  b2h264_enc_get_recon (b2h264_enc* e, int stream, uint8_t* h_dst);

/* timing of the last collected batch, microseconds: [0] source padding + macroblock wavefront kernel,
 * [1] deblocking wavefront + border expansion (both from CUDA events on the encoder's stream),
 * [2] host entropy coding (wall clock) */
int  b2h264_enc_last_timing (b2h264_enc* e, float* us3);
/* bytes the device handed to the host for the batch collected last: the index table plus the records of the
 * coded (non P_SKIP) macroblocks, written by the GPU straight into mapped pinned memory */
int  b2h264_enc_last_d2h_bytes (b2h264_enc* e, unsigned long long* bytes);
/* statistics: macroblocks of the last collected batch that were coded (not P_SKIP), over all its streams */
int  b2h264_enc_last_coded_mbs (b2h264_enc* e, unsigned long long* count);

/* makes the encoder issue all its GPU work on the caller's CUDA stream (cudaStream_t as void*), e.g. so
 * that a harness can bracket it with its own events; only while nothing is in flight */
int  b2h264_enc_set_stream (b2h264_enc* e, void* stream);

/* layer 3 (WelsCreateSVCEncoder / ISVCEncoder, codec_api.h:272-339,545-586) is declared in b2h264_wels_api.h */

/* ---- batched decoder (first device version of the decoder construct path; DESIGN.md section 9) -----------------
 * Replaces, for Baseline / Main / High streams with CAVLC or CABAC slice data (I and P slices, several slices per picture in raster
 * order, up to 16 reference frames with list modification, sliding-window and memory-management marking incl. long-term pictures,
 * all partition shapes down to 4x4, I_PCM, constrained intra prediction, per-slice deblocking control, non-reference pictures, B slices with
 * spatial / temporal direct prediction and implicit weights, the 8x8 transform with Intra_8x8, explicit weights in P and B slices, a
 * chroma QP offset; no FMO / ASO, interlace, scaling lists, SVC extensions), ISVCDecoder::DecodeFrameNoDelay
 * (codec/api/wels/codec_api.h:383; codec/decoder/plus/src/welsDecoderExt.cpp:~700).  The host parses, the GPU
 * reconstructs, deblocks and pads.  Anything else is rejected: -101 truncated, -102 unsupported stream feature,
 * -103 invalid syntax, -104 slice before its parameter sets, -105 the slices given do not cover the picture; -2 picture size differs from the configuration. */
typedef struct b2h264_dec b2h264_dec;
typedef struct {
  int32_t width, height;        /* cropped picture size the streams must have */
  int32_t n_streams;            /* independent streams decoded per call */
  int32_t device;               /* CUDA device ordinal */
} b2h264_dec_config;
int  b2h264_dec_create (const b2h264_dec_config* cfg, b2h264_dec** out);
void b2h264_dec_destroy (b2h264_dec* d);
/* au[s] / au_bytes[s]: one access unit ([SPS PPS] slice, Annex B) of stream s; yuv[s]: host buffer for the decoded
 * picture, tightly packed I420 of width x height.  Synchronous. */
int  b2h264_dec_decode (b2h264_dec* d, const uint8_t* const* au, const int32_t* au_bytes, uint8_t* const* yuv);
/* as b2h264_dec_decode; streams whose au[s] is NULL or carries no slice (parameter sets only) sit the call out:
 * got_picture[s] = 1 where yuv[s] was written, else 0 (the parameter sets are kept for the stream) */
int  b2h264_dec_decode2 (b2h264_dec* d, const uint8_t* const* au, const int32_t* au_bytes, uint8_t* const* yuv, int32_t* got_picture);
/* for callers that batch UNRELATED streams (the ISVCDecoder broker of layer 3): status[s] = 1 picture decoded, 0 no slice in the unit (or
 * au[s] == NULL), < 0 that stream's own error (-101 .. -105 as above, -2 size mismatch) — it sits the batch out, the other streams are
 * decoded.  The return value only reports errors of the call as a whole (CUDA). */
int  b2h264_dec_decode3 (b2h264_dec* d, const uint8_t* const* au, const int32_t* au_bytes, uint8_t* const* yuv, int32_t* status);
/* As b2h264_dec_decode3 (same parsing, same status[s], same error codes), with the pictures left in HBM: yuv_dev[s] is a device
 * pointer on the decoder's device that receives the cropped, tightly packed I420 picture of stream s (w*h*3/2 bytes, any byte
 * alignment).  yuv_dev[s] may be NULL only where au[s] is NULL.  A stream that sits the call out or fails keeps its destination
 * untouched.  Host pointers and pointers on another device are refused with -1 before anything is launched.
 * ASYNCHRONOUS: the call returns once its work is enqueued on the decoder's stream (b2h264_dec_set_stream); the pictures are
 * complete when that stream reaches them, so work issued on the same stream afterwards reads finished pictures, and anything else
 * must wait for the stream.  Each destination must stay allocated until then.  The access units are parsed inside the call and
 * may be reused on return.  The next call's parse overlaps this call's kernels; the synchronous entry points above may follow a
 * device call at any time. */
int  b2h264_dec_decode_device (b2h264_dec* d, const uint8_t* const* au, const int32_t* au_bytes, uint8_t* const* yuv_dev, int32_t* status);
/* moves all of the decoder's GPU work to the caller's CUDA stream (cudaStream_t as void*), after waiting for the work already
 * issued on the decoder's current stream (as b2h264_enc_set_stream; the caller keeps the stream alive while the decoder uses it) */
int  b2h264_dec_set_stream (b2h264_dec* d, void* stream);
/* Pictures come back in DECODING order.  Of the picture stream `stream` decoded last: its picture order count inside its coded video
 * sequence, *flags (bit 0: an IDR picture — a new sequence starts; bit 1: the picture holds B slices), and the stream's reorder depth (num_ref_frames; 0 for Baseline streams,
 * whose decoding order is the output order).  The reference reorders inside DecodeFrameNoDelay (welsDecoderExt.cpp: ReorderPicturesInDisplay);
 * layer 3 does the same with these values. */
int  b2h264_dec_last_picture_order (b2h264_dec* d, int stream, int32_t* poc, int32_t* flags, int32_t* reorder_depth);
/* stream `stream` starts over: parameter sets, frame numbering and reference pictures are forgotten (the next unit must carry SPS / PPS / IDR) */
int  b2h264_dec_reset_stream (b2h264_dec* d, int stream);
/* stateless look at an access unit: *has_slice, and — if it carries an SPS of the supported class — the cropped picture
 * size (so that a caller can create the decoder for it: ISVCDecoder learns the size from the stream) */
int  b2h264_dec_probe (const uint8_t* au, int32_t au_bytes, int32_t* width, int32_t* height, int32_t* has_slice);

/* Page-locked host memory for pictures handed to b2h264_enc_submit / received from b2h264_dec_decode: copies to and from such
 * memory run at PCIe speed and asynchronously; ordinary (pageable) buffers work too, at roughly a third of the rate.
 * The reference's callers own their picture buffers (SSourcePicture::pData, codec_app_def.h) - this is the allocator for them. */
void* b2h264_host_alloc (size_t bytes);
void  b2h264_host_free (void* p);

#ifdef __cplusplus
}
#endif
#endif
