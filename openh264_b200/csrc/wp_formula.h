// wp_formula.h — weighted sample prediction (Rec. H.264 8.4.2.3), written once for the decoder's construct stage (dec_mb.cuh),
// the layer-1 kernel k_weighted_pred (k_pixel.cu, pinned to the reference by tests/test_cross_weighted.py) and the host parser,
// which resolves the offsets of a two-list prediction (h264_motion.h).  Reference counterparts: WeightPrediction and
// BiWeightPrediction (codec/decoder/core/src/rec_mb.cpp:298, :366).  The results are not clipped; the caller clips to 0..255.
#pragma once

#ifdef __CUDACC__
#define WP_HD __host__ __device__ __forceinline__
#else
#define WP_HD inline
#endif

// one list: ((p * w + 2^(ld - 1)) >> ld) + o, and p * w + o for ld 0
WP_HD int wp_single(int p, int w, int o, int ld) { return (ld >= 1 ? (p * w + (1 << (ld - 1))) >> ld : p * w) + o; }
// two lists: ((a * w0 + b * w1 + 2^ld) >> (ld + 1)) + o, with o = wp_bi_offset(o0, o1)
WP_HD int wp_bi(int a, int b, int w0, int w1, int o, int ld) { return ((a * w0 + b * w1 + (1 << ld)) >> (ld + 1)) + o; }
WP_HD int wp_bi_offset(int o0, int o1) { return (o0 + o1 + 1) >> 1; }

// What the explicit weights of B slices reached while decoding: counted per 8x8 by the parser (emit_resolved) and, for the clipping,
// per sample by the construct stage.  Read and reset through b2h264_dec_wp_stats (h264_parse.cpp); the tests use them to show that
// their streams exercise every case of the weighting.  Only the host build of the decoder (tests/emu, single-threaded) counts: the
// product library is compiled with B2H264_NO_WP_STATS (openh264_b200/csrc/Makefile), so its parser threads carry neither the
// counting nor the query.
enum {
  WPS_SINGLE_L0, WPS_SINGLE_L1,                      // one-list formula from list 0 / list 1
  WPS_BI_16x16, WPS_BI_16x8, WPS_BI_8x16, WPS_BI_SUB,  // 8x8s of two-list partitions (B_8x8: sub-macroblocks, direct 8x8s excluded)
  WPS_QUIRK_FIRST, WPS_QUIRK_SECOND,                 // two-list 16x8 / 8x16 partitions whose luma weights do not sum to 2^(ld+1)
                                                     // and whose offsets are not both 0: first / second partition
  WPS_SPATIAL_DIRECT, WPS_TEMPORAL_DIRECT, WPS_B_SKIP,
  WPS_REF_L0_GT0, WPS_REF_L1_GT0,                    // a weighted 8x8 with refIdxL0 > 0 / refIdxL1 > 0
  WPS_DENOM_Y0, WPS_DENOM_Y7, WPS_DENOM_C0, WPS_DENOM_C7,
  WPS_WEIGHT_MIN, WPS_WEIGHT_MAX, WPS_OFFSET_MIN, WPS_OFFSET_MAX,   // a table entry in use holds -128 / 127
  WPS_DEFAULTED,                                     // a table entry in use whose luma or chroma flag is 0
  WPS_HALF,                                          // one-list 8x4 / 4x8 sub-macroblock: only its second half is weighted
  WPS_CLIP_LOW, WPS_CLIP_HIGH,                       // weighted samples of such macroblocks clipped at 0 / 255
  WPS_N
};
#if !defined(B2H264_NO_WP_STATS) && !defined(__CUDA_ARCH__)
#define B2H264_WP_STATS 1
void b2h264_wp_stat(int which, long long n);
// copies min(n, WPS_N) counters to out, resets all of them when `reset`; returns WPS_N
extern "C" int b2h264_dec_wp_stats(long long* out, int n, int reset);
#endif
