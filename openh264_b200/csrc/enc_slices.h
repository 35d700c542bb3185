// enc_slices.h — the slice partition of the encoder's pictures: SSliceArgument resolved as the reference resolves it, for the
// two modes whose partition is fixed before a picture is coded (SM_FIXEDSLCNUM_SLICE and SM_RASTER_SLICE).  Host only and free
// of CUDA: layer 2 (b2h264_enc_set_slices) and layer 3 (InitializeExt, GetOption) both resolve through it.
//
// Behavioural model (codec/encoder/core/src): ParamValidationExt (encoder_ext.cpp:540-612) with
// SliceArgumentValidationFixedSliceMode (:173-250) for RC_OFF_MODE, CheckFixedSliceNumMultiSliceSetting and
// CheckRasterMultiSliceSetting (svc_enc_slice_segment.cpp:125,166), and InitSliceSettings (encoder_ext.cpp:2010-2056), which
// sets the slice-coding thread count and turns loop filter idc 0 into 2 when more than one thread codes slices.
// Slices are raster runs (no FMO): a macroblock's neighbour is in its slice exactly when the neighbour lies inside the picture
// and its address is at least the first address of the macroblock's slice.
#pragma once
#include <stdint.h>

namespace b2h264 {

enum { kSmSingle = 0, kSmFixedNum = 1, kSmRaster = 2, kSmSizeLimited = 3 };   // SliceModeEnum (codec_app_def.h:337-342)
enum { kMaxSlicesNum = 35,                   // MAX_SLICES_NUM (svc_enc_slice_segment.h:61-62) = MAX_SLICES_NUM_TMP (codec_app_def.h:45-56)
       kMinMbPerSlice = 48,                  // MIN_NUM_MB_PER_SLICE
       kMaxThreadsNum = 4 };                 // MAX_THREADS_NUM (wels_const.h:69)

struct SliceConfig {
  int mode = kSmSingle;                      // resolved uiSliceMode
  int num = 1;                               // resolved uiSliceNum
  uint32_t mb_num[kMaxSlicesNum] = {};       // resolved uiSliceMbNum, entries past the slices as the reference leaves them

  int slices() const { return mode == kSmSingle ? 1 : num; }
  // first macroblock of each slice, and n_mb after the last: slices() + 1 entries
  void starts(int n_mb, int32_t* first) const {
    first[0] = 0;
    for (int i = 1; i < slices(); i++) first[i] = first[i - 1] + (int32_t)mb_num[i - 1];
    first[slices()] = n_mb;
  }

  // Resolves a request on a picture of mb_w x mb_h macroblocks.  mb_num: the caller's uiSliceMbNum (kMaxSlicesNum entries; NULL
  // reads as zeros).  Returns false for a request this encoder refuses, with the reason in *why: what the reference refuses
  // (one slice per row with more rows than kMaxSlicesNum, explicit runs that cannot be completed), what depends on the machine
  // (fixed slices with uiSliceNum 0 take the CPU core count), and the modes whose partition depends on the bits spent.
  static bool resolve(int mode, int num, const uint32_t* mb_num, int mb_w, int mb_h, SliceConfig* out, const char** why) {
    SliceConfig c;
    const int n_mb = mb_w * mb_h;
    if (mb_num) for (int i = 0; i < kMaxSlicesNum; i++) c.mb_num[i] = mb_num[i];
    c.mode = mode; c.num = num;
    auto single = [&](bool clear_runs) {
      c.mode = kSmSingle; c.num = 1;
      if (clear_runs) for (int i = 0; i < kMaxSlicesNum; i++) c.mb_num[i] = 0;
    };
    if (mb_w == 1 && mb_h == 1) c.mode = kSmSingle;                  // a one-macroblock picture (encoder_ext.cpp:541-544)
    if (c.mode == kSmSingle) {
      single(true);
    } else if (c.mode == kSmFixedNum) {
      if (num == 0) { *why = "SM_FIXEDSLCNUM_SLICE with uiSliceNum 0 (the reference takes the CPU core count)"; return false; }
      if (num <= 1 || n_mb <= kMinMbPerSlice) single(true);
      else {
        if (c.num > kMaxSlicesNum) c.num = kMaxSlicesNum;
        const int per = n_mb / c.num;
        for (int i = 0; i + 1 < c.num; i++) c.mb_num[i] = (uint32_t)per;
        const int left = n_mb - per * (c.num - 1);
        c.mb_num[c.num - 1] = (uint32_t)left;
        if (left <= 0 || per <= 0) single(true);
      }
    } else if (c.mode == kSmRaster) {
      if (c.mb_num[0] == 0) {                                          // one slice per macroblock row
        if (mb_h > kMaxSlicesNum) { *why = "SM_RASTER_SLICE with one slice per row and more rows than MAX_SLICES_NUM (35)"; return false; }
        c.num = mb_h;
        for (int j = 0; j < mb_h; j++) c.mb_num[j] = (uint32_t)mb_w;
      } else {
        // CheckRasterMultiSliceSetting: the runs up to the first 0 (or the picture's end), the last cut or a remainder added
        int count = 0, total = 0, i = 0;
        while (i < kMaxSlicesNum && c.mb_num[i] > 0) {
          total += (int)c.mb_num[i];
          count = i + 1;
          if (total >= n_mb) break;
          i++;
        }
        if (total > n_mb) c.mb_num[count - 1] -= (uint32_t)(total - n_mb);
        else if (total < n_mb) {
          if (count >= kMaxSlicesNum) { *why = "SM_RASTER_SLICE runs that leave macroblocks over after MAX_SLICES_NUM slices"; return false; }
          c.mb_num[count++] = (uint32_t)(n_mb - total);
        }
        c.num = count;
        if (c.num == 1 || n_mb <= kMinMbPerSlice) { c.mode = kSmSingle; c.num = 1; }
      }
    } else {
      *why = c.mode == kSmSizeLimited ? "SM_SIZELIMITED_SLICE (its slice boundaries depend on the bits coded so far)" : "uiSliceMode";
      return false;
    }
    *out = c;
    return true;
  }

  // Slices of one picture are coded by min(iMultipleThreadIdc clipped to 1..MAX_THREADS_NUM, uiSliceNum) threads
  // (GetMultipleThreadIdc, InitSliceSettings: encoder_ext.cpp:2213-2225,2051).  Fixed slices with load balancing move their
  // boundaries by measured coding times (encoder_ext.cpp:3564-3574, slice_multi_threading.cpp:168), and iMultipleThreadIdc 0
  // takes the machine's core count: false for these, whose bytes depend on the machine.
  bool reproducible(int multiple_thread_idc, bool load_balancing) const {
    if (slices() < 2) return true;
    if (multiple_thread_idc == 0) return false;
    const int t = threads(multiple_thread_idc);
    return !(mode == kSmFixedNum && t > 1 && load_balancing && t >= num);
  }
  // iLoopFilterDisableIdc as coded: 0 becomes 2 (slice edges unfiltered) when more than one thread codes the picture's slices
  int loop_filter_idc(int idc, int multiple_thread_idc) const {
    const int t = threads(multiple_thread_idc);
    return idc == 0 && (t < slices() ? t : slices()) > 1 ? 2 : idc;
  }
  static int threads(int multiple_thread_idc) {
    return multiple_thread_idc < 1 ? 1 : multiple_thread_idc > kMaxThreadsNum ? kMaxThreadsNum : multiple_thread_idc;
  }
};

}  // namespace b2h264
