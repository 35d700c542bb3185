// enc_host.h — host-side stream control for one encoder instance: parameter sets, frame numbering,
// slice serialisation from the device's MbOut records.  Mirrors the small part of
// codec/encoder/core/src/encoder_ext.cpp (WelsEncoderEncodeExt :3441, frame_num / idr_pic_id handling
// :3131,:3253) that the supported configuration exercises: CAMERA_VIDEO_REAL_TIME, 1 spatial + 1
// temporal layer, RC_OFF_MODE, fixed slice partitions, CAVLC, 1 reference frame, IDR only at the start
// (uiIntraPeriod = 0) or on ForceIntraFrame.
#pragma once
#include <vector>

#include "enc_refs.h"
#include "enc_types.h"
#include "h264_bitstream.h"

namespace b2h264 {

// Host twin of k_pack_records (enc_kernels.cu): compacts n records into `dst` (worst case n * sizeof(MbOut) bytes) and fills idx[mb] =
// offset of the macroblock's record in 32-byte units, or -1 - qp for a P_SKIP macroblock (the decoder's hand-over keeps the
// quantiser of a skipped macroblock: deblocking needs it; the encoder's reader only tests the sign).  Returns the units written.
// Record: 128-byte head (MbOut bytes [0, 112) + chroma_dc, presence mask of the 24 residual blocks in pad0) + 32 bytes per present block.
int pack_records_compact(const MbOut* mbs, int n, uint8_t* dst, int32_t* idx);

// A padded picture (picture_handle.cpp:60-85): Y, then Cb, then Cr, luma padded by 32 samples on every side and chroma by 16, so
// sample (0, 0) lies at row 32, column 32 of the luma plane and at row 16, column 16 of each chroma plane.  Built from the picture
// size in macroblocks, or from given strides and the height in macroblocks.
struct PicLayout {
  int stride_y = 0, stride_c = 0, rows_y = 0, rows_c = 0;
  PicLayout() = default;
  PicLayout(int mb_w, int mb_h) : PicLayout(mb_w * 16 + 64, mb_w * 8 + 32, mb_h) {}
  PicLayout(int sty, int stc, int mb_h) : stride_y(sty), stride_c(stc), rows_y(mb_h * 16 + 64), rows_c(mb_h * 8 + 32) {}
  int stride(int pl) const { return pl ? stride_c : stride_y; }
  size_t y_bytes() const { return (size_t)stride_y * rows_y; }
  size_t c_bytes() const { return (size_t)stride_c * rows_c; }
  size_t bytes() const { return y_bytes() + 2 * c_bytes(); }
  // offset of sample (0, 0) of plane pl (0 Y, 1 Cb, 2 Cr) from the first byte of the picture
  size_t plane0(int pl) const { return pl == 0 ? (size_t)32 * stride_y + 32 : y_bytes() + (size_t)(pl - 1) * c_bytes() + (size_t)16 * stride_c + 16; }
};

struct StreamCtl {
  StreamParams sp;
  float fps;
  // numbering of the picture written last; write_access_unit_packed takes both from the picture's RefDecision (StreamRefs numbers
  // the pictures), write_access_unit (one-reference host path) counts them here
  int frame_num = 0;
  int idr_pic_id = 0;
  long frames_coded = 0;
  bool force_idr = true;
  // eSpsPpsIdStrategy: INCREASING_ID (the reference default) gives every emitted SPS/PPS pair the next id
  // (mod MAX_SPS_COUNT 32 / MAX_PPS_COUNT 57, paraset_strategy.cpp:338-369); CONSTANT_ID keeps 0/0
  bool increasing_ids = true;
  int parasets_written = 0;
  bool fast_mode = false;                   // iComplexityMode == LOW_COMPLEXITY
  bool record_mb_bits = false;              // keep the writer's bits per macroblock of the last picture (parity of the device count)
  std::vector<int32_t> last_mb_bits;

  void init(int width, int height, int qp, float fps_, int target_bitrate, int entropy_cabac = 0, int profile_idc = 0);
  bool next_is_idr() const { return force_idr; }
  // first macroblock of every slice of a picture (enc_slices.h: SliceConfig::starts), set before set_loop_filter; empty: one slice
  std::vector<int32_t> slice_first;
  // iLoopFilterDisableIdc / iLoopFilterAlphaC0Offset / iLoopFilterBetaOffset (after init): with one slice per picture idc 2 is
  // idc 0 (encoder_ext.cpp:1109-1114); false if a value is out of range (encoder_ext.cpp:316-318)
  bool set_loop_filter(int idc, int alpha_c0_offset, int beta_offset) {
    if (idc < 0 || idc > 2 || alpha_c0_offset < -6 || alpha_c0_offset > 6 || beta_offset < -6 || beta_offset > 6) return false;
    sp.dbk_idc = idc == 2 && slice_first.size() < 2 ? 0 : idc; sp.dbk_alpha_div2 = alpha_c0_offset; sp.dbk_beta_div2 = beta_offset;
    return true;
  }
  // geometry of the padded pictures (PicLayout)
  int rec_stride_y() const { return PicLayout(sp.mb_w, sp.mb_h).stride_y; }
  int rec_stride_c() const { return PicLayout(sp.mb_w, sp.mb_h).stride_c; }
  int rec_rows_y() const { return PicLayout(sp.mb_w, sp.mb_h).rows_y; }
  int rec_rows_c() const { return PicLayout(sp.mb_w, sp.mb_h).rows_c; }
  EncFrameParams frame_params(bool idr, bool ref_is_p) const;
  // serialises the access unit of the frame just coded (SPS+PPS+IDR slices, or P slices: one NAL unit per slice)
  void write_access_unit(bool idr, const MbOut* mbs, std::vector<uint8_t>* au);                 // one record per MB
  // compact form (k_pack_records): idx[mb] = offset of the macroblock's record in `packed` in 32-byte units, or -1 for P_SKIP;
  // refs: the picture's reference syntax (enc_refs.h), NULL for the one-reference stream's
  void write_access_unit_packed(bool idr, const MbOut* packed, const int32_t* idx, std::vector<uint8_t>* au,
                                const RefDecision* refs = nullptr);
  // max_num_ref_frames of the SPS; the level follows from it (after init)
  void set_num_ref_frames(int n, int target_bitrate) { sp.num_ref_frames = n; select_level(&sp, fps, target_bitrate); }
 private:
  void write_au(bool idr, const MbOut* const* recs, std::vector<uint8_t>* au, const RefDecision* refs = nullptr);
  std::vector<const MbOut*> recs_;
  std::vector<uint8_t> rbsp_;               // payload of the NAL being written (reused from picture to picture)
  std::vector<MbOut> expand_;               // compact records of the coded macroblocks, expanded for the slice writer
 public:
  int last_coded_mbs = 0;                   // macroblocks of the last picture that were not P_SKIP (write_access_unit_packed)
};

// copies a w x h I420 picture into MB-aligned planes; rows/cols beyond the picture are 0 (luma) / 0x80
// (chroma) like CWelsPreProcess::Padding (wels_preprocess.cpp:1250)
void pad_source(const uint8_t* yuv, int w, int h, int mb_w, int mb_h, uint8_t* y, uint8_t* u, uint8_t* v);

}  // namespace b2h264
