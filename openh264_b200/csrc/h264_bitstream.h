// h264_bitstream.h — host-side bitstream serialisation (stays on the CPU by design, north_star):
// parameter sets, slice headers, CAVLC macroblock syntax, NAL encapsulation.  It consumes the MbOut
// records the device pipeline copies back.  Syntax follows Rec. H.264 7.3 / 9.2; the field values
// follow what the reference emits for the supported configuration
// (codec/encoder/core/src/au_set.cpp:197-470, svc_encode_slice.cpp:275-346,
//  svc_set_mb_syn_cavlc.cpp:60-420, set_mb_syn_cavlc.cpp:84-250, nal_encap.cpp).
#pragma once
#include <stdint.h>
#include <stddef.h>
#include <vector>

#include "enc_types.h"

namespace b2h264 {

class BitWriter {
 public:
  explicit BitWriter(std::vector<uint8_t>* out) : out_(out) {}
  // n <= 32 bits, MSB first.  Bits gather in a 64-bit accumulator; whole bytes go to the buffer at once (a byte is in the buffer as
  // soon as it is complete, so bit_pos() / the buffer's size always tell the truth)
  void put(int n, uint32_t v) {
    if (n <= 0) return;
    acc_ = (acc_ << n) | (n >= 32 ? (uint64_t)v : (uint64_t)(v & ((1u << n) - 1u)));
    nbits_ += n;
    while (nbits_ >= 8) { nbits_ -= 8; out_->push_back((uint8_t)(acc_ >> nbits_)); }
  }
  void bit(int b) { put(1, (uint32_t)(b != 0)); }
  void ue(uint32_t v) {
    const int len = 31 - __builtin_clz(v + 1);     // v + 1 >= 1; v < 2^32 - 1
    if (len > 16) { put(len, 0); put(len + 1, v + 1); }
    else put(2 * len + 1, v + 1);
  }
  void se(int32_t v) { ue(v > 0 ? (uint32_t)(2 * v - 1) : (uint32_t)(-2 * v)); }
  void trailing() { bit(1); if (nbits_) put(8 - nbits_, 0); }
  size_t bit_pos() const { return out_->size() * 8 + nbits_; }
 private:
  std::vector<uint8_t>* out_;
  uint64_t acc_ = 0;             // the low nbits_ bits are pending
  int nbits_ = 0;                // < 8 between calls
};

struct StreamParams {
  int width, height;            // picture size in luma samples (coded size = MB aligned)
  int mb_w, mb_h;
  int num_ref_frames;
  int level_idc;
  bool constraint_set3;
  int qp;
  bool crop;
  int crop_right, crop_bottom;  // in units of 2 luma samples
  int sps_id, pps_id;           // ids written into the parameter sets / slice headers (paraset_strategy.cpp)
  int profile_idc = 66;         // 66 Baseline (CAVLC); with CABAC the reference picks High (100) unless the layer asks for Main (77)
  bool entropy_cabac = false;   // entropy_coding_mode_flag
  // slice header: disable_deblocking_filter_idc (0 / 1), slice_alpha_c0_offset_div2, slice_beta_offset_div2 (-6..6)
  int dbk_idc = 0, dbk_alpha_div2 = 0, dbk_beta_div2 = 0;
};

// level selection (WelsGetLevelIdc, au_set.cpp:51-195; limits = H.264 Table A-1)
void select_level(StreamParams* sp, float fps, int target_bitrate);

// appends one NAL unit (4-byte start code + header + emulation-prevented payload)
void append_nal(std::vector<uint8_t>* dst, int nal_ref_idc, int nal_type, const std::vector<uint8_t>& rbsp);

void write_sps(const StreamParams& sp, std::vector<uint8_t>* rbsp);
void write_pps(const StreamParams& sp, std::vector<uint8_t>* rbsp);

struct SliceState {
  bool idr;
  int frame_num;
  int idr_pic_id;
  int qp;
  // reference syntax (enc_refs.h: RefDecision); the defaults are the one-reference stream's: the previous picture, no marking
  int mod_idc = 0, mod_val = 0;         // P: ref_pic_list_modification, idc 0 (abs_diff_pic_num_minus1) or 2 (long_term_pic_num)
  bool long_term_reference_flag = false;  // IDR
  int n_mmco = 0;                       // P: adaptive_ref_pic_marking_mode_flag = n_mmco > 0
  int mmco[3][3] = {};                  // operation and its values, in the order they are written
  int first_mb = 0, end_mb = -1;        // the slice's macroblocks [first_mb, end_mb) (raster run; -1: to the picture's end)
};
// slice header up to slice_beta_offset_div2 (svc_encode_slice.cpp:275-346); both entropy modes write it
void write_slice_header(BitWriter& w, const StreamParams& sp, const SliceState& ss);
// coded_block_pattern me(v) mapping (Rec. H.264 Table 9-4, chroma_format_idc 1): codeNum indexed by cbp (48 entries)
const uint8_t* cbp_me_table(bool intra);

// slice header + the slice's macroblocks (ss.first_mb .. ss.end_mb) + trailing bits.  A neighbour outside the slice is not
// available.  recs[i] = the record of macroblock i of the picture (P_SKIP macroblocks may all point at one shared all-zero-nnz record)
// mb_bits (optional, sized to the picture): bits of macroblock_layer() of the slice's macroblocks (0 for P_SKIP; mb_skip_run not included)
void write_slice(const StreamParams& sp, const SliceState& ss, const MbOut* const* recs, std::vector<uint8_t>* rbsp,
                 std::vector<int32_t>* mb_bits = nullptr);

// the same slice through CABAC (entropy_coding_mode_flag = 1; contexts initialised per slice): h264_cabac.cpp
void write_slice_cabac(const StreamParams& sp, const SliceState& ss, const MbOut* const* recs, std::vector<uint8_t>* rbsp);

}  // namespace b2h264
