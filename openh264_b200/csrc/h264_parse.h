// h264_parse.h — host-side bitstream PARSER: the inverse of h264_bitstream.{h,cpp} for the stream class this
// library decodes: Baseline / Main / High (8x8 transform, flat scaling lists), CAVLC or CABAC, I, P and B slices (several per picture, in raster order: no FMO / ASO),
// up to 16 reference frames, all partition shapes down to 4x4, direct prediction and implicit weights in B slices (h264_motion.h), non-reference pictures, constrained intra prediction, per-slice deblocking control.  Groundwork for the decoder construct path (SURVEY.md section 8f / DESIGN.md section 9): the
// reference parses on the host too (codec/decoder/core/src/{au_parser,parse_mb_syn_cavlc,decode_slice}.cpp) and
// hands macroblock arrays to the pixel stage; here the macroblock array is the same MbOut record the encoder's
// entropy coder consumes, so "parse(write(x)) == x" is checked for every picture the host build encodes
// (tests/emu) and the device-side construct stage can be the mirror image of the encoder's reconstruction.
// Anything outside that stream class is REJECTED with an error code, never guessed.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <vector>

#include "enc_types.h"
#include "h264_bitstream.h"

namespace b2h264 {

enum ParseError {
  PARSE_OK = 0,
  PARSE_NO_PICTURE = 1,        // the access unit was parsed (parameter sets taken) but holds no slice
  PARSE_TRUNCATED = -1,        // ran out of bits
  PARSE_UNSUPPORTED = -2,      // valid H.264 outside the supported class (FMO, scaling lists, interlace, ...)
  PARSE_INVALID = -3,          // not valid H.264 syntax / values out of range
  PARSE_NO_PARAMETER_SETS = -4,// a slice before its SPS / PPS
  PARSE_INCOMPLETE = -5        // the slices seen so far do not cover the picture (more slices of the access unit to come, or lost)
};

// what an SPS / a PPS contributes; streams may carry several of each (selected per slice through pic_parameter_set_id)
struct SpsFields {
  bool valid = false;
  StreamParams sp{};
  int log2_max_frame_num = 0, poc_type = 2, log2_max_poc_lsb = 0, n_slots = 2, crop_left = 0, crop_top = 0;
  bool delta_pic_order_always_zero = false;
  int profile = 66;
  bool direct_8x8_inference = true;
};
struct PpsFields {
  bool valid = false;
  int sps_id = 0, pic_init_qp = 26, num_ref_idx_default = 1, num_ref_idx_l1_default = 1, weighted_bipred_idc = 0;
  bool deblocking_control = true, constrained_intra_pred = false, entropy_cabac = false;
  int chroma_qp_offset = 0;            // chroma_qp_index_offset (= second_chroma_qp_index_offset, else the PPS is rejected)
  bool transform_8x8 = false, weighted_pred = false;
};

// CABAC only: what later macroblocks of the slice need to know about a parsed macroblock (context selection, 9.3.3.1.1)
struct CabacMbInfo {
  uint8_t type, skip, intra, cbp, chroma_mode, ref_gt0;   // ref_gt0: bit q = ref_idx_l0 of 8x8 block q is > 0
  uint8_t ref_gt0_l1;               // the same for list 1 (B slices); direct-predicted blocks count as 0 in both (9.3.3.1.1.6)
  uint8_t direct;                   // B_Skip or B_Direct_16x16 (ctxIdxInc of mb_type in B slices)
  uint8_t t8;                       // transform_size_8x8_flag (ctxIdxInc of the neighbours' flag)
  uint8_t pad1[3];
  uint32_t cbf;                     // bit 0..15 luma 4x4 (raster), 16..19 Cb AC, 20..23 Cr AC, 24 luma DC, 25 Cb DC, 26 Cr DC
  uint8_t mvd[16][2];               // min(|mvd|, 255) per 4x4 block (raster); the context only distinguishes sums up to 33
  uint8_t mvd_l1[16][2];            // list 1 (B slices)
};

// What the parser keeps per decoded picture when the stream may hold B slices (any profile but Baseline): the motion field —
// the co-located picture of direct prediction (8.4.1.2) and, inside the picture being parsed, the neighbours of the host-side
// vector prediction of B macroblocks.  Raster 4x4 order inside a macroblock.
struct MotionStore {
  std::vector<int16_t> mv[2];        // [list][(mb * 16 + blk) * 2 + c]
  std::vector<int8_t> ref[2];        // [list][mb * 16 + blk]: reference index as coded / inferred, -1: list not used or intra
  std::vector<int32_t> ref_id[2];    // [list][mb * 16 + blk]: identity (decoding counter) of the referenced picture, -1 if none
  std::vector<uint8_t> intra;        // [mb]
  int poc = 0, pic_id = -1;
  void size_for(int n_mb) {
    for (int l = 0; l < 2; l++) { mv[l].assign((size_t)n_mb * 32, 0); ref[l].assign((size_t)n_mb * 16, -1); ref_id[l].assign((size_t)n_mb * 16, -1); }
    intra.assign(n_mb, 0);
  }
};

// parameter sets carried from access unit to access unit
struct ParserState {
  SpsFields sps_tab[32];
  PpsFields pps_tab[256];
  int crop_left = 0, crop_top = 0;   // of the active SPS, in units of 2 luma samples
  bool have_sps = false, have_pps = false;
  StreamParams sp{};             // width / height / mb_w / mb_h / crop / level / ids (num_ref_frames)
  int log2_max_frame_num = 0;
  int poc_type = 2, log2_max_poc_lsb = 0;
  bool delta_pic_order_always_zero = false;
  int pic_init_qp = 26;
  bool deblocking_control = true;
  bool constrained_intra_pred = false;
  bool entropy_cabac = false;
  int num_ref_idx_default = 1;
  bool have_ref = false;         // a picture has been decoded (a P slice has something to predict from)
  int last_frame_num = 0;
  // decoded picture buffer bookkeeping (8.2.4, 8.2.5.3): the short-term reference pictures in decoding order, each in one
  // of n_slots picture slots of the construct stage (num_ref_frames + 1: the picture being decoded needs one too)
  struct RefPic { int slot, frame_num; bool long_term; int lt_idx; int poc; int pic_id; };
  std::vector<RefPic> refs;
  int n_slots = 2;
  // B slices: picture order count (type 0, 8.2.1.1), motion fields by picture slot
  int profile = 66, weighted_bipred_idc = 0, num_ref_idx_l1_default = 1;
  int chroma_qp_offset = 0;
  bool transform_8x8 = false, weighted_pred = false;
  bool direct_8x8_inference = true;
  int prev_poc_msb = 0, prev_poc_lsb = 0;      // of the previous reference picture
  int next_pic_id = 0;
  int decode_count = 0;                        // pictures so far (output order of streams whose POC is not type 0)
  std::vector<MotionStore> motion;             // [slot]; empty for Baseline streams
};

struct ParsedPicture {
  SliceState ss;                 // idr, frame_num, idr_pic_id, slice qp
  bool is_ref = true;            // nal_ref_idc != 0
  int crop_left = 0, crop_top = 0;   // luma samples to drop at the left / top of the decoded picture
  std::vector<MbOut> mbs;        // mb_w * mb_h records, same meaning as the encoder's hand-over records
  std::vector<DecMbAux> aux;     // one per macroblock: slice membership, sub-macroblock partitions, deblocking control
  int next_mb = 0;               // macroblocks parsed so far (slices arrive in raster order)
  int n_slices = 0;
  int poc = 0;                   // picture order count (output order); decoding order x 2 where the stream has no type-0 POC
  int poc_msb = 0, poc_lsb = 0;
  int pic_id = 0;                // decoding counter: identity of the picture in other pictures' motion fields
  int max_reorder = 0;           // pictures that may have to wait for an earlier-output picture (0: output order = decoding order)
  bool has_b = false;            // some slice is a B slice: aux_b is filled
  bool has_t8 = false;           // the picture's PPS allows the 8x8 transform (the filter must look at MbInfo::t8x8)
  int chroma_qp_offset = 0;      // chroma_qp_index_offset of the picture's PPS
  std::vector<DecMbAuxB> aux_b;  // list 1 of the B macroblocks (sized like aux when has_b)
  int cur_slot = 0;              // picture slot this picture is reconstructed into
  int n_slots = 2;               // slots the stream needs (from its SPS)
  // dec_ref_pic_marking of the picture (first slice): sliding window, or memory_management_control_operation 1 commands
  bool adaptive_marking = false;
  struct Mmco { int op, a, b; };  // memory_management_control_operation with its operands
  std::vector<Mmco> mmco;
  bool idr_long_term = false;    // long_term_reference_flag of an IDR picture
  bool any_deblock = false;      // some slice wants its macroblocks filtered
  std::vector<CabacMbInfo> cabac_info;   // scratch of the CABAC slice-data parser (one per macroblock)
};

// Parses one access unit: [SPS] [PPS] slice, each NAL behind a 3- or 4-byte start code, into a fresh *pic (whose record arrays keep
// their storage).  Returns PARSE_OK or an error.
int parse_access_unit(const uint8_t* au, size_t len, ParserState* st, ParsedPicture* pic);
// without state: is there a slice, and the cropped size of the SPS the unit carries (0 x 0 if none)
int probe_access_unit(const uint8_t* au, size_t len, int* width, int* height, int* has_slice);

}  // namespace b2h264
