// enc_launch.h — host-callable launchers of the encoder kernels (enc_kernels.cu)
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "enc_types.h"

struct StreamFrame {            // one stream's frame job, array in device memory
  EncFrameParams p;
  EncFramePtrs f;
};

int enc_upload_deblock_tables();
// pad (if d_src != NULL) + wavefront macroblock kernel for n_streams pictures of identical geometry
int enc_launch_frame(const StreamFrame* d_sf, const uint8_t* const* d_src, int n_streams, int w, int h, int mb_w, int mb_h,
                     int* d_sched_ws, void* d_stash,
                     const void* tmap_ref /* CUtensorMap of the reference luma planes or NULL: the search reads the planes directly */,
                     int fast_mode /* LOW_COMPLEXITY: also computes the VAA 8x8 SADs */, cudaStream_t st);
// wavefront deblocking + border expansion of the pictures just reconstructed
int enc_launch_deblock_expand(const StreamFrame* d_sf, int n_streams, int mb_w, int mb_h, cudaStream_t st);
// number of ints of scheduler workspace (dependency counters, ready lists) for a batch
size_t enc_sched_ints(int n_streams, int mb_w, int mb_h);
size_t enc_stash_bytes(int n_streams, int mb_h);      // parked macroblock scratches (one per stream and MB row)
size_t enc_scratch_bytes();
// decoder construct path: reconstruct + deblock (if `deblock`) + expand one picture per stream from parsed records
size_t dec_sched_ints(int n_streams, int mb_w, int mb_h);
int dec_launch_frame(const StreamFrame* d_sf, int n_streams, int mb_w, int mb_h, int* d_ws, const MbOut* d_recs, const DecMbAux* d_aux, int deblock,
                     cudaStream_t st, int b_slices /* some picture of the batch holds B slices */);
// compacts the records of the picture just coded into (mapped pinned) `pack`; idx / cnt likewise host-visible
int dec_launch_unpack(const void* d_pack, size_t stream_stride_bytes, const int32_t* d_idx, MbOut* d_recs, int n_streams, int n_mb, cudaStream_t st);
int enc_launch_pack(const StreamFrame* d_sf, int n_streams, int n_mb, MbOut* pack, int32_t* idx, int32_t* cnt, cudaStream_t st);
