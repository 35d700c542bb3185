// mbk_common.cuh — shared device helpers for the macroblock kernels (sm_90a).
//
// Execution model used throughout: ONE WARP OWNS ONE MACROBLOCK (or one block-level job).
// Every warp-level routine below must be called by all 32 lanes of a converged warp; results
// are returned to all lanes.  Pixel pointers are generic (shared or global).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define MBK_FULL 0xffffffffu

// ---- host/device portability ------------------------------------------------------------------
// The macroblock code is written once.  Compiled for the device, a routine is executed by the 32
// lanes of one warp (lane-strided loops + REDUX).  Compiled for the host (tests/emu only: a
// debugging build that is NOT part of the product library) the same source runs as a "1-lane warp":
// MBK_WS == 1, so every lane-strided loop visits all indices and warp reductions are the identity.
#define MBK_HD __host__ __device__ __forceinline__
// Warp-level routines are real functions, not inlined: one inlined copy per call site grew the encode
// kernel several-fold and the warps (each in a different phase of a different macroblock) spent most
// of their cycles waiting for instruction fetch.
// External (weak, ODR-merged) linkage on purpose: with `static`, ptxas specialises the calling convention of each
// function inside the translation unit, and one such specialisation returned a stale register for a field the
// callee had just stored through a pointer into the caller's frame (me_refine -> MeState::mv_y).  Externally visible functions follow the standard ABI.  Every
// translation unit is compiled with the same register cap because nvlink keeps one copy of each function.
#define MBK_FN inline __host__ __device__ __noinline__
// stage entry points have ONE call site each: inlined there, they cost no code and save the callee-saved register
// spill / reload of a real call (a few dozen STL + LDL per call)
#ifdef B2H264_STAGE_CALLS                  // profiling variant: stage entry points as real calls
#define MBK_STAGE MBK_FN
#else
#define MBK_STAGE __host__ __device__ __forceinline__
#endif
// loops around calls to the big warp routines are kept rolled: the macroblock kernel is bound by instruction fetch (the code one
// stage walks through does not fit the instruction cache), so code size is time
#ifdef __CUDACC__
#define MBK_NO_UNROLL _Pragma("unroll 1")
#else
#define MBK_NO_UNROLL
#endif
// Re-alignment points of a lock-step batch (device, experiment B2H264_BATCH_SYNC): the warps of a batch drift apart inside a long
// stage (different search lengths) and stop sharing instruction-cache fills; a named barrier over the n warps of the batch pulls
// them together again.  Every warp of the batch passes each point exactly once: mbk_batch_sync waits, a warp that leaves the
// stage early calls mbk_batch_leave for the points it will not reach.  Barrier ids 2.. (0 = __syncthreads, 1 = the batch barrier).
#ifdef __CUDA_ARCH__
__device__ __forceinline__ void mbk_batch_sync(int id, int n) { if (n > 1) asm volatile("barrier.sync %0, %1;" ::"r"(id), "r"(32 * n) : "memory"); }
__device__ __forceinline__ void mbk_batch_leave(int id, int n) { if (n > 1) asm volatile("barrier.arrive %0, %1;" ::"r"(id), "r"(32 * n) : "memory"); }
#else
inline void mbk_batch_sync(int, int) {}
inline void mbk_batch_leave(int, int) {}
#endif
#ifdef __CUDA_ARCH__
#define MBK_WS 32
#else
#define MBK_WS 1
#endif

namespace mbk {

MBK_HD int lane_id() {
#ifdef __CUDA_ARCH__
  return threadIdx.x & 31;
#else
  return 0;
#endif
}
MBK_HD int warp_sum(int v) {
#ifdef __CUDA_ARCH__
  return __reduce_add_sync(MBK_FULL, v);
#else
  return v;
#endif
}
MBK_HD int warp_min(int v) {
#ifdef __CUDA_ARCH__
  return __reduce_min_sync(MBK_FULL, v);
#else
  return v;
#endif
}
MBK_HD void warp_sync() {
#ifdef __CUDA_ARCH__
  __syncwarp();
#endif
}
MBK_HD uint32_t vsadu4(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
  return __vsadu4(a, b);
#else
  uint32_t s = 0;
  for (int i = 0; i < 4; i++) { const int d = (int)((a >> (8 * i)) & 0xff) - (int)((b >> (8 * i)) & 0xff); s += d < 0 ? -d : d; }
  return s;
#endif
}
// per-byte rounded average (a + b + 1) >> 1 of packed bytes
MBK_HD uint32_t vavgu4(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
  return __vavgu4(a, b);
#else
  uint32_t r = 0;
  for (int i = 0; i < 4; i++) r |= ((((a >> (8 * i)) & 0xff) + ((b >> (8 * i)) & 0xff) + 1) >> 1) << (8 * i);
  return r;
#endif
}
MBK_HD int clz32(uint32_t v) {
#ifdef __CUDA_ARCH__
  return __clz((int)v);
#else
  return v ? __builtin_clz(v) : 32;
#endif
}

// quantiser tables live in constant memory, filled once by b2h264 init (closed forms, see tables.cu)
// host copies of the same tables (tables.cu); the device reads constant memory, the host build reads these
extern int16_t h_quant_ff[58][8];
extern int16_t h_quant_mf[52][8];
extern uint16_t h_dequant[52][8];
extern uint8_t h_lambda[52];
extern uint8_t h_chroma_qp[52];
#ifdef __CUDACC__
extern __constant__ int16_t c_quant_ff[58][8];   // g_kiQuantInterFF (intra = row qp+6)
extern __constant__ int16_t c_quant_mf[52][8];   // g_kiQuantMF
extern __constant__ uint16_t c_dequant[52][8];   // g_kuiDequantCoeff
extern __constant__ uint8_t c_lambda[52];        // g_kiQpCostTable
extern __constant__ uint8_t c_chroma_qp[52];     // g_kuiChromaQpTable
#endif
#ifdef __CUDA_ARCH__
#define MBK_TBL(dev, host) dev
#else
#define MBK_TBL(dev, host) host
#endif
MBK_HD const int16_t* tbl_quant_ff(int q) { return MBK_TBL(c_quant_ff, h_quant_ff)[q]; }
MBK_HD const int16_t* tbl_quant_mf(int q) { return MBK_TBL(c_quant_mf, h_quant_mf)[q]; }
MBK_HD const uint16_t* tbl_dequant(int q) { return MBK_TBL(c_dequant, h_dequant)[q]; }
MBK_HD int tbl_lambda(int q) { return MBK_TBL(c_lambda, h_lambda)[q]; }
MBK_HD int tbl_chroma_qp(int q) { return MBK_TBL(c_chroma_qp, h_chroma_qp)[q]; }

MBK_HD int iabs(int v) { return v < 0 ? -v : v; }
MBK_HD int clip3(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
MBK_HD int clip255(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

// block-size ids follow the reference (encoder/core/inc/wels_const.h:139-148)
enum { BLK_16x16 = 0, BLK_16x8, BLK_8x16, BLK_8x8, BLK_4x4, BLK_8x4, BLK_4x8 };
MBK_HD int blk_lw(int blk) { return (0x2323344 >> (blk * 4)) & 0xf; }  // log2(width)
MBK_HD int blk_lh(int blk) { return (0x3223434 >> (blk * 4)) & 0xf; }  // log2(height)
MBK_HD int blk_w(int blk) { return 1 << blk_lw(blk); }
MBK_HD int blk_h(int blk) { return 1 << blk_lh(blk); }

// 4 consecutive bytes at an arbitrary byte address as a little-endian word: two aligned 32-bit
// loads + funnel shift (never reads past the aligned word that holds byte p+3).
MBK_HD uint32_t ld4u(const uint8_t* p) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
  const uint32_t sh = (uint32_t)(a & 3) * 8;
  const uint32_t lo = w[0];
  const uint32_t hi = sh ? w[1] : 0u;
#ifdef __CUDA_ARCH__
  return __funnelshift_r(lo, hi, sh);
#else
  return sh ? (lo >> sh) | (hi << (32 - sh)) : lo;
#endif
}

// bits of the signed Exp-Golomb code of v (encoder/core/inc/svc_enc_golomb.h:84-95)
MBK_HD int se_bits(int v) {
  const uint32_t code = v > 0 ? (uint32_t)(2 * v - 1) : (uint32_t)(-2 * v);
  return 2 * (31 - clz32(code + 1)) + 1;
}
// COST_MVD(table, dx, dy) with table[d] = (uint16)(lambda * bits(se(d)))  (md.cpp:797-824)
MBK_HD int mvd_cost(int lambda, int dx, int dy) {
  return ((lambda * se_bits(dx)) & 0xffff) + ((lambda * se_bits(dy)) & 0xffff);
}

}  // namespace mbk
