// k_pixel.cu — batched pixel-domain kernels behind include/b2h264.h: SAD/SATD, sub-pel MC, deblocking
// edge filters, border expansion, integer motion search, and the MC+SAD roofline unit.
// One warp per job; 8 warps per CTA; grid sized to cover n jobs.
#include <cuda.h>               // CUtensorMap (the encode entry point is fetched through the runtime)

#include "b2h264_internal.h"
#include "mbk_deblock.cuh"
#include "mbk_mc.cuh"
#include "mbk_me.cuh"
#include "mbk_pix8.cuh"
#include "mbk_sad.cuh"
#include "wp_formula.h"

using namespace mbk;

#define WARPS_PER_CTA 8
#define JOB_GRID(n) dim3(((n) + WARPS_PER_CTA - 1) / WARPS_PER_CTA), dim3(32 * WARPS_PER_CTA)
__device__ __forceinline__ int warp_job() { return blockIdx.x * WARPS_PER_CTA + (threadIdx.x >> 5); }

// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_sad(const uint8_t* __restrict__ a, int sa, const int32_t* __restrict__ a_off,
                                             const uint8_t* __restrict__ b, int sb, const int32_t* __restrict__ b_off, int blk,
                                             int n, int32_t* sad, int32_t* satd, int32_t* sad4) {
  const int j = warp_job();
  if (j >= n) return;
  const uint8_t* pa = a + a_off[j];
  const uint8_t* pb = b + b_off[j];
  const int lw = blk_lw(blk), lh = blk_lh(blk);
  if (sad) { const int v = warp_sad(pa, sa, pb, sb, lw, lh); if (lane_id() == 0) sad[j] = v; }
  if (satd) { const int v = warp_satd(pa, sa, pb, sb, lw, lh); if (lane_id() == 0) satd[j] = v; }
  if (sad4) {
    int s[4];
    warp_sad_four(pa, sa, pb, sb, lw, lh, s);
    if (lane_id() < 4) sad4[4 * j + lane_id()] = s[lane_id()];   // s[] is warp-uniform
  }
}

__global__ void __launch_bounds__(256) k_mc_luma(const uint8_t* __restrict__ src, int ss, const int32_t* __restrict__ off,
                                                 const int16_t* __restrict__ mv, int w, int h, int n, uint8_t* dst) {
  const int j = warp_job();
  if (j >= n) return;
  warp_mc_luma(src + off[j], ss, dst + 256 * j, 16, mv[2 * j], mv[2 * j + 1], w, h);
}
__global__ void __launch_bounds__(256) k_mc_chroma(const uint8_t* __restrict__ src, int ss, const int32_t* __restrict__ off,
                                                   const int16_t* __restrict__ mv, int w, int h, int n, uint8_t* dst) {
  const int j = warp_job();
  if (j >= n) return;
  warp_mc_chroma(src + off[j], ss, dst + 64 * j, 8, mv[2 * j], mv[2 * j + 1], w, h);
}
__global__ void __launch_bounds__(256) k_halfpel(int which, const uint8_t* __restrict__ src, int ss,
                                                 const int32_t* __restrict__ off, int w, int h, int n, uint8_t* dst) {
  const int j = warp_job();
  if (j >= n) return;
  warp_halfpel(which, src + off[j], ss, dst + 289 * j, 17, w, h);
}
__global__ void __launch_bounds__(256) k_pixel_avg(const uint8_t* __restrict__ a, int sa, const int32_t* __restrict__ a_off,
                                                   const uint8_t* __restrict__ b, int sb, const int32_t* __restrict__ b_off,
                                                   int w, int h, int n, uint8_t* dst) {
  const int j = warp_job();
  if (j >= n) return;
  warp_pixel_avg(dst + 256 * j, 16, a + a_off[j], sa, b + b_off[j], sb, w, h);
}

// ------------------------------------------------------------------------------------------------
// deblocking: one warp per edge job, one lane per pixel line (16 luma lines / 8 chroma lines x 2 planes)
__global__ void __launch_bounds__(256) k_deblock_luma(uint8_t* pic, const b2h264_edge_job* __restrict__ jobs, int n) {
  const int j = warp_job();
  if (j >= n) return;
  const b2h264_edge_job e = jobs[j];
  const int l = lane_id();
  if (l < 16) {
    uint8_t* p = pic + e.off + l * e.sy;
    if (e.strong) deblock_luma_eq4_line(p, e.sx, e.alpha, e.beta);
    else deblock_luma_lt4_line(p, e.sx, e.alpha, e.beta, e.tc[l >> 2]);
  }
}
__global__ void __launch_bounds__(256) k_deblock_chroma(uint8_t* cb, uint8_t* cr, const b2h264_edge_job* __restrict__ jobs,
                                                        int n) {
  const int j = warp_job();
  if (j >= n) return;
  const b2h264_edge_job e = jobs[j];
  const int l = lane_id();
  if (l < 16) {
    uint8_t* p = (l < 8 ? cb : cr) + e.off + (l & 7) * e.sy;
    if (e.strong) deblock_chroma_eq4_line(p, e.sx, e.alpha, e.beta);
    else deblock_chroma_lt4_line(p, e.sx, e.alpha, e.beta, e.tc[(l & 7) >> 1]);
  }
}

// ------------------------------------------------------------------------------------------------
// border replication: phase 1 left/right of every row, phase 2 top/bottom bands (incl. corners)
__global__ void k_expand_lr(uint8_t* pic, int stride, int w, int h, int pad) { expand_rows(pic, stride, w, h, pad); }
__global__ void k_expand_tb(uint8_t* pic, int stride, int w, int h, int pad) { expand_bands(pic, stride, w, h, pad); }

// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_me_search(const uint8_t* __restrict__ cur, int cs, const uint8_t* __restrict__ ref,
                                                   int rs, const b2h264_me_job* __restrict__ jobs, int n,
                                                   b2h264_me_result* out) {
  const int j = warp_job();
  if (j >= n) return;
  const b2h264_me_job* jb = jobs + j;
  MeIn in;
  in.enc = cur + jb->cur_off; in.enc_stride = cs;
  in.ref = ref + jb->ref_off; in.ref_stride = rs;
  in.blk = jb->blk;
  in.mvp_x = jb->mvp_x; in.mvp_y = jb->mvp_y;
  in.min_x = jb->mv_min_x; in.min_y = jb->mv_min_y; in.max_x = jb->mv_max_x; in.max_y = jb->mv_max_y;
  in.n_mvc = jb->n_mvc; in.mvc = &jb->mvc[0][0];
  in.sad_pred = jb->sad_pred;
  in.lambda = c_lambda[jb->qp];
  in.calc_satd = jb->calc_satd != 0;
  in.win = nullptr; in.win_w = in.win_h = in.win_dx = in.win_dy = 0;
  MeOut o;
  warp_me_search(in, o);
  if (lane_id() == 0) {
    b2h264_me_result r;
    r.mv_x = (int16_t)o.mv_x; r.mv_y = (int16_t)o.mv_y;
    r.sad_cost = o.sad_cost; r.satd_cost = o.satd_cost;
    r.ref_off = (int32_t)(o.ref_best - ref);
    out[j] = r;
  }
}

// ------------------------------------------------------------------------------------------------
// WelsMotionCrossSearch / LineFullSearch_c (svc_motion_estimate.cpp:568-643).  One warp per job; a LANE per candidate position:
// the positions of a line are independent (the reference walks them serially and keeps the first minimum), so every lane scores
// whole blocks at its positions with packed SADs and the warp takes the minimum of (cost << 12 | index): the smallest index wins a
// tie, like the reference's strict `<` in ascending order.
__device__ __forceinline__ uint32_t lane_block_sad(const uint8_t* a, int sa, const uint8_t* b, int sb, int w, int h) {
  uint32_t s = 0;
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x += 4) s += vsadu4(ld4u(a + y * sa + x), ld4u(b + y * sb + x));
  return s;
}
__device__ __forceinline__ void line_search(const uint8_t* enc, int cs, const uint8_t* colo, const uint8_t* plane, int rs, int w, int h, int lambda,
                                            int mvp_x, int mvp_y, int min_mv, int max_mv, bool vertical, b2h264_me_result& io) {
  const int n = max_mv - min_mv;
  if (n <= 0) return;
  const int fixed = (lambda * se_bits(vertical ? -mvp_x : -mvp_y)) & 0xffff;
  const int stride = vertical ? rs : 1;
  unsigned long long best = ~0ull;
  for (int i = lane_id(); i < n; i += 32) {
    const int mv = min_mv + i;
    const uint32_t cost = lane_block_sad(enc, cs, colo + (ptrdiff_t)mv * stride, rs, w, h) +
                          (uint32_t)(fixed + ((lambda * se_bits(mv * 4 - (vertical ? mvp_y : mvp_x))) & 0xffff));
    const unsigned long long key = ((unsigned long long)cost << 16) | (unsigned)i;
    best = key < best ? key : best;
  }
  for (int o = 16; o; o >>= 1) { const unsigned long long other = __shfl_xor_sync(MBK_FULL, best, o); best = other < best ? other : best; }
  const uint32_t cost = (uint32_t)(best >> 16);
  const int mv = min_mv + (int)(best & 0xffff);
  if (cost < io.sad_cost) {                              // UpdateMeResults (:60)
    io.mv_x = (int16_t)(vertical ? 0 : mv); io.mv_y = (int16_t)(vertical ? mv : 0);
    io.sad_cost = cost;
    io.ref_off = (int32_t)(colo + (ptrdiff_t)io.mv_y * rs + io.mv_x - plane);
  }
}
__global__ void __launch_bounds__(256) k_me_cross_search(const uint8_t* __restrict__ cur, int cs, const uint8_t* __restrict__ ref, int rs,
                                                         const b2h264_cross_job* __restrict__ jobs, int n, b2h264_me_result* io) {
  const int j = warp_job();
  if (j >= n) return;
  const b2h264_cross_job jb = jobs[j];
  b2h264_me_result r = io[j];
  const int w = 1 << blk_lw(jb.blk), h = 1 << blk_lh(jb.blk), lambda = c_lambda[jb.qp];
  const uint8_t* enc = cur + jb.cur_off;
  const uint8_t* colo = ref + jb.ref_off;
  line_search(enc, cs, colo, ref, rs, w, h, lambda, jb.mvp_x, jb.mvp_y, jb.mv_min_y, jb.mv_max_y, true, r);
  if (r.sad_cost >= jb.sad_cost_threshold) line_search(enc, cs, colo, ref, rs, w, h, lambda, jb.mvp_x, jb.mvp_y, jb.mv_min_x, jb.mv_max_x, false, r);
  if (lane_id() == 0) io[j] = r;
}

// rec_mb.cpp:298-460: explicit weighted, bi-weighted (explicit / implicit) and averaged prediction, one plane of a block per warp
__global__ void __launch_bounds__(256) k_weighted_pred(int mode, uint8_t* __restrict__ dst, const uint8_t* __restrict__ tmp, int stride,
                                                       const int32_t* __restrict__ dst_off, const int32_t* __restrict__ tmp_off,
                                                       const b2h264_weight_job* __restrict__ jobs, int w, int h, int n) {
  const int j = warp_job();
  if (j >= n) return;
  uint8_t* d = dst + dst_off[j];
  const uint8_t* t = mode ? tmp + tmp_off[j] : nullptr;
  const b2h264_weight_job jb = mode == 2 ? b2h264_weight_job{0, 0, 0, 0, 0} : jobs[j];
  for (int i = lane_id(); i < w * h; i += 32) {
    const int y = i / w, x = i - y * w;
    const int p = d[y * stride + x];
    int v;
    if (mode == 0) v = wp_single(p, jb.w1, jb.o1, jb.log2_denom);
    else if (mode == 1) v = wp_bi(p, t[y * stride + x], jb.w1, jb.w2, wp_bi_offset(jb.o1, jb.o2), jb.log2_denom);
    else v = wp_bi(p, t[y * stride + x], 1, 1, 0, 0);                   // the plain average (p + q + 1) >> 1
    d[y * stride + x] = (uint8_t)min(max(v, 0), 255);
  }
}

// ------------------------------------------------------------------------------------------------
// MC + SAD roofline unit.  One warp per macroblock.  The warp stages the reference window that all
// of the macroblock's k candidates can touch ([-R-2, 16+R+3) in both axes, R = 8 integer pels) and
// the current macroblock into shared memory once (coalesced 4-byte loads of 128-B-aligned rows from
// HBM/L2), then evaluates every candidate from shared memory: quarter-pel interpolation fused with
// the SAD accumulation, no intermediate prediction buffer.  HBM traffic per MB = cur 256 B + its
// share of the reference plane (each reference byte is fetched from DRAM once; window overlaps
// between neighbouring MBs hit L2) + 4k bytes of costs  ->  ~512 B + 4k per MB algorithmic.
#define MCS_R 8
#define MCS_WIN (16 + 2 * MCS_R + 5)       // 37 rows/cols touched
#define MCS_WSTRIDE 44                     // smem row pitch: 37 + alignment slack, multiple of 4
__global__ void __launch_bounds__(256) k_mc_sad(const uint8_t* __restrict__ cur, int cs, const uint8_t* __restrict__ ref,
                                                int rs, int mb_w, int mb_h, const int16_t* __restrict__ mv, int k,
                                                int32_t* __restrict__ cost) {
  __shared__ __align__(16) uint8_t s_win[WARPS_PER_CTA][MCS_WIN * MCS_WSTRIDE + 16];
  __shared__ __align__(16) uint8_t s_cur[WARPS_PER_CTA][256];
  const int m = warp_job();
  if (m >= mb_w * mb_h) return;
  const int wi = threadIdx.x >> 5, l = lane_id();
  const int mbx = m % mb_w, mby = m / mb_w;
  uint8_t* win = s_win[wi];
  uint8_t* cm = s_cur[wi];
  // current MB: 16 rows x 16 B = 64 words, 2 per lane
  for (int i = l; i < 64; i += 32) {
    const int row = i >> 2, c4 = (i & 3) << 2;
    *reinterpret_cast<uint32_t*>(cm + row * 16 + c4) =
        *reinterpret_cast<const uint32_t*>(cur + (size_t)(mby * 16 + row) * cs + mbx * 16 + c4);
  }
  // reference window: origin (mbx*16 - R - 2, mby*16 - R - 2); load whole aligned words covering it
  const int ox = mbx * 16 - MCS_R - 2, oy = mby * 16 - MCS_R - 2;
  const uint8_t* wsrc = ref + (ptrdiff_t)oy * rs + ox;
  const int mis = (int)(reinterpret_cast<uintptr_t>(wsrc) & 3);     // same for every row when rs % 4 == 0
  const int words = (mis + MCS_WIN + 3) >> 2;                      // <= 11
  for (int i = l; i < MCS_WIN * words; i += 32) {
    const int row = i / words, wd = i - row * words;
    *reinterpret_cast<uint32_t*>(win + row * MCS_WSTRIDE + 4 * wd) =
        *reinterpret_cast<const uint32_t*>(wsrc - mis + (ptrdiff_t)row * rs + 4 * wd);
  }
  __syncwarp();
  const uint8_t* w0 = win + mis + (MCS_R + 2) * MCS_WSTRIDE + (MCS_R + 2);   // pixel (0,0) of the co-located block
  for (int c = 0; c < k; c++) {
    const int mvx = mv[(size_t)(m * k + c) * 2], mvy = mv[(size_t)(m * k + c) * 2 + 1];
    const uint8_t* p = w0 + (mvy >> 2) * MCS_WSTRIDE + (mvx >> 2);
    const int fx = mvx & 3, fy = mvy & 3;
    int s = 0;
#pragma unroll 2
    for (int i = l; i < 256; i += 32) {
      const int y = i >> 4, x = i & 15;
      s += iabs((int)cm[i] - luma_qpel_sample(p + y * MCS_WSTRIDE + x, MCS_WSTRIDE, fx, fy));
    }
    s = warp_sum(s);
    if (l == 0) cost[(size_t)m * k + c] = s;
  }
}

// ------------------------------------------------------------------------------------------------
// Tile geometry of the TMA form of the MC + SAD unit (k_mc_sad_tma, the one launched when the planes are 16-byte aligned):
// a CTA owns a tile of 8 x 4 macroblocks (128 x 64 luma samples), one warp per macroblock column.  The CTA stages the
// current tile and the reference tile with its search halo ([-16, +144) x [-10, +75): 160 B x 85 rows) into shared memory
// (every reference byte of the tile is read from HBM once, the halo rows / columns shared with the neighbouring tiles come
// from L2), then every warp evaluates the candidates of its column of 4 macroblocks from shared memory.  Algorithmic HBM
// bytes per macroblock: 256 (cur) + 256 (ref) + 8k (vectors, costs).
#define MCT_W 8
#define MCT_H 4
#define MCT_HALO_X 16                       // left/right halo in bytes (>= R + 3, multiple of 16)
#define MCT_TOP (MCS_R + 2)                 // rows above the tile
#define MCT_ROWS (16 * MCT_H + MCS_R + 2 + MCS_R + 3)
#define MCT_PITCH (16 * MCT_W + 2 * MCT_HALO_X)

// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint2 g8(uint32_t p) {
  uint32_t s[2];
  seg_words<2>(p, s);
  return make_uint2(s[0], s[1]);
}
__device__ __forceinline__ uint2 avg8(uint2 a, uint2 b) { return make_uint2(__vavgu4(a.x, b.x), __vavgu4(a.y, b.y)); }
// eight prediction samples at quarter-sample phase (fx, fy); p = address of integer sample (x0, row) in the tile
__device__ __forceinline__ uint2 qpel8(uint32_t p, int P, int fx, int fy) {
  if (fy == 0) {
    const uint2 b = h8(p);
    return fx == 2 ? b : avg8(b, g8(p + (fx == 3)));
  }
  if (fx == 0) {
    const uint2 h = v8(p, P);
    return fy == 2 ? h : avg8(h, g8(p + (fy == 3 ? P : 0)));
  }
  if (fx == 2 && fy == 2) return c8(p, P);
  if (fx == 2) return avg8(h8(p + (fy == 3 ? P : 0)), c8(p, P));
  if (fy == 2) return avg8(v8(p + (fx == 3), P), c8(p, P));
  return avg8(h8(p + (fy == 3 ? P : 0)), v8(p + (fx == 3), P));
}

// ------------------------------------------------------------------------------------------------
// TMA form of the tiled unit (sm_90a: cp.async.bulk.tensor + mbarrier complete_tx).  ONE thread issues two bulk tensor
// copies (current tile 128 x 64, reference tile + halo 160 x 85) and every warp waits on the mbarrier: no per-thread address
// arithmetic for staging, out-of-picture parts are zero-filled by the copy engine.  (A form that staged the tile with 16-byte
// cp.async copies left the SMs issue-bound, with about a third of the warp instructions per macroblock spent on staging
// arithmetic.)
// 6 CTAs per SM (40 registers): the packed interpolation needs them; the integer path loses nothing measurable against 8
__global__ void __launch_bounds__(32 * MCT_W, 6)
k_mc_sad_tma(const __grid_constant__ CUtensorMap tm_cur, const __grid_constant__ CUtensorMap tm_ref, int mb_w, int mb_h,
             const int16_t* __restrict__ mv, int k, int32_t* __restrict__ cost) {
  __shared__ __align__(128) uint8_t t_cur[16 * MCT_H][16 * MCT_W];
  __shared__ __align__(128) uint8_t t_ref[MCT_ROWS][MCT_PITCH];
  __shared__ __align__(8) unsigned long long bar;
  const int mbx0 = blockIdx.x * MCT_W, mby0 = blockIdx.y * MCT_H;
  const uint32_t bar_a = (uint32_t)__cvta_generic_to_shared(&bar);
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    constexpr uint32_t kBytes = sizeof(t_cur) + sizeof(t_ref);
    asm volatile("{ .reg .b64 st; mbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1; }" ::"r"(bar_a), "r"(kBytes) : "memory");
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"((uint32_t)__cvta_generic_to_shared(&t_cur[0][0])), "l"(&tm_cur), "r"(mbx0 * 16), "r"(mby0 * 16), "r"(bar_a)
                 : "memory");
    // the reference map starts at the padded origin (-32, -32)
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"((uint32_t)__cvta_generic_to_shared(&t_ref[0][0])), "l"(&tm_ref), "r"(mbx0 * 16 - MCT_HALO_X + 32),
                   "r"(mby0 * 16 - MCT_TOP + 32), "r"(bar_a)
                 : "memory");
  }
  // while the copies fly: lane ty fetches the first vector of macroblock (tx, ty) of this warp's column
  const int tx = threadIdx.x >> 5, l = threadIdx.x & 31;
  const int mbx = mbx0 + tx;
  int first_mv = 0;
  if (l < MCT_H && mbx < mb_w && mby0 + l < mb_h)
    first_mv = __ldg(reinterpret_cast<const int*>(mv + (size_t)((mby0 + l) * mb_w + mbx) * k * 2));
  __syncthreads();                                   // the barrier object is initialised for everybody
  {
    uint32_t ok = 0;
    while (!ok)
      asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }"
                   : "=r"(ok) : "r"(bar_a) : "memory");
  }
  if (mbx >= mb_w) return;
  const uint32_t cur_s = (uint32_t)__cvta_generic_to_shared(&t_cur[0][16 * tx]);
  const uint32_t ref_s = (uint32_t)__cvta_generic_to_shared(&t_ref[MCT_TOP][MCT_HALO_X + 16 * tx]);
  for (int ty = 0; ty < MCT_H; ty++) {
    const int mby = mby0 + ty;
    if (mby >= mb_h) break;
    const int m = mby * mb_w + mbx;
    const int mv0 = __shfl_sync(0xffffffffu, first_mv, ty);
    for (int c = 0; c < k; c++) {
      const int mvw = c == 0 ? mv0 : __ldg(reinterpret_cast<const int*>(mv + (size_t)(m * k + c) * 2));
      const int mvx = (int16_t)(mvw & 0xffff), mvy = mvw >> 16;
      const int fx = mvx & 3, fy = mvy & 3;
      int s = 0;
      if ((fx | fy) == 0) {                    // integer vector: packed SAD on shared-space addresses, 2 words per lane
        const uint32_t pb = ref_s + (16 * ty + (mvy >> 2)) * MCT_PITCH + (mvx >> 2);
        const uint32_t sh = (pb & 3) * 8, pa = pb & ~3u;
#pragma unroll
        for (int i = 0; i < 2; i++) {
          const int y = (l >> 2) + 8 * i, x = (l & 3) << 2;
          uint32_t cw, lo, hi;
          asm volatile("ld.shared.u32 %0, [%1];" : "=r"(cw) : "r"(cur_s + (16 * ty + y) * (16 * MCT_W) + x));
          asm volatile("ld.shared.u32 %0, [%1];" : "=r"(lo) : "r"(pa + y * MCT_PITCH + x));
          asm volatile("ld.shared.u32 %0, [%1];" : "=r"(hi) : "r"(pa + y * MCT_PITCH + x + 4));
          s += __vsadu4(cw, __funnelshift_r(lo, hi, sh));
        }
      } else {                                 // fractional vector: lane = (row, 8-sample half), packed interpolation, packed SAD
        const int r = l >> 1, x0 = (l & 1) * 8;
        const uint32_t p = ref_s + (16 * ty + r + (mvy >> 2)) * MCT_PITCH + x0 + (mvx >> 2);
        const uint2 pr = qpel8(p, MCT_PITCH, fx, fy);
        uint2 cw;
        asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(cw.x), "=r"(cw.y) : "r"(cur_s + (16 * ty + r) * (16 * MCT_W) + x0));
        s = (int)(__vsadu4(cw.x, pr.x) + __vsadu4(cw.y, pr.y));
      }
      s = warp_sum(s);
      if (l == 0) cost[(size_t)m * k + c] = s;
    }
  }
}

// tensor maps of the two planes (host): uint8, rank 2, no swizzle, zero fill outside the extents
typedef CUresult (*tmap_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static tmap_encode_fn tmap_encoder() {
  static tmap_encode_fn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (tmap_encode_fn)p;
    (void)cudaGetLastError();
  }
  return fn;
}
static bool make_plane_map(CUtensorMap* tm, const uint8_t* base, uint64_t w, uint64_t h, uint64_t stride, uint32_t bw, uint32_t bh) {
  tmap_encode_fn enc = tmap_encoder();
  if (!enc) return false;
  const cuuint64_t dims[2] = {w, h}, strides[1] = {stride};
  const cuuint32_t box[2] = {bw, bh}, es[2] = {1, 1};
  return enc(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<uint8_t*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// rank-3 map over a stack of n equally sized byte planes (x, y, plane): the encoder's reference pictures of all
// streams of a batch (enc_batch.cu); `out` = 128 bytes, 64-byte aligned
int b2h264_make_tmap_planes(void* out, const void* base, uint64_t w, uint64_t h, uint64_t n, uint64_t stride_y, uint64_t stride_plane,
                            uint32_t box_w, uint32_t box_h) {
  tmap_encode_fn enc = tmap_encoder();
  if (!enc) return -1;
  const cuuint64_t dims[3] = {w, h, n}, strides[2] = {stride_y, stride_plane};
  const cuuint32_t box[3] = {box_w, box_h, 1}, es[3] = {1, 1, 1};
  return enc(reinterpret_cast<CUtensorMap*>(out), CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), dims, strides, box, es,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS ? 0 : -1;
}

// ================================================================================================
// C-ABI
// ================================================================================================
extern "C" {

int b2h264_k_sad(const uint8_t* a, int sa, const int32_t* a_off, const uint8_t* b, int sb, const int32_t* b_off, int blk,
                 int n, int32_t* sad, int32_t* satd, int32_t* sad4, void* stream) {
  if (n <= 0) return 0;
  k_sad<<<JOB_GRID(n), 0, (cudaStream_t)stream>>>(a, sa, a_off, b, sb, b_off, blk, n, sad, satd, sad4);
  return b2h264_launched();
}
int b2h264_k_mc_luma(const uint8_t* src, int ss, const int32_t* off, const int16_t* mv, int w, int h, int n, uint8_t* dst,
                     void* stream) {
  if (n <= 0) return 0;
  k_mc_luma<<<JOB_GRID(n), 0, (cudaStream_t)stream>>>(src, ss, off, mv, w, h, n, dst);
  return b2h264_launched();
}
int b2h264_k_mc_chroma(const uint8_t* src, int ss, const int32_t* off, const int16_t* mv, int w, int h, int n,
                       uint8_t* dst, void* stream) {
  if (n <= 0) return 0;
  k_mc_chroma<<<JOB_GRID(n), 0, (cudaStream_t)stream>>>(src, ss, off, mv, w, h, n, dst);
  return b2h264_launched();
}
int b2h264_k_halfpel(int which, const uint8_t* src, int ss, const int32_t* off, int w, int h, int n, uint8_t* dst,
                     void* stream) {
  if (n <= 0) return 0;
  k_halfpel<<<JOB_GRID(n), 0, (cudaStream_t)stream>>>(which, src, ss, off, w, h, n, dst);
  return b2h264_launched();
}
int b2h264_k_pixel_avg(const uint8_t* a, int sa, const int32_t* a_off, const uint8_t* b, int sb, const int32_t* b_off,
                       int w, int h, int n, uint8_t* dst, void* stream) {
  if (n <= 0) return 0;
  k_pixel_avg<<<JOB_GRID(n), 0, (cudaStream_t)stream>>>(a, sa, a_off, b, sb, b_off, w, h, n, dst);
  return b2h264_launched();
}
int b2h264_k_deblock_luma(uint8_t* pic, const b2h264_edge_job* jobs, int n, void* stream) {
  if (n <= 0) return 0;
  k_deblock_luma<<<JOB_GRID(n), 0, (cudaStream_t)stream>>>(pic, jobs, n);
  return b2h264_launched();
}
int b2h264_k_deblock_chroma(uint8_t* cb, uint8_t* cr, const b2h264_edge_job* jobs, int n, void* stream) {
  if (n <= 0) return 0;
  k_deblock_chroma<<<JOB_GRID(n), 0, (cudaStream_t)stream>>>(cb, cr, jobs, n);
  return b2h264_launched();
}
int b2h264_k_expand_plane(uint8_t* pic, int stride, int w, int h, int pad, void* stream) {
  k_expand_lr<<<dim3((h + 7) / 8), dim3(32, 8), 0, (cudaStream_t)stream>>>(pic, stride, w, h, pad);
  int rc = b2h264_launched();
  if (rc) return rc;
  k_expand_tb<<<dim3((w + 2 * pad + 127) / 128, 4), dim3(128), 0, (cudaStream_t)stream>>>(pic, stride, w, h, pad);
  return b2h264_launched();
}
int b2h264_k_me_search(const uint8_t* cur, int cs, const uint8_t* ref, int rs, const b2h264_me_job* jobs, int n,
                       b2h264_me_result* out, void* stream) {
  if (n <= 0) return 0;
  k_me_search<<<JOB_GRID(n), 0, (cudaStream_t)stream>>>(cur, cs, ref, rs, jobs, n, out);
  return b2h264_launched();
}
int b2h264_k_me_cross_search(const uint8_t* cur, int cs, const uint8_t* ref, int rs, const b2h264_cross_job* jobs, int n,
                             b2h264_me_result* io, void* stream) {
  if (n <= 0) return 0;
  k_me_cross_search<<<JOB_GRID(n), 0, (cudaStream_t)stream>>>(cur, cs, ref, rs, jobs, n, io);
  return b2h264_launched();
}
int b2h264_k_weighted_pred(int mode, uint8_t* dst, const uint8_t* tmp, int stride, const int32_t* dst_off, const int32_t* tmp_off,
                           const b2h264_weight_job* jobs, int w, int h, int n, void* stream) {
  if (n <= 0) return 0;
  if (mode < 0 || mode > 2 || w <= 0 || h <= 0 || (mode != 2 && !jobs) || (mode != 0 && (!tmp || !tmp_off))) return cudaErrorInvalidValue;
  k_weighted_pred<<<JOB_GRID(n), 0, (cudaStream_t)stream>>>(mode, dst, tmp, stride, dst_off, tmp_off, jobs, w, h, n);
  return b2h264_launched();
}
int b2h264_k_mc_sad(const uint8_t* cur, int cs, const uint8_t* ref, int rs, int mb_w, int mb_h, const int16_t* mv, int k,
                    int32_t* cost, void* stream) {
  const int n = mb_w * mb_h;
  if (n <= 0 || k <= 0) return 0;
  if ((rs & 3) || (cs & 3)) return cudaErrorInvalidValue;
  const bool aligned = !((rs | cs) & 15) && !((reinterpret_cast<uintptr_t>(cur) | reinterpret_cast<uintptr_t>(ref)) & 15);
  if (aligned) {
    // TMA: the reference plane is described from its padded origin (pad >= 32 is part of the contract)
    CUtensorMap tc, tr;
    if (make_plane_map(&tc, cur, (uint64_t)mb_w * 16, (uint64_t)mb_h * 16, (uint64_t)cs, 16 * MCT_W, 16 * MCT_H) &&
        make_plane_map(&tr, ref - (ptrdiff_t)32 * rs - 32, (uint64_t)mb_w * 16 + 64, (uint64_t)mb_h * 16 + 64, (uint64_t)rs, MCT_PITCH,
                       MCT_ROWS)) {
      k_mc_sad_tma<<<dim3((mb_w + MCT_W - 1) / MCT_W, (mb_h + MCT_H - 1) / MCT_H), 32 * MCT_W, 0, (cudaStream_t)stream>>>(
          tc, tr, mb_w, mb_h, mv, k, cost);
      return b2h264_launched();
    }
  }
  // unaligned planes, or planes no tensor map can describe: one warp per macroblock
  k_mc_sad<<<JOB_GRID(n), 0, (cudaStream_t)stream>>>(cur, cs, ref, rs, mb_w, mb_h, mv, k, cost);
  return b2h264_launched();
}

}  // extern "C"
