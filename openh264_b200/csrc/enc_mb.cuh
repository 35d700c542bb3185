// enc_mb.cuh — one macroblock, one warp: scratch layout, neighbour plumbing, intra mode decision and
// intra residual coding.  (Inter: enc_inter.cuh.)  See enc_intra.cuh for the reference map.
#pragma once
#include <stddef.h>

#include "enc_intra.cuh"
#include "enc_types.h"

namespace mbk {

#define REF_NOT_AVAIL (-2)
#define REF_NOT_IN_LIST (-1)

// per-warp mbarrier of the search-window copy (static shared memory of the encode kernel; never parked)
struct WinBar { unsigned long long bar; uint32_t phase; uint32_t pad; };

struct MbCtx {
  EncFrameParams p;
  EncFramePtrs f;
  int mbx, mby, nb;             // position, neighbour availability (NB_*)
  int qp, qp_c, lambda;
  // device only (null elsewhere): TMA descriptor of the reference luma planes of all streams of the launch
  // (x, y from the padded origin, z = stream) and this warp's mbarrier; no descriptor: the search reads the plane directly
  const void* tmap_ref;
  WinBar* wbar;
  int batch_n;                  // device: worker warps of the lock-step batch this macroblock runs in (re-alignment points of stage B)
};

struct MeState {            // the parts of SWelsME the later steps of a partition need
  int mv_x, mv_y;           // quarter-pel
  int mvp_x, mvp_y;
  uint32_t sad_cost, satd_cost;
  int satd;                 // raw SATD at the integer position (uSadPredISatd.uiSatd)
  const uint8_t* ref;       // integer-position block in the reference plane
};

// values of a P macroblock that cross a stage boundary (enc_inter.cuh: inter_stage_a/b/c); warp-uniform
struct InterState {
  int32_t is_skip, cost_luma, cost_skip_mb, p16_mvx, p16_mvy, final_type, cost16, bb;
};

// integer-search window of stage B: WIN_W x WIN_H reference luma samples around the 16x16 start point, staged by
// ONE cp.async.bulk.tensor copy per macroblock (svc_motion_estimate.cpp:222-386 runs out of it: the 16-step
// diamond never leaves +-16 samples around its start)
// The bulk tensor copy needs a 16-byte aligned start in the plane: the window is 64 wide and starts at the aligned
// address at or below (start - 16), which still covers [start - 16, start + 32).
enum { WIN_W = 64, WIN_H = 48 };

// Per-warp working set (shared memory on the device, a plain struct in the host emulation build).
// Plain data only: the device scheduler parks the LIVE PART in global memory between stages — the prefix up to
// and including the header of `out` (kParkCore) plus pred_y when the macroblock goes on to stage C;
// everything behind is dead across a stage boundary (cur_y / cur_c are re-read from the source picture).
struct alignas(128) MbScratch {
  // ---- parked prefix -------------------------------------------------------------------------------------
  RecTile tile;                 // reconstruction tile incl. neighbour samples
  InterState st;
  int16_t mvc[30][2];           // motion vector cache (6 wide: col 0 = left MB, row 0 = top MBs)
  int8_t  refc[30];             // reference index cache (REF_NOT_AVAIL -2 / REF_NOT_IN_LIST -1)
  int8_t  i4m[25];              // intra4x4 mode cache: (by+1)*5+(bx+1), -1 = unavailable
  int8_t  skip_flag[4];
  int32_t sadc[4];              // neighbour SAD costs (topleft, top, topright, left)
  int32_t sad_skip[4];
  MbInfo  info;                 // staged MbInfo
  MbInfo  nbi[4];               // neighbours' MbInfo: 0 top-left, 1 top, 2 top-right, 3 left (valid per c.nb)
  int32_t nb_sad[4];            // neighbours' persistent SAD cost (pSadCost[0])
  int32_t nb_skip_sad[4];       // neighbours' skip SAD of THIS picture (pMbSkipSad)
  alignas(16) MbOut out;        // staged output record: the header (MBOUT_HEADER_WORDS) is live, the levels are not
  // ---- not parked (except pred_y, see above) -----------------------------------------------------------------
  alignas(16) uint8_t pred_y[2][256];       // luma prediction ping-pong (pMemPredMb)
  // The next four are contiguous and double as the search window (3072 of their 3136 bytes, 128-byte aligned for
  // the bulk tensor copy): the window lives from the start of stage B's 16x16 search to the last sub-partition
  // search; pred_c / qplane / coef are first written by the refinement that follows, skip_pred is dead on that path.
  alignas(128) uint8_t pred_c[2][128];      // chroma prediction ping-pong (Cb, Cr)
  uint8_t skip_pred[384];       // P-skip prediction (pSkipMb): Y 256, Cb 64, Cr 64
  uint8_t qplane[3][18 * 32];   // fractional refinement: half-sample planes H, V, C of the partition, stride 32
                                // (pBufferInterPredMe, md.cpp:505-510)
  int16_t coef[384];            // pCoeffLevel: transform coefficients (coding order, 16 per 4x4)
  alignas(16) uint8_t cur_y[256];           // current MB, stride 16
  uint8_t cur_c[128];           // Cb 0..63, Cr 64..127, stride 8
  int16_t dc16[16];
  int32_t red[32];              // small scratch
  RefMbInfo col;                // the reference picture's record of this macroblock (P pictures; read by stage A)
  // kept in the scratch rather than on the per-thread stack: the stack of 768 threads does not fit L1 next to the
  // scratches, and these are touched all the time
  MbCtx ctx;                    // frame parameters / pointers / position of the macroblock being coded
  MeState me[9];                // 16x16, 16x8 x2, 8x16 x2, 8x8 x4 (warp-uniform; written by lane 0)
  int16_t mvcand[5][2];         // 16x16 search candidates
  int32_t win_x0, win_y0, win_ok;   // search window: origin relative to the macroblock, valid flag
  uint32_t t_last;              // phase timer (profiling builds only)
};
static_assert(offsetof(MbScratch, skip_pred) == offsetof(MbScratch, pred_c) + 256 &&
              offsetof(MbScratch, qplane) == offsetof(MbScratch, skip_pred) + 384 && offsetof(MbScratch, coef) == offsetof(MbScratch, qplane) + 3 * 18 * 32 &&
              256 + 384 + 3 * 18 * 32 + 768 >= WIN_W * WIN_H,
              "pred_c / skip_pred / qplane / coef double as the search window");
static_assert(offsetof(MbScratch, pred_c) % 128 == 0 && offsetof(MbScratch, skip_pred) % 16 == 0 && offsetof(MbScratch, pred_y) % 16 == 0 &&
              offsetof(MbScratch, out) % 16 == 0, "alignment of the parked ranges / the bulk copy destination");
// bytes of the scratch that cross every stage boundary
constexpr int kParkCore = (int)((offsetof(MbScratch, out) + 4 * MBOUT_HEADER_WORDS + 15) / 16 * 16);
constexpr int kParkExtra = 512;                               // pred_y (A or B -> C)
constexpr int kParkSlot = kParkCore + kParkExtra;
MBK_HD uint8_t* scratch_win(MbScratch& s) { return &s.pred_c[0][0]; }

// phase timing, compiled in only with -DB2H264_PHASE_STATS (profiling build): cycles since the previous mark
#if defined(B2H264_PHASE_STATS) && defined(__CUDA_ARCH__)
extern __device__ unsigned long long g_phase[32];
__device__ __forceinline__ void phase_mark(MbScratch& s, int i) {
  if ((threadIdx.x & 31) == 0) { const uint32_t t = (uint32_t)clock(); atomicAdd(&g_phase[i], (unsigned long long)(uint32_t)(t - s.t_last)); s.t_last = t; }
}
#else
MBK_HD void phase_mark(MbScratch&, int) {}
#endif


// position of 4x4 block k (coding / z order) in units of 4 pixels
MBK_HD int blk_x(int k) { return (k & 1) | ((k >> 1) & 2); }
MBK_HD int blk_y(int k) { return ((k >> 1) & 1) | ((k >> 2) & 2); }
MBK_HD int blk_raster(int k) { return blk_y(k) * 4 + blk_x(k); }

// loads from memory written by OTHER warps (previous MB row): bypass L1 on the device
MBK_HD uint8_t ld_cg_u8(const uint8_t* p) {
#ifdef __CUDA_ARCH__
  return __ldcg(p);
#else
  return *p;
#endif
}

MBK_HD uint32_t ld_cg_u32(const uint32_t* p) {
#ifdef __CUDA_ARCH__
  return __ldcg(p);
#else
  return *p;
#endif
}

// Neighbour records into the scratch.  Neighbouring macroblocks are coded by other warps, possibly on
// other SMs, during the same launch: they are fetched with L1-bypassing loads (after the scheduler's fence).
MBK_HD void mb_load_neighbors(const MbCtx& c, MbScratch& s) {
  const int mbw = c.p.mb_w, idx = c.mby * mbw + c.mbx;
  const int offs[4] = {-mbw - 1, -mbw, -mbw + 1, -1};
  const int bits[4] = {NB_TOPLEFT, NB_TOP, NB_TOPRIGHT, NB_LEFT};
  // 4 records x 30 words: one pass, all loads in flight together
  for (int i = lane_id(); i < 4 * (int)(sizeof(MbInfo) / 4); i += MBK_WS) {
    const int k = i / (int)(sizeof(MbInfo) / 4), w = i - k * (int)(sizeof(MbInfo) / 4);
    if (c.nb & bits[k])
      reinterpret_cast<uint32_t*>(&s.nbi[k])[w] = ld_cg_u32(reinterpret_cast<const uint32_t*>(c.f.mbi + idx + offs[k]) + w);
  }
  for (int k = lane_id(); k < 8; k += MBK_WS) {
    const int j = k & 3;
    const bool av = (c.nb & bits[j]) != 0;
    if (k < 4) s.nb_sad[j] = av ? (int32_t)ld_cg_u32(reinterpret_cast<const uint32_t*>(c.f.sad_cost + idx + offs[j])) : 0;
    else s.nb_skip_sad[j] = av ? (int32_t)ld_cg_u32(reinterpret_cast<const uint32_t*>(&c.f.rec_info[idx + offs[j]].skip_sad)) : 0;
  }
  warp_sync();
}

// ---- MB setup ------------------------------------------------------------------------------------
MBK_HD void mb_load_cur(const MbCtx& c, MbScratch& s) {
  const uint8_t* y = c.f.cur[0] + (size_t)(c.mby * 16) * c.p.cur_stride_y + c.mbx * 16;
  for (int i = lane_id(); i < 64; i += MBK_WS) {
    const int r = i >> 2, c4 = (i & 3) << 2;
    *reinterpret_cast<uint32_t*>(s.cur_y + r * 16 + c4) = *reinterpret_cast<const uint32_t*>(y + (size_t)r * c.p.cur_stride_y + c4);
  }
  for (int i = lane_id(); i < 32; i += MBK_WS) {
    const int pl = i >> 4, r = (i >> 1) & 7, c4 = (i & 1) << 2;
    const uint8_t* src = c.f.cur[1 + pl] + (size_t)(c.mby * 8 + r) * c.p.cur_stride_c + c.mbx * 8 + c4;
    *reinterpret_cast<uint32_t*>(s.cur_c + pl * 64 + r * 8 + c4) = *reinterpret_cast<const uint32_t*>(src);
  }
  warp_sync();
}

// neighbour samples into the tile borders, from the picture being reconstructed (written by other warps)
MBK_HD void mb_load_borders(const MbCtx& c, MbScratch& s) {
  RecTile& t = s.tile;
  const uint8_t* ry = c.f.rec[0] + (ptrdiff_t)(c.mby * 16 - 1) * c.p.rec_stride_y + c.mbx * 16;
  const uint8_t* ru = c.f.rec[1] + (ptrdiff_t)(c.mby * 8 - 1) * c.p.rec_stride_c + c.mbx * 8;
  const uint8_t* rv = c.f.rec[2] + (ptrdiff_t)(c.mby * 8 - 1) * c.p.rec_stride_c + c.mbx * 8;
  // 43 top samples (luma x = -1..23, chroma x = -1..7 twice) + 32 left samples (16 luma, 8 + 8 chroma)
  for (int i = lane_id(); i < 43 + 32; i += MBK_WS) {
    if (i < 25) {
      const int x = i - 1;
      const bool ok = x < 0 ? (c.nb & NB_TOPLEFT) : x < 16 ? (c.nb & NB_TOP) : (c.nb & NB_TOPRIGHT);
      *tile_y(t, x, -1) = ok ? ld_cg_u8(ry + x) : 0;
    } else if (i < 34) {
      const int x = i - 26;
      const bool ok = x < 0 ? (c.nb & NB_TOPLEFT) : (c.nb & NB_TOP);
      *tile_c(t.u, x, -1) = ok ? ld_cg_u8(ru + x) : 0;
    } else if (i < 43) {
      const int x = i - 35;
      const bool ok = x < 0 ? (c.nb & NB_TOPLEFT) : (c.nb & NB_TOP);
      *tile_c(t.v, x, -1) = ok ? ld_cg_u8(rv + x) : 0;
    } else {
      const int j = i - 43;
      const bool ok = (c.nb & NB_LEFT) != 0;
      if (j < 16) *tile_y(t, -1, j) = ok ? ld_cg_u8(ry + (ptrdiff_t)(j + 1) * c.p.rec_stride_y - 1) : 0;
      else if (j < 24) *tile_c(t.u, -1, j - 16) = ok ? ld_cg_u8(ru + (ptrdiff_t)(j - 15) * c.p.rec_stride_c - 1) : 0;
      else *tile_c(t.v, -1, j - 24) = ok ? ld_cg_u8(rv + (ptrdiff_t)(j - 23) * c.p.rec_stride_c - 1) : 0;
    }
  }
  warp_sync();
}

// Fused form of mb_load_neighbors + mb_load_cur + mb_load_borders: every lane first ISSUES all of its loads
// (12 independent global loads in flight: neighbour records, SAD history, the reference picture's co-located record,
// current MB, border samples) and only
// then stores to the scratch, so the macroblock pays one memory latency here instead of five serialized ones.
MBK_STAGE void mb_load_all(const MbCtx& c, MbScratch& s) {
  const int mbw = c.p.mb_w, idx = c.mby * mbw + c.mbx, l = lane_id();
  constexpr int kW = (int)(sizeof(MbInfo) / 4);
#ifdef __CUDA_ARCH__
  // neighbour k = 0..3: top-left, top, top-right, left.  Computed, not looked up: a lane-indexed local array lives in local memory
  // (12 dependent LDL per macroblock in the round-2 profile of this routine)
  auto nb_off = [&](int k) { return k == 3 ? -1 : -mbw - 1 + k; };
  auto nb_bit = [](int k) { return (int)((((uint32_t)NB_TOPLEFT) | ((uint32_t)NB_TOP << 8) | ((uint32_t)NB_TOPRIGHT << 16) | ((uint32_t)NB_LEFT << 24)) >> (8 * k)) & 0xff; };
  // ---- issue ----
  uint32_t nbw[4];
#pragma unroll
  for (int r = 0; r < 4; r++) {
    const int i = l + 32 * r, k = i / kW, w = i - k * kW;
    nbw[r] = (i < 4 * kW && (c.nb & nb_bit(k & 3))) ? ld_cg_u32(reinterpret_cast<const uint32_t*>(c.f.mbi + idx + nb_off(k & 3)) + w) : 0u;
  }
  uint32_t hist = 0;
  if (l < 8 && (c.nb & nb_bit(l & 3)))
    hist = l < 4 ? ld_cg_u32(reinterpret_cast<const uint32_t*>(c.f.sad_cost + idx + nb_off(l & 3)))
                 : ld_cg_u32(reinterpret_cast<const uint32_t*>(&c.f.rec_info[idx + nb_off(l & 3)].skip_sad));
  constexpr int kC = (int)(sizeof(RefMbInfo) / 4);
  uint32_t colw = 0;
  if (c.p.ref_is_p && l >= 8 && l < 8 + kC) colw = reinterpret_cast<const uint32_t*>(c.f.ref_info + idx)[l - 8];
  const uint8_t* cy = c.f.cur[0] + (size_t)(c.mby * 16) * c.p.cur_stride_y + c.mbx * 16;
  const uint32_t cy0 = *reinterpret_cast<const uint32_t*>(cy + (size_t)(l >> 2) * c.p.cur_stride_y + ((l & 3) << 2));
  const uint32_t cy1 = *reinterpret_cast<const uint32_t*>(cy + (size_t)(8 + (l >> 2)) * c.p.cur_stride_y + ((l & 3) << 2));
  const uint32_t cc = *reinterpret_cast<const uint32_t*>(c.f.cur[1 + (l >> 4)] + (size_t)(c.mby * 8 + ((l >> 1) & 7)) * c.p.cur_stride_c +
                                                          c.mbx * 8 + ((l & 1) << 2));
  const uint8_t* ry = c.f.rec[0] + (ptrdiff_t)(c.mby * 16 - 1) * c.p.rec_stride_y + c.mbx * 16;
  const uint8_t* ru = c.f.rec[1] + (ptrdiff_t)(c.mby * 8 - 1) * c.p.rec_stride_c + c.mbx * 8;
  const uint8_t* rv = c.f.rec[2] + (ptrdiff_t)(c.mby * 8 - 1) * c.p.rec_stride_c + c.mbx * 8;
  uint8_t tb[2] = {0, 0};
#pragma unroll
  for (int r = 0; r < 2; r++) {
    const int i = l + 32 * r;
    if (i < 25) {
      const int x = i - 1;
      if (x < 0 ? (c.nb & NB_TOPLEFT) : x < 16 ? (c.nb & NB_TOP) : (c.nb & NB_TOPRIGHT)) tb[r] = ld_cg_u8(ry + x);
    } else if (i < 34) {
      const int x = i - 26;
      if (x < 0 ? (c.nb & NB_TOPLEFT) : (c.nb & NB_TOP)) tb[r] = ld_cg_u8(ru + x);
    } else if (i < 43) {
      const int x = i - 35;
      if (x < 0 ? (c.nb & NB_TOPLEFT) : (c.nb & NB_TOP)) tb[r] = ld_cg_u8(rv + x);
    }
  }
  uint8_t lb = 0;
  if (c.nb & NB_LEFT)
    lb = l < 16 ? ld_cg_u8(ry + (ptrdiff_t)(l + 1) * c.p.rec_stride_y - 1)
                : l < 24 ? ld_cg_u8(ru + (ptrdiff_t)(l - 15) * c.p.rec_stride_c - 1) : ld_cg_u8(rv + (ptrdiff_t)(l - 23) * c.p.rec_stride_c - 1);
  // ---- commit ----
#pragma unroll
  for (int r = 0; r < 4; r++) {
    const int i = l + 32 * r;
    if (i < 4 * kW) reinterpret_cast<uint32_t*>(&s.nbi[0])[i] = nbw[r];
  }
  if (l < 4) s.nb_sad[l] = (int32_t)hist;
  else if (l < 8) s.nb_skip_sad[l - 4] = (int32_t)hist;
  else if (l < 8 + kC) reinterpret_cast<uint32_t*>(&s.col)[l - 8] = colw;
  *reinterpret_cast<uint32_t*>(s.cur_y + (l >> 2) * 16 + ((l & 3) << 2)) = cy0;
  *reinterpret_cast<uint32_t*>(s.cur_y + (8 + (l >> 2)) * 16 + ((l & 3) << 2)) = cy1;
  *reinterpret_cast<uint32_t*>(s.cur_c + (l >> 4) * 64 + ((l >> 1) & 7) * 8 + ((l & 1) << 2)) = cc;
  RecTile& t = s.tile;
#pragma unroll
  for (int r = 0; r < 2; r++) {
    const int i = l + 32 * r;
    if (i < 25) *tile_y(t, i - 1, -1) = tb[r];
    else if (i < 34) *tile_c(t.u, i - 26, -1) = tb[r];
    else if (i < 43) *tile_c(t.v, i - 35, -1) = tb[r];
  }
  if (l < 16) *tile_y(t, -1, l) = lb;
  else if (l < 24) *tile_c(t.u, -1, l - 16) = lb;
  else *tile_c(t.v, -1, l - 24) = lb;
  warp_sync();
#else
  (void)l;
  if (c.p.ref_is_p) s.col = c.f.ref_info[idx];
  else memset(&s.col, 0, sizeof(s.col));
  mb_load_neighbors(c, s);
  mb_load_cur(c, s);
  mb_load_borders(c, s);
#endif
}

// P_SKIP: the reconstruction IS the skip prediction (s.skip_pred: 16x16 luma, 8x8 Cb, 8x8 Cr, dense and word aligned) — stored
// straight from there: 3 word loads + 3 word stores per lane instead of a byte-wise copy into the tile and a byte-wise gather out of it
// (five of six macroblocks of the bench clip end this way)
MBK_HD void mb_store_recon_skip(const MbCtx& c, MbScratch& s) {
  uint8_t* ry = c.f.rec[0] + (size_t)(c.mby * 16) * c.p.rec_stride_y + c.mbx * 16;
  for (int i = lane_id(); i < 64; i += MBK_WS) {
    const int r = i >> 2, c4 = (i & 3) << 2;
    *reinterpret_cast<uint32_t*>(ry + (size_t)r * c.p.rec_stride_y + c4) = *reinterpret_cast<const uint32_t*>(s.skip_pred + r * 16 + c4);
  }
  for (int i = lane_id(); i < 32; i += MBK_WS) {
    const int pl = i >> 4, r = (i >> 1) & 7, c4 = (i & 1) << 2;
    uint8_t* dst = c.f.rec[1 + pl] + (size_t)(c.mby * 8 + r) * c.p.rec_stride_c + c.mbx * 8 + c4;
    *reinterpret_cast<uint32_t*>(dst) = *reinterpret_cast<const uint32_t*>(s.skip_pred + 256 + 64 * pl + r * 8 + c4);
  }
  warp_sync();
}

// reconstructed tile -> picture
MBK_STAGE void mb_store_recon(const MbCtx& c, MbScratch& s) {
  uint8_t* ry = c.f.rec[0] + (size_t)(c.mby * 16) * c.p.rec_stride_y + c.mbx * 16;
  for (int i = lane_id(); i < 64; i += MBK_WS) {
    const int r = i >> 2, c4 = (i & 3) << 2;
    const uint8_t* src = tile_y(s.tile, c4, r);
    *reinterpret_cast<uint32_t*>(ry + (size_t)r * c.p.rec_stride_y + c4) =
        (uint32_t)src[0] | ((uint32_t)src[1] << 8) | ((uint32_t)src[2] << 16) | ((uint32_t)src[3] << 24);
  }
  for (int i = lane_id(); i < 32; i += MBK_WS) {
    const int pl = i >> 4, r = (i >> 1) & 7, c4 = (i & 1) << 2;
    const uint8_t* src = tile_c(pl ? s.tile.v : s.tile.u, c4, r);
    uint8_t* dst = c.f.rec[1 + pl] + (size_t)(c.mby * 8 + r) * c.p.rec_stride_c + c.mbx * 8 + c4;
    *reinterpret_cast<uint32_t*>(dst) = (uint32_t)src[0] | ((uint32_t)src[1] << 8) | ((uint32_t)src[2] << 16) | ((uint32_t)src[3] << 24);
  }
  warp_sync();
}

// ---- I16x16 mode decision (WelsMdI16x16, svc_base_layer_md.cpp:365; pfMdCost = SATD) -------------
// returns the cost; s.out.i16_mode = raw mode id; the winning prediction is in s.pred_y[*best_buf]
// All modes are costed in one warp pass: lane l takes the (mode, 4x4 block) pairs l and l + 32 (mode = pair / 16) and forms
// the block's prediction in registers from the tile border; the modes are then taken in list order with strict '<', and
// only the winner's prediction is written.
MBK_HD int md_i16x16_inl(const MbCtx& c, MbScratch& s, int* best_buf) {
  int modes[4] = {0, 0, 0, 0};
  const int n = i16_modes(c.nb & 7, modes);
  const uint32_t packed = (uint32_t)modes[0] | ((uint32_t)modes[1] << 8) | ((uint32_t)modes[2] << 16) | ((uint32_t)modes[3] << 24);   // no indexed local array
  const uint8_t* org = tile_y(s.tile, 0, 0);
  // border sums of the DC modes (the samples of a missing neighbour are read but not used)
  int st = 0, sl = 0;
  for (int i = lane_id(); i < 32; i += MBK_WS) {
    if (i < 16) st += org[-TY_PITCH + i];
    else sl += org[(i - 16) * TY_PITCH - 1];
  }
  st = warp_sum(st); sl = warp_sum(sl);
  const PlaneCoef pc = n == 4 ? plane_coef(org, TY_PITCH, 16) : PlaneCoef{0, 0, 0};   // I16_P is in the list only with all three neighbours
#ifdef __CUDA_ARCH__
  int s0 = 0, s1 = 0;
#else
  int acc[4] = {0, 0, 0, 0};
#endif
  MBK_NO_UNROLL
  for (int p = lane_id(); p < 16 * n; p += MBK_WS) {
    const int mode = (int)((packed >> (8 * (p >> 4))) & 0xffu);
    const int bx = p & 3, by = (p >> 2) & 3;
    uint32_t r[4];
    if (mode == I16_V) {
      const uint32_t t = ld4u(org - TY_PITCH + 4 * bx);
#pragma unroll
      for (int y = 0; y < 4; y++) r[y] = t;
    } else if (mode == I16_H) {
#pragma unroll
      for (int y = 0; y < 4; y++) r[y] = 0x01010101u * org[(4 * by + y) * TY_PITCH - 1];
    } else if (mode == I16_P) {
#pragma unroll
      for (int y = 0; y < 4; y++) {
        const int v = pc.a + pc.b * (4 * bx - 7) + pc.c * (4 * by + y - 7) + 16;
        r[y] = clip_pack4(v >> 5, (v + pc.b) >> 5, (v + 2 * pc.b) >> 5, (v + 3 * pc.b) >> 5);
      }
    } else {
      const int dc = mode == I16_DC ? (st + sl + 16) >> 5 : mode == I16_DC_L ? (sl + 8) >> 4 : mode == I16_DC_T ? (st + 8) >> 4 : 128;
#pragma unroll
      for (int y = 0; y < 4; y++) r[y] = 0x01010101u * (uint32_t)dc;
    }
    const uint8_t* cur = s.cur_y + 64 * by + 4 * bx;
    int v;
    if (c.p.fast_mode) {                     // pfMdCost: SAD in LOW_COMPLEXITY (encoder_ext.cpp:2618)
      v = 0;
#pragma unroll
      for (int y = 0; y < 4; y++) v += (int)vsadu4(ld4u(cur + 16 * y), r[y]);
    } else {
      v = satd4x4_rows(cur, 16, r);
    }
#ifdef __CUDA_ARCH__
    if (p < 32) s0 = v; else s1 = v;
#else
    acc[p >> 4] += v;
#endif
  }
#ifdef __CUDA_ARCH__
  const int4 tot = cand_totals(s0, s1, 4);
#else
  const int4 tot = make_int4(acc[0], acc[1], acc[2], acc[3]);
#endif
  int best = 0x7fffffff, best_mode = modes[0];
  MBK_NO_UNROLL
  for (int i = 0; i < n; i++) {
    const int mode = (int)((packed >> (8 * i)) & 0xffu);
    const int cost = (i == 0 ? tot.x : i == 1 ? tot.y : i == 2 ? tot.z : tot.w) + c.lambda * ue_bits(map_i16(mode));
    if (cost < best) { best = cost; best_mode = mode; }
  }
  pred_i16(s.pred_y[0], org, TY_PITCH, best_mode);
  s.out.i16_mode = (uint8_t)map_i16(best_mode);
  *best_buf = 0;
  return best;
}
// the shared (real-call) copy of the intra paths; stages A and B of a P picture, which run it for every skip candidate and every
// macroblock they search, inline it
MBK_FN int md_i16x16(const MbCtx& c, MbScratch& s, int* best_buf) { return md_i16x16_inl(c, s, best_buf); }

// ---- intra chroma mode decision (WelsMdIntraChroma, :867) ---------------------------------------
// returns the cost; s.out.chroma_mode = the coded mode; the winning prediction (Cb, Cr at +64) is in s.pred_c[*best_buf]
// Device: all modes of both planes in one warp pass.  Lane l takes (mode l / 8, plane, 4x4 block) and forms its block's
// prediction in registers from the tile border; the eight lanes of a mode sum their costs by shuffles; the modes are then
// taken in list order with strict '<', and only the winner's lanes write their prediction (to s.pred_c[0]).
MBK_FN int md_chroma(const MbCtx& c, MbScratch& s, int* best_buf) {
  int modes[4] = {0, 0, 0, 0};
  const int n = chroma_modes(c.nb & 7, modes);
#ifdef __CUDA_ARCH__
  const uint32_t packed = (uint32_t)modes[0] | ((uint32_t)modes[1] << 8) | ((uint32_t)modes[2] << 16) | ((uint32_t)modes[3] << 24);
  const int l = lane_id(), mi = l >> 3, pl = (l >> 2) & 1, bx = l & 1, by = (l >> 1) & 1;
  const int mode = (int)((packed >> (8 * mi)) & 0xffu);           // lanes of an unused list entry cost C_DC, never taken
  const uint8_t* org = tile_c(pl ? s.tile.v : s.tile.u, 0, 0);
  uint32_t r[4];
  if (mode == C_V) {
    const uint32_t t = ld4u(org - TC_PITCH + 4 * bx);
#pragma unroll
    for (int y = 0; y < 4; y++) r[y] = t;
  } else if (mode == C_H) {
#pragma unroll
    for (int y = 0; y < 4; y++) r[y] = 0x01010101u * org[(4 * by + y) * TC_PITCH - 1];
  } else if (mode == C_P) {
    const PlaneCoef pc = plane_coef(org, TC_PITCH, 8);
#pragma unroll
    for (int y = 0; y < 4; y++) {
      const int v = pc.a + pc.b * (4 * bx - 3) + pc.c * (4 * by + y - 3) + 16;
      r[y] = clip_pack4(v >> 5, (v + pc.b) >> 5, (v + 2 * pc.b) >> 5, (v + 3 * pc.b) >> 5);
    }
  } else {                                   // the DC modes: one value per 4x4 quadrant (pred_chroma)
    const int t0 = (int)vsadu4(ld4u(org - TC_PITCH), 0u), t1 = (int)vsadu4(ld4u(org - TC_PITCH + 4), 0u);
    int l0 = 0, l1 = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) { l0 += org[i * TC_PITCH - 1]; l1 += org[(4 + i) * TC_PITCH - 1]; }
    int dc = 128;
    if (mode == C_DC) dc = bx ? (by ? (t1 + l1 + 4) >> 3 : (t1 + 2) >> 2) : (by ? (l1 + 2) >> 2 : (t0 + l0 + 4) >> 3);
    else if (mode == C_DC_L) dc = by ? (l1 + 2) >> 2 : (l0 + 2) >> 2;
    else if (mode == C_DC_T) dc = bx ? (t1 + 2) >> 2 : (t0 + 2) >> 2;
#pragma unroll
    for (int y = 0; y < 4; y++) r[y] = 0x01010101u * (uint32_t)dc;
  }
  const uint8_t* cur = s.cur_c + 64 * pl + 32 * by + 4 * bx;
  uint32_t w[4];
#pragma unroll
  for (int y = 0; y < 4; y++) w[y] = *reinterpret_cast<const uint32_t*>(cur + 8 * y);
  int v = 0;
  if (c.p.fast_mode) {                       // SAD in LOW_COMPLEXITY
#pragma unroll
    for (int y = 0; y < 4; y++) v += (int)vsadu4(w[y], r[y]);
  } else {
    v = satd4x4_words(w, r);
  }
  v += __shfl_xor_sync(MBK_FULL, v, 1);
  v += __shfl_xor_sync(MBK_FULL, v, 2);
  v += __shfl_xor_sync(MBK_FULL, v, 4);
  int best = 0x7fffffff, best_i = 0;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int cost = __shfl_sync(MBK_FULL, v, 8 * i) + c.lambda * ue_bits(map_chroma((int)((packed >> (8 * i)) & 0xffu)));
    if (i < n && cost < best) { best = cost; best_i = i; }
  }
  if (mi == best_i) {
    uint8_t* d = s.pred_c[0] + 64 * pl + 32 * by + 4 * bx;
#pragma unroll
    for (int y = 0; y < 4; y++) *reinterpret_cast<uint32_t*>(d + 8 * y) = r[y];
  }
  s.out.chroma_mode = (uint8_t)map_chroma((int)((packed >> (8 * best_i)) & 0xffu));
  *best_buf = 0;
  warp_sync();
  return best;
#else
  int best = 0x7fffffff, best_mode = modes[0], bb = 1;
  for (int i = 0; i < n; i++) {
    uint8_t* dst = s.pred_c[1 - bb];
    pred_chroma(dst, tile_c(s.tile.u, 0, 0), TC_PITCH, modes[i]);
    pred_chroma(dst + 64, tile_c(s.tile.v, 0, 0), TC_PITCH, modes[i]);
    const int cost = (c.p.fast_mode ? warp_sad(dst, 8, s.cur_c, 8, 3, 3) + warp_sad(dst + 64, 8, s.cur_c + 64, 8, 3, 3)
                                     : warp_satd(dst, 8, s.cur_c, 8, 3, 3) + warp_satd(dst + 64, 8, s.cur_c + 64, 8, 3, 3)) +
                     c.lambda * ue_bits(map_chroma(modes[i]));
    if (cost < best) { best = cost; best_mode = modes[i]; bb = 1 - bb; }
    warp_sync();
  }
  s.out.chroma_mode = (uint8_t)map_chroma(best_mode);
  *best_buf = bb;
  return best;
#endif
}

// ---- I16x16 residual coding + reconstruction (WelsEncRecI16x16Y, svc_encode_mb.cpp:54) ----------
// Device: ONE warp pass from registers.  Lane l < 16 takes block l (coding order): transform, AC quantisation and scan; the 16
// DC terms reach every lane by shuffles, so each lane runs the DC Hadamard, its quantisation, scan and inverse itself and
// picks its own block's DC; then every block is reconstructed onto the prediction (with no AC level the inverse transform of
// a DC-only block is the rounded DC the reference adds, and nothing at all without DC levels).  Lanes 16..31 mirror 0..15
// and write nothing.
MBK_FN void enc_rec_i16x16(const MbCtx& c, MbScratch& s, const uint8_t* pred) {
  const int qp = c.qp;
  const int16_t* ff = tbl_quant_ff(qp + 6);
  const int16_t* mf = tbl_quant_mf(qp);
#ifdef __CUDA_ARCH__
  const int l = lane_id(), k = l & 15, o = blk_y(k) * 64 + blk_x(k) * 4;
  uint32_t a[4], p[4];
#pragma unroll
  for (int y = 0; y < 4; y++) {
    a[y] = *reinterpret_cast<const uint32_t*>(s.cur_y + o + 16 * y);
    p[y] = *reinterpret_cast<const uint32_t*>(pred + o + 16 * y);
  }
  int16_t d[16], dcq[16], lv[16];
  dct4x4_rows(d, a, p);
#pragma unroll
  for (int j = 0; j < 16; j++) lv[j] = (int16_t)__shfl_sync(MBK_FULL, (int)d[0], j);
  hadamard_t4_dc(dcq, lv);
  quant4x4_dc(dcq, ff[0] << 1, mf[0] >> 1);
  scan4x4_dcac(lv, dcq);
  const int n_dc = nonzero_count(lv);
  auto store16 = [](int16_t* dst, const int16_t v[16]) {
    uint32_t w[8];
#pragma unroll
    for (int i = 0; i < 8; i++) w[i] = (uint32_t)(uint16_t)v[2 * i] | ((uint32_t)(uint16_t)v[2 * i + 1] << 16);
    uint4* q = reinterpret_cast<uint4*>(dst);
    q[0] = make_uint4(w[0], w[1], w[2], w[3]);
    q[1] = make_uint4(w[4], w[5], w[6], w[7]);
  };
  if (l == 0) store16(s.out.luma_dc, lv);
  quant4x4(d, ff, mf);
  scan4x4_ac(lv, d);
  const int nz = nonzero_count(lv);
  if (l < 16) { store16(s.out.luma[k], lv); s.info.nnz[blk_raster(k)] = (int8_t)nz; }
  const int nz_ac = warp_sum(l < 16 ? nz : 0);
  if (n_dc > 0) {
    if (qp < 12) { ihadamard4x4(dcq); dequant_luma_dc4x4(dcq, qp); }
    else dequant_ihadamard4x4(dcq, (uint16_t)(tbl_dequant(qp)[0] >> 2));
  }
  int16_t dc = 0;                                        // this block's DC, selected without an indexed local array
  const int rk = blk_raster(k);
#pragma unroll
  for (int i = 0; i < 16; i++) if (i == rk) dc = dcq[i];
  if (nz_ac > 0) dequant4x4(d, tbl_dequant(qp));
  else {
#pragma unroll
    for (int i = 0; i < 16; i++) d[i] = 0;
  }
  d[0] = dc;
  if (l < 16) idct4x4_rec_rows(tile_y(s.tile, 4 * blk_x(k), 4 * blk_y(k)), TY_PITCH, p, d);
  if (l == 0 && nz_ac > 0) s.info.cbp = 15;
  warp_sync();
#else
  // forward transform of the 16 blocks
  for (int k = lane_id(); k < 16; k += MBK_WS) {
    int16_t d[16];
    const int o = blk_y(k) * 4 * 16 + blk_x(k) * 4;
    dct4x4(d, s.cur_y + o, 16, pred + o, 16);
    for (int i = 0; i < 16; i++) s.coef[16 * k + i] = d[i];
  }
  warp_sync();
  // DC path: one lane (serial in the reference too)
  int16_t dcq[16];
  {
    int16_t in[16];
    for (int k = 0; k < 16; k++) in[k] = s.coef[16 * k];
    hadamard_t4_dc(dcq, in);
    quant4x4_dc(dcq, ff[0] << 1, mf[0] >> 1);
  }
  int16_t lv[16];
  scan4x4_dcac(lv, dcq);
  const int n_dc = nonzero_count(lv);
  for (int i = lane_id(); i < 16; i += MBK_WS) s.out.luma_dc[i] = lv[i];
  // AC quantisation + scan + counts
  int nz_ac = 0;
  for (int k = lane_id(); k < 16; k += MBK_WS) {
    int16_t d[16], l[16];
    for (int i = 0; i < 16; i++) d[i] = s.coef[16 * k + i];
    quant4x4(d, ff, mf);
    scan4x4_ac(l, d);
    const int nz = nonzero_count(l);
    for (int i = 0; i < 16; i++) { s.coef[16 * k + i] = d[i]; s.out.luma[k][i] = l[i]; }
    s.info.nnz[blk_raster(k)] = (int8_t)nz;
    nz_ac += nz;
  }
  nz_ac = warp_sum(nz_ac);
  if (n_dc > 0) {
    if (qp < 12) { ihadamard4x4(dcq); dequant_luma_dc4x4(dcq, qp); }
    else dequant_ihadamard4x4(dcq, (uint16_t)(tbl_dequant(qp)[0] >> 2));
  }
  warp_sync();
  uint8_t* rec = tile_y(s.tile, 0, 0);
  if (nz_ac > 0) {
    s.info.cbp = 15;
    for (int k = lane_id(); k < 16; k += MBK_WS) {
      int16_t d[16];
      for (int i = 0; i < 16; i++) d[i] = s.coef[16 * k + i];
      dequant4x4(d, tbl_dequant(qp));
      d[0] = dcq[blk_raster(k)];
      const int o = blk_y(k) * 4, ox = blk_x(k) * 4;
      idct4x4_rec(rec + o * TY_PITCH + ox, TY_PITCH, pred + o * 16 + ox, 16, d);
    }
  } else if (n_dc > 0) {
    for (int i = lane_id(); i < 256; i += MBK_WS) {
      const int y = i >> 4, x = i & 15;
      rec[y * TY_PITCH + x] = (uint8_t)clip255(pred[i] + ((dcq[(y & 12) + (x >> 2)] + 32) >> 6));
    }
  } else {
    for (int i = lane_id(); i < 256; i += MBK_WS) rec[(i >> 4) * TY_PITCH + (i & 15)] = pred[i];
  }
  warp_sync();
#endif
}

// Host build: how the I4x4 try of the intra tail ended, so that tests can show which ends their cases reach.
//   I4_END_BREAK     the running cost reached the limit before the 16th block
//   I4_END_COMPLETE  all 16 blocks were coded
//   I4_END_WON       ... and the I4x4 cost beat the I16x16 cost
enum { I4_END_BREAK = 0, I4_END_COMPLETE, I4_END_WON, I4_END_OUTCOMES };
inline uint64_t g_i4_end[I4_END_OUTCOMES];

// ---- I4x4 mode decision with in-loop coding (WelsMdI4x4 :418 + WelsEncRecI4x4Y svc_encode_mb.cpp:139)
// returns the I4x4 cost; reconstructs into the tile as it goes; stops early once the running cost
// reaches `cost_limit` (the I16x16 / inter cost), exactly like the reference.
// Device: lane j costs candidate j with its prediction formed in registers; the lane that holds the winner codes the block
// from those registers (transform, quantisation, scan, inverse) and writes the reconstruction into the tile, so the next
// block waits on one warp_sync only.  The host build re-predicts the winner and codes it through the serial helpers.
MBK_FN int md_enc_i4x4(const MbCtx& c, MbScratch& s, int cost_limit) {
  const int qp = c.qp;
  const int16_t* ff = tbl_quant_ff(qp + 6);
  const int16_t* mf = tbl_quant_mf(qp);
  const int lam4 = c.lambda << 2, lam1 = c.lambda;
  int total = 0;
  MBK_NO_UNROLL
  for (int k = 0; k < 16; k++) {
    const int bx = blk_x(k), by = blk_y(k);
    uint8_t* org = tile_y(s.tile, bx * 4, by * 4);
    const uint8_t* cur = s.cur_y + by * 4 * 16 + bx * 4;
    // predicted mode (PredIntra4x4Mode :246)
    const int lm = s.i4m[(by + 1) * 5 + bx], tm = s.i4m[by * 5 + bx + 1];
    const int pm = (lm == -1 || tm == -1) ? 2 : (lm < tm ? lm : tm);
    int best_cost, best_mode;
#ifdef __CUDA_ARCH__
    const int l = lane_id();
    const uint64_t list = i4_modes_packed(i4_avail(c.nb, k));
    const int n = (int)(list >> 60);
    const int mj = (int)((list >> (4 * (l & 15))) & 15);     // lane l < n: candidate l
    uint32_t w[4], r[4] = {0u, 0u, 0u, 0u};                  // source rows, prediction rows
#pragma unroll
    for (int y = 0; y < 4; y++) w[y] = *reinterpret_cast<const uint32_t*>(cur + 16 * y);
    int key = 0x7fffffff;
    if (l < n) {
      uint8_t p[16];
      pred_i4_inl(p, org, TY_PITCH, mj);
#pragma unroll
      for (int y = 0; y < 4; y++)
        r[y] = (uint32_t)p[4 * y] | ((uint32_t)p[4 * y + 1] << 8) | ((uint32_t)p[4 * y + 2] << 16) | ((uint32_t)p[4 * y + 3] << 24);
      int dist;
      if (c.p.fast_mode) {                   // LOW_COMPLEXITY: SAD
        dist = 0;
#pragma unroll
        for (int y = 0; y < 4; y++) dist += (int)vsadu4(w[y], r[y]);
      } else {
        dist = satd4x4_words(w, r);
      }
      const int cost = dist + (pm == map_i4(mj) ? lam1 : lam4);
      if (c.p.fast_mode) s.red[mj] = cost;
      key = (cost << 4) | l;
    }
    if (!c.p.fast_mode) {
      // ties resolve to the earliest list entry like the serial '<'
      key = warp_min(key);
      best_cost = key >> 4; best_mode = (int)((list >> (4 * (key & 15))) & 15);
    } else {
      auto mode_at = [&](int j) { return (int)((list >> (4 * j)) & 15); };
#else
    int modes[9];
    const int n = i4_modes(i4_avail(c.nb, k), modes);
    if (!c.p.fast_mode) {
      // all candidates in parallel (one lane each); ties resolve to the earliest list entry like the serial '<'
      int key = 0x7fffffff;
      for (int j = lane_id(); j < n; j += MBK_WS) {
        uint8_t p[16];
        pred_i4(p, org, TY_PITCH, modes[j]);
        const int cost = satd4x4_pred(p, cur, 16) + (pm == map_i4(modes[j]) ? lam1 : lam4);
        const int kj = (cost << 4) | j;
        if (kj < key) key = kj;
      }
      key = warp_min(key);
      best_cost = key >> 4; best_mode = modes[key & 15];
    } else {
      // LOW_COMPLEXITY (WelsMdI4x4Fast, svc_base_layer_md.cpp:548): SAD costs and a pruned candidate tree.  Every
      // candidate's cost is computed (one lane each, into s.red); the tree is then walked on the costs — a cost is a
      // pure function of the mode, so evaluating more modes than the reference cannot change which one it picks.
      for (int j = lane_id(); j < n; j += MBK_WS) {
        uint8_t p[16];
        pred_i4(p, org, TY_PITCH, modes[j]);
        int sad = 0;
        for (int q = 0; q < 16; q++) sad += iabs((int)p[q] - (int)cur[(q >> 2) * 16 + (q & 3)]);
        s.red[modes[j]] = sad + (pm == map_i4(modes[j]) ? lam1 : lam4);
      }
      auto mode_at = [&](int j) { return modes[j]; };
#endif
      warp_sync();
      const int32_t* cst = s.red;
      if (n == 9 || n == 7) {
        best_mode = I4_DC; best_cost = cst[I4_DC];
        const int cH = cst[I4_H], cV = cst[I4_V];
        if (cH < best_cost) { best_cost = cH; best_mode = I4_H; }
        if (cV < best_cost) { best_cost = cV; best_mode = I4_V; }
#define I4_TRY(m) do { if (cst[m] < best_cost) { best_cost = cst[m]; best_mode = (m); } } while (0)
        if (cV < cH) {
          if (n == 9) {
            I4_TRY(I4_VR); I4_TRY(I4_VL);
            if (cst[I4_VR] < cV || cst[I4_VL] < cV) {               // vertical is not the (fake) best: go on
              if (cst[I4_VR] < cst[I4_VL]) I4_TRY(I4_DDR); else I4_TRY(I4_DDL);
            }
          } else { I4_TRY(I4_DDR); I4_TRY(I4_VR); }
        } else {
          I4_TRY(I4_HD); I4_TRY(I4_HU);
          if (cst[I4_HD] < cH || cst[I4_HU] < cH) {
            if (cst[I4_HD] < cst[I4_HU]) I4_TRY(I4_DDR);
            else if (n == 9) I4_TRY(I4_DDL);
          }
        }
#undef I4_TRY
      } else {
        best_cost = 0x7fffffff; best_mode = mode_at(0);
        for (int j = 0; j < n; j++) if (cst[mode_at(j)] < best_cost) { best_cost = cst[mode_at(j)]; best_mode = mode_at(j); }
      }
      warp_sync();
    }
    total += best_cost;
    if (total >= cost_limit) {
#ifndef __CUDA_ARCH__
      g_i4_end[I4_END_BREAK]++;
#endif
      break;
    }
#ifndef __CUDA_ARCH__
    if (k == 15) g_i4_end[I4_END_COMPLETE]++;
#endif
    const int fm = map_i4(best_mode);
    s.out.prev_i4_flag[k] = (int8_t)(pm == fm);
    s.out.rem_i4_mode[k] = (int8_t)(fm < pm ? fm : fm - 1);
    s.i4m[(by + 1) * 5 + bx + 1] = (int8_t)fm;
    s.info.i4_mode[by * 4 + bx] = (int8_t)fm;
#ifdef __CUDA_ARCH__
    // the lane of the winning candidate codes the block from its registers (modes of a list are distinct)
    if (l < n && mj == best_mode) {
      int16_t d[16], lv[16];
      dct4x4_rows(d, w, r);
      quant4x4(d, ff, mf);
      scan4x4_dcac(lv, d);
      const int nz = nonzero_count(lv);
      uint32_t q[8];
#pragma unroll
      for (int i = 0; i < 8; i++) q[i] = (uint32_t)(uint16_t)lv[2 * i] | ((uint32_t)(uint16_t)lv[2 * i + 1] << 16);
      uint4* ol = reinterpret_cast<uint4*>(s.out.luma[k]);
      ol[0] = make_uint4(q[0], q[1], q[2], q[3]);
      ol[1] = make_uint4(q[4], q[5], q[6], q[7]);
      s.info.nnz[by * 4 + bx] = (int8_t)nz;
      if (nz > 0) s.info.cbp |= (uint8_t)(1 << (k >> 2));
      dequant4x4(d, tbl_dequant(qp));                    // all zero without levels: the reconstruction is the prediction
      idct4x4_rec_rows(org, TY_PITCH, r, d);
    }
#else
    // encode + reconstruct this block (single lane: 16 samples)
    if (lane_id() == 0) {
      uint8_t p[16];
      int16_t d[16], l[16];
      pred_i4(p, org, TY_PITCH, best_mode);
      dct4x4(d, cur, 16, p, 4);
      quant4x4(d, ff, mf);
      scan4x4_dcac(l, d);
      const int nz = nonzero_count(l);
      for (int i = 0; i < 16; i++) s.out.luma[k][i] = l[i];
      s.info.nnz[by * 4 + bx] = (int8_t)nz;
      if (nz > 0) {
        s.info.cbp |= (uint8_t)(1 << (k >> 2));
        dequant4x4(d, tbl_dequant(qp));
        idct4x4_rec(org, TY_PITCH, p, 4, d);
      } else {
        for (int i = 0; i < 16; i++) org[(i >> 2) * TY_PITCH + (i & 3)] = p[i];
      }
    }
#endif
    warp_sync();
  }
  return total + 24 * c.lambda;       // 4*6*lambda (JVT SATD0)
}

// ---- host build: the serial chroma residual, the specification of residual_pass's chroma lanes (enc_inter.cuh) ----
#ifndef __CUDA_ARCH__
// ---- chroma residual of one plane (WelsEncRecUV, svc_encode_mb.cpp:244); res = s.coef + 256 + 64*uv
MBK_FN void enc_rec_uv(const MbCtx& c, MbScratch& s, int uv, bool inter) {
  int16_t* res = s.coef + 256 + 64 * uv;
  const int qpc = c.qp_c;
  const int16_t* ff = tbl_quant_ff(qpc + (inter ? 0 : 6));
  const int16_t* mf = tbl_quant_mf(qpc);
  // chroma DC 2x2 (all lanes compute the same 4 values)
  const int16_t dcin[4] = {res[0], res[16], res[32], res[48]};
  int16_t dc[4];
  const int nz_dc = hadamard_quant2x2(dcin, (int16_t)(ff[0] << 1), (int16_t)(mf[0] >> 1), dc);
  warp_sync();
  // AC of the 4 blocks: one lane each (the DC position is quantised as 0, as after pfQuantizationHadamard2x2)
  for (int j = lane_id(); j < 4; j += MBK_WS) {
    int16_t d[16], l[16];
    for (int i = 0; i < 16; i++) d[i] = res[16 * j + i];
    d[0] = 0;
    const int16_t mx = quant4x4_max(d, ff, mf);
    if (mx == 0) { for (int i = 0; i < 16; i++) l[i] = 0; }
    else scan4x4_ac(l, d);
    for (int i = 0; i < 16; i++) { res[16 * j + i] = d[i]; s.out.chroma_ac[4 * uv + j][i] = l[i]; }
    s.red[j] = mx;
    s.red[4 + j] = mx == 0 ? 0 : single_ctr4x4(l);
    s.red[8 + j] = nonzero_count(l);
  }
  if (lane_id() == 0) for (int i = 0; i < 4; i++) s.out.chroma_dc[uv][i] = dc[i];
  warp_sync();
  // JVT-O079 decision in the reference's block order (uniform)
  int ctr = 0;
  for (int j = 0; j < 4; j++) {
    const int mx = s.red[j];
    if (mx == 0) continue;
    if (inter) {
      if (mx > 1) ctr += 9;
      else if (ctr < 7) ctr += s.red[4 + j];
    } else ctr = 0x7fffffff;
  }
  if (ctr < 7) {
    for (int i = lane_id(); i < 64; i += MBK_WS) res[i] = 0;
    if (lane_id() == 0) for (int j = 0; j < 4; j++) s.info.nnz[16 + 4 * uv + j] = 0;
  } else {
    for (int j = lane_id(); j < 4; j += MBK_WS) {
      s.info.nnz[16 + 4 * uv + j] = (int8_t)s.red[8 + j];
      int16_t d[16];
      for (int i = 0; i < 16; i++) d[i] = res[16 * j + i];
      dequant4x4(d, tbl_dequant(qpc));
      for (int i = 0; i < 16; i++) res[16 * j + i] = d[i];
    }
    if (lane_id() == 0) s.info.cbp = (uint8_t)((s.info.cbp & 0x0F) | 0x20);
  }
  warp_sync();
  if (nz_dc > 0 && lane_id() == 0) {
    dequant_ihadamard2x2_dc(dc, tbl_dequant(qpc)[0]);
    if (2 != (s.info.cbp >> 4)) s.info.cbp |= 0x10;
    res[0] = dc[0]; res[16] = dc[1]; res[32] = dc[2]; res[48] = dc[3];
  }
  warp_sync();
}

// chroma transform of both planes against prediction `pred` (Cb 0..63, Cr 64..127)
MBK_FN void dct_chroma(MbScratch& s, const uint8_t* pred) {
  for (int t = lane_id(); t < 8; t += MBK_WS) {
    const int uv = t >> 2, j = t & 3, ox = (j & 1) * 4, oy = (j >> 1) * 4;
    int16_t d[16];
    dct4x4(d, s.cur_c + 64 * uv + oy * 8 + ox, 8, pred + 64 * uv + oy * 8 + ox, 8);
    for (int i = 0; i < 16; i++) s.coef[256 + 64 * uv + 16 * j + i] = d[i];
  }
  warp_sync();
}
#endif
// chroma reconstruction of both planes into the tile: pred + IDCT(coef)
MBK_FN void rec_chroma(MbScratch& s, const uint8_t* pred) {
  for (int t = lane_id(); t < 8; t += MBK_WS) {
    const int uv = t >> 2, j = t & 3, ox = (j & 1) * 4, oy = (j >> 1) * 4;
    int16_t d[16];
    for (int i = 0; i < 16; i++) d[i] = s.coef[256 + 64 * uv + 16 * j + i];
    idct4x4_rec(tile_c(uv ? s.tile.v : s.tile.u, ox, oy), TC_PITCH, pred + 64 * uv + oy * 8 + ox, 8, d);
  }
  warp_sync();
}

// ---- intra4x4 mode cache from the neighbours (FillNeighborCacheIntra, md.cpp:51) -----------------
MBK_FN void fill_i4_cache(const MbCtx& c, MbScratch& s) {
  if (lane_id() == 0) {
    for (int i = 0; i < 25; i++) s.i4m[i] = -1;
    if (c.nb & NB_LEFT) {
      const MbInfo* l = &s.nbi[3];
      for (int y = 0; y < 4; y++) s.i4m[(y + 1) * 5] = l->mb_type == MBT_I4x4 ? l->i4_mode[y * 4 + 3] : 2;
    }
    if (c.nb & NB_TOP) {
      const MbInfo* t = &s.nbi[1];
      for (int x = 0; x < 4; x++) s.i4m[x + 1] = t->mb_type == MBT_I4x4 ? t->i4_mode[12 + x] : 2;
    }
  }
  warp_sync();
}

// LOW_COMPLEXITY tries I4x4 only on textured macroblocks (WelsMdIntraFinePartitionVaa :942, MdIntraAnalysisVaaInfo /
// AnalysisVaaInfoIntra_c md.cpp:435-500): variance of the sixteen 4x4 block means of the SOURCE macroblock >= 150
MBK_FN bool intra_try_i4x4(const MbCtx& c, MbScratch& s) {
  if (!c.p.fast_mode) return true;
  int sum = 0, sqr = 0;
  for (int k = lane_id(); k < 16; k += MBK_WS) {
    const uint8_t* p = s.cur_y + (k >> 2) * 4 * 16 + (k & 3) * 4;
    int a = 0;
    for (int q = 0; q < 16; q++) a += p[(q >> 2) * 16 + (q & 3)];
    a >>= 4;
    sum += a; sqr += a * a;
  }
  sum = warp_sum(sum); sqr = warp_sum(sqr);
  return sqr - ((sum * sum) >> 4) >= 150;                // INTRA_VARIANCE_SAD_THRESHOLD
}

// publishes MbInfo / RefMbInfo / MbOut of a finished macroblock
MBK_STAGE void mb_publish(const MbCtx& c, MbScratch& s) {
  const int idx = c.mby * c.p.mb_w + c.mbx;
  if (lane_id() == 0) {
    s.info.qp = (uint8_t)c.qp; s.info.qp_c = (uint8_t)c.qp_c;
    s.out.mb_type = s.info.mb_type; s.out.cbp = s.info.cbp; s.out.qp = (uint8_t)c.qp;
    for (int i = 0; i < 24; i++) s.out.nnz[i] = s.info.nnz[i];
  }
  warp_sync();
  // word copies
  const uint32_t* si = reinterpret_cast<const uint32_t*>(&s.info);
  uint32_t* di = reinterpret_cast<uint32_t*>(c.f.mbi + idx);
  for (int i = lane_id(); i < (int)(sizeof(MbInfo) / 4); i += MBK_WS) di[i] = si[i];
  const uint32_t* so = reinterpret_cast<const uint32_t*>(&s.out);
  uint32_t* dout = reinterpret_cast<uint32_t*>(c.f.out + idx);
  const int n_out = s.info.mb_type == MBT_PSKIP ? MBOUT_HEADER_WORDS : (int)(sizeof(MbOut) / 4);
  for (int i = lane_id(); i < n_out; i += MBK_WS) dout[i] = so[i];
  warp_sync();
}

}  // namespace mbk
