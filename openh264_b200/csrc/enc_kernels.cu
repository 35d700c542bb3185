// enc_kernels.cu — frame-level CUDA kernels of the encoder path (sm_90a):
//   k_pad_source     source I420 -> MB-aligned current picture
//   k_encode_mbs     macroblock mode decision + coding + reconstruction, ONE WARP PER MACROBLOCK; the MBs of
//                    all streams of the batch are scheduled by dependency (ready list, persistent warps)
//   k_deblock_mbs    in-loop deblocking, same scheduling
//   k_expand_*       border replication of the new reference picture (ExpandReferencingPicture)
// Why a wavefront: MB(x,y) needs the FINAL state of (x-1,y), (x,y-1), (x+1,y-1) — motion-vector / SAD
// predictors, intra neighbours, skip context (SURVEY.md §7 hard part 1); bit-exactness forbids breaking
// that chain, so parallelism comes from rows (2-MB lag) x independent streams of the batch.
#include <cuda.h>
#include <type_traits>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>

#include "b2h264_internal.h"
#define B2H264_WITH_INTER 1
#include "enc_deblock.cuh"
#include "enc_frame.cuh"
#include "dec_mb.cuh"
#include "enc_launch.h"

using namespace mbk;

namespace mbk {
__constant__ uint8_t c_alpha[52];
__constant__ uint8_t c_beta[52];
__constant__ uint8_t c_tc0[52][3];
}  // namespace mbk

#define DEC_WPC 24         // warps per CTA of the decoder's macroblock kernel (one CTA per SM at 80 registers)
#ifndef ENC_WPC
#define ENC_WPC 23         // WORKER warps per CTA of the encode kernel; one more warp schedules (24 x 32 x 80 registers = one CTA per SM)
#endif

__device__ __forceinline__ int ld_volatile(const int* p) { return *reinterpret_cast<const volatile int*>(p); }

// ---- source padding (CWelsPreProcess::Padding, wels_preprocess.cpp:1250) --------------------------------
__global__ void k_pad_source(const StreamFrame* __restrict__ sf, const uint8_t* const* __restrict__ src, int w, int h) {
  const StreamFrame& F = sf[blockIdx.z];
  const uint8_t* yuv = src[blockIdx.z];
  const int W = F.p.mb_w * 16, H = F.p.mb_h * 16;
  const int x = (blockIdx.x * blockDim.x + threadIdx.x) * 4, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= W || y >= H) return;
  uchar4 v = make_uchar4(0, 0, 0, 0);
  if (y < h) {
    const uint8_t* r = yuv + (size_t)y * w;
    if (x + 3 < w) v = *reinterpret_cast<const uchar4*>(r + x);          // w % 4 == 0 is required at create time
  }
  *reinterpret_cast<uchar4*>(const_cast<uint8_t*>(F.f.cur[0]) + (size_t)y * F.p.cur_stride_y + x) = v;
  if (y < H / 2 && x < W / 2) {
    const int cw = w / 2, ch = h / 2;
    for (int pl = 0; pl < 2; pl++) {
      uchar4 c = make_uchar4(0x80, 0x80, 0x80, 0x80);
      const uint8_t* p = yuv + (size_t)w * h + (size_t)pl * cw * ch + (size_t)y * cw;
      if (y < ch) {
        uint8_t t[4];
        for (int i = 0; i < 4; i++) t[i] = (x + i < cw) ? p[x + i] : 0x80;
        c = make_uchar4(t[0], t[1], t[2], t[3]);
      }
      *reinterpret_cast<uchar4*>(const_cast<uint8_t*>(F.f.cur[1 + pl]) + (size_t)y * F.p.cur_stride_c + x) = c;
    }
  }
}

// ---- VAA statistics of LOW_COMPLEXITY (VAACalcSad_c, codec/processing/src/vaacalc/vaacalcfuncs.cpp:254) -------------------------
// SAD of the four 8x8 blocks of every macroblock between the current and the PREVIOUS source picture (both MB-aligned,
// stride 16 * mb_w): one warp per macroblock, lane = (row, 8-pixel half), two packed SADs per lane, three shuffles.
// out[(stream, mb) * 4 + k], k = 0 top-left, 1 top-right, 2 bottom-left, 3 bottom-right.  Pure streaming: 512 B read, 16 B written per MB.
__global__ void __launch_bounds__(256) k_vaa_sad8x8(const StreamFrame* __restrict__ sf, int n_mb) {
  const int lane = threadIdx.x & 31, mb = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (mb >= n_mb) return;
  const StreamFrame& F = sf[blockIdx.y];
  if (F.f.vaa_sad8x8 == nullptr || F.f.prev_luma == nullptr) return;
  const int st = F.p.cur_stride_y, mbx = mb % F.p.mb_w, mby = mb / F.p.mb_w;
  const size_t off = (size_t)(mby * 16 + (lane >> 1)) * st + mbx * 16 + (lane & 1) * 8;
  const uint2 a = *reinterpret_cast<const uint2*>(F.f.cur[0] + off), b = *reinterpret_cast<const uint2*>(F.f.prev_luma + off);
  int v = (int)(__vsadu4(a.x, b.x) + __vsadu4(a.y, b.y));
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  v += __shfl_xor_sync(0xffffffffu, v, 8);                 // lanes 0, 1, 16, 17 hold the four block sums
  if ((lane & 14) == 0) const_cast<int32_t*>(F.f.vaa_sad8x8)[(size_t)mb * 4 + (lane >> 4) * 2 + (lane & 1)] = v;
}

// ---- dependency-driven macroblock scheduling -------------------------------------------------------------
// MB(x,y) may start when (x-1,y) and (x+1,y-1) [(x,y-1) on the last column] are final; those two imply the
// top and top-left neighbours.  Every finished MB notifies its right neighbour and its bottom-left
// neighbour; the second notification pushes the MB onto a global ready list.  Persistent warps pop the
// list: no warp ever holds an SM slot while a row it depends on is still busy (a row-per-warp wavefront
// spent most of its issue slots spinning).
struct Sched {
  int* dep;        // per (stream, mb): notifications received so far
  int* queue;      // ready list, capacity = n_streams * n_mb, -1 = not yet pushed
  int* head;       // next entry to pop
  int* tail;       // next free entry
};

__device__ __forceinline__ void sched_push(const Sched& q, int id) {
  const int slot = atomicAdd(q.tail, 1);
  *reinterpret_cast<volatile int*>(q.queue + slot) = id;
}
__device__ __forceinline__ void sched_notify(const Sched& q, int id, int need) {
  if (atomicAdd(q.dep + id, 1) + 1 == need) sched_push(q, id);
}

template <class Body>
__device__ __forceinline__ void run_mbs(const StreamFrame* sf, int n_streams, const Sched q, Body body) {
  const int lane = threadIdx.x & 31;
  const int mb_w = sf[0].p.mb_w, mb_h = sf[0].p.mb_h, n_mb = mb_w * mb_h, total = n_streams * n_mb;
  for (;;) {
    int id = 0;
    if (lane == 0) {
      const int t = atomicAdd(q.head, 1);
      id = -1;
      if (t < total) {
        while ((id = ld_volatile(q.queue + t)) < 0) __nanosleep(100);
      }
    }
    id = __shfl_sync(MBK_FULL, id, 0);
    if (id < 0) break;
    __threadfence();
    const int si = id / n_mb, mb = id - si * n_mb, y = mb / mb_w, x = mb - y * mb_w;
    body(sf[si], x, y);
    __threadfence();
    __syncwarp();
    if (lane == 0) {
      if (x + 1 < mb_w) sched_notify(q, id + 1, 1 + (y > 0));                    // right neighbour: we are its left
      if (y + 1 < mb_h) {
        if (x > 0) sched_notify(q, id + mb_w - 1, 1 + (x - 1 > 0));              // bottom-left: we are its top-right
        if (x == mb_w - 1) sched_notify(q, id + mb_w, 1 + (x > 0));              // last column: we are its top
      }
    }
  }
}

// ---- staged lock-step scheduler of the encode kernel -------------------------------------------------------------
// The SM's instruction cache holds ~32 KB; the code one macroblock walks through is several times that.  Warps
// that execute different code thrash it, warps that start the same code together
// share every fill.  So (1) the CTA claims up to ENC_WPC tasks AT ONCE, its warps start them together and meet
// again before the next batch, and (2) a batch is homogeneous: a macroblock is coded in stages (enc_inter.cuh:
// A skip test, B motion search + inter coding, C intra branch; I = a whole IDR-picture macroblock), every stage has
// its own ready list, and a batch comes from ONE list.  A macroblock that needs another stage parks its scratch in
// global memory (one slot per stream and macroblock ROW: at most one macroblock of a row is in flight) and is
// pushed onto the next stage's list; whichever CTA takes it continues from the parked scratch.
enum { NQ = MBS_COUNT - 1 };                       // ready lists, index = stage - 1
struct EncSched {
  int* dep;          // per (stream, mb): notifications received so far
  int* queue;        // NQ ready lists of capacity `total` each, -1 = slot not yet written
  int* ctl;          // one 128-byte line per ready list: [32 k] head, [32 k + 1] tail; line NQ: [32 NQ] macroblocks finished
  uint4* stash;      // parked scratches
  int* rowprog;      // per (stream, macroblock row): macroblocks finished (rows complete left to right) — the deblocking kernel that
                     // runs beside this one follows it
};
// The control words are spread over NQ + 1 lines (different L2 slices): every finished macroblock, every push and every
// scheduler look / claim of one CTA per SM used to hit ONE line, and the queueing there slowed the workers' own atomics.
__device__ __forceinline__ int* ctl_head(const EncSched& q, int k) { return q.ctl + 32 * k; }
__device__ __forceinline__ int* ctl_tail(const EncSched& q, int k) { return q.ctl + 32 * k + 1; }
__device__ __forceinline__ int* ctl_done(const EncSched& q) { return q.ctl + 32 * NQ; }
constexpr int kCtlInts = 32 * (NQ + 1);
// Only the live part of a scratch is parked (enc_mb.cuh: kParkCore + skip_pred or pred_y): slot = kParkSlot bytes
constexpr int kStashU4 = kParkSlot / 16, kCoreU4 = kParkCore / 16;
static_assert(kParkSlot % 16 == 0 && kParkCore % 16 == 0, "parked ranges are copied as uint4");
// second parked range of a macroblock that continues at `stage`: offset (uint4 units) and length
__device__ __forceinline__ void park_extra(int stage, int* off, int* n) {
  if (stage == MBS_BSKIP) { *off = (int)(offsetof(MbScratch, skip_pred) / 16); *n = 384 / 16; }
  else if (stage == MBS_C) { *off = (int)(offsetof(MbScratch, pred_y) / 16); *n = 512 / 16; }
  else { *off = 0; *n = 0; }
}

__device__ __forceinline__ void esched_push(const EncSched& q, int total, int stage, int id) {
  const int k = stage - 1;
  const int slot = atomicAdd(ctl_tail(q, k), 1);
  *reinterpret_cast<volatile int*>(q.queue + (size_t)k * total + slot) = id;
}

// optional batch statistics (debug, B2H264_ENC_STATS): per ready list [batches, tasks, batch cycles]; [NQ] = leader wait cycles
__device__ unsigned long long g_batch_stats[NQ + 1][3];
__device__ unsigned long long g_task_wall[NQ][2];                    // per list: cycles from the batch barrier to the end of run_task, tasks
__device__ unsigned long long g_fill_stats[NQ][ENC_WPC + 1][2];      // per list and batch fill: [batches, cycles]
extern "C" int b2h264_debug_task_wall(unsigned long long* out, int reset) {
  cudaError_t e = cudaMemcpyFromSymbol(out, g_task_wall, sizeof(g_task_wall));
  if (e == cudaSuccess && reset) { unsigned long long z[NQ][2] = {}; e = cudaMemcpyToSymbol(g_task_wall, z, sizeof(z)); }
  return (int)e;
}
extern "C" int b2h264_debug_fill_stats(unsigned long long* out, int* n_lists, int* wpc, int reset) {
  *n_lists = NQ; *wpc = ENC_WPC;
  cudaError_t e = cudaMemcpyFromSymbol(out, g_fill_stats, sizeof(g_fill_stats));
  if (reset) { void* a = nullptr; if (cudaGetSymbolAddress(&a, g_fill_stats) == cudaSuccess) cudaMemset(a, 0, sizeof(g_fill_stats)); }
  return (int)e;
}
extern "C" int b2h264_debug_batch_stats(unsigned long long* out, int reset) {
  cudaError_t e = cudaMemcpyFromSymbol(out, g_batch_stats, sizeof(g_batch_stats));
  if (e == cudaSuccess && reset) { unsigned long long z[NQ + 1][3] = {}; e = cudaMemcpyToSymbol(g_batch_stats, z, sizeof(z)); }
  return (int)e;
}

// one task: (continue) macroblock `id` at `stage`; notify the dependants or park it for its next stage
template <class Body>
__device__ __forceinline__ void run_task(const StreamFrame* sf, const EncSched& q, MbScratch& s, int id, int stage, int mb_w, int mb_h,
                                         int total, int batch_n, Body& body) {
  const int lane = threadIdx.x & 31, n_mb = mb_w * mb_h;
  __threadfence();
  const int si = id / n_mb, mb = id - si * n_mb, y = mb / mb_w, x = mb - y * mb_w;
  uint4* park = q.stash + (size_t)(si * mb_h + y) * kStashU4;
  uint4* sc = reinterpret_cast<uint4*>(&s);
  if (stage != MBS_A && stage != MBS_I) {            // continue a parked macroblock
    int xo, xn;
    park_extra(stage, &xo, &xn);
    for (int i = lane; i < kCoreU4 + xn; i += 32) {
      const uint4 v = __ldcg(park + i);
      if (i < kCoreU4) sc[i] = v; else sc[xo + i - kCoreU4] = v;
    }
    __syncwarp();
  }
  const int next = body(sf[si], x, y, stage, batch_n);
  __syncwarp();
  if (next == MBS_DONE) {
    __threadfence();
    if (lane == 0) {
      // the (up to three) notifications are independent: issue the atomics together, one L2 round trip instead of three
      const int first = sf[si].p.is_idr ? MBS_I : MBS_A;
      const bool nr = x + 1 < mb_w;                                              // right neighbour: we are its left
      const bool nbl = y + 1 < mb_h && x > 0;                                    // bottom-left: we are its top-right
      const bool nb = y + 1 < mb_h && x == mb_w - 1;                             // last column: we are its top
      const int r0 = nr ? atomicAdd(q.dep + id + 1, 1) : 0;
      const int r1 = nbl ? atomicAdd(q.dep + id + mb_w - 1, 1) : 0;
      const int r2 = nb ? atomicAdd(q.dep + id + mb_w, 1) : 0;
      if (nr && r0 + 1 == 1 + (y > 0)) esched_push(q, total, first, id + 1);
      if (nbl && r1 + 1 == 1 + (x - 1 > 0)) esched_push(q, total, first, id + mb_w - 1);
      if (nb && r2 + 1 == 1 + (x > 0)) esched_push(q, total, first, id + mb_w);
      if (q.rowprog) atomicAdd(q.rowprog + si * mb_h + y, 1);
      atomicAdd(ctl_done(q), 1);
    }
  } else {
    int xo, xn;
    park_extra(next, &xo, &xn);
    for (int i = lane; i < kCoreU4 + xn; i += 32) park[i] = i < kCoreU4 ? sc[i] : sc[xo + i - kCoreU4];
    __threadfence();
    __syncwarp();
    if (lane == 0) esched_push(q, total, next, id);
  }
}

// The batches are claimed by a SCHEDULER WARP (warp ENC_WPC of the CTA, no macroblock scratch): while the ENC_WPC workers run
// batch i it watches the ready lists and claims batch i + 1, so the claim (a look at the control block plus a contended
// CAS: ~18 k cycles per batch when thread 0 did it between two batches, a fifth of the kernel) is off the workers' path
// and a batch costs ONE CTA barrier instead of two.  Claimed macroblocks wait until the running batch ends, so the scheduler
// only claims ahead when that cannot starve anybody: a FULL batch once the first worker has finished (or at any time when
// the list holds two batches' worth); a partial batch only when the workers are already waiting — exactly the decision
// thread 0 used to take at that moment.  (Experiments that gave up the common start of a batch — warp-asynchronous
// draws, 2 x 12 and 3 x 8 warp groups — lost more than they saved to instruction-cache misses.)
struct BatchSlot { int k, base, n, pad; };
constexpr int kEncThreads = 32 * (ENC_WPC + 1);
__device__ __forceinline__ void enc_cta_barrier() { asm volatile("barrier.sync 1, %0;" ::"n"(kEncThreads) : "memory"); }

template <class Body>
__device__ __forceinline__ void run_stages(const StreamFrame* sf, int n_streams, const EncSched q, MbScratch& s, int stats, bool legacy_claim, Body body) {
  __shared__ BatchSlot s_slot[2];
  __shared__ int s_ids[2][ENC_WPC];        // the claimed macroblocks of slot p, read off the ready list by the scheduler warp
  __shared__ int s_fin[2];                 // workers of the batch in slot p that have finished their macroblock
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int mb_w = sf[0].p.mb_w, mb_h = sf[0].p.mb_h, n_mb = mb_w * mb_h, total = n_streams * n_mb;
  if (warp == ENC_WPC) {
    // ---- scheduler warp: lane 0 claims, the warp meets the workers at the barrier ----
    int p = 0, run_n = 0;                  // run_n: macroblocks of the batch the workers are running (slot p ^ 1)
    for (;;) {
      if (lane == 0) {
        int k = 0, h = 0, n = 0;
        long long t_exposed = 0;
        bool exposed = false;
        unsigned long long n_poll = 0, n_fail = 0, n_idle = 0;
        for (;;) {
          const int fin = run_n ? *reinterpret_cast<volatile int*>(&s_fin[p ^ 1]) : 0;
          const bool all_done = fin >= run_n;
          if (stats && all_done && !exposed) { exposed = true; t_exposed = clock64(); }
          n_poll++;
          // ONE look at the control words: NQ + 1 independent loads (a line per list), one L2 round trip
          int c[2 * NQ + 1];
#pragma unroll
          for (int kk = 0; kk < NQ; kk++)
            asm volatile("ld.volatile.global.v2.s32 {%0, %1}, [%2];" : "=r"(c[kk]), "=r"(c[NQ + kk]) : "l"(ctl_head(q, kk)) : "memory");
          asm volatile("ld.volatile.global.s32 %0, [%1];" : "=r"(c[2 * NQ]) : "l"(ctl_done(q)) : "memory");
          if (c[2 * NQ] >= total) { n = -1; break; }
          // later stages first (they finish macroblocks others wait for); a FULL batch beats a partial one
          int best = -1, best_avail = 0;
#pragma unroll
          for (int kk = NQ - 1; kk >= 0; kk--) {
            const int avail = c[NQ + kk] - c[kk];
            if (avail >= ENC_WPC && best_avail < ENC_WPC) { best = kk; best_avail = avail; }
            else if (best_avail < ENC_WPC && avail > best_avail) { best = kk; best_avail = avail; }
          }
          const bool full = best_avail >= ENC_WPC;
          const bool take = best >= 0 && (all_done || (!legacy_claim && full && (fin > 0 || best_avail >= 2 * ENC_WPC)));
          if (take) {
            int tail = 0;
#pragma unroll
            for (int kk = 0; kk < NQ; kk++) if (kk == best) { h = c[kk]; tail = c[NQ + kk]; }
            bool got = false;
            for (;;) {                     // a lost race returns the new head: claim from there instead of looking at every list again
              n = min(ENC_WPC, tail - h);
              if (n <= 0 || (n < ENC_WPC && !all_done)) break;
              const int old = atomicCAS(ctl_head(q, best), h, h + n);
              if (old == h) { got = true; break; }
              n_fail++;
              h = old;
            }
            if (got) { k = best; break; }
            __nanosleep(100 + 40 * (blockIdx.x & 7));        // lost the batch to another CTA: do not hammer the list's line
            continue;
          }
          n_idle++;
          __nanosleep(all_done ? 100 : fin > 0 ? 400 : 1500);
        }
        s_slot[p].k = k; s_slot[p].base = h; s_slot[p].n = n;
        s_fin[p] = 0;
        if (stats) {
          if (exposed) atomicAdd(&g_batch_stats[NQ][2], (unsigned long long)(clock64() - t_exposed));   // what the workers waited for the claim
          atomicAdd(&g_batch_stats[NQ][0], n_poll + (n_fail << 32));        // low word: looks, high word: failed claims
          atomicAdd(&g_batch_stats[NQ][1], n_idle);
        }
      }
      __syncwarp();
      {
        // lane i fetches the i-th claimed macroblock (its producer may still be writing the entry: spin), so that the workers
        // start from shared memory instead of each paying an L2 round trip after the barrier
        const int kk = s_slot[p].k, nn = s_slot[p].n;
        if (lane < nn) {
          int id;
          while ((id = ld_volatile(q.queue + (size_t)kk * total + s_slot[p].base + lane)) < 0) {}
          s_ids[p][lane] = id;
        }
      }
      __syncwarp();
      enc_cta_barrier();                   // slot p is published; the workers have finished the batch of slot p ^ 1
      run_n = s_slot[p].n;
      if (run_n < 0) break;
      p ^= 1;
    }
    return;
  }
  // ---- workers ----
  int p = 0, prev_k = -1, prev_n = 0;
  long long t_prev = 0;
  for (;;) {
    enc_cta_barrier();
    const int k = s_slot[p].k, n = s_slot[p].n;
    if (stats && threadIdx.x == 0) {
      const long long t = clock64();
      if (prev_k >= 0) {
        const unsigned long long dt = (unsigned long long)(t - t_prev);     // barrier to barrier: the batch plus whatever the claim left exposed
        atomicAdd(&g_batch_stats[prev_k][0], 1ull);
        atomicAdd(&g_batch_stats[prev_k][1], (unsigned long long)prev_n);
        atomicAdd(&g_batch_stats[prev_k][2], dt);
        atomicAdd(&g_fill_stats[prev_k][min(prev_n, ENC_WPC)][0], 1ull);
        atomicAdd(&g_fill_stats[prev_k][min(prev_n, ENC_WPC)][1], dt);
      }
      t_prev = t; prev_k = k; prev_n = n;
    }
    if (n < 0) break;
    if (warp < n) {
      const long long t_task = stats ? clock64() : 0;
      const int id = s_ids[p][warp];
      run_task(sf, q, s, id, k + 1, mb_w, mb_h, total, n, body);
      if (lane == 0) atomicAdd(&s_fin[p], 1);
      if (stats && lane == 0) { atomicAdd(&g_task_wall[k][0], (unsigned long long)(clock64() - t_task)); atomicAdd(&g_task_wall[k][1], 1ull); }
    }
    p ^= 1;
  }
}

__global__ void k_esched_init(EncSched q, const StreamFrame* __restrict__ sf, int n_streams, int n_mb) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) {
    // MB (0,0) of every stream is ready: IDR pictures on list I, P pictures on list A
    int na = 0, ni = 0;
    const int total = n_streams * n_mb;
    for (int s = 0; s < n_streams; s++) {
      if (sf[s].p.is_idr) q.queue[(size_t)(MBS_I - 1) * total + ni++] = s * n_mb;
      else q.queue[(size_t)(MBS_A - 1) * total + na++] = s * n_mb;
    }
    for (int k = 0; k < kCtlInts; k++) q.ctl[k] = 0;
    *ctl_tail(q, MBS_A - 1) = na;
    *ctl_tail(q, MBS_I - 1) = ni;
  }
}

__global__ void k_sched_init(Sched q, int n_streams, int n_mb) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_streams) q.queue[i] = i * n_mb;        // MB (0,0) of every stream is ready
  if (i == 0) { *q.head = 0; *q.tail = n_streams; }
}

// optional per-MB-type cycle statistics (debug): [type*2] = cycles, [type*2+1] = count
__device__ unsigned long long g_enc_stats[16];
#ifdef B2H264_PHASE_STATS
namespace mbk { __device__ unsigned long long g_phase[32]; }
extern "C" int b2h264_debug_phase_stats(unsigned long long* out32, int reset) {
  cudaError_t e = cudaMemcpyFromSymbol(out32, mbk::g_phase, sizeof(mbk::g_phase));
  if (e == cudaSuccess && reset) { unsigned long long z[32] = {0}; e = cudaMemcpyToSymbol(mbk::g_phase, z, sizeof(z)); }
  return (int)e;
}
#endif

#ifndef ENC_MIN_CTAS
#define ENC_MIN_CTAS 1
#endif
// dynamic shared memory of the macroblock kernels: ENC_WPC scratches from a 128-byte aligned base (+128 bytes of slack)
constexpr size_t kScratchSmem = sizeof(MbScratch) * DEC_WPC + 128;          // DEC_WPC >= ENC_WPC
static_assert(DEC_WPC >= ENC_WPC, "one scratch area size for both kernels");
__device__ __forceinline__ MbScratch& my_scratch(uint8_t* smem) {
  const uintptr_t a = (reinterpret_cast<uintptr_t>(smem) + 127) & ~uintptr_t(127);
  return reinterpret_cast<MbScratch*>(a)[threadIdx.x >> 5];      // (the encode kernel's scheduler warp gets one it never touches)
}

// tm_ref: reference luma planes of all streams (x, y from the padded origin, z = stream); stage B stages its
// search window out of it with one bulk tensor copy per macroblock (enc_inter.cuh: win_issue / win_wait)
__global__ void __launch_bounds__(kEncThreads, ENC_MIN_CTAS) k_encode_mbs(const StreamFrame* __restrict__ sf, int n_streams, EncSched q, int stats,
                                                                          const __grid_constant__ CUtensorMap tm_ref, const void* tm_global,
                                                                          int win_mode /* 0 none, 1 TMA (descriptor = kernel parameter), 2 warp loads, 3 TMA (descriptor in global memory) */,
                                                                          int* started /* tells the resident deblocking CTAs that this kernel is running */) {
  extern __shared__ __align__(128) uint8_t smem[];
  if (threadIdx.x == 0 && started) *reinterpret_cast<volatile int*>(started) = 1;
  __shared__ WinBar s_wbar[ENC_WPC];
  MbScratch& s = my_scratch(smem);
  WinBar* wb = &s_wbar[min((int)(threadIdx.x >> 5), ENC_WPC - 1)];
  if ((threadIdx.x & 31) == 0 && threadIdx.x < 32 * ENC_WPC) {
    wb->phase = 0;
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"((uint32_t)__cvta_generic_to_shared(&wb->bar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const void* tmap = win_mode == 1 ? (const void*)&tm_ref : win_mode == 3 ? tm_global : nullptr;
  const int wmode = win_mode == 3 ? 1 : win_mode;
  run_stages(sf, n_streams, q, s, stats & 1, (stats & 4) != 0, [&](const StreamFrame& F, int x, int y, int stage, int batch_n) {
    const long long t0 = (stats & 1) ? clock64() : 0;
    mb_ctx(s.ctx, F.p, F.f, x, y);
    if ((threadIdx.x & 31) == 0) { s.ctx.tmap_ref = tmap; s.ctx.wbar = wb; s.ctx.win_mode = wmode; s.ctx.batch_n = (stats & (stage == MBS_A ? 16 : 8)) ? batch_n : 0; s.ctx.batch_n_fine = (stats & 32) ? batch_n : 0; }
    __syncwarp();
    int next = mb_run_stage(s.ctx, s, stage);
    if (stats & 2) while (next != MBS_DONE) next = mb_run_stage(s.ctx, s, next);      // debugging: all stages in one task
    if ((stats & 1) && (threadIdx.x & 31) == 0) {          // cycles and count per stage
      atomicAdd(&g_enc_stats[2 * stage], (unsigned long long)(clock64() - t0));
      atomicAdd(&g_enc_stats[2 * stage + 1], 1ull);
    }
    return next;
  });
  if (threadIdx.x == 0 && started) reinterpret_cast<volatile int*>(started)[1] = 1;      // (every CTA leaves when all macroblocks are coded)
}

// In-loop deblocking: ONE WARP PER MACROBLOCK ROW.  The tasks are short and uniform (a few microseconds each), so the
// dependency bookkeeping of the general scheduler (two global atomics, a fence and a polled ready list per macroblock) cost
// more than the filtering itself: 9.4 ms per 256 x 1080p pictures, 1900 warp instructions per macroblock.  Here a warp walks
// its row left to right and only has to stay two macroblocks behind the row above (MB(x, y) needs (x - 1, y) — the warp's own
// previous step — and (x + 1, y - 1)); progress is one int per row.  Rows are handed out row-major over the streams (all
// rows 0 first), so a row is only ever claimed after the row it waits for: no deadlock whatever the number of resident warps.
// Two instantiations.  <8, 6>: the full-size grid (6 CTAs of 8 warps per SM), launched behind the encode kernel.
// <4, 16>: an EXPERIMENT (B2H264_RESIDENT_DEBLOCK=1), kept because its result is instructive: ONE 4-warp CTA per SM at <= 32
// registers, sized to be resident BESIDE the encode kernel's CTA (768 threads x 80 registers leave 4096 registers and ~9 KB of
// shared memory per SM).  Launched with k_encode_mbs it follows the encode wavefront through `enc_prog` (macroblock (x, y) may be
// filtered once (x + 1, y + 1) is coded: nothing reads its unfiltered samples any more); both instantiations draw rows from
// the same counter, so the full-size grid finishes what the resident CTAs have not claimed.  It works (bit-exact, sanitizer
// clean, steps aside where kernels are serialised) and it does hide the filter, but the encode
// kernel beside it slows down by more: a fifth instruction stream on every SM evicts the lock-step batch's code from the
// instruction caches, the same effect as splitting the batch.  Slower per step overall: off by default.
#define DBK_WPC 8
#define DBK_CO_WPC 4
template <int WPC, int MIN_CTAS, bool BSL = false /* decoder: the pictures may hold B macroblocks (two reference lists in the strength rule) */>
__global__ void __launch_bounds__(32 * WPC, MIN_CTAS) k_deblock_rows(const StreamFrame* __restrict__ sf, int n_streams, int* prog, int* counter,
                                                                      const int* enc_prog /* NULL: every macroblock is coded already */,
                                                                      const int* enc_started /* resident form only, see below */) {
  using Tile = typename std::conditional<BSL, DbkTileB, DbkTile>::type;
  __shared__ Tile tiles[WPC];
  // The resident form waits for a kernel that runs AT THE SAME TIME.  Where kernels are serialised (compute-sanitizer, ncu replay,
  // a debugger) that kernel cannot start while this one spins: a CTA that does not see the encode kernel running within ~0.3 ms leaves
  // without claiming a row, and the full-size grid launched behind the encode kernel does all the work.
  if (enc_started != nullptr) {
    __shared__ int s_go;
    if (threadIdx.x == 0) {
      int go = 0;
      for (int i = 0; i < 300 && !(go = ld_volatile(enc_started)); i++) __nanosleep(1000);
      // ... and one that only starts when the encode kernel is already DONE (serialised after it) leaves too: the full-size grid
      // behind it is the faster way through the rows then
      if (go && ld_volatile(enc_started + 1)) go = 0;
      s_go = go;
    }
    __syncthreads();
    if (!s_go) return;
  }
  Tile& t = tiles[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  const int mb_w = sf[0].p.mb_w, mb_h = sf[0].p.mb_h, units = n_streams * mb_h;
  for (;;) {
    int u = 0;
    if (lane == 0) u = atomicAdd(counter, 1);
    u = __shfl_sync(MBK_FULL, u, 0);
    if (u >= units) break;
    const int row = u / n_streams, si = u - row * n_streams;
    const StreamFrame& F = sf[si];
    int* mine = prog + si * mb_h + row;
    const int* up = mine - 1;
    const int* coded = enc_prog ? enc_prog + si * mb_h + (row + 1 < mb_h ? row + 1 : row) : nullptr;
    int seen = row > 0 ? 0 : mb_w, seen_enc = coded ? 0 : mb_w;
    for (int x = 0; x < mb_w; x++) {
      const int need = x + 2 < mb_w ? x + 2 : mb_w;
      if (seen < need || seen_enc < need) {
        if (lane == 0) {
          while (seen < need && (seen = ld_volatile(up)) < need) __nanosleep(40);
          while (seen_enc < need && (seen_enc = ld_volatile(coded)) < need) __nanosleep(200);
        }
        seen = __shfl_sync(MBK_FULL, seen, 0);
        seen_enc = __shfl_sync(MBK_FULL, seen_enc, 0);
        __threadfence();
      }
      deblock_one_mb_t<BSL>(F.p, F.f, x, row, t);
      __threadfence();
      __syncwarp();
      if (lane == 0) *reinterpret_cast<volatile int*>(mine) = x + 1;
    }
  }
}

// ---- decoder construct path (groundwork of the next SURVEY row: dec_mb.cuh) ------------------------------------------------
// One warp reconstructs one macroblock from its parsed record (h264_parse.h); the macroblocks of all streams are
// scheduled by the same dependency rule as the encoder (left + top-right done), with the simple per-warp ready list.
__global__ void __launch_bounds__(32 * DEC_WPC) k_decode_mbs(const StreamFrame* __restrict__ sf, int n_streams, Sched q,
                                                            const MbOut* __restrict__ recs, const DecMbAux* __restrict__ aux) {
  extern __shared__ __align__(128) uint8_t smem[];
  MbScratch& s = my_scratch(smem);
  run_mbs(sf, n_streams, q, [&](const StreamFrame& F, int x, int y) {
    const int n_mb = F.p.mb_w * F.p.mb_h, si = (int)(&F - sf);
    const size_t r = (size_t)si * n_mb + y * F.p.mb_w + x;
    dec_one_mb(F.p, F.f, s, x, y, recs[r], aux[r]);
  });
}

// ---- border replication, all planes of all streams in two launches -------------------------------------------
__global__ void k_expand_lr_batch(const StreamFrame* __restrict__ sf) {
  const StreamFrame& F = sf[blockIdx.z / 3];
  const int pl = blockIdx.z % 3;
  const int pad = pl ? 16 : 32, st = pl ? F.p.rec_stride_c : F.p.rec_stride_y;
  const int w = (pl ? 8 : 16) * F.p.mb_w, h = (pl ? 8 : 16) * F.p.mb_h;
  const int y = blockIdx.x * blockDim.y + threadIdx.y;
  if (y >= h) return;
  uint8_t* row = F.f.rec[pl] + (size_t)y * st;
  const uint8_t l = row[0], r = row[w - 1];
  for (int x = threadIdx.x; x < pad; x += blockDim.x) { row[x - pad] = l; row[w + x] = r; }
}
__global__ void k_expand_tb_batch(const StreamFrame* __restrict__ sf) {
  const StreamFrame& F = sf[blockIdx.z / 3];
  const int pl = blockIdx.z % 3;
  const int pad = pl ? 16 : 32, st = pl ? F.p.rec_stride_c : F.p.rec_stride_y;
  const int w = (pl ? 8 : 16) * F.p.mb_w, h = (pl ? 8 : 16) * F.p.mb_h;
  const int x = blockIdx.x * blockDim.x + threadIdx.x - pad;
  if (x >= w + pad) return;
  uint8_t* pic = F.f.rec[pl];
  const uint8_t t = pic[x], b = pic[(size_t)(h - 1) * st + x];
  for (int y = 1 + blockIdx.y; y <= pad; y += gridDim.y) {
    pic[x - (ptrdiff_t)y * st] = t;
    pic[(size_t)(h - 1 + y) * st + x] = b;
  }
}

// ================================================================================================
// H.264 Tables 8-16 / 8-17 (host copies; the device reads the constant-memory twins)
namespace mbk {
uint8_t h_alpha[52] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 4, 4, 5, 6, 7, 8, 9, 10, 12, 13, 15, 17, 20, 22, 25, 28,
                       32, 36, 40, 45, 50, 56, 63, 71, 80, 90, 101, 113, 127, 144, 162, 182, 203, 226, 255, 255};
uint8_t h_beta[52] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 6, 6, 7, 7, 8, 8,
                      9, 9, 10, 10, 11, 11, 12, 12, 13, 13, 14, 14, 15, 15, 16, 16, 17, 17, 18, 18};
uint8_t h_tc0[52][3] = {
    {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0},
    {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 1}, {0, 0, 1}, {0, 0, 1}, {0, 0, 1}, {0, 1, 1},
    {0, 1, 1}, {1, 1, 1}, {1, 1, 1}, {1, 1, 1}, {1, 1, 1}, {1, 1, 2}, {1, 1, 2}, {1, 1, 2}, {1, 1, 2}, {1, 2, 3}, {1, 2, 3},
    {2, 2, 3}, {2, 2, 4}, {2, 3, 4}, {2, 3, 4}, {3, 3, 5}, {3, 4, 6}, {3, 4, 6}, {4, 5, 7}, {4, 5, 8}, {4, 6, 9}, {5, 7, 10},
    {6, 8, 11}, {6, 8, 13}, {7, 10, 14}, {8, 11, 16}, {9, 12, 18}, {10, 13, 20}, {11, 15, 23}, {13, 17, 25}};
}  // namespace mbk

int enc_upload_deblock_tables() {
  cudaError_t e;
  if ((e = cudaMemcpyToSymbol(mbk::c_alpha, mbk::h_alpha, sizeof(mbk::h_alpha))) != cudaSuccess) return (int)e;
  if ((e = cudaMemcpyToSymbol(mbk::c_beta, mbk::h_beta, sizeof(mbk::h_beta))) != cudaSuccess) return (int)e;
  if ((e = cudaMemcpyToSymbol(mbk::c_tc0, mbk::h_tc0, sizeof(mbk::h_tc0))) != cudaSuccess) return (int)e;
  return 0;
}

// Persistent grids: exactly what the chip can hold.  cudaFuncSetAttribute and the occupancy are PER DEVICE: cached per
// device ordinal under a lock (encoders / decoders on several devices and threads of one process).
#include <mutex>
template <class K>
static int grid_blocks_for(K kernel, int threads, int* cache /*[64]*/) {
  static std::mutex mu;
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lock(mu);
  if (dev < 0 || dev >= 64) dev = 0;
  if (cache[dev]) return cache[dev];
  cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kScratchSmem);
  int sms = 0, per_sm = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, kScratchSmem);
  if (per_sm < 1) per_sm = 1;
  return cache[dev] = sms * per_sm;
}
static int enc_grid_blocks() {
  static int cache[64];
  return grid_blocks_for(k_encode_mbs, kEncThreads, cache);
}
static int dec_grid_blocks() {
  static int cache[64];
  return grid_blocks_for(k_decode_mbs, 32 * DEC_WPC, cache);
}

// scheduler workspace layout (ints): [0..3] head/tail of the deblock list; from 32: dep[2][total] (encode, deblock), then
// queue[1 + NQ][total] (deblock list, encode lists); then, 128-byte aligned, the encode lists' control lines (kCtlInts)
static size_t enc_ctl_offset(size_t total) { return (32 + (3 + NQ) * total + 31) / 32 * 32; }       // 128-byte aligned, behind the lists
// ... then the coded-rows counters the deblocking kernels follow (n_streams * mb_h ints; n_streams * n_mb reserved)
size_t enc_sched_ints(int n_streams, int n_mb) { return enc_ctl_offset((size_t)n_streams * n_mb) + kCtlInts + (size_t)n_streams * n_mb; }
size_t enc_stash_bytes(int n_streams, int mb_h) { return (size_t)n_streams * mb_h * kStashU4 * sizeof(uint4); }

static Sched make_sched(int* ws, int which, int total) {
  Sched q;
  q.head = ws + 2 * which; q.tail = ws + 2 * which + 1;
  (void)which;                                     // only the deblock list (1) uses the simple scheduler
  q.dep = ws + 32 + (size_t)total;
  q.queue = ws + 32 + (size_t)2 * total;
  return q;
}
static EncSched make_esched(int* ws, int total, void* stash) {
  EncSched q;
  q.ctl = ws + enc_ctl_offset((size_t)total);
  q.dep = ws + 32;
  q.queue = ws + 32 + (size_t)3 * total;
  q.stash = reinterpret_cast<uint4*>(stash);
  q.rowprog = nullptr;
  return q;
}

// prog: n_streams * mb_h progress counters, zero; counter: the row hand-out counter (zeroed by the caller)
static int launch_deblock_rows(const StreamFrame* d_sf, int n_streams, int mb_h, int* prog, int* counter, const int* enc_prog, cudaStream_t st,
                               bool b_slices = false) {
  static int per_dev[64];
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (!per_dev[dev]) {
    int per_sm = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_deblock_rows<DBK_WPC, 6>, 32 * DBK_WPC, 0);
    per_dev[dev] = sms * (per_sm < 1 ? 1 : per_sm);
  }
  const int units = n_streams * mb_h;
  int blocks = per_dev[dev];
  if (blocks > (units + DBK_WPC - 1) / DBK_WPC) blocks = (units + DBK_WPC - 1) / DBK_WPC;
  if (b_slices) k_deblock_rows<DBK_WPC, 6, true><<<blocks, 32 * DBK_WPC, 0, st>>>(d_sf, n_streams, prog, counter, enc_prog, nullptr);
  else k_deblock_rows<DBK_WPC, 6><<<blocks, 32 * DBK_WPC, 0, st>>>(d_sf, n_streams, prog, counter, enc_prog, nullptr);
  return b2h264_launched();
}
// the resident companion of the encode kernel: one small CTA per SM
static int launch_deblock_rows_resident(const StreamFrame* d_sf, int n_streams, int mb_h, int* prog, int* counter, const int* enc_prog,
                                        const int* enc_started, cudaStream_t st) {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  // An SM changes its L1 / shared-memory split only when it is empty.  Should one of these CTAs ever reach an SM before the encode
  // kernel's CTA, it must leave the SM configured for the encoder's 186 KB — otherwise the encoder could not join it and this CTA
  // would wait for an encoder that waits for the SM to drain (seen as a hang when this kernel was launched FIRST).
  static bool carve_set[64];
  if (dev >= 0 && dev < 64 && !carve_set[dev]) {
    cudaFuncSetAttribute(k_deblock_rows<DBK_CO_WPC, 16>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    carve_set[dev] = true;
  }
  const int units = n_streams * mb_h;
  int blocks = sms;
  if (blocks > (units + DBK_CO_WPC - 1) / DBK_CO_WPC) blocks = (units + DBK_CO_WPC - 1) / DBK_CO_WPC;
  k_deblock_rows<DBK_CO_WPC, 16><<<blocks, 32 * DBK_CO_WPC, 0, st>>>(d_sf, n_streams, prog, counter, enc_prog, enc_started);
  return b2h264_launched();
}

// B2H264_BATCH_SYNC: bit 0 stage B (default: measured +5.5 %), bit 1 stage A (measured: no gain, -1.5 % together with B), bit 2 finer points in stage B
static int batch_sync_bits() {
  const char* v = getenv("B2H264_BATCH_SYNC");
  const int m = v ? atoi(v) : 1;
  return ((m & 1) ? 8 : 0) | ((m & 2) ? 16 : 0) | ((m & 4) ? 32 : 0);
}

int enc_launch_frame(const StreamFrame* d_sf, const uint8_t* const* d_src, int n_streams, int w, int h, int mb_w, int mb_h,
                     int* d_ws, void* d_stash, const void* tmap_ref, const void* d_tmap, int fast_mode, cudaStream_t st,
                     cudaStream_t st_dbk, cudaEvent_t ev_ready, cudaEvent_t ev_dbk) {
  int rc;
  if (d_src) {
    dim3 b(32, 8), g((mb_w * 4 + 31) / 32, (mb_h * 16 + 7) / 8, n_streams);
    k_pad_source<<<g, b, 0, st>>>(d_sf, d_src, w, h);
    if ((rc = b2h264_launched())) return rc;
  }
  if (fast_mode) {                                    // LOW_COMPLEXITY: the partition choice reads these statistics
    const int n_mb = mb_w * mb_h;
    k_vaa_sad8x8<<<dim3((n_mb + 7) / 8, n_streams), 256, 0, st>>>(d_sf, n_mb);
    if ((rc = b2h264_launched())) return rc;
  }
  const int total = n_streams * mb_w * mb_h;
  cudaMemsetAsync(d_ws + 32, 0, 2 * (size_t)total * sizeof(int), st);                                     // dep counters
  cudaMemsetAsync(d_ws + 32 + 2 * (size_t)total, 0xff, (size_t)(1 + NQ) * total * sizeof(int), st);       // ready lists
  EncSched qe = make_esched(d_ws, total, d_stash);
  // progress counters: rows deblocked in the deblocking list's (zeroed) counter area, rows coded behind the control lines
  int* dbk_prog = d_ws + 32 + (size_t)total;
  static const bool resident_dbk = getenv("B2H264_RESIDENT_DEBLOCK") != nullptr;     // experiment, off: see k_deblock_rows
  const bool co = resident_dbk && st_dbk != nullptr;
  if (co) {                                          // the coded-rows counters are only kept for the resident deblocking CTAs
    qe.rowprog = d_ws + enc_ctl_offset((size_t)total) + kCtlInts;
    cudaMemsetAsync(qe.rowprog, 0, (size_t)n_streams * mb_h * sizeof(int), st);
  }
  k_esched_init<<<1, 32, 0, st>>>(qe, d_sf, n_streams, mb_w * mb_h);
  cudaMemsetAsync(d_ws + 2, 0, 3 * sizeof(int), st);               // the deblocking row hand-out counter; [3] = "the encode kernel is running", [4] = "... has finished"
  int blocks = enc_grid_blocks();
  const int need = (total + ENC_WPC - 1) / ENC_WPC;
  if (blocks > need) blocks = need;
  static const int stats = (getenv("B2H264_ENC_STATS") ? 1 : 0) | (getenv("B2H264_FUSE_STAGES") ? 2 : 0) | (getenv("B2H264_LEGACY_CLAIM") ? 4 : 0) |
                           batch_sync_bits();      // 8 / 16: re-alignment points inside stages B / A (mbk_batch_sync)
  CUtensorMap tm;
  memset(&tm, 0, sizeof(tm));
  // B2H264_ENC_WIN: 0 = search out of the plane, 1 = TMA window, descriptor passed as kernel parameter (default),
  // 2 = window staged by the warp's own loads, 3 = TMA window, descriptor read from global memory
  static const int win_env = getenv("B2H264_ENC_WIN") ? atoi(getenv("B2H264_ENC_WIN")) : 1;
  int win_mode = win_env;
  if ((win_mode == 1 || win_mode == 3) && tmap_ref == nullptr) win_mode = 2;
  if (win_mode == 3 && d_tmap == nullptr) win_mode = 2;
  if (win_mode == 1) memcpy(&tm, tmap_ref, sizeof(tm));
  if (co && cudaEventRecord(ev_ready, st) != cudaSuccess) return (int)cudaGetLastError();
  k_encode_mbs<<<blocks, kEncThreads, kScratchSmem, st>>>(d_sf, n_streams, qe, stats, tm, d_tmap, win_mode, co ? d_ws + 3 : nullptr);
  if ((rc = b2h264_launched())) return rc;
  if (co) {
    // the resident deblocking CTAs are launched BEHIND the encode kernel (its CTAs take their SMs first) and follow its wavefront
    if (cudaStreamWaitEvent(st_dbk, ev_ready, 0) != cudaSuccess) return (int)cudaGetLastError();
    if ((rc = launch_deblock_rows_resident(d_sf, n_streams, mb_h, dbk_prog, d_ws + 2, qe.rowprog, d_ws + 3, st_dbk))) return rc;
    if (cudaEventRecord(ev_dbk, st_dbk) != cudaSuccess) return (int)cudaGetLastError();
  }
  return 0;
}

int enc_launch_deblock_expand(const StreamFrame* d_sf, int n_streams, int mb_w, int mb_h, int* d_ws, cudaStream_t st, cudaEvent_t ev_dbk) {
  int rc;
  const int total = n_streams * mb_w * mb_h;
  int* dbk_prog = d_ws + 32 + (size_t)total;      // the deblocking list's counters: zeroed per picture (enc_launch_frame)
  // the full-size grid takes the rows the resident CTAs have not claimed (same hand-out counter, same progress words)
  static const bool resident_dbk = getenv("B2H264_RESIDENT_DEBLOCK") != nullptr;     // experiment, off: see k_deblock_rows
  if ((rc = launch_deblock_rows(d_sf, n_streams, mb_h, dbk_prog, d_ws + 2, resident_dbk ? d_ws + enc_ctl_offset((size_t)total) + kCtlInts : nullptr, st))) return rc;
  if (resident_dbk && ev_dbk && cudaStreamWaitEvent(st, ev_dbk, 0) != cudaSuccess) return (int)cudaGetLastError();
  k_expand_lr_batch<<<dim3((mb_h * 16 + 7) / 8, 1, 3 * n_streams), dim3(32, 8), 0, st>>>(d_sf);
  if ((rc = b2h264_launched())) return rc;
  k_expand_tb_batch<<<dim3((mb_w * 16 + 64 + 127) / 128, 4, 3 * n_streams), dim3(128), 0, st>>>(d_sf);
  return b2h264_launched();
}

// decoder: workspace (ints) = [0..3] heads / tails, then dep[2][total], then queue[2][total] (construct, deblock)
size_t dec_sched_ints(int n_streams, int n_mb) { return 8 + 4 * (size_t)n_streams * n_mb; }
static Sched make_dec_sched(int* ws, int which, int total) {
  Sched q;
  q.head = ws + 2 * which; q.tail = ws + 2 * which + 1;
  q.dep = ws + 8 + (size_t)which * total;
  q.queue = ws + 8 + (size_t)(2 + which) * total;
  return q;
}
int dec_launch_frame(const StreamFrame* d_sf, int n_streams, int mb_w, int mb_h, int* d_ws, const MbOut* d_recs, const DecMbAux* d_aux, int deblock,
                     cudaStream_t st, int b_slices) {
  const int blocks_per_launch = dec_grid_blocks();
  int rc;
  const int total = n_streams * mb_w * mb_h;
  cudaMemsetAsync(d_ws + 8, 0, 2 * (size_t)total * sizeof(int), st);
  cudaMemsetAsync(d_ws + 8 + 2 * (size_t)total, 0xff, 2 * (size_t)total * sizeof(int), st);
  const Sched qc = make_dec_sched(d_ws, 0, total), qd = make_dec_sched(d_ws, 1, total);
  k_sched_init<<<(n_streams + 127) / 128, 128, 0, st>>>(qc, n_streams, mb_w * mb_h);
  k_sched_init<<<(n_streams + 127) / 128, 128, 0, st>>>(qd, n_streams, mb_w * mb_h);
  const int need = (total + DEC_WPC - 1) / DEC_WPC;
  k_decode_mbs<<<blocks_per_launch < need ? blocks_per_launch : need, 32 * DEC_WPC, kScratchSmem, st>>>(d_sf, n_streams, qc, d_recs, d_aux);
  if ((rc = b2h264_launched())) return rc;
  if (deblock) {
    cudaMemsetAsync(d_ws + 2, 0, sizeof(int), st);
    if ((rc = launch_deblock_rows(d_sf, n_streams, mb_h, d_ws + 8 + (size_t)total, d_ws + 2, nullptr, st, b_slices != 0))) return rc;
  }
  k_expand_lr_batch<<<dim3((mb_h * 16 + 7) / 8, 1, 3 * n_streams), dim3(32, 8), 0, st>>>(d_sf);
  if ((rc = b2h264_launched())) return rc;
  k_expand_tb_batch<<<dim3((mb_w * 16 + 64 + 127) / 128, 4, 3 * n_streams), dim3(128), 0, st>>>(d_sf);
  return b2h264_launched();
}

// ---- record hand-over: only coded macroblocks travel, and of those only the residual blocks that carry levels ------
// One CTA per stream, a warp per coded macroblock.  `pack` is MAPPED PINNED HOST memory: the SMs' 16-byte stores go over
// PCIe as posted writes, there is no separate copy and no size round trip.  The hand-over is PCIe-bound (whole 896-byte
// records of the coded macroblocks were 326 MB per 256 x 1080p pictures, ~11 ms at the ~28 GB/s such stores reach), so a
// record is compacted before it travels (enc_types.h: MbRecHead):
//   128-byte head = MbOut bytes [0, 112) + chroma_dc, with the presence mask of the 24 residual blocks in pad0[3]
//   32 bytes per PRESENT block (luma in coding order 0..15, chroma AC 16..23): inside a coded 8x8 / chroma AC set and not all zero
// idx[mb] = offset of the macroblock's record in 32-byte units, or -1 for P_SKIP; cnt[stream] = units written.
// Records land in whatever order the warps finish (one shared-memory atomic hands out the space); the host goes through idx.
#define PACK_THREADS 256          // small CTAs: the kernel is PCIe-bound and must leave the SMs to the deblocking kernel
__global__ void __launch_bounds__(PACK_THREADS) k_pack_records(const StreamFrame* __restrict__ sf, int n_mb, uint4* __restrict__ pack,
                                                               int32_t* __restrict__ idx, int32_t* __restrict__ cnt) {
  __shared__ int s_units;
  const int s = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wi = tid >> 5;
  const MbOut* out = sf[s].f.out;
  int32_t* my_idx = idx + (size_t)s * n_mb;
  uint4* dst0 = pack + (size_t)s * n_mb * (sizeof(MbOut) / 16);
  if (tid == 0) s_units = 0;
  __syncthreads();
  for (int c0 = wi * 32; c0 < n_mb; c0 += PACK_THREADS) {
    const int mb = c0 + lane;
    const bool coded = mb < n_mb && out[mb].mb_type != MBT_PSKIP;
    unsigned m = __ballot_sync(0xffffffffu, coded);
    if (mb < n_mb && !coded) my_idx[mb] = -1;
    while (m) {
      const int j = __ffs(m) - 1;
      m &= m - 1;
      const MbOut* rec = out + c0 + j;
      const uint4* rq = reinterpret_cast<const uint4*>(rec);
      const int type = rec->mb_type, cbp = rec->cbp;
      uint4 a = make_uint4(0, 0, 0, 0), b = a;
      bool want = false;
      if (lane < 16) want = type == MBT_I16x16 ? (cbp & 15) != 0 : ((cbp >> (lane >> 2)) & 1) != 0;
      else if (lane < 24) want = (cbp >> 4) == 2;
      if (want) {
        const int q = lane < 16 ? 7 + 2 * lane : 40 + 2 * (lane - 16);      // luma at byte 112, chroma_ac at byte 640
        a = rq[q]; b = rq[q + 1];
        want = (a.x | a.y | a.z | a.w | b.x | b.y | b.z | b.w) != 0;
      }
      const unsigned mask = __ballot_sync(0xffffffffu, want);
      int off = 0;
      if (lane == 0) off = atomicAdd(&s_units, 4 + __popc(mask));
      off = __shfl_sync(0xffffffffu, off, 0);
      uint4* dst = dst0 + (size_t)off * 2;
      if (lane < 8) {
        uint4 v = rq[lane < 7 ? lane : 39];                                    // chroma_dc at byte 624
        if (lane == 0) v.y = (v.y & 0xffu) | (mask << 8);                      // pad0[3] = presence mask
        dst[lane] = v;
      }
      if (want) {
        const int pos = 8 + 2 * __popc(mask & ((1u << lane) - 1));
        dst[pos] = a; dst[pos + 1] = b;
      }
      if (lane == 0) my_idx[c0 + j] = off;
    }
  }
  __syncthreads();
  if (tid == 0) cnt[s] = s_units;
}

int enc_launch_pack(const StreamFrame* d_sf, int n_streams, int n_mb, MbOut* pack, int32_t* idx, int32_t* cnt, cudaStream_t st) {
  static_assert(sizeof(MbOut) == 896 && offsetof(MbOut, luma) == 112 && offsetof(MbOut, chroma_dc) == 624 && offsetof(MbOut, chroma_ac) == 640 &&
                offsetof(MbOut, pad0) == 5, "compact record layout");
  k_pack_records<<<n_streams, PACK_THREADS, 0, st>>>(d_sf, n_mb, reinterpret_cast<uint4*>(pack), idx, cnt);
  return b2h264_launched();
}

// ---- decoder hand-over: compact records (host: pack_records_compact, enc_host.cpp) -> the MbOut array k_decode_mbs reads ----
// One warp per macroblock.  idx < 0: a P_SKIP macroblock, only its header is (re)written (type, quantiser = -1 - idx); the
// levels of such a record are never read.  Otherwise the 128-byte head goes back to its two places and each of the 24
// residual blocks is copied or zeroed.  7.3 MB per 1080p picture used to cross PCIe; a typical P picture now sends ~0.3 MB.
__global__ void __launch_bounds__(256) k_unpack_records(const uint4* __restrict__ pack, size_t stream_stride_u4, const int32_t* __restrict__ idx,
                                                        MbOut* __restrict__ recs, int n_mb) {
  const int s = blockIdx.y, lane = threadIdx.x & 31, mb = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (mb >= n_mb) return;
  const int32_t o = idx[(size_t)s * n_mb + mb];
  uint4* dst = reinterpret_cast<uint4*>(recs + (size_t)s * n_mb + mb);
  const uint4 z = make_uint4(0, 0, 0, 0);
  if (o < 0) {
    if (lane < 7) dst[lane] = lane == 0 ? make_uint4((uint32_t)MBT_PSKIP | ((uint32_t)(-1 - o) << 16), 0, 0, 0) : z;
    else if (lane == 7) dst[39] = z;
    return;
  }
  const uint4* src = pack + (size_t)s * stream_stride_u4 + (size_t)o * 2;
  const uint32_t mask = src[0].y >> 8;
  if (lane < 7) {
    uint4 v = src[lane];
    if (lane == 0) v.y &= 0xffu;                                   // pad0 carried the presence mask
    dst[lane] = v;
  } else if (lane == 7) {
    dst[39] = src[7];                                              // chroma_dc
  } else {
    const int b = lane - 8, q = b < 16 ? 7 + 2 * b : 40 + 2 * (b - 16);
    uint4 v0 = z, v1 = z;
    if ((mask >> b) & 1) { const int pos = 8 + 2 * __popc(mask & ((1u << b) - 1)); v0 = src[pos]; v1 = src[pos + 1]; }
    dst[q] = v0; dst[q + 1] = v1;
  }
}
int dec_launch_unpack(const void* d_pack, size_t stream_stride_bytes, const int32_t* d_idx, MbOut* d_recs, int n_streams, int n_mb, cudaStream_t st) {
  k_unpack_records<<<dim3((n_mb + 7) / 8, n_streams), 256, 0, st>>>(reinterpret_cast<const uint4*>(d_pack), stream_stride_bytes / 16, d_idx, d_recs, n_mb);
  return b2h264_launched();
}

size_t enc_scratch_bytes() { return sizeof(MbScratch); }

extern "C" int b2h264_debug_enc_stats(unsigned long long* out16, int reset) {
  cudaError_t e = cudaMemcpyFromSymbol(out16, g_enc_stats, sizeof(g_enc_stats));
  if (e != cudaSuccess) return (int)e;
  if (reset) { unsigned long long z[16] = {0}; e = cudaMemcpyToSymbol(g_enc_stats, z, sizeof(z)); }
  return (int)e;
}
