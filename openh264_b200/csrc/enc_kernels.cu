// enc_kernels.cu — frame-level CUDA kernels of the encoder path (sm_90a):
//   k_pad_source     source I420 -> MB-aligned current picture
//   k_encode_mbs     macroblock mode decision + coding + reconstruction, ONE WARP PER MACROBLOCK; the MBs of
//                    all streams of the batch are scheduled by dependency (ready lists, persistent warps)
//   k_deblock_pictures  in-loop deblocking, one CTA per picture, one warp per macroblock row (encoder and decoder)
//   k_decode_mbs     the decoder's macroblock reconstruction, scheduled like the encoder's macroblocks
//   k_expand_*       border replication of the new reference picture (ExpandReferencingPicture)
// Why a wavefront: MB(x,y) needs the FINAL state of (x-1,y), (x,y-1), (x+1,y-1) — motion-vector / SAD
// predictors, intra neighbours, skip context (SURVEY.md §7 hard part 1); bit-exactness forbids breaking
// that chain, so parallelism comes from rows (2-MB lag) x independent streams of the batch.
#include <cuda.h>
#include <type_traits>
#include <vector>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>

#include "b2h264_internal.h"
#include "enc_deblock.cuh"
#include "enc_frame.cuh"
#include "dec_mb.cuh"
#include "dec_records_check.h"
#include "stage_hooks.cuh"
#include "enc_launch.h"
#include "enc_host.h"
#include "cuda_owned.h"

using namespace mbk;
using b2h264::DeviceBuf;

namespace mbk {
__constant__ uint8_t c_alpha[52];
__constant__ uint8_t c_beta[52];
__constant__ uint8_t c_tc0[52][3];
}  // namespace mbk

#define DEC_WPC 24         // warps per CTA of the decoder's macroblock kernel (one CTA per SM at 80 registers)
#define ENC_WPC 23         // WORKER warps per CTA of the encode kernel; one more warp schedules (24 x 32 x 80 registers = one CTA per SM)
// A full batch of a PULLED list claims up to ENC_PULL x ENC_WPC tasks; a warp that finishes its task takes the next unstarted
// one of the block (run_stages).  Pulled: A (skip test), bit enc_list(stage) of the mask.
// ENC_PULL = 1 is the plain one-task-per-warp batch.
#ifndef ENC_PULL
#define ENC_PULL 2
#endif
#ifndef ENC_PULL_LISTS
#define ENC_PULL_LISTS (1 << enc_list(MBS_A))
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
// spent most of its issue slots spinning).  The encoder has one ready list per stage (below), the decoder one list.
// the encoder's ready lists: one per stage (MBP_SKIPCAND_INTRA is not a stage), index enc_list(stage)
enum { NQ = MBS_COUNT - 2 };
__host__ __device__ constexpr int enc_list(int stage) { return stage < MBP_SKIPCAND_INTRA ? stage - 1 : stage - 2; }
__host__ __device__ constexpr int enc_stage(int list) { return list < MBP_SKIPCAND_INTRA - 1 ? list + 1 : list + 2; }
static_assert(enc_stage(enc_list(MBS_C)) == MBS_C && enc_list(MBS_C) == NQ - 1, "one list per stage");
struct MbSched {
  int* dep;          // per (stream, mb): notifications received so far
  int* queue;        // ready lists of capacity `total` each, -1 = slot not yet written
  int* ctl;          // one 128-byte line per ready list: [32 k] head, [32 k + 1] tail; the encoder's line NQ: [32 NQ] macroblocks finished
  uint4* stash;      // the encoder's parked scratches
};
// The control words are spread over NQ + 1 lines (different L2 slices): every finished macroblock, every push and every
// scheduler look / claim of one CTA per SM used to hit ONE line, and the queueing there slowed the workers' own atomics.
__device__ __forceinline__ int* ctl_head(const MbSched& q, int k) { return q.ctl + 32 * k; }
__device__ __forceinline__ int* ctl_tail(const MbSched& q, int k) { return q.ctl + 32 * k + 1; }
__device__ __forceinline__ int* ctl_done(const MbSched& q) { return q.ctl + 32 * NQ; }

__device__ __forceinline__ void ready_push(const MbSched& q, int total, int k, int id) {
  const int slot = atomicAdd(ctl_tail(q, k), 1);
  *reinterpret_cast<volatile int*>(q.queue + (size_t)k * total + slot) = id;
}
// macroblock `id` at (x, y) is final: notify its dependants and push those now ready onto list k (one lane)
__device__ __forceinline__ void notify_dependants(const MbSched& q, int total, int k, int id, int x, int y, int mb_w, int mb_h) {
  // the (up to three) notifications are independent: issue the atomics together, one L2 round trip instead of three
  const bool nr = x + 1 < mb_w;                                              // right neighbour: we are its left
  const bool nbl = y + 1 < mb_h && x > 0;                                    // bottom-left: we are its top-right
  const bool nb = y + 1 < mb_h && x == mb_w - 1;                             // last column: we are its top
  const int r0 = nr ? atomicAdd(q.dep + id + 1, 1) : 0;
  const int r1 = nbl ? atomicAdd(q.dep + id + mb_w - 1, 1) : 0;
  const int r2 = nb ? atomicAdd(q.dep + id + mb_w, 1) : 0;
  if (nr && r0 + 1 == 1 + (y > 0)) ready_push(q, total, k, id + 1);
  if (nbl && r1 + 1 == 1 + (x - 1 > 0)) ready_push(q, total, k, id + mb_w - 1);
  if (nb && r2 + 1 == 1 + (x > 0)) ready_push(q, total, k, id + mb_w);
}

// the decoder's policy: every warp pops one macroblock from list 0 at a time
template <class Body>
__device__ __forceinline__ void run_mbs(const StreamFrame* sf, int n_streams, const MbSched q, Body body) {
  const int lane = threadIdx.x & 31;
  const int mb_w = sf[0].p.mb_w, mb_h = sf[0].p.mb_h, n_mb = mb_w * mb_h, total = n_streams * n_mb;
  for (;;) {
    int id = 0;
    if (lane == 0) {
      const int t = atomicAdd(ctl_head(q, 0), 1);
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
    if (lane == 0) notify_dependants(q, total, 0, id, x, y, mb_w, mb_h);
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
// Only the live part of a scratch is parked (enc_mb.cuh: kParkCore, + pred_y for stage C): slot = kParkSlot bytes
constexpr int kStashU4 = kParkSlot / 16, kCoreU4 = kParkCore / 16;
static_assert(kParkSlot % 16 == 0 && kParkCore % 16 == 0, "parked ranges are copied as uint4");
// second parked range of a macroblock that continues at `stage`: offset (uint4 units) and length
__device__ __forceinline__ void park_extra(int stage, int* off, int* n) {
  if (stage == MBS_C) { *off = (int)(offsetof(MbScratch, pred_y) / 16); *n = 512 / 16; }
  else { *off = 0; *n = 0; }
}

// optional batch statistics (debug, B2H264_ENC_STATS): per ready list [batches, tasks, batch cycles]; [NQ] = leader wait cycles
__device__ unsigned long long g_batch_stats[NQ + 1][3];
// per list: cycles from the batch barrier (a pulled task: from the end of the warp's previous task) to the end of run_task, tasks
__device__ unsigned long long g_task_wall[NQ][2];
// per list and batch fill (tasks claimed, up to ENC_PULL x ENC_WPC for a pulled list): [batches, cycles]
constexpr int kMaxClaim = ENC_PULL * ENC_WPC;
__device__ unsigned long long g_fill_stats[NQ][kMaxClaim + 1][2];
extern "C" int b2h264_debug_task_wall(unsigned long long* out, int reset) {
  cudaError_t e = cudaMemcpyFromSymbol(out, g_task_wall, sizeof(g_task_wall));
  if (e == cudaSuccess && reset) { unsigned long long z[NQ][2] = {}; e = cudaMemcpyToSymbol(g_task_wall, z, sizeof(z)); }
  return (int)e;
}
// out: NQ x (*wpc + 1) x 2 words, *wpc = the largest batch fill (ENC_PULL x ENC_WPC)
extern "C" int b2h264_debug_fill_stats(unsigned long long* out, int* n_lists, int* wpc, int reset) {
  *n_lists = NQ; *wpc = kMaxClaim;
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
__device__ __forceinline__ void run_task(const StreamFrame* sf, const MbSched& q, MbScratch& s, int id, int stage, int mb_w, int mb_h,
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
      notify_dependants(q, total, enc_list(sf[si].p.is_idr ? MBS_I : MBS_A), id, x, y, mb_w, mb_h);
      atomicAdd(ctl_done(q), 1);
    }
  } else {
    int xo, xn;
    park_extra(next, &xo, &xn);
    for (int i = lane; i < kCoreU4 + xn; i += 32) park[i] = i < kCoreU4 ? sc[i] : sc[xo + i - kCoreU4];
    __threadfence();
    __syncwarp();
    if (lane == 0) ready_push(q, total, enc_list(next), id);
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
// The short stage (A: ENC_PULL_LISTS) paid the batch barrier, the claim and the slowest warp once per ENC_WPC tasks of
// ~20 k cycles each.  A full batch of such a list claims up to ENC_PULL x ENC_WPC tasks: every warp starts on task `warp`
// together as before, then takes the next unstarted task of the block (a shared counter per slot) until the block is
// empty; the warps drift apart inside the stage, which costs nothing measurable there (DESIGN.md §2).  "The first worker
// has finished" becomes "a worker found the block empty" (counter > n).  List B stays one task per warp: its
// re-alignment points (mbk_batch_sync) count the batch's warps.
static_assert(!(ENC_PULL_LISTS & (1 << enc_list(MBS_B))), "stage B's re-alignment barriers need one task per warp");
static_assert(ENC_PULL >= 1, "a pulled batch holds up to ENC_PULL x ENC_WPC tasks");
struct BatchSlot { int k, base, n, pad; };
constexpr int kEncThreads = 32 * (ENC_WPC + 1);
__device__ __forceinline__ void enc_cta_barrier() { asm volatile("barrier.sync 1, %0;" ::"n"(kEncThreads) : "memory"); }

template <class Body>
__device__ __forceinline__ void run_stages(const StreamFrame* sf, int n_streams, const MbSched q, MbScratch& s, int stats, Body body) {
  __shared__ BatchSlot s_slot[2];
  __shared__ int s_ids[2][kMaxClaim];      // the claimed macroblocks of slot p, read off the ready list by the scheduler warp
  __shared__ int s_fin[2];                 // tasks of the batch in slot p that have finished
  __shared__ int s_next[2];                // next unstarted task of slot p (starts at the batch's warp count; > n: a warp found it empty)
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
          // the running batch nears its end: a worker has finished its task (one task per warp) or found the block empty
          const bool ending = run_n > ENC_WPC ? *reinterpret_cast<volatile int*>(&s_next[p ^ 1]) > run_n : fin > 0;
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
          const bool take = best >= 0 && (all_done || (full && (ending || best_avail >= 2 * ENC_WPC)));
          if (take) {
            int tail = 0;
#pragma unroll
            for (int kk = 0; kk < NQ; kk++) if (kk == best) { h = c[kk]; tail = c[NQ + kk]; }
            const int cap = (ENC_PULL_LISTS >> best) & 1 ? kMaxClaim : ENC_WPC;
            bool got = false;
            for (;;) {                     // a lost race returns the new head: claim from there instead of looking at every list again
              n = min(cap, tail - h);
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
          __nanosleep(all_done ? 100 : ending ? 400 : 1500);
        }
        s_slot[p].k = k; s_slot[p].base = h; s_slot[p].n = n;
        s_fin[p] = 0;
        s_next[p] = min(n, ENC_WPC);
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
        for (int i = lane; i < nn; i += 32) {
          int id;
          while ((id = ld_volatile(q.queue + (size_t)kk * total + s_slot[p].base + i)) < 0) {}
          s_ids[p][i] = id;
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
  // One loop and one run_task call site for the first and the pulled tasks: a task loop nested in the batch loop, or k and
  // n kept in registers across the inlined body, cost the kernel more spills.
  int p = 0, prev_k = -1, prev_n = 0, t = -1;        // t >= 0: the task of the batch in slot p this warp runs next
  long long t_prev = 0;
  for (;;) {
    if (t < 0) {
      enc_cta_barrier();
      if (stats && threadIdx.x == 0) {
        const long long tc = clock64();
        if (prev_k >= 0) {
          const unsigned long long dt = (unsigned long long)(tc - t_prev);  // barrier to barrier: the batch plus whatever the claim left exposed
          atomicAdd(&g_batch_stats[prev_k][0], 1ull);
          atomicAdd(&g_batch_stats[prev_k][1], (unsigned long long)prev_n);
          atomicAdd(&g_batch_stats[prev_k][2], dt);
          atomicAdd(&g_fill_stats[prev_k][min(prev_n, kMaxClaim)][0], 1ull);
          atomicAdd(&g_fill_stats[prev_k][min(prev_n, kMaxClaim)][1], dt);
        }
        t_prev = tc; prev_k = s_slot[p].k; prev_n = s_slot[p].n;
      }
      if (s_slot[p].n < 0) break;
      t = warp;
    }
    const int k = s_slot[p].k, n = s_slot[p].n;
    if (t < n) {
      const long long t_task = stats ? clock64() : 0;
      run_task(sf, q, s, s_ids[p][t], enc_stage(k), mb_w, mb_h, total, min(n, ENC_WPC) /* batch_n: warps, not tasks */, body);
      const int kt = ld_volatile(&s_slot[p].k), nt = ld_volatile(&s_slot[p].n);
      if (lane == 0) atomicAdd(&s_fin[p], 1);
      if (stats && lane == 0) { atomicAdd(&g_task_wall[kt][0], (unsigned long long)(clock64() - t_task)); atomicAdd(&g_task_wall[kt][1], 1ull); }
      if (nt > ENC_WPC) {                               // a pulled block: take its next unstarted task
        int tn = 0;
        if (lane == 0) tn = atomicAdd(&s_next[p], 1);
        t = __shfl_sync(MBK_FULL, tn, 0);
        if (t < nt) continue;
      }
    }
    t = -1;                                             // this warp is done with the batch: meet the others at the barrier
    p ^= 1;
  }
}

// MB (0,0) of every stream is ready.  The encoder (n_lists = NQ) puts IDR pictures on list I and P pictures on list A, the
// decoder (n_lists = 1) every stream on list 0, which is list A's index.
static_assert(enc_list(MBS_A) == 0, "list 0 is list A");
__global__ void k_ready_init(MbSched q, const StreamFrame* __restrict__ sf, int n_streams, int n_mb, int n_lists) {
  if (threadIdx.x != 0) return;
  int na = 0, ni = 0;
  const int total = n_streams * n_mb;
  for (int s = 0; s < n_streams; s++) {
    if (n_lists > 1 && sf[s].p.is_idr) q.queue[(size_t)enc_list(MBS_I) * total + ni++] = s * n_mb;
    else q.queue[(size_t)enc_list(MBS_A) * total + na++] = s * n_mb;
  }
  for (int k = 0; k < 32 * (n_lists + 1); k++) q.ctl[k] = 0;
  *ctl_tail(q, enc_list(MBS_A)) = na;
  if (n_lists > 1) *ctl_tail(q, enc_list(MBS_I)) = ni;
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

// dynamic shared memory of the macroblock kernels: ENC_WPC scratches from a 128-byte aligned base (+128 bytes of slack)
constexpr size_t kScratchSmem = sizeof(MbScratch) * DEC_WPC + 128;          // DEC_WPC >= ENC_WPC
static_assert(DEC_WPC >= ENC_WPC, "one scratch area size for both kernels");
__device__ __forceinline__ MbScratch& my_scratch(uint8_t* smem) {
  const uintptr_t a = (reinterpret_cast<uintptr_t>(smem) + 127) & ~uintptr_t(127);
  return reinterpret_cast<MbScratch*>(a)[threadIdx.x >> 5];      // (the encode kernel's scheduler warp gets one it never touches)
}

// tm_ref: reference luma planes of all streams (x, y from the padded origin, z = stream); stage B stages its
// search window out of it with one bulk tensor copy per macroblock (enc_inter.cuh: win_issue / win_wait).
// has_window = 0: there is no such descriptor, the search reads the reference plane directly.
// stats: B2H264_ENC_STATS, cycle and batch counters (g_enc_stats, g_batch_stats, g_task_wall, g_fill_stats).
__global__ void __launch_bounds__(kEncThreads, 1) k_encode_mbs(const StreamFrame* __restrict__ sf, int n_streams, MbSched q, int stats,
                                                               const __grid_constant__ CUtensorMap tm_ref, int has_window) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ WinBar s_wbar[ENC_WPC];
  MbScratch& s = my_scratch(smem);
  WinBar* wb = &s_wbar[min((int)(threadIdx.x >> 5), ENC_WPC - 1)];
  if ((threadIdx.x & 31) == 0 && threadIdx.x < 32 * ENC_WPC) {
    wb->phase = 0;
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"((uint32_t)__cvta_generic_to_shared(&wb->bar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const void* tmap = has_window ? (const void*)&tm_ref : nullptr;
  run_stages(sf, n_streams, q, s, stats, [&](const StreamFrame& F, int x, int y, int stage, int batch_n) {
    const long long t0 = stats ? clock64() : 0;
    mb_ctx(s.ctx, F.p, F.f, x, y);
    if ((threadIdx.x & 31) == 0) { s.ctx.tmap_ref = tmap; s.ctx.wbar = wb; s.ctx.batch_n = batch_n; }
    __syncwarp();
    const int next = mb_run_stage(s.ctx, s, stage);
    if (stats && (threadIdx.x & 31) == 0) {          // cycles and count per stage
      atomicAdd(&g_enc_stats[2 * stage], (unsigned long long)(clock64() - t0));
      atomicAdd(&g_enc_stats[2 * stage + 1], 1ull);
    }
    return next;
  });
}

// In-loop deblocking: ONE CTA PER PICTURE, ONE WARP PER MACROBLOCK ROW AT A TIME.  The warps of a CTA take the rows of
// their picture round-robin; a warp walks its row left to right and only has to stay two macroblocks behind the row above
// (MB(x, y) needs (x - 1, y) — the warp's own previous step — and (x + 1, y - 1)).  Progress is one word per warp in shared
// memory, ordered with CTA-scope release / acquire: the whole wavefront of a picture lives on one SM, so no GPU-scope fence,
// no global counter and no L1 invalidation are needed (the round-1 version spread the rows of all pictures over the chip
// and paid two GPU-scope fences per macroblock; the staged filter waited mostly for its loads).  Per macroblock a warp
// fetches the next macroblock's own samples and records asynchronously before it filters this one (deblock_row_t), so only
// the 4 rows above wait on another warp.  Launched behind the encode kernel.  (Deblocking CTAs resident beside the encode
// kernel, following its wavefront, hid the filter but slowed the encode kernel by more: DESIGN.md §7.)
#define DBK_MAX_WARPS 32
#define DBK_WARPS_SHARED 17       // two CTAs per SM: 68-row (1080p) pictures give every warp 4 rows
__device__ __forceinline__ int ld_acquire_cta(const int* p) {
  int v;
  asm volatile("ld.acquire.cta.shared.b32 %0, [%1];" : "=r"(v) : "r"((unsigned)__cvta_generic_to_shared(p)) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_cta(int* p, int v) {
  asm volatile("st.release.cta.shared.b32 [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(p)), "r"(v) : "memory");
}
// __maxnreg__(56): two CTAs of DBK_WARPS_SHARED warps fit the register file (60 registers, the uncapped count, allow one)
template <bool BSL = false /* decoder: the pictures may hold B macroblocks (two reference lists in the strength rule) */>
__global__ void __maxnreg__(56) k_deblock_pictures(const StreamFrame* __restrict__ sf) {
  using Tile = typename std::conditional<BSL, DbkTileB, DbkTile>::type;
  extern __shared__ __align__(16) uint8_t dbk_smem[];
  __shared__ int s_done[DBK_MAX_WARPS];                    // macroblocks finished by each warp, counted as row * mb_w + x + 1
  const int nw = blockDim.x >> 5, w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const StreamFrame& F = sf[blockIdx.x];
  const int mb_w = F.p.mb_w, mb_h = F.p.mb_h;
  Tile* t = reinterpret_cast<Tile*>(dbk_smem) + 2 * w;
  if (threadIdx.x < DBK_MAX_WARPS) s_done[threadIdx.x] = 0;
  __syncthreads();
  const int* above = &s_done[w > 0 ? w - 1 : nw - 1];
  int* mine = &s_done[w];
  for (int row = w; row < mb_h; row += nw) {
    const int base = (row - 1) * mb_w;
    deblock_row_t<BSL>(F.p, F.f, row, t,
        [&](int need) {
          if (lane == 0)
            while (ld_acquire_cta(above) < base + need) __nanosleep(32);
          __syncwarp();
        },
        [&](int x) {
          __syncwarp();
          if (lane == 0) st_release_cta(mine, base + mb_w + x + 1);
        });
  }
}
template <bool BSL>
static size_t dbk_tile_bytes() { return sizeof(typename std::conditional<BSL, DbkTileB, DbkTile>::type); }

// ---- decoder construct path (groundwork of the next SURVEY row: dec_mb.cuh) ------------------------------------------------
// One warp reconstructs one macroblock from its parsed record (h264_parse.h); the macroblocks of all streams are
// scheduled by the same dependency rule and ready-list structure as the encoder's (left + top-right done), on one list
// that every warp pops a macroblock at a time from (run_mbs).
__global__ void __launch_bounds__(32 * DEC_WPC) k_decode_mbs(const StreamFrame* __restrict__ sf, int n_streams, MbSched q,
                                                            const MbOut* __restrict__ recs, const DecMbAux* __restrict__ aux) {
  extern __shared__ __align__(128) uint8_t smem[];
  MbScratch& s = my_scratch(smem);
  run_mbs(sf, n_streams, q, [&](const StreamFrame& F, int x, int y) {
    const int n_mb = F.p.mb_w * F.p.mb_h, si = (int)(&F - sf);
    const size_t r = (size_t)si * n_mb + y * F.p.mb_w + x;
    dec_one_mb(F.p, F.f, s, x, y, recs[r], aux[r]);
  });
}

// ---- border replication, all planes of all streams in two launches (blockIdx.z = 3 * stream + plane) -----------
struct ExpandPlane { uint8_t* pic; int stride, w, h, pad; };
__device__ __forceinline__ ExpandPlane expand_plane(const StreamFrame* sf) {
  const StreamFrame& F = sf[blockIdx.z / 3];
  const int pl = blockIdx.z % 3;
  return {F.f.rec[pl], pl ? F.p.rec_stride_c : F.p.rec_stride_y, (pl ? 8 : 16) * F.p.mb_w, (pl ? 8 : 16) * F.p.mb_h, pl ? 16 : 32};
}
__global__ void k_expand_lr_batch(const StreamFrame* __restrict__ sf) {
  const ExpandPlane e = expand_plane(sf);
  expand_rows(e.pic, e.stride, e.w, e.h, e.pad);
}
__global__ void k_expand_tb_batch(const StreamFrame* __restrict__ sf) {
  const ExpandPlane e = expand_plane(sf);
  expand_bands(e.pic, e.stride, e.w, e.h, e.pad);
}
static int launch_expand(const StreamFrame* d_sf, int n_streams, int mb_w, int mb_h, cudaStream_t st) {
  k_expand_lr_batch<<<dim3((mb_h * 16 + 7) / 8, 1, 3 * n_streams), dim3(32, 8), 0, st>>>(d_sf);
  const int rc = b2h264_launched();
  if (rc) return rc;
  k_expand_tb_batch<<<dim3((mb_w * 16 + 64 + 127) / 128, 4, 3 * n_streams), dim3(128), 0, st>>>(d_sf);
  return b2h264_launched();
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

// ---- scheduler workspace (ints), one layout for the encoder (NQ ready lists) and the decoder (one list) ------------------
//   dep[total]                notifications received per macroblock (total = n_streams * n_mb)
//   queue[n_lists][total]     ready lists, -1 = slot not yet written
//   ctl[32 * (n_lists + 1)]   control lines (MbSched)
// Every part starts on a 128-byte line.  Per picture [0, queue) is zeroed and the lists are set to -1 (sched_ws_reset); the
// control lines are written by k_ready_init.
struct SchedWs { size_t dep, queue, ctl, ints; };
static size_t ws_lines(size_t n) { return (n + 31) / 32 * 32; }
static SchedWs sched_ws(int n_streams, int mb_w, int mb_h, int n_lists) {
  const size_t total = (size_t)n_streams * mb_w * mb_h;
  SchedWs w;
  w.dep = 0;
  w.queue = w.dep + ws_lines(total);
  w.ctl = w.queue + ws_lines((size_t)n_lists * total);
  w.ints = w.ctl + 32 * ((size_t)n_lists + 1);
  return w;
}
static void sched_ws_reset(int* ws, const SchedWs& w, cudaStream_t st) {
  cudaMemsetAsync(ws, 0, w.queue * sizeof(int), st);
  cudaMemsetAsync(ws + w.queue, 0xff, (w.ctl - w.queue) * sizeof(int), st);
}
size_t enc_sched_ints(int n_streams, int mb_w, int mb_h) { return sched_ws(n_streams, mb_w, mb_h, NQ).ints; }
size_t enc_stash_bytes(int n_streams, int mb_h) { return (size_t)n_streams * mb_h * kStashU4 * sizeof(uint4); }

static MbSched make_sched(int* ws, const SchedWs& w, void* stash) {
  MbSched q;
  q.dep = ws + w.dep;
  q.queue = ws + w.queue;
  q.ctl = ws + w.ctl;
  q.stash = reinterpret_cast<uint4*>(stash);
  return q;
}

// One CTA per picture.  With enough pictures for two CTAs per SM a CTA has DBK_WARPS_SHARED warps; a small batch (a single
// encoder or decoder object) has the SMs to itself and gives each picture DBK_MAX_WARPS warps, which shortens the row pipeline
// of a picture.  n_warps > 0 replaces that choice (still capped at mb_h); *warps_used receives the count launched.
template <bool BSL>
static int launch_deblock_t(const StreamFrame* d_sf, int n_streams, int mb_h, cudaStream_t st, int n_warps = 0, int* warps_used = nullptr) {
  static std::mutex mu;
  static int sms_dev[64];
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  int sms;
  {
    std::lock_guard<std::mutex> lock(mu);
    if (!sms_dev[dev]) {
      cudaFuncSetAttribute(k_deblock_pictures<BSL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(2 * DBK_MAX_WARPS * dbk_tile_bytes<BSL>()));
      cudaDeviceGetAttribute(&sms_dev[dev], cudaDevAttrMultiProcessorCount, dev);
      if (sms_dev[dev] < 1) sms_dev[dev] = 1;
    }
    sms = sms_dev[dev];
  }
  int nw = n_warps > 0 ? n_warps : 2 * n_streams > sms ? DBK_WARPS_SHARED : DBK_MAX_WARPS;
  if (nw > mb_h) nw = mb_h;
  if (warps_used) *warps_used = nw;
  k_deblock_pictures<BSL><<<n_streams, 32 * nw, 2 * nw * dbk_tile_bytes<BSL>(), st>>>(d_sf);
  return b2h264_launched();
}

// Test hook (not part of the public headers): deblocks n pictures given as device planes and records, through the same
// launcher as the encoder and the decoder.  planes[3 * i + pl] = sample (0, 0) of plane pl of picture i; geo[4 * i] = luma
// stride, chroma stride, mb_w, mb_h; mbi[i] = its MbInfo records, aux_b[i] = its DecMbAuxB records or NULL (aux_b itself may
// be NULL).  dec_mode 1 reads the slice control from the records, 0 uses idc / off_a / off_b.  bsl selects the two-list
// instantiation (required for B records and the 8x8 transform).  n_warps 0 lets the launcher choose.  Returns -1 without
// launching when an argument does not fit the kernel's accesses (16-byte luma rows, 8-byte chroma rows, 16-byte aligned
// plane origins); otherwise the CUDA status after the kernel finished, with the warp count in *warps_used.
extern "C" int b2h264_debug_deblock_pictures(int n, uint8_t* const* planes, const int* geo, MbInfo* const* mbi,
                                             const DecMbAuxB* const* aux_b, int dec_mode, int idc, int off_a, int off_b, int bsl,
                                             int n_warps, int* warps_used) {
  if (n < 1 || !planes || !geo || !mbi || n_warps < 0 || n_warps > DBK_MAX_WARPS) return -1;
  int max_h = 1;
  for (int i = 0; i < n; i++) {
    const int sy = geo[4 * i], sc = geo[4 * i + 1], mb_w = geo[4 * i + 2], mb_h = geo[4 * i + 3];
    if (mb_w < 1 || mb_h < 1 || sy % 16 || sc % 8 || sy < 16 * mb_w || sc < 8 * mb_w || !mbi[i]) return -1;
    for (int pl = 0; pl < 3; pl++)
      if (!planes[3 * i + pl] || reinterpret_cast<uintptr_t>(planes[3 * i + pl]) % 16) return -1;
    if (aux_b && aux_b[i] && !bsl) return -1;
    if (mb_h > max_h) max_h = mb_h;
  }
  int rc = enc_upload_deblock_tables();            // as b2h264_enc_create / b2h264_dec_create do
  if (rc) return rc;
  std::vector<StreamFrame> h(n);
  memset(h.data(), 0, sizeof(StreamFrame) * n);
  for (int i = 0; i < n; i++) {
    EncFrameParams& p = h[i].p;
    p.rec_stride_y = geo[4 * i]; p.rec_stride_c = geo[4 * i + 1]; p.mb_w = geo[4 * i + 2]; p.mb_h = geo[4 * i + 3];
    p.dec_mode = dec_mode; p.dbk_idc = idc; p.dbk_off_a = off_a; p.dbk_off_b = off_b;
    for (int pl = 0; pl < 3; pl++) h[i].f.rec[pl] = planes[3 * i + pl];
    h[i].f.mbi = mbi[i];
    h[i].f.dec_aux_b = aux_b ? aux_b[i] : nullptr;
  }
  DeviceBuf<StreamFrame> d_sf;
  rc = (int)d_sf.alloc(sizeof(StreamFrame) * n);
  if (rc) return rc;
  rc = (int)cudaMemcpy(d_sf.get(), h.data(), sizeof(StreamFrame) * n, cudaMemcpyHostToDevice);
  int used = 0;
  if (!rc)
    rc = bsl ? launch_deblock_t<true>(d_sf.get(), n, max_h, 0, n_warps, &used) : launch_deblock_t<false>(d_sf.get(), n, max_h, 0, n_warps, &used);
  if (!rc) rc = (int)cudaDeviceSynchronize();
  if (warps_used) *warps_used = used;
  return rc;
}
// Test hook (not part of the public headers): stage B's residual step (inter_residual_pass) on n cases, one warp each.  Host
// arrays: src_pred[768 * i] = case i's source (luma 16x16, Cb 8x8, Cr 8x8, dense) then its prediction in the same layout;
// qp[i] = its luma QP (the chroma QP follows from the table, as in the encoder); out[kInterResOut * i] = the MbOut record
// (896 bytes: levels, chroma DC; the rest zero), MbInfo::nnz (24), MbInfo::cbp, 7 zero bytes, the reconstruction (luma 16x16,
// Cb 8x8, Cr 8x8).  Returns -1 without launching for a bad argument (stage_hooks.cuh), else the CUDA status.
__global__ void k_debug_inter_residual(const uint8_t* in, const int* qp, uint8_t* out) {
  extern __shared__ __align__(128) uint8_t smem[];
  MbScratch& s = *reinterpret_cast<MbScratch*>(smem);
  const int i = blockIdx.x;
  for (int w = threadIdx.x; w < (int)(sizeof(MbScratch) / 4); w += 32) reinterpret_cast<uint32_t*>(&s)[w] = 0;
  __syncwarp();
  inter_residual_case(in + 768 * i, qp[i], out + (size_t)kInterResOut * i, s);
}
extern "C" int b2h264_debug_inter_residual(int n, const uint8_t* src_pred, const int* qp, uint8_t* out) {
  if (!inter_residual_args_ok(n, src_pred, qp, out)) return -1;
  DeviceBuf<uint8_t> d_in, d_out;
  DeviceBuf<int> d_qp;
  int rc = (int)d_in.alloc((size_t)768 * n);
  if (!rc) rc = (int)d_qp.alloc(sizeof(int) * n);
  if (!rc) rc = (int)d_out.alloc((size_t)kInterResOut * n);
  if (!rc) rc = (int)cudaMemcpy(d_in.get(), src_pred, (size_t)768 * n, cudaMemcpyHostToDevice);
  if (!rc) rc = (int)cudaMemcpy(d_qp.get(), qp, sizeof(int) * n, cudaMemcpyHostToDevice);
  if (!rc) {
    k_debug_inter_residual<<<n, 32, sizeof(MbScratch)>>>(d_in.get(), d_qp.get(), d_out.get());
    rc = b2h264_launched();
  }
  if (!rc) rc = (int)cudaMemcpy(out, d_out.get(), (size_t)kInterResOut * n, cudaMemcpyDeviceToHost);
  return rc;
}
// Test hook (not part of the public headers): the intra tail (md_i16x16, then intra_mb_finish, as stage I runs them) on n
// cases, one warp each.  Host arrays: in[kIntraTailIn * i] = case i's reconstruction tile with its neighbour samples (RecTile),
// its source (luma 16x16, Cb 8x8, Cr 8x8, dense), int32 QP / neighbour availability (NB_* bits) / LOW complexity / cost limit
// of the I4x4 try (< 0: the I16x16 cost), then int8 I4x4 modes of the left neighbour's right column and of the top
// neighbour's bottom row (a neighbour whose first entry is < 0 is not I4x4), 8 bytes padding.  out[kIntraTailOut * i] = the
// MbOut record, the MbInfo record, int32 cost limit used / I4x4 cost returned / lambda / 0, the tile.  Returns -1 without
// launching for a bad argument (stage_hooks.cuh), else the CUDA status.
__global__ void k_debug_intra_tail(const uint8_t* in, int32_t* sad, uint8_t* out) {
  extern __shared__ __align__(128) uint8_t smem[];
  MbScratch& s = *reinterpret_cast<MbScratch*>(smem);
  const int i = blockIdx.x;
  for (int w = threadIdx.x; w < (int)(sizeof(MbScratch) / 4); w += 32) reinterpret_cast<uint32_t*>(&s)[w] = 0;
  __syncwarp();
  intra_tail_case(in + (size_t)kIntraTailIn * i, sad + i, out + (size_t)kIntraTailOut * i, s);
}
extern "C" int b2h264_debug_intra_tail(int n, const uint8_t* in, uint8_t* out) {
  if (!intra_tail_args_ok(n, in, out)) return -1;
  DeviceBuf<uint8_t> d_in, d_out;
  DeviceBuf<int32_t> d_sad;
  int rc = (int)d_in.alloc((size_t)kIntraTailIn * n);
  if (!rc) rc = (int)d_sad.alloc(sizeof(int32_t) * n);
  if (!rc) rc = (int)d_out.alloc((size_t)kIntraTailOut * n);
  if (!rc) rc = (int)cudaMemcpy(d_in.get(), in, (size_t)kIntraTailIn * n, cudaMemcpyHostToDevice);
  if (!rc) {
    k_debug_intra_tail<<<n, 32, sizeof(MbScratch)>>>(d_in.get(), d_sad.get(), d_out.get());
    rc = b2h264_launched();
  }
  if (!rc) rc = (int)cudaMemcpy(out, d_out.get(), (size_t)kIntraTailOut * n, cudaMemcpyDeviceToHost);
  return rc;
}
// Test hook (not part of the public headers): stage B's motion search of one partition shape on n macroblock jobs, one warp
// each, in stage B's order: me_start_point -> win_issue -> win_wait, me_partition for every partition, then me_refine and
// mc_chroma_part for every partition (the first refinement may stage out of the window; it clears win_ok).
// d_planes (DEVICE memory): job i's padded, expanded reference planes at d_planes + i * set_bytes: Y (stride_y, 16 mb_h + 64
// rows, sample (0, 0) at 32 rows + 32), then Cb and Cr (stride_c, 8 mb_h + 32 rows, sample (0, 0) at 16 rows + 16).
// window = 1 stages the search window with the bulk tensor copy out of a tensor map over those planes (z = job), as the
// encoder does; 0 passes no map (the searches read the planes, as after a skip candidate).
// jobs[kMeJobIn * i] (host), int32: mb_w, mb_h, stride_y, stride_c, mv_range, mbx, mby, qp, LOW complexity, 16x16 predictor
// (x, y: places the window), shape (0 16x16, 1 16x8, 2 8x16, 3 8x8); per partition p (in the order stage B visits them) at
// word 12 + 16 p: search predictor (x, y), candidate count (0..5), sad_pred, five candidates (x, y), refinement predictor
// (x, y); padding to word 80; then the current macroblock's luma (16 x 16, dense).  Vectors in quarter samples.
// out[kMeJobOut * i] (host), int32: per partition p at word 12 p: the MeState after the search (mv x, y, mvp x, y, sad_cost,
// satd_cost, satd, ref - luma sample (0, 0) in bytes), then mv x, y and satd_cost after the refinement, 0; at word 48:
// win_x0, win_y0, win_ok as issued (win_x0 / win_y0 0 without a window); padding to word 64; then the luma prediction
// (16 x 16) and the chroma prediction (Cb 8 x 8, Cr 8 x 8).
// Returns -1 without launching for a bad argument (stage_hooks.cuh; and see below), else the CUDA status.
__global__ void k_debug_me_partitions(const uint8_t* planes, long long set_bytes, const uint8_t* jobs, uint8_t* out,
                                      const __grid_constant__ CUtensorMap tm_ref, int has_window) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ WinBar wb;
  MbScratch& s = my_scratch(smem);
  const int i = blockIdx.x;
  for (int w = threadIdx.x; w < (int)(sizeof(MbScratch) / 4); w += 32) reinterpret_cast<uint32_t*>(&s)[w] = 0;
  if (threadIdx.x == 0) {
    wb.phase = 0;
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"((uint32_t)__cvta_generic_to_shared(&wb.bar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  me_partitions_case(i, planes + (size_t)set_bytes * i, jobs + (size_t)kMeJobIn * i, out + (size_t)kMeJobOut * i, s,
                     has_window ? (const void*)&tm_ref : nullptr, &wb);
}
extern "C" int b2h264_debug_me_partitions(int n, const uint8_t* d_planes, long long set_bytes, const uint8_t* jobs, int window,
                                          uint8_t* out) {
  if (!me_partitions_args_ok(n, d_planes, set_bytes, jobs, out)) return -1;
  // Device only: one tensor map covers the planes of every job, so the jobs share stride_y, stride_c and mb_h and the sets
  // start on 16-byte boundaries; the window copy needs a luma stride that is a multiple of 16 and a chroma one of 8.
  const int32_t* J0 = reinterpret_cast<const int32_t*>(jobs);
  if (set_bytes % 16) return -1;
  for (int i = 0; i < n; i++) {
    const int32_t* J = reinterpret_cast<const int32_t*>(jobs + (size_t)kMeJobIn * i);
    if (J[2] % 16 || J[3] % 8 || J[2] != J0[2] || J[3] != J0[3] || J[1] != J0[1]) return -1;
  }
  alignas(64) CUtensorMap tm;
  memset(&tm, 0, sizeof(tm));
  if (window) {
    const int sy = J0[2], rows = 16 * J0[1] + 64;
    if (b2h264_make_tmap_planes(&tm, d_planes, (uint64_t)sy, (uint64_t)rows, (uint64_t)n, (uint64_t)sy, (uint64_t)set_bytes, WIN_W, WIN_H))
      return -1;
  }
  DeviceBuf<uint8_t> d_jobs, d_out;
  int rc = (int)d_jobs.alloc((size_t)kMeJobIn * n);
  if (!rc) rc = (int)d_out.alloc((size_t)kMeJobOut * n);
  if (!rc) rc = (int)cudaMemcpy(d_jobs.get(), jobs, (size_t)kMeJobIn * n, cudaMemcpyHostToDevice);
  if (!rc) {
    k_debug_me_partitions<<<n, 32, sizeof(MbScratch) + 128>>>(d_planes, set_bytes, d_jobs.get(), d_out.get(), tm, window != 0);
    rc = b2h264_launched();
  }
  if (!rc) rc = (int)cudaMemcpy(out, d_out.get(), (size_t)kMeJobOut * n, cudaMemcpyDeviceToHost);
  return rc;
}
// Test hook (not part of the public headers): stage A's P-skip test on n macroblock jobs, one warp each, in stage A's order:
// fill_inter_cache -> predict_sad_skip -> pskip_enc.
// planes (host): ONE set of reference planes that every job reads, laid out for the job's own geometry: Y (stride_y, 16 mb_h
// + 64 rows, sample (0, 0) at 32 rows + 32), then Cb and Cr (stride_c, 8 mb_h + 32 rows, sample (0, 0) at 16 rows + 16).  The
// hook does not expand the borders: whatever the padding holds is read.
// jobs[kSkipJobIn * i] (host), int32: mb_w, mb_h, stride_y, stride_c, mbx, mby, qp, LOW complexity, neighbour availability
// (NB_* bits, replaces the one mb_ctx derives from the position), ref_is_p, the co-located macroblock's type and skip SAD;
// per neighbour k (0 top-left, 1 top, 2 top-right, 3 left) at word 12 + 5 k: mb_type, vector (x, y, quarter samples, every 4x4
// block), SAD cost, skip SAD; padding to word 32; then the current macroblock (Y 16 x 16, Cb 8 x 8, Cr 8 x 8, dense).
// out[kSkipJobOut * i] (host), int32: ok, skip vector (x, y), the SAD predictor used, cost_luma, cost_skip, the macroblock's
// sad_cost slot (kSkipSadUnset unless pskip_enc wrote it), 0; then s.skip_pred (384 bytes).
// Returns -1 without launching for a bad argument (stage_hooks.cuh), else the CUDA status.
__global__ void k_debug_skip_test(const uint8_t* planes, const uint8_t* jobs, int32_t* sad, uint8_t* out) {
  extern __shared__ __align__(128) uint8_t smem[];
  MbScratch& s = my_scratch(smem);
  const int i = blockIdx.x;
  for (int w = threadIdx.x; w < (int)(sizeof(MbScratch) / 4); w += 32) reinterpret_cast<uint32_t*>(&s)[w] = 0;
  __syncwarp();
  skip_test_case(jobs + (size_t)kSkipJobIn * i, planes, sad + i, out + (size_t)kSkipJobOut * i, s);
}
extern "C" int b2h264_debug_skip_test(int n, const uint8_t* planes, long long set_bytes, const uint8_t* jobs, uint8_t* out) {
  if (!skip_test_args_ok(n, planes, set_bytes, jobs, out)) return -1;
  DeviceBuf<uint8_t> d_planes, d_jobs, d_out;
  DeviceBuf<int32_t> d_sad;
  int rc = (int)d_planes.alloc((size_t)set_bytes);
  if (!rc) rc = (int)d_jobs.alloc((size_t)kSkipJobIn * n);
  if (!rc) rc = (int)d_sad.alloc(sizeof(int32_t) * n);
  if (!rc) rc = (int)d_out.alloc((size_t)kSkipJobOut * n);
  if (!rc) rc = (int)cudaMemcpy(d_planes.get(), planes, (size_t)set_bytes, cudaMemcpyHostToDevice);
  if (!rc) rc = (int)cudaMemcpy(d_jobs.get(), jobs, (size_t)kSkipJobIn * n, cudaMemcpyHostToDevice);
  if (!rc) rc = (int)cudaMemset(d_sad.get(), kSkipSadUnset & 0xff, sizeof(int32_t) * n);
  if (!rc) {
    k_debug_skip_test<<<n, 32, sizeof(MbScratch) + 128>>>(d_planes.get(), d_jobs.get(), d_sad.get(), d_out.get());
    rc = b2h264_launched();
  }
  if (!rc) rc = (int)cudaMemcpy(out, d_out.get(), (size_t)kSkipJobOut * n, cudaMemcpyDeviceToHost);
  return rc;
}
static int launch_deblock(const StreamFrame* d_sf, int n_streams, int mb_h, cudaStream_t st, bool b_slices = false) {
  return b_slices ? launch_deblock_t<true>(d_sf, n_streams, mb_h, st) : launch_deblock_t<false>(d_sf, n_streams, mb_h, st);
}

int enc_launch_frame(const StreamFrame* d_sf, const uint8_t* const* d_src, int n_streams, int w, int h, int mb_w, int mb_h,
                     int* d_ws, void* d_stash, const void* tmap_ref, int fast_mode, cudaStream_t st) {
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
  const SchedWs ws = sched_ws(n_streams, mb_w, mb_h, NQ);
  sched_ws_reset(d_ws, ws, st);
  const MbSched qe = make_sched(d_ws, ws, d_stash);
  k_ready_init<<<1, 32, 0, st>>>(qe, d_sf, n_streams, mb_w * mb_h, NQ);
  int blocks = enc_grid_blocks();
  const int need = (total + ENC_WPC - 1) / ENC_WPC;
  if (blocks > need) blocks = need;
  static const int stats = getenv("B2H264_ENC_STATS") ? 1 : 0;
  CUtensorMap tm;
  memset(&tm, 0, sizeof(tm));
  if (tmap_ref) memcpy(&tm, tmap_ref, sizeof(tm));
  k_encode_mbs<<<blocks, kEncThreads, kScratchSmem, st>>>(d_sf, n_streams, qe, stats, tm, tmap_ref != nullptr);
  return b2h264_launched();
}

int enc_launch_deblock_expand(const StreamFrame* d_sf, int n_streams, int mb_w, int mb_h, cudaStream_t st) {
  int rc;
  if ((rc = launch_deblock(d_sf, n_streams, mb_h, st))) return rc;
  return launch_expand(d_sf, n_streams, mb_w, mb_h, st);
}

size_t dec_sched_ints(int n_streams, int mb_w, int mb_h) { return sched_ws(n_streams, mb_w, mb_h, 1).ints; }
int dec_launch_frame(const StreamFrame* d_sf, int n_streams, int mb_w, int mb_h, int* d_ws, const MbOut* d_recs, const DecMbAux* d_aux, int deblock,
                     cudaStream_t st, int b_slices) {
  const int blocks_per_launch = dec_grid_blocks();
  int rc;
  const int total = n_streams * mb_w * mb_h;
  const SchedWs ws = sched_ws(n_streams, mb_w, mb_h, 1);
  sched_ws_reset(d_ws, ws, st);
  const MbSched qc = make_sched(d_ws, ws, nullptr);
  k_ready_init<<<1, 32, 0, st>>>(qc, d_sf, n_streams, mb_w * mb_h, 1);
  const int need = (total + DEC_WPC - 1) / DEC_WPC;
  k_decode_mbs<<<blocks_per_launch < need ? blocks_per_launch : need, 32 * DEC_WPC, kScratchSmem, st>>>(d_sf, n_streams, qc, d_recs, d_aux);
  if ((rc = b2h264_launched())) return rc;
  if (deblock && (rc = launch_deblock(d_sf, n_streams, mb_h, st, b_slices != 0))) return rc;
  return launch_expand(d_sf, n_streams, mb_w, mb_h, st);
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

// Test hook (not part of the public headers): the decoder's construct stage on given records, with the production hand-over and
// launches: pack_records_compact -> dec_launch_unpack, border replication of the reference pictures, dec_launch_frame without
// deblocking.  n streams of mb_w x mb_h macroblocks; host arrays, stream-major: recs / aux = n * mb_w * mb_h records, aux_b = as
// many list-1 records or NULL (required when a record is B), cqp_off[s] = chroma_qp_index_offset of stream s, refs = n * n_refs
// dense I420 pictures (16 mb_w x 16 mb_h luma) that become picture slots 0 .. n_refs - 1; the picture is decoded into slot n_refs.
// Out (host): planes = n padded pictures (Y: (16 mb_w + 64) x (16 mb_h + 64), sample (0, 0) at row 32, column 32; Cb, Cr:
// (8 mb_w + 32) x (8 mb_h + 32) at 16, 16), mbi = the n * mb_w * mb_h MbInfo records.  Returns -1 without launching for a bad
// argument (dec_records_check.h), else the CUDA status.
extern "C" int b2h264_debug_decode_records(int n, int mb_w, int mb_h, const int* cqp_off, const MbOut* recs, const DecMbAux* aux,
                                           const DecMbAuxB* aux_b, int n_refs, const uint8_t* refs, uint8_t* planes, MbInfo* mbi) {
  if (!dec_records_ok(n, mb_w, mb_h, cqp_off, recs, aux, aux_b, n_refs, refs, planes, mbi)) return -1;
  const int n_mb = mb_w * mb_h;
  bool has_b = false;
  for (size_t i = 0; i < (size_t)n * n_mb; i++) has_b = has_b || MBT_IS_B(recs[i].mb_type);
  const b2h264::PicLayout lay(mb_w, mb_h);
  const size_t pic_bytes = lay.bytes();
  const size_t slots = (size_t)n_refs + 1, dense = (size_t)n_mb * 384;
  DeviceBuf<uint8_t> d_pic, d_pack;
  DeviceBuf<int32_t> d_idx;
  DeviceBuf<int> d_ws;
  DeviceBuf<MbOut> d_recs;
  DeviceBuf<DecMbAux> d_aux;
  DeviceBuf<DecMbAuxB> d_aux_b;
  DeviceBuf<MbInfo> d_mbi;
  DeviceBuf<StreamFrame> d_sf;
  std::vector<uint8_t> pack((size_t)n * n_mb * sizeof(MbOut));
  std::vector<int32_t> idx((size_t)n * n_mb);
  std::vector<StreamFrame> h((size_t)n * n_refs);
  auto plane0 = [&](uint8_t* base, size_t s, size_t slot, int pl) { return base + (s * slots + slot) * pic_bytes + lay.plane0(pl); };
  int rc = (int)d_pic.alloc((size_t)n * slots * pic_bytes + 256);
  if (!rc) rc = (int)cudaMemset(d_pic.get(), 0, (size_t)n * slots * pic_bytes + 256);
  if (!rc) rc = (int)d_pack.alloc(pack.size());
  if (!rc) rc = (int)d_idx.alloc(idx.size() * sizeof(int32_t));
  if (!rc) rc = (int)d_recs.alloc((size_t)n * n_mb * sizeof(MbOut));
  if (!rc) rc = (int)d_aux.alloc((size_t)n * n_mb * sizeof(DecMbAux));
  if (!rc && has_b) rc = (int)d_aux_b.alloc((size_t)n * n_mb * sizeof(DecMbAuxB));
  if (!rc) rc = (int)d_mbi.alloc((size_t)n * n_mb * sizeof(MbInfo));
  if (!rc) rc = (int)cudaMemset(d_mbi.get(), 0, (size_t)n * n_mb * sizeof(MbInfo));
  if (!rc) rc = (int)d_sf.alloc(h.size() * sizeof(StreamFrame));
  if (!rc) rc = (int)d_ws.alloc(dec_sched_ints(n, mb_w, mb_h) * sizeof(int));
  // the reference pictures into their slots, then their borders as the decoder replicates them after decoding a picture
  for (size_t s = 0; s < (size_t)n && !rc; s++)
    for (size_t r = 0; r < (size_t)n_refs && !rc; r++) {
      const uint8_t* src = refs + (s * n_refs + r) * dense;
      for (int pl = 0; pl < 3 && !rc; pl++) {
        const int w = pl ? 8 * mb_w : 16 * mb_w, hh = pl ? 8 * mb_h : 16 * mb_h;
        rc = (int)cudaMemcpy2D(plane0(d_pic.get(), s, r, pl), lay.stride(pl), src + (pl ? (size_t)n_mb * 256 + (size_t)(pl - 1) * n_mb * 64 : 0), w, w, hh,
                               cudaMemcpyHostToDevice);
      }
      StreamFrame& F = h[s * n_refs + r];
      memset(&F, 0, sizeof(F));
      F.p.mb_w = mb_w; F.p.mb_h = mb_h; F.p.rec_stride_y = lay.stride_y; F.p.rec_stride_c = lay.stride_c;
      for (int pl = 0; pl < 3; pl++) F.f.rec[pl] = plane0(d_pic.get(), s, r, pl);
    }
  if (!rc) rc = (int)cudaMemcpy(d_sf.get(), h.data(), h.size() * sizeof(StreamFrame), cudaMemcpyHostToDevice);
  if (!rc) rc = launch_expand(d_sf.get(), n * n_refs, mb_w, mb_h, 0);
  if (!rc) rc = (int)cudaDeviceSynchronize();
  // the records: compact form per stream, unpacked on the device as b2h264_dec_decode does it
  for (int s = 0; s < n && !rc; s++) {
    const int units = b2h264::pack_records_compact(recs + (size_t)s * n_mb, n_mb, pack.data() + (size_t)s * n_mb * sizeof(MbOut), idx.data() + (size_t)s * n_mb);
    if (units > 0)
      rc = (int)cudaMemcpy(d_pack.get() + (size_t)s * n_mb * sizeof(MbOut), pack.data() + (size_t)s * n_mb * sizeof(MbOut), (size_t)units * 32, cudaMemcpyHostToDevice);
  }
  if (!rc) rc = (int)cudaMemcpy(d_idx.get(), idx.data(), idx.size() * sizeof(int32_t), cudaMemcpyHostToDevice);
  if (!rc) rc = dec_launch_unpack(d_pack.get(), (size_t)n_mb * sizeof(MbOut), d_idx.get(), d_recs.get(), n, n_mb, 0);
  if (!rc) rc = (int)cudaMemcpy(d_aux.get(), aux, (size_t)n * n_mb * sizeof(DecMbAux), cudaMemcpyHostToDevice);
  if (!rc && has_b) rc = (int)cudaMemcpy(d_aux_b.get(), aux_b, (size_t)n * n_mb * sizeof(DecMbAuxB), cudaMemcpyHostToDevice);
  for (int s = 0; s < n && !rc; s++) {
    StreamFrame& F = h[s];
    memset(&F, 0, sizeof(F));
    F.p.mb_w = mb_w; F.p.mb_h = mb_h; F.p.rec_stride_y = lay.stride_y; F.p.rec_stride_c = lay.stride_c;
    F.p.mv_range = 64; F.p.dec_mode = 1; F.p.dec_cqp_off = cqp_off[s];
    for (int pl = 0; pl < 3; pl++) { F.f.rec[pl] = plane0(d_pic.get(), s, n_refs, pl); F.f.ref[pl] = F.f.dpb0[pl] = plane0(d_pic.get(), s, 0, pl); }
    F.f.dpb_stride = (int64_t)pic_bytes;
    F.f.mbi = d_mbi.get() + (size_t)s * n_mb;
    F.f.dec_aux_b = has_b ? d_aux_b.get() + (size_t)s * n_mb : nullptr;
  }
  if (!rc) rc = (int)cudaMemcpy(d_sf.get(), h.data(), (size_t)n * sizeof(StreamFrame), cudaMemcpyHostToDevice);
  if (!rc) rc = dec_launch_frame(d_sf.get(), n, mb_w, mb_h, d_ws.get(), d_recs.get(), d_aux.get(), 0, 0, has_b ? 1 : 0);
  if (!rc) rc = (int)cudaDeviceSynchronize();
  for (int s = 0; s < n && !rc; s++)
    rc = (int)cudaMemcpy(planes + (size_t)s * pic_bytes, d_pic.get() + ((size_t)s * slots + n_refs) * pic_bytes, pic_bytes, cudaMemcpyDeviceToHost);
  if (!rc) rc = (int)cudaMemcpy(mbi, d_mbi.get(), (size_t)n * n_mb * sizeof(MbInfo), cudaMemcpyDeviceToHost);
  return rc;
}

extern "C" int b2h264_debug_enc_stats(unsigned long long* out16, int reset) {
  cudaError_t e = cudaMemcpyFromSymbol(out16, g_enc_stats, sizeof(g_enc_stats));
  if (e != cudaSuccess) return (int)e;
  if (reset) { unsigned long long z[16] = {0}; e = cudaMemcpyToSymbol(g_enc_stats, z, sizeof(z)); }
  return (int)e;
}
