// k_vpp.cu — pre-processing kernels in front of the macroblock pipeline (SURVEY.md 8f rank 3): the bilinear
// down-sampler that produces the lower spatial / simulcast layers from the source picture.
// Replaces (semantics of) DyadicBilinearDownsampler_c / ...Quarter... / ...OneThird... / GeneralBilinearFastDownsampler_c /
// GeneralBilinearAccurateDownsampler_c (codec/processing/src/downsample/downsamplefuncs.cpp:47-250) and the dispatch of
// CDownsampling::Process (downsample.cpp:143-300).  One thread per 4 destination samples of one row; a launch covers
// up to 24 destination planes (8 rungs x 3 planes of a picture, each with its own mode and geometry) of a range of pictures,
// so the work is a pure HBM stream:
// algorithmic bytes per destination sample = 4 source bytes (2x2) + 1 (modes 0, 3, 4), 4 of 16 / 4 of 9 source bytes + 1 (modes 1, 2).
#include "b2h264_internal.h"

namespace {

__device__ __forceinline__ uint32_t avg2x2(const uint8_t* p, int ss) {
  const int r1 = (p[0] + p[1] + 1) >> 1, r2 = (p[ss] + p[ss + 1] + 1) >> 1;
  return (uint32_t)((r1 + r2 + 1) >> 1);
}

struct LadderArgs {
  b2h264_ds_plane p[B2H264_LADDER_MAX_PLANES];
  int n, rows;
};

// destination samples x0 .. x0 + 3 (fewer at the row's end) of row y of plane a: s = the picture's source plane, d = &row[x0]
__device__ __forceinline__ void downsample4(const b2h264_ds_plane& a, const uint8_t* __restrict__ s, uint8_t* __restrict__ d, int x0, int y) {
  const int ss = a.src_stride;
  uint32_t v[4] = {0, 0, 0, 0};
  const int n = min(4, a.dst_w - x0);
  if (a.mode == 0) {      // half: 8 source bytes per row as one 8-byte load when both rows are 8-aligned and the 4 samples one word
    const uint8_t* p = s + (size_t)(2 * y) * ss + 2 * x0;
    if (n == 4 && ((reinterpret_cast<uintptr_t>(p) | (uintptr_t)ss) & 7) == 0 && (reinterpret_cast<uintptr_t>(d) & 3) == 0) {
      const uint2 r0 = *reinterpret_cast<const uint2*>(p), r1 = *reinterpret_cast<const uint2*>(p + ss);
      // bytes (0,1),(2,3) of each word: rounded average of neighbours = __vavgu4 of the word and itself shifted by 8
      const uint32_t h0a = __vavgu4(r0.x, r0.x >> 8), h0b = __vavgu4(r0.y, r0.y >> 8);
      const uint32_t h1a = __vavgu4(r1.x, r1.x >> 8), h1b = __vavgu4(r1.y, r1.y >> 8);
      const uint32_t va = __vavgu4(h0a, h1a), vb = __vavgu4(h0b, h1b);       // bytes 0 and 2 hold the results
      *reinterpret_cast<uint32_t*>(d) = (va & 0xff) | ((va >> 8) & 0xff00) | ((vb & 0xff) << 16) | ((vb << 8) & 0xff000000u);
      return;
    }
    for (int i = 0; i < n; i++) v[i] = avg2x2(p + 2 * i, ss);
  } else if (a.mode == 1 || a.mode == 2) {
    const int step = a.mode == 1 ? 4 : 3;
    const uint8_t* p = s + (size_t)(step * y) * ss + step * x0;
    for (int i = 0; i < n; i++) v[i] = avg2x2(p + step * i, ss);
  } else {
    const int bw = a.mode == 3 ? 16 : 15, bh = 15;
    const int yinv = (1 << (bh - 1)) + y * a.sy;
    const int yy = yinv >> bh, fv = yinv & ((1 << bh) - 1);
    const uint8_t* row = s + (size_t)yy * ss;
    for (int i = 0; i < n; i++) {
      const int j = x0 + i;
      const int xinv = (1 << (bw - 1)) + j * a.sx;
      const int xx = xinv >> bw, fu = xinv & ((1 << bw) - 1);
      if (y == a.dst_h - 1 || j == a.dst_w - 1) { v[i] = row[xx]; continue; }     // last row / column: nearest sample
      const uint32_t pa = row[xx], pb = row[xx + 1], pc = row[xx + ss], pd = row[xx + ss + 1];
      if (a.mode == 3) {
        const uint32_t Wd = 1u << bw, Hh = 1u << bh;
        uint32_t x = (((uint32_t)(Wd - 1 - fu)) * (Hh - 1 - fv) >> bw) * pa;
        x += (((uint32_t)fu) * (Hh - 1 - fv) >> bw) * pb;
        x += (((uint32_t)(Wd - 1 - fu)) * (uint32_t)fv >> bw) * pc;
        x += (((uint32_t)fu) * (uint32_t)fv >> bw) * pd;
        x >>= (bh - 1);
        x += 1;
        x >>= 1;
        v[i] = x > 255 ? 255 : x;
      } else {
        const long long S = 1 << 15;
        long long x = ((S - 1 - fu) * (S - 1 - fv) * pa + (long long)fu * (S - 1 - fv) * pb + (S - 1 - fu) * fv * pc + (long long)fu * fv * pd +
                       (1ll << 29)) >> 30;
        v[i] = (uint32_t)(x < 0 ? 0 : x > 255 ? 255 : x);
      }
    }
  }
  if (n == 4 && ((reinterpret_cast<uintptr_t>(d)) & 3) == 0) *reinterpret_cast<uint32_t*>(d) = v[0] | (v[1] << 8) | (v[2] << 16) | (v[3] << 24);
  else for (int i = 0; i < n; i++) d[i] = (uint8_t)v[i];
}

// one warp per destination row, 4 rows per block: grid y = the rows of all planes in descriptor order (concatenated), z = pictures
// lo, lo + 1, ...; each lane takes 4 samples per step along the row.  A warp finds its plane by the descriptors' row0 (a running sum
// of dst_h, in kernel-parameter space).  Whole rows per warp keep the block count at rows / 4 per picture: with a block per 256
// samples of a row (a third of the blocks idle on the ladder's narrow chroma rows) the 1080p ladder's nine planes of 256 pictures
// took 2.50 ms, against 1.31 ms this way (H100, DESIGN.md §7).
__global__ void __launch_bounds__(128) k_downsample_ladder(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, size_t dst_pitch,
                                                           size_t src_pitch, int lo, LadderArgs la) {
  const int row = blockIdx.y * 4 + (threadIdx.x >> 5);
  if (row >= la.rows) return;
  int k = 0;
  while (k + 1 < la.n && row >= la.p[k + 1].row0) k++;
  const b2h264_ds_plane& a = la.p[k];
  const int y = row - a.row0;
  const size_t pic = (size_t)lo + blockIdx.z;
  const uint8_t* s = src + pic * src_pitch + a.src_offset;
  uint8_t* d = dst + pic * dst_pitch + a.dst_offset + (size_t)y * a.dst_stride;
  for (int x0 = (threadIdx.x & 31) * 4; x0 < a.dst_w; x0 += 128) downsample4(a, s, d + x0, x0, y);
}

int round_ratio(int src, int dst, int scale) { return (int)(0.5 + ((float)src / (float)dst * scale)); }   // WELS_ROUND, macros.h:120

}  // namespace

extern "C" {

int b2h264_k_downsample_ladder(const b2h264_ds_plane* h_planes, int n_planes, uint8_t* dst, size_t dst_pitch, const uint8_t* src,
                               size_t src_pitch, int lo, int cnt, void* stream) {
  if (!h_planes || n_planes < 1 || n_planes > B2H264_LADDER_MAX_PLANES || lo < 0 || cnt < 1 || cnt > 65535) return cudaErrorInvalidValue;
  LadderArgs la;
  la.n = n_planes;
  int rows = 0;
  for (int k = 0; k < n_planes; k++) {
    const b2h264_ds_plane& p = h_planes[k];
    if (p.mode < 0 || p.mode > 4 || p.dst_w < 1 || p.dst_h < 1 || p.row0 != rows) return cudaErrorInvalidValue;
    la.p[k] = p;
    rows += p.dst_h;
  }
  la.rows = rows;
  if ((rows + 3) / 4 > 65535) return cudaErrorInvalidValue;
  k_downsample_ladder<<<dim3(1, (rows + 3) / 4, cnt), 128, 0, (cudaStream_t)stream>>>(dst, src, dst_pitch, src_pitch, lo, la);
  return b2h264_launched();
}

// n_planes planes of one geometry: a ladder of one descriptor whose "pictures" are the planes
int b2h264_k_downsample(int mode, uint8_t* dst, int dst_stride, int dst_w, int dst_h, const uint8_t* src, int src_stride, int src_w,
                        int src_h, int n_planes, size_t dst_plane_bytes, size_t src_plane_bytes, void* stream) {
  if (mode < 0 || mode > 4 || dst_w < 1 || dst_h < 1 || n_planes < 1) return cudaErrorInvalidValue;
  b2h264_ds_plane p = {};
  p.mode = mode; p.dst_stride = dst_stride; p.dst_w = dst_w; p.dst_h = dst_h; p.src_stride = src_stride; p.src_w = src_w; p.src_h = src_h;
  p.sx = mode >= 3 ? round_ratio(src_w, dst_w, 1 << (mode == 3 ? 16 : 15)) : 0;
  p.sy = mode >= 3 ? round_ratio(src_h, dst_h, 1 << 15) : 0;
  return b2h264_k_downsample_ladder(&p, 1, dst, dst_plane_bytes, src, src_plane_bytes, 0, n_planes, stream);
}

// which function CDownsampling::Process (downsample.cpp:143-215, the direct branch) applies to a plane pair:
// 0 half, 1 quarter, 2 one third, else the general ratio (3 for luma, 4 for chroma)
int b2h264_downsample_mode(int src_w, int src_h, int dst_w, int dst_h, int is_chroma) {
  if ((src_w >> 1) == dst_w && (src_h >> 1) == dst_h) return 0;
  if ((src_w >> 2) == dst_w && (src_h >> 2) == dst_h) return 1;
  if ((src_w / 3) == dst_w && (src_h / 3) == dst_h) return 2;
  return is_chroma ? 4 : 3;
}

}  // extern "C"
