/*
 * oracle/h264_oracle.c — scalar CPU restatement of the cisco/openh264 macroblock pixel kernels.
 * TEST INFRASTRUCTURE ONLY (see h264_oracle.h).  Plain C, no SIMD, written for clarity; each
 * function names the reference file:line (relative to /root/reference/codec) it follows.
 * Pinned against oracle/_ref/libopenh264_ref.so by tests/test_oracle_vs_ref.py.
 */
#include "h264_oracle.h"
#include <stdlib.h>
#include <string.h>

static inline int iabs (int v) { return v < 0 ? -v : v; }
static inline int clip3 (int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
static inline uint8_t clip255 (int v) { return (uint8_t) (v < 0 ? 0 : (v > 255 ? 255 : v)); }

void orc_blk_dims (int blk, int* w, int* h) {
  static const int8_t kW[ORC_BLK_ALL] = {16, 16, 8, 8, 4, 8, 4};
  static const int8_t kH[ORC_BLK_ALL] = {16, 8, 16, 8, 4, 4, 8};
  *w = kW[blk];
  *h = kH[blk];
}

/* ------------------------------------------------------------------------------------------
 * Tables.  The reference stores these as literal arrays; they are closed forms of the H.264
 * quantiser design, generated here and verified equal to the reference's arrays in the tests.
 * ------------------------------------------------------------------------------------------ */
/* 2x the standard's quantiser multipliers for qp%6 at positions (0,0) / (0,1) / (1,1) */
static const int32_t kMfBase[6][3] = {
  {26214, 16132, 10486}, {23832, 14980, 9320}, {20164, 13108, 8388},
  {18724, 11650, 7294},  {16384, 10486, 6710}, {14564, 9118, 5786}
};
static const uint8_t kDequantBase[6][3] = {
  {10, 13, 16}, {11, 14, 18}, {13, 16, 20}, {14, 18, 23}, {16, 20, 25}, {18, 23, 29}
};
/* position class inside an 8-entry row: the reference indexes FF/MF/dequant with (i & 7) */
static const uint8_t kPosClass[8] = {0, 1, 0, 1, 1, 2, 1, 2};

static int16_t  g_ff[58][8];
static int16_t  g_mf[52][8];
static uint16_t g_dq[52][8];
static int      g_tables_ready = 0;

static void build_tables (void) {
  if (g_tables_ready) return;
  for (int qp = 0; qp < 58; qp++) {
    const int s = qp / 6;
    for (int j = 0; j < 8; j++) {
      const int64_t base = kMfBase[qp % 6][kPosClass[j]];
      /* encode_mb_aux.cpp:38-101: rounding offset ~ (1/6)·2^16/MF (intra rows are qp+6 => ~1/3) */
      const int64_t num = 65536LL << s, den = 6 * base;
      g_ff[qp][j] = (int16_t) ((2 * num + den) / (2 * den));
      if (qp < 52) {
        /* encode_mb_aux.cpp:103-156 */
        g_mf[qp][j] = (int16_t) ((base + (s ? (1 << (s - 1)) : 0)) >> s);
        /* common_tables.cpp:208-235 */
        g_dq[qp][j] = (uint16_t) (kDequantBase[qp % 6][kPosClass[j]] << s);
      }
    }
  }
  g_tables_ready = 1;
}
const int16_t* orc_quant_ff (int q) { build_tables(); return g_ff[q]; }
const int16_t* orc_quant_mf (int q) { build_tables(); return g_mf[q]; }
const uint16_t* orc_dequant_coeff (int q) { build_tables(); return g_dq[q]; }

/* encoder_data_tables.cpp:59-67 — lambda(qp) = max(1, round(2^((qp-12)/6))) */
int orc_qp_lambda (int qp) {
  static const uint8_t k[52] = {
    1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 4, 4, 4, 5, 6,
    6, 7, 8, 9, 10, 11, 13, 14, 16, 18, 20, 23, 25, 29, 32, 36, 40, 45, 51, 57, 64, 72, 81, 91
  };
  return k[qp];
}
/* H.264 Table 8-15 (QPc as a function of qPI); reference: common_tables.cpp g_kuiChromaQpTable */
int orc_chroma_qp (int qp) {
  static const uint8_t k[22] = {29, 30, 31, 32, 32, 33, 34, 34, 35, 35, 36, 36, 37, 37, 37, 38, 38, 38, 39, 39, 39, 39};
  return qp < 30 ? qp : k[qp - 30];
}

/* bits of a signed Exp-Golomb code — encoder/core/inc/svc_enc_golomb.h:58-95 */
static int se_bits (int v) {
  uint32_t code = v > 0 ? (uint32_t) (2 * v - 1) : (uint32_t) (-2 * v);
  int n = 0;
  for (uint32_t t = code + 1; t > 1; t >>= 1) n++;
  return 2 * n + 1;
}
/* md.cpp:797-824: cost[mvd] = lambda(qp) * bits(se(mvd)), table centred on mvd = 0 */
void orc_mvd_cost_init (uint16_t* centre, int sz, int qp) {
  const int lambda = orc_qp_lambda (qp);
  for (int d = -sz; d <= sz; d++) centre[d] = (uint16_t) (lambda * se_bits (d));
}

/* ------------------------------------------------------------------------------------------
 * SAD / SATD
 * ------------------------------------------------------------------------------------------ */
/* sad_common.cpp:44-120 */
int32_t orc_sad (int blk, const uint8_t* a, int sa, const uint8_t* b, int sb) {
  int w, h, sum = 0;
  orc_blk_dims (blk, &w, &h);
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) sum += iabs (a[y * sa + x] - b[y * sb + x]);
  return sum;
}
/* sad_common.cpp:122-165: order is up, down, left, right */
void orc_sad_four (int blk, const uint8_t* a, int sa, const uint8_t* b, int sb, int32_t out[4]) {
  out[0] = orc_sad (blk, a, sa, b - sb, sb);
  out[1] = orc_sad (blk, a, sa, b + sb, sb);
  out[2] = orc_sad (blk, a, sa, b - 1, sb);
  out[3] = orc_sad (blk, a, sa, b + 1, sb);
}
/* sample.cpp:48-96: 4x4 Hadamard of the difference, sum |.|, (sum+1)>>1 PER 4x4 block */
static int satd4x4 (const uint8_t* a, int sa, const uint8_t* b, int sb) {
  int d[4][4], t[4][4], sum = 0;
  for (int y = 0; y < 4; y++)
    for (int x = 0; x < 4; x++) d[y][x] = a[y * sa + x] - b[y * sb + x];
  for (int y = 0; y < 4; y++) {
    const int e0 = d[y][0] + d[y][2], e1 = d[y][1] + d[y][3], e2 = d[y][0] - d[y][2], e3 = d[y][1] - d[y][3];
    t[y][0] = e0 + e1; t[y][1] = e2 + e3; t[y][2] = e2 - e3; t[y][3] = e0 - e1;
  }
  for (int x = 0; x < 4; x++) {
    const int e0 = t[0][x] + t[2][x], e1 = t[1][x] + t[3][x], e2 = t[0][x] - t[2][x], e3 = t[1][x] - t[3][x];
    sum += iabs (e0 + e1) + iabs (e2 + e3) + iabs (e2 - e3) + iabs (e0 - e1);
  }
  return (sum + 1) >> 1;
}
/* sample.cpp:98-148 */
int32_t orc_satd (int blk, const uint8_t* a, int sa, const uint8_t* b, int sb) {
  int w, h, sum = 0;
  orc_blk_dims (blk, &w, &h);
  for (int y = 0; y < h; y += 4)
    for (int x = 0; x < w; x += 4) sum += satd4x4 (a + y * sa + x, sa, b + y * sb + x, sb);
  return sum;
}

/* ------------------------------------------------------------------------------------------
 * Motion compensation
 * ------------------------------------------------------------------------------------------ */
/* mc.cpp:150-160: taps (1,-5,20,20,-5,1) around p[0],p[step] */
static int tap6 (const uint8_t* p, int step) {
  return (p[-2 * step] + p[3 * step]) - 5 * (p[-step] + p[2 * step]) + 20 * (p[0] + p[step]);
}
/* mc.cpp:187-231 */
static void half_h (const uint8_t* s, int ss, uint8_t* d, int ds, int w, int h) {
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) d[y * ds + x] = clip255 ((tap6 (s + y * ss + x, 1) + 16) >> 5);
}
static void half_v (const uint8_t* s, int ss, uint8_t* d, int ds, int w, int h) {
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) d[y * ds + x] = clip255 ((tap6 (s + y * ss + x, ss) + 16) >> 5);
}
static void half_c (const uint8_t* s, int ss, uint8_t* d, int ds, int w, int h) {
  for (int y = 0; y < h; y++) {
    int16_t col[17 + 5];   /* vertical pass kept unrounded in 16 bits, as mc.cpp:218 */
    for (int x = 0; x < w + 5; x++) col[x] = (int16_t) tap6 (s + y * ss + x - 2, ss);
    for (int x = 0; x < w; x++) {
      const int v = (col[x] + col[x + 5]) - 5 * (col[x + 1] + col[x + 4]) + 20 * (col[x + 2] + col[x + 3]);
      d[y * ds + x] = clip255 ((v + 512) >> 10);
    }
  }
}
/* mc.cpp:162-172 */
void orc_pixel_avg (uint8_t* dst, int ds, const uint8_t* a, int sa, const uint8_t* b, int sb, int w, int h) {
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) dst[y * ds + x] = (uint8_t) ((a[y * sa + x] + b[y * sb + x] + 1) >> 1);
}
/* mc.cpp:234-347: the 16 quarter-sample positions.  Position (fx,fy):
 *   integer -> copy; one half-sample plane -> that plane; otherwise rounded average of two of
 *   {integer sample G / neighbours, horizontal half b, vertical half h, centre j}. */
void orc_mc_luma (const uint8_t* src, int ss, uint8_t* dst, int ds, int mvx, int mvy, int w, int h) {
  const int fx = mvx & 3, fy = mvy & 3;
  uint8_t t0[17 * 17], t1[17 * 17];
  if (fx == 0 && fy == 0) {
    for (int y = 0; y < h; y++) memcpy (dst + y * ds, src + y * ss, (size_t) w);
    return;
  }
  if (fy == 0) {                       /* (1,0) (2,0) (3,0) */
    if (fx == 2) { half_h (src, ss, dst, ds, w, h); return; }
    half_h (src, ss, t0, 17, w, h);
    orc_pixel_avg (dst, ds, src + (fx == 3), ss, t0, 17, w, h);
    return;
  }
  if (fx == 0) {                       /* (0,1) (0,2) (0,3) */
    if (fy == 2) { half_v (src, ss, dst, ds, w, h); return; }
    half_v (src, ss, t0, 17, w, h);
    orc_pixel_avg (dst, ds, src + (fy == 3 ? ss : 0), ss, t0, 17, w, h);
    return;
  }
  if (fx == 2 && fy == 2) { half_c (src, ss, dst, ds, w, h); return; }
  if (fx == 2) {                       /* (2,1) (2,3): centre + horizontal half of row y / y+1 */
    half_h (src + (fy == 3 ? ss : 0), ss, t0, 17, w, h);
    half_c (src, ss, t1, 17, w, h);
  } else if (fy == 2) {                /* (1,2) (3,2): centre + vertical half of column x / x+1 */
    half_v (src + (fx == 3), ss, t0, 17, w, h);
    half_c (src, ss, t1, 17, w, h);
  } else {                             /* diagonals: horizontal half (row y or y+1) + vertical half (col x or x+1) */
    half_h (src + (fy == 3 ? ss : 0), ss, t0, 17, w, h);
    half_v (src + (fx == 3), ss, t1, 17, w, h);
  }
  orc_pixel_avg (dst, ds, t0, 17, t1, 17, w, h);
}
/* mc.cpp:349-380: bilinear eighth-sample chroma */
void orc_mc_chroma (const uint8_t* src, int ss, uint8_t* dst, int ds, int mvx, int mvy, int w, int h) {
  const int dx = mvx & 7, dy = mvy & 7;
  const int A = (8 - dx) * (8 - dy), B = dx * (8 - dy), C = (8 - dx) * dy, D = dx * dy;
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) {
      const uint8_t* p = src + y * ss + x;
      if (dx == 0 && dy == 0) dst[y * ds + x] = p[0];
      else dst[y * ds + x] = (uint8_t) ((A * p[0] + B * p[1] + C * p[ss] + D * p[ss + 1] + 32) >> 6);
    }
}

/* ------------------------------------------------------------------------------------------
 * Forward transform, quantisation, scan
 * ------------------------------------------------------------------------------------------ */
/* encode_mb_aux.cpp:313-356: residual then H.264 4x4 core transform (rows, then columns), int16 */
void orc_dct4x4 (int16_t* dct, const uint8_t* p1, int s1, const uint8_t* p2, int s2) {
  int16_t m[16];
  for (int y = 0; y < 4; y++) {
    int16_t r[4];
    for (int x = 0; x < 4; x++) r[x] = (int16_t) (p1[y * s1 + x] - p2[y * s2 + x]);
    const int16_t a = r[0] + r[3], b = r[1] + r[2], c = r[1] - r[2], d = r[0] - r[3];
    m[4 * y + 0] = a + b; m[4 * y + 2] = a - b;
    m[4 * y + 1] = (int16_t) (2 * d + c); m[4 * y + 3] = (int16_t) (d - 2 * c);
  }
  for (int x = 0; x < 4; x++) {
    const int16_t a = m[x] + m[12 + x], b = m[4 + x] + m[8 + x], c = m[4 + x] - m[8 + x], d = m[x] - m[12 + x];
    dct[x] = a + b; dct[8 + x] = a - b;
    dct[4 + x] = (int16_t) (2 * d + c); dct[12 + x] = (int16_t) (d - 2 * c);
  }
}
/* encode_mb_aux.cpp:358-366: 8x8 region as four 4x4 blocks in z order */
void orc_dct_four4x4 (int16_t* dct, const uint8_t* p1, int s1, const uint8_t* p2, int s2) {
  for (int k = 0; k < 4; k++) {
    const int ox = (k & 1) * 4, oy = (k >> 1) * 4;
    orc_dct4x4 (dct + 16 * k, p1 + oy * s1 + ox, s1, p2 + oy * s2 + ox, s2);
  }
}
/* encode_mb_aux.cpp:161-163: sign * (((ff + |x|) * mf) >> 16), stored to int16 */
static int16_t quant1 (int16_t x, int ff, int mf) {
  const int sign = x < 0 ? -1 : 0;
  const int32_t mag = ((ff + ((sign ^ x) - sign)) * mf) >> 16;
  return (int16_t) ((sign ^ mag) - sign);
}
void orc_quant4x4 (int16_t* d, const int16_t* ff, const int16_t* mf) {
  for (int i = 0; i < 16; i++) d[i] = quant1 (d[i], ff[i & 7], mf[i & 7]);
}
void orc_quant4x4_dc (int16_t* d, int16_t ff, int16_t mf) {
  for (int i = 0; i < 16; i++) d[i] = quant1 (d[i], ff, mf);
}
void orc_quant_four4x4 (int16_t* d, const int16_t* ff, const int16_t* mf) {
  for (int i = 0; i < 64; i++) d[i] = quant1 (d[i], ff[i & 7], mf[i & 7]);
}
/* encode_mb_aux.cpp:209-224: also reports the largest magnitude of each 4x4 block.
 * NB the magnitude passes through int16 before the comparison. */
void orc_quant_four4x4_max (int16_t* d, const int16_t* ff, const int16_t* mf, int16_t* max4) {
  for (int k = 0; k < 4; k++) {
    int16_t mx = 0;
    for (int i = 0; i < 16; i++) {
      const int16_t x = d[16 * k + i];
      const int sign = x < 0 ? -1 : 0;
      const int16_t mag = (int16_t) (((ff[i & 7] + ((sign ^ x) - sign)) * mf[i & 7]) >> 16);
      if (mx < mag) mx = mag;
      d[16 * k + i] = (int16_t) ((sign ^ mag) - sign);
    }
    max4[k] = mx;
  }
}
/* encode_mb_aux.cpp:226-242: would any chroma DC survive quantisation? (DCs sit at 0,16,32,48) */
int32_t orc_hadamard_quant2x2_skip (const int16_t* rs, int16_t ff, int16_t mf) {
  const int16_t thr = (int16_t) (((1 << 16) - 1) / mf - ff);
  const int16_t s0 = rs[0] + rs[32], s1 = rs[0] - rs[32], s2 = rs[16] + rs[48], s3 = rs[16] - rs[48];
  const int16_t d[4] = { (int16_t) (s0 + s2), (int16_t) (s0 - s2), (int16_t) (s1 + s3), (int16_t) (s1 - s3) };
  return iabs (d[0]) > thr || iabs (d[1]) > thr || iabs (d[2]) > thr || iabs (d[3]) > thr;
}
/* encode_mb_aux.cpp:244-277 */
int32_t orc_hadamard_quant2x2 (int16_t* rs, int16_t ff, int16_t mf, int16_t* dct, int16_t* block) {
  const int16_t s0 = rs[0] + rs[32], s1 = rs[0] - rs[32], s2 = rs[16] + rs[48], s3 = rs[16] - rs[48];
  int nz = 0;
  rs[0] = rs[16] = rs[32] = rs[48] = 0;
  dct[0] = quant1 ((int16_t) (s0 + s2), ff, mf);
  dct[1] = quant1 ((int16_t) (s0 - s2), ff, mf);
  dct[2] = quant1 ((int16_t) (s1 + s3), ff, mf);
  dct[3] = quant1 ((int16_t) (s1 - s3), ff, mf);
  for (int i = 0; i < 4; i++) { block[i] = dct[i]; nz += block[i] != 0; }
  return nz;
}
/* encode_mb_aux.cpp:280-309: gather the 16 luma DCs of an I16x16 MB (coefficient 0 of each 4x4,
 * MB stored as 4 groups of 64) and apply the 4x4 Hadamard with (x+1)>>1, saturated to int16 */
void orc_hadamard_t4_dc (int16_t* luma_dc, const int16_t* dct) {
  int32_t p[16];
  for (int i = 0; i < 16; i += 4) {
    const int idx = ((i & 8) << 4) + ((i & 4) << 3);
    const int a = dct[idx] + dct[idx + 80], d = dct[idx] - dct[idx + 80];
    const int b = dct[idx + 16] + dct[idx + 64], c = dct[idx + 16] - dct[idx + 64];
    p[i] = a + b; p[i + 2] = a - b; p[i + 1] = d + c; p[i + 3] = d - c;
  }
  for (int i = 0; i < 4; i++) {
    const int a = p[i] + p[i + 12], d = p[i] - p[i + 12], b = p[i + 4] + p[i + 8], c = p[i + 4] - p[i + 8];
    luma_dc[i]      = (int16_t) clip3 ((a + b + 1) >> 1, -32768, 32767);
    luma_dc[i + 8]  = (int16_t) clip3 ((a - b + 1) >> 1, -32768, 32767);
    luma_dc[i + 4]  = (int16_t) clip3 ((d + c + 1) >> 1, -32768, 32767);
    luma_dc[i + 12] = (int16_t) clip3 ((d - c + 1) >> 1, -32768, 32767);
  }
}
/* encode_mb_aux.cpp:371-401: frame zig-zag */
static const uint8_t kZigzag[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};
void orc_scan4x4_dcac (int16_t* level, const int16_t* dct) {
  for (int i = 0; i < 16; i++) level[i] = dct[kZigzag[i]];
}
void orc_scan4x4_ac (int16_t* level, const int16_t* dct) {
  for (int i = 1; i < 16; i++) level[i - 1] = dct[kZigzag[i]];
  level[15] = 0;
}
/* encode_mb_aux.cpp:418-435 (JVT-O079): cost of isolated small coefficients by preceding zero run */
int32_t orc_single_ctr4x4 (const int16_t* d) {
  static const int8_t kRunCost[16] = {3, 2, 2, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  int idx = 15, total = 0;
  while (idx >= 0 && d[idx] == 0) idx--;
  while (idx >= 0) {
    int run;
    idx--;
    run = idx;
    while (idx >= 0 && d[idx] == 0) idx--;
    total += kRunCost[run - idx];
  }
  return total;
}
/* encode_mb_aux.cpp:437-451 */
int32_t orc_nonzero_count (const int16_t* level) {
  int n = 0;
  for (int i = 0; i < 16; i++) n += level[i] != 0;
  return n;
}

/* ------------------------------------------------------------------------------------------
 * Dequantisation and inverse transforms (encoder side)
 * ------------------------------------------------------------------------------------------ */
/* decode_mb_aux.cpp:40-77: 4x4 inverse Hadamard in place, int16 arithmetic */
void orc_ihadamard4x4_dc (int16_t* r) {
  for (int i = 3; i >= 0; i--) {
    int16_t* q = r + 4 * i;
    const int16_t a = q[0] + q[2], b = q[0] - q[2], c = q[1] - q[3], d = q[1] + q[3];
    q[0] = a + d; q[1] = b + c; q[2] = b - c; q[3] = a - d;
  }
  for (int i = 3; i >= 0; i--) {
    const int16_t a = r[i] + r[8 + i], b = r[i] - r[8 + i], c = r[4 + i] - r[12 + i], d = r[4 + i] + r[12 + i];
    r[i] = a + d; r[4 + i] = b + c; r[8 + i] = b - c; r[12 + i] = a - d;
  }
}
/* decode_mb_aux.cpp:80-95: luma DC scaling for qp < 12 */
void orc_dequant_luma_dc4x4 (int16_t* r, int qp) {
  const int v = orc_dequant_coeff (qp % 6)[0];
  const int qf0 = qp / 6, sh = 2 - qf0, rnd = 1 << (1 - qf0);
  for (int i = 0; i < 16; i++) r[i] = (int16_t) ((r[i] * v + (int16_t) rnd) >> sh);
}
/* decode_mb_aux.cpp:98-125: inverse Hadamard then *mf (qp >= 12), wrapping in int16 */
void orc_dequant_ihadamard4x4 (int16_t* r, uint16_t mf) {
  for (int i = 0; i < 16; i += 4) {
    int16_t* q = r + i;
    const int16_t a = q[0] + q[2], b = q[0] - q[2], c = q[1] - q[3], d = q[1] + q[3];
    q[0] = a + d; q[1] = b + c; q[2] = b - c; q[3] = a - d;
  }
  for (int i = 0; i < 4; i++) {
    const int16_t a = r[i] + r[8 + i], b = r[i] - r[8 + i], c = r[4 + i] - r[12 + i], d = r[4 + i] + r[12 + i];
    r[i] = (int16_t) ((a + d) * mf); r[4 + i] = (int16_t) ((b + c) * mf);
    r[8 + i] = (int16_t) ((b - c) * mf); r[12 + i] = (int16_t) ((a - d) * mf);
  }
}
/* decode_mb_aux.cpp:127-137 */
void orc_dequant_ihadamard2x2_dc (int16_t* d, uint16_t mf) {
  const int16_t su = d[0] + d[2], du = d[0] - d[2], sd = d[1] + d[3], dd = d[1] - d[3];
  d[0] = (int16_t) (((su + sd) * mf) >> 1);
  d[1] = (int16_t) (((su - sd) * mf) >> 1);
  d[2] = (int16_t) (((du + dd) * mf) >> 1);
  d[3] = (int16_t) (((du - dd) * mf) >> 1);
}
/* decode_mb_aux.cpp:139-160: level * scale, product truncated to int16 */
void orc_dequant4x4 (int16_t* r, const uint16_t* mf) {
  for (int i = 0; i < 16; i++) r[i] = (int16_t) (r[i] * mf[i & 7]);
}
void orc_dequant_four4x4 (int16_t* r, const uint16_t* mf) {
  for (int i = 0; i < 64; i++) r[i] = (int16_t) (r[i] * mf[i & 7]);
}
/* decode_mb_aux.cpp:164-197: inverse core transform, (x+32)>>6, add prediction, clip.
 * The row pass is stored in int16. */
void orc_idct4x4_rec (uint8_t* rec, int rs, const uint8_t* pred, int ps, const int16_t* dct) {
  int16_t t[16];
  for (int y = 0; y < 4; y++) {
    const int16_t* c = dct + 4 * y;
    const int su = c[0] + c[2], du = c[0] - c[2], sd = c[1] + (c[3] >> 1), dd = (c[1] >> 1) - c[3];
    t[4 * y] = (int16_t) (su + sd); t[4 * y + 1] = (int16_t) (du + dd);
    t[4 * y + 2] = (int16_t) (du - dd); t[4 * y + 3] = (int16_t) (su - sd);
  }
  for (int x = 0; x < 4; x++) {
    const int sl = t[x] + t[8 + x], dl = t[x] - t[8 + x], dr = (t[4 + x] >> 1) - t[12 + x], sr = t[4 + x] + (t[12 + x] >> 1);
    rec[x]          = clip255 (pred[x]          + ((sl + sr + 32) >> 6));
    rec[rs + x]     = clip255 (pred[ps + x]     + ((dl + dr + 32) >> 6));
    rec[2 * rs + x] = clip255 (pred[2 * ps + x] + ((dl - dr + 32) >> 6));
    rec[3 * rs + x] = clip255 (pred[3 * ps + x] + ((sl - sr + 32) >> 6));
  }
}
/* decode_mb_aux.cpp:199-207 */
void orc_idct_four4x4_rec (uint8_t* rec, int rs, const uint8_t* pred, int ps, const int16_t* dct) {
  for (int k = 0; k < 4; k++) {
    const int ox = (k & 1) * 4, oy = (k >> 1) * 4;
    orc_idct4x4_rec (rec + oy * rs + ox, rs, pred + oy * ps + ox, ps, dct + 16 * k);
  }
}
/* decode_mb_aux.cpp:223-233: I16x16 with DC-only residual; dc[] indexed by 4x4 block raster */
void orc_idct_rec_i16x16_dc (uint8_t* rec, int rs, const uint8_t* pred, int ps, const int16_t* dc) {
  for (int y = 0; y < 16; y++)
    for (int x = 0; x < 16; x++)
      rec[y * rs + x] = clip255 (pred[y * ps + x] + ((dc[(y & 12) + (x >> 2)] + 32) >> 6));
}

/* ------------------------------------------------------------------------------------------
 * Decoder reconstruction (decoder/core/src/decode_mb_aux.cpp)
 * ------------------------------------------------------------------------------------------ */
/* decode_mb_aux.cpp:42-77: in-place residual add; row pass stored in int16 */
void orc_idct_res_add_pred (uint8_t* pred, int stride, const int16_t* rs) {
  int16_t t[16];
  for (int y = 0; y < 4; y++) {
    const int16_t* c = rs + 4 * y;
    const int e0 = c[0] + c[2], e1 = c[0] - c[2], e2 = (c[1] >> 1) - c[3], e3 = c[1] + (c[3] >> 1);
    t[4 * y] = (int16_t) (e0 + e3); t[4 * y + 1] = (int16_t) (e1 + e2);
    t[4 * y + 2] = (int16_t) (e1 - e2); t[4 * y + 3] = (int16_t) (e0 - e3);
  }
  for (int x = 0; x < 4; x++) {
    const int a = t[x] + t[8 + x], b = t[4 + x] + (t[12 + x] >> 1);
    const int c = t[x] - t[8 + x], d = (t[4 + x] >> 1) - t[12 + x];
    pred[x]              = clip255 (((32 + a + b) >> 6) + pred[x]);
    pred[3 * stride + x] = clip255 (((32 + a - b) >> 6) + pred[3 * stride + x]);
    pred[stride + x]     = clip255 (((32 + c + d) >> 6) + pred[stride + x]);
    pred[2 * stride + x] = clip255 (((32 + c - d) >> 6) + pred[2 * stride + x]);
  }
}
/* one 8-point inverse butterfly of the High-profile 8x8 transform, all in int16 as the reference */
static void idct8_1d (const int16_t p[8], int16_t out[8]) {
  int16_t a[4], b[8];
  a[0] = p[0] + p[4]; a[1] = p[0] - p[4]; a[2] = p[6] - (p[2] >> 1); a[3] = p[2] + (p[6] >> 1);
  b[0] = a[0] + a[3]; b[2] = a[1] - a[2]; b[4] = a[1] + a[2]; b[6] = a[0] - a[3];
  a[0] = -p[3] + p[5] - p[7] - (p[7] >> 1);
  a[1] = p[1] + p[7] - p[3] - (p[3] >> 1);
  a[2] = -p[1] + p[7] + p[5] + (p[5] >> 1);
  a[3] = p[3] + p[5] + p[1] + (p[1] >> 1);
  b[1] = a[0] + (a[3] >> 2); b[3] = a[1] + (a[2] >> 2); b[5] = a[2] - (a[1] >> 2); b[7] = a[3] - (a[0] >> 2);
  out[0] = b[0] + b[7]; out[1] = b[2] - b[5]; out[2] = b[4] + b[3]; out[3] = b[6] + b[1];
  out[4] = b[6] - b[1]; out[5] = b[4] - b[3]; out[6] = b[2] + b[5]; out[7] = b[0] - b[7];
}
/* decode_mb_aux.cpp:79-190 */
void orc_idct_res_add_pred8x8 (uint8_t* pred, int stride, const int16_t* rs) {
  int16_t tmp[64], res[64], in[8], out[8];
  for (int y = 0; y < 8; y++) {
    idct8_1d (rs + 8 * y, out);
    for (int x = 0; x < 8; x++) tmp[8 * y + x] = out[x];
  }
  for (int x = 0; x < 8; x++) {
    for (int y = 0; y < 8; y++) in[y] = tmp[8 * y + x];
    idct8_1d (in, out);
    for (int y = 0; y < 8; y++) res[8 * y + x] = out[y];
  }
  for (int y = 0; y < 8; y++)
    for (int x = 0; x < 8; x++)
      pred[y * stride + x] = clip255 (pred[y * stride + x] + ((32 + res[8 * y + x]) >> 6));
}

/* ------------------------------------------------------------------------------------------
 * Deblocking edge filters (common/src/deblocking_common.cpp)
 * ------------------------------------------------------------------------------------------ */
/* deblocking_common.cpp:5-38: bS < 4, 16 lines, tc0 per group of 4 lines (negative = skip) */
void orc_deblock_luma_lt4 (uint8_t* pix, int sx, int sy, int alpha, int beta, const int8_t tc4[4]) {
  for (int i = 0; i < 16; i++, pix += sy) {
    const int tc0 = tc4[i >> 2];
    if (tc0 < 0) continue;
    const int p0 = pix[-sx], p1 = pix[-2 * sx], p2 = pix[-3 * sx], q0 = pix[0], q1 = pix[sx], q2 = pix[2 * sx];
    if (!(iabs (p0 - q0) < alpha && iabs (p1 - p0) < beta && iabs (q1 - q0) < beta)) continue;
    int tc = tc0;
    if (iabs (p2 - p0) < beta) {
      pix[-2 * sx] = (uint8_t) (p1 + clip3 ((p2 + ((p0 + q0 + 1) >> 1) - 2 * p1) >> 1, -tc0, tc0));
      tc++;
    }
    if (iabs (q2 - q0) < beta) {
      pix[sx] = (uint8_t) (q1 + clip3 ((q2 + ((p0 + q0 + 1) >> 1) - 2 * q1) >> 1, -tc0, tc0));
      tc++;
    }
    const int delta = clip3 ((4 * (q0 - p0) + (p1 - q1) + 4) >> 3, -tc, tc);
    pix[-sx] = clip255 (p0 + delta);
    pix[0] = clip255 (q0 - delta);
  }
}
/* deblocking_common.cpp:39-79: bS == 4 strong filter */
void orc_deblock_luma_eq4 (uint8_t* pix, int sx, int sy, int alpha, int beta) {
  for (int i = 0; i < 16; i++, pix += sy) {
    const int p0 = pix[-sx], p1 = pix[-2 * sx], p2 = pix[-3 * sx], q0 = pix[0], q1 = pix[sx], q2 = pix[2 * sx];
    const int d = iabs (p0 - q0);
    if (!(d < alpha && iabs (p1 - p0) < beta && iabs (q1 - q0) < beta)) continue;
    if (d < (alpha >> 2) + 2) {
      if (iabs (p2 - p0) < beta) {
        const int p3 = pix[-4 * sx];
        pix[-sx]     = (uint8_t) ((p2 + 2 * p1 + 2 * p0 + 2 * q0 + q1 + 4) >> 3);
        pix[-2 * sx] = (uint8_t) ((p2 + p1 + p0 + q0 + 2) >> 2);
        pix[-3 * sx] = (uint8_t) ((2 * p3 + 3 * p2 + p1 + p0 + q0 + 4) >> 3);
      } else {
        pix[-sx] = (uint8_t) ((2 * p1 + p0 + q1 + 2) >> 2);
      }
      if (iabs (q2 - q0) < beta) {
        const int q3 = pix[3 * sx];
        pix[0]      = (uint8_t) ((p1 + 2 * p0 + 2 * q0 + 2 * q1 + q2 + 4) >> 3);
        pix[sx]     = (uint8_t) ((p0 + q0 + q1 + q2 + 2) >> 2);
        pix[2 * sx] = (uint8_t) ((2 * q3 + 3 * q2 + q1 + q0 + p0 + 4) >> 3);
      } else {
        pix[0] = (uint8_t) ((2 * q1 + q0 + p1 + 2) >> 2);
      }
    } else {
      pix[-sx] = (uint8_t) ((2 * p1 + p0 + q1 + 2) >> 2);
      pix[0]   = (uint8_t) ((2 * q1 + q0 + p1 + 2) >> 2);
    }
  }
}
static void chroma_lt4_line (uint8_t* pix, int sx, int alpha, int beta, int tc) {
  const int p0 = pix[-sx], p1 = pix[-2 * sx], q0 = pix[0], q1 = pix[sx];
  if (iabs (p0 - q0) < alpha && iabs (p1 - p0) < beta && iabs (q1 - q0) < beta) {
    const int delta = clip3 ((4 * (q0 - p0) + (p1 - q1) + 4) >> 3, -tc, tc);
    pix[-sx] = clip255 (p0 + delta);
    pix[0] = clip255 (q0 - delta);
  }
}
/* deblocking_common.cpp:93-133: 8 lines, tc per pair of lines, filtered only when tc > 0 */
void orc_deblock_chroma_lt4 (uint8_t* cb, uint8_t* cr, int sx, int sy, int alpha, int beta, const int8_t tc4[4]) {
  for (int i = 0; i < 8; i++, cb += sy, cr += sy) {
    const int tc = tc4[i >> 1];
    if (tc <= 0) continue;
    chroma_lt4_line (cb, sx, alpha, beta, tc);
    chroma_lt4_line (cr, sx, alpha, beta, tc);
  }
}
static void chroma_eq4_line (uint8_t* pix, int sx, int alpha, int beta) {
  const int p0 = pix[-sx], p1 = pix[-2 * sx], q0 = pix[0], q1 = pix[sx];
  if (iabs (p0 - q0) < alpha && iabs (p1 - p0) < beta && iabs (q1 - q0) < beta) {
    pix[-sx] = (uint8_t) ((2 * p1 + p0 + q1 + 2) >> 2);
    pix[0]   = (uint8_t) ((2 * q1 + q0 + p1 + 2) >> 2);
  }
}
/* deblocking_common.cpp:135-168 */
void orc_deblock_chroma_eq4 (uint8_t* cb, uint8_t* cr, int sx, int sy, int alpha, int beta) {
  for (int i = 0; i < 8; i++, cb += sy, cr += sy) {
    chroma_eq4_line (cb, sx, alpha, beta);
    chroma_eq4_line (cr, sx, alpha, beta);
  }
}

/* ------------------------------------------------------------------------------------------
 * Whole-picture deblocking, H.264 8.7, macroblocks in raster order.  Boundary strengths follow
 * 8.7.2.1 with the departures of the reference decoder (decoder/core/src/deblocking.cpp) marked
 * where they occur; the edge filters are the ones above.
 * ------------------------------------------------------------------------------------------ */
/* Table 8-16: alpha' and beta' by indexA / indexB */
static const uint8_t kDbkAlpha[52] = {
  0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 4, 4, 5, 6, 7, 8, 9, 10, 12, 13,
  15, 17, 20, 22, 25, 28, 32, 36, 40, 45, 50, 56, 63, 71, 80, 90, 101, 113, 127, 144, 162, 182, 203, 226, 255, 255};
static const uint8_t kDbkBeta[52] = {
  0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4,
  6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13, 14, 14, 15, 15, 16, 16, 17, 17, 18, 18};
/* Table 8-17: tC0 by bS (rows 1..3) and indexA */
static const uint8_t kDbkTc0[3][52] = {
  {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1,
   1, 1, 1, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 4, 4, 4, 5, 6, 6, 7, 8, 9, 10, 11, 13},
  {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1,
   1, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 4, 4, 5, 5, 6, 7, 8, 8, 10, 11, 12, 13, 15, 17},
  {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1,
   1, 2, 2, 2, 2, 3, 3, 3, 4, 4, 4, 5, 6, 6, 7, 8, 9, 10, 11, 13, 14, 16, 18, 20, 23, 25}};

static int dbk_is_intra (int t) { return t == ORC_MB_I4x4 || t == ORC_MB_I16x16 || t == ORC_MB_IPCM; }
static int dbk_is_b (int t) { return t == ORC_MB_B || t == ORC_MB_BSKIP; }
static int dbk_mv_far (const int32_t* a, const int32_t* b) { return iabs (a[0] - b[0]) >= 4 || iabs (a[1] - b[1]) >= 4; }
static void dbk_motion (const int32_t* ref, const int32_t* mv, int mb, int blk, int* r, int32_t m[2]) {
  *r = ref ? ref[16 * mb + blk] : -1;
  m[0] = *r < 0 ? 0 : mv[32 * mb + 2 * blk];            /* a list that is not used has no vector */
  m[1] = *r < 0 ? 0 : mv[32 * mb + 2 * blk + 1];
}

/* 8.7.2.1: bS of the edge between 4x4 block bq of macroblock q and block bp of macroblock p (p == q inside a macroblock) */
static int dbk_strength (const orc_dbk_pic* d, int q, int bq, int p, int bp, int mb_edge) {
  const int tq = d->type[q], tp = d->type[p];
  if (dbk_is_intra (tq) || dbk_is_intra (tp)) return mb_edge ? 4 : 3;
  /* Reference departure: the inner edges of a skipped macroblock get bS 0 (deblocking.cpp:1184, IS_SKIP).  For P_Skip the
   * spec agrees (one vector, no coefficients); for B_Skip the spec would derive bS from the direct-mode motion of each block. */
  if (!mb_edge && (tq == ORC_MB_PSKIP || tq == ORC_MB_BSKIP)) return 0;
  if (d->nnz[16 * q + bq] || d->nnz[16 * p + bp]) return 2;
  if (dbk_is_b (tq) || dbk_is_b (tp)) {
    /* two lists: DeblockingBSliceBsMarginalMBAvcbase (deblocking.cpp:544) / IN_SMB_EDGE_MV (:95).  bS 1 unless both blocks
     * use the same pair of reference pictures; then the vectors are compared picture by picture, and when both lists of q
     * name the same picture, both pairings must be far for bS 1 */
    int rq0, rq1, rp0, rp1;
    int32_t mq0[2], mq1[2], mp0[2], mp1[2];
    dbk_motion (d->ref0, d->mv0, q, bq, &rq0, mq0);
    dbk_motion (d->ref1, d->mv1, q, bq, &rq1, mq1);
    dbk_motion (d->ref0, d->mv0, p, bp, &rp0, mp0);
    dbk_motion (d->ref1, d->mv1, p, bp, &rp1, mp1);
    const int straight = rq0 == rp0 && rq1 == rp1, crossed = rq0 == rp1 && rq1 == rp0;
    if (!straight && !crossed) return 1;
    if (rq0 != rq1) return straight ? (dbk_mv_far (mq0, mp0) || dbk_mv_far (mq1, mp1)) : (dbk_mv_far (mq0, mp1) || dbk_mv_far (mq1, mp0));
    return (dbk_mv_far (mq0, mp0) || dbk_mv_far (mq1, mp1)) && (dbk_mv_far (mq0, mp1) || dbk_mv_far (mq1, mp0));
  }
  if (d->compare_refs && d->ref0[16 * q + bq] != d->ref0[16 * p + bp]) return 1;
  return dbk_mv_far (&d->mv0[32 * q + 2 * bq], &d->mv0[32 * p + 2 * bp]);
}

/* counts what the edge filter is about to do to one line (the lines of one edge are independent) */
static void dbk_count_luma (const uint8_t* pix, int sx, int alpha, int beta, int bs, int32_t* st) {
  const int p0 = pix[-sx], p1 = pix[-2 * sx], p2 = pix[-3 * sx], q0 = pix[0], q1 = pix[sx], q2 = pix[2 * sx];
  if (!(iabs (p0 - q0) < alpha && iabs (p1 - p0) < beta && iabs (q1 - q0) < beta)) return;
  st[ORC_DBK_LUMA_BS1 + bs - 1]++;
  const int ap = iabs (p2 - p0) < beta, aq = iabs (q2 - q0) < beta;
  if (bs == 4) {
    if (iabs (p0 - q0) < (alpha >> 2) + 2) { st[ORC_DBK_STRONG]++; st[ORC_DBK_STRONG_AP] += ap; st[ORC_DBK_STRONG_AQ] += aq; }
  } else {
    st[ORC_DBK_LT4_AP] += ap; st[ORC_DBK_LT4_AQ] += aq;
  }
}
static void dbk_count_chroma (const uint8_t* pix, int sx, int alpha, int beta, int bs, int32_t* st) {
  const int p0 = pix[-sx], p1 = pix[-2 * sx], q0 = pix[0], q1 = pix[sx];
  if (iabs (p0 - q0) < alpha && iabs (p1 - p0) < beta && iabs (q1 - q0) < beta) st[ORC_DBK_CHROMA_BS1 + bs - 1]++;
}

void orc_deblock_picture (uint8_t* y, uint8_t* cb, uint8_t* cr, int stride_y, int stride_c, int mb_w, int mb_h,
                          const orc_dbk_pic* d, int32_t* stats) {
  int32_t dummy[ORC_DBK_NSTATS];
  int32_t* st = stats ? stats : dummy;
  for (int mby = 0; mby < mb_h; mby++)
    for (int mbx = 0; mbx < mb_w; mbx++) {
      const int q = mby * mb_w + mbx;
      /* every rule reads the q macroblock's own slice controls */
      const int idc = d->idc[q], off_a = d->off_a[q], off_b = d->off_b[q];
      if (idc == 1) { st[ORC_DBK_OFF_IDC1] += 8; continue; }
      for (int dir = 0; dir < 2; dir++) {                 /* 0: vertical edges (p to the left), 1: horizontal (p above) */
        const int at_border = dir ? mby == 0 : mbx == 0;
        const int nb = dir ? q - mb_w : q - 1;
        for (int e = 0; e < 4; e++) {
          if (e == 0 && at_border) { st[ORC_DBK_OFF_BORDER]++; continue; }
          /* idc 2 (deblocking.cpp:671-681): macroblock edges toward another slice stay unfiltered */
          if (e == 0 && idc == 2 && d->slice[nb] != d->slice[q]) { st[ORC_DBK_OFF_IDC2]++; continue; }
          /* 8.7: with the 8x8 transform the luma edges at 4 and 12 are no transform block edges */
          if ((e & 1) && d->t8x8[q]) { st[ORC_DBK_OFF_T8X8]++; continue; }
          const int p = e == 0 ? nb : q;
          int bs[4], any = 0;
          for (int s = 0; s < 4; s++) {
            const int bq = dir ? 4 * e + s : 4 * s + e;
            const int bp = dir ? (e == 0 ? 12 + s : bq - 4) : (e == 0 ? 4 * s + 3 : bq - 1);
            bs[s] = dbk_strength (d, q, bq, p, bp, e == 0);
            any |= bs[s];
          }
          if (!any) continue;
          /* 8.7.2.2: a macroblock edge uses the mean QP of the two macroblocks (luma and chroma separately) */
          for (int chroma = 0; chroma < 2; chroma++) {
            if (chroma && (e & 1)) continue;            /* chroma edges lie at luma edges 0 and 2 */
            const int32_t* qpa = chroma ? d->qp_c : d->qp;
            const int qpav = e == 0 ? (qpa[q] + qpa[p] + 1) >> 1 : qpa[q];
            const int ia = clip3 (qpav + off_a, 0, 51), ib = clip3 (qpav + off_b, 0, 51);
            const int alpha = kDbkAlpha[ia], beta = kDbkBeta[ib];
            int8_t tc[4];
            if (!chroma) {
              uint8_t* pix = y + (size_t) (16 * mby + (dir ? 4 * e : 0)) * stride_y + 16 * mbx + (dir ? 0 : 4 * e);
              const int sx = dir ? stride_y : 1, sy = dir ? 1 : stride_y;
              for (int l = 0; l < 16; l++) if (bs[l >> 2]) dbk_count_luma (pix + l * sy, sx, alpha, beta, bs[l >> 2], st);
              if (bs[0] == 4) {                           /* bS 4 only on macroblock edges with an intra side: all 4 segments */
                orc_deblock_luma_eq4 (pix, sx, sy, alpha, beta);
              } else {
                for (int s = 0; s < 4; s++) tc[s] = (int8_t) (bs[s] ? kDbkTc0[bs[s] - 1][ia] : -1);
                orc_deblock_luma_lt4 (pix, sx, sy, alpha, beta, tc);   /* tc = tC0 + ap + aq inside the filter */
              }
            } else {
              const size_t off = (size_t) (8 * mby + (dir ? 2 * e : 0)) * stride_c + 8 * mbx + (dir ? 0 : 2 * e);
              const int sx = dir ? stride_c : 1, sy = dir ? 1 : stride_c;
              for (int l = 0; l < 8; l++)
                if (bs[l >> 1]) {
                  dbk_count_chroma (cb + off + l * sy, sx, alpha, beta, bs[l >> 1], st);
                  dbk_count_chroma (cr + off + l * sy, sx, alpha, beta, bs[l >> 1], st);
                }
              if (bs[0] == 4) {
                orc_deblock_chroma_eq4 (cb + off, cr + off, sx, sy, alpha, beta);
              } else {
                for (int s = 0; s < 4; s++) tc[s] = (int8_t) (bs[s] ? kDbkTc0[bs[s] - 1][ia] + 1 : 0);   /* chroma: tC = tC0 + 1 */
                orc_deblock_chroma_lt4 (cb + off, cr + off, sx, sy, alpha, beta, tc);
              }
            }
          }
        }
      }
    }
}

/* ------------------------------------------------------------------------------------------
 * expand_pic.cpp:40-340,388: replicate the picture border `pad` pixels outwards on all sides
 * ------------------------------------------------------------------------------------------ */
void orc_expand_plane (uint8_t* pic, int stride, int w, int h, int pad) {
  for (int y = 0; y < h; y++) {
    uint8_t* row = pic + y * stride;
    memset (row - pad, row[0], (size_t) pad);
    memset (row + w, row[w - 1], (size_t) pad);
  }
  for (int y = 1; y <= pad; y++) {
    memcpy (pic - y * stride - pad, pic - pad, (size_t) (w + 2 * pad));
    memcpy (pic + (h - 1 + y) * stride - pad, pic + (h - 1) * stride - pad, (size_t) (w + 2 * pad));
  }
}

/* ------------------------------------------------------------------------------------------
 * Integer-pel motion search: initial point test + small-diamond descent (+ SATD of the winner)
 * svc_motion_estimate.cpp:170-181 (driver), :222-284 (initial point), :300-386 (diamond)
 * ------------------------------------------------------------------------------------------ */
#define ORC_MVD_SZ 1100   /* |mvd| bound in quarter-pel for the oracle's private cost table */
void orc_me_search (const uint8_t* cur, int cs, const uint8_t* ref, int rs, const orc_me_job* j, orc_me_result* out) {
  static uint16_t cost_tbl[52][2 * ORC_MVD_SZ + 1];
  static uint8_t cost_ready[52];
  if (!cost_ready[j->qp]) { orc_mvd_cost_init (cost_tbl[j->qp] + ORC_MVD_SZ, ORC_MVD_SZ, j->qp); cost_ready[j->qp] = 1; }
  const uint16_t* mvd = cost_tbl[j->qp] + ORC_MVD_SZ;
  const uint8_t* enc = cur + j->cur_off;
  const uint8_t* col = ref + j->ref_off;
  const int px = j->mvp_x, py = j->mvp_y;

  /* initial point: rounded predictor, clamped to the search window (:242-250) */
  int mx = clip3 ((2 + px) >> 2, j->mv_min_x, j->mv_max_x);
  int my = clip3 ((2 + py) >> 2, j->mv_min_y, j->mv_max_y);
  const uint8_t* best_ref = col + my * rs + mx;
  int best = orc_sad (j->blk, enc, cs, best_ref, rs) + mvd[mx * 4 - px] + mvd[my * 4 - py];
  for (int i = 0; i < j->n_mvc; i++) {               /* candidate predictors (:252-270) */
    const int cx = clip3 ((2 + j->mvc[i][0]) >> 2, j->mv_min_x, j->mv_max_x);
    const int cy = clip3 ((2 + j->mvc[i][1]) >> 2, j->mv_min_y, j->mv_max_y);
    if (cx == mx && cy == my) continue;
    const uint8_t* r = col + cy * rs + cx;
    const int c = orc_sad (j->blk, enc, cs, r, rs) + mvd[cx * 4 - px] + mvd[cy * 4 - py];
    if (c < best) { best = c; mx = cx; my = cy; best_ref = r; }
  }
  if (!(best < (int32_t) j->sad_pred)) {             /* no early stop (:278) -> diamond (:335-386) */
    int dx = mx * 4 - px, dy = my * 4 - py;
    for (int iter = 0; iter < 16; iter++) {
      const int tx = (dx + px) >> 2, ty = (dy + py) >> 2;
      /* half-open range test; an out-of-range centre just burns the iteration (:357-359) */
      if (!(tx >= j->mv_min_x && tx < j->mv_max_x && ty >= j->mv_min_y && ty < j->mv_max_y)) continue;
      int32_t s[4];
      orc_sad_four (j->blk, enc, cs, best_ref, rs, s);
      const int c_up = s[0] + mvd[dx] + mvd[dy - 4], c_dn = s[1] + mvd[dx] + mvd[dy + 4];
      const int c_lf = s[2] + mvd[dx - 4] + mvd[dy], c_rt = s[3] + mvd[dx + 4] + mvd[dy];
      int sx = 0, sy = 0, moved = 0;                 /* strict <, tested up, down, left, right (:309-331) */
      if (c_up < best) { best = c_up; sx = 0; sy = -1; moved = 1; }
      if (c_dn < best) { best = c_dn; sx = 0; sy = 1; moved = 1; }
      if (c_lf < best) { best = c_lf; sx = -1; sy = 0; moved = 1; }
      if (c_rt < best) { best = c_rt; sx = 1; sy = 0; moved = 1; }
      if (!moved) break;
      dx += 4 * sx; dy += 4 * sy;
      best_ref += sx + sy * rs;
    }
    mx = (dx + px) >> 2; my = (dy + py) >> 2;
  }
  out->mv_x = (int16_t) (mx * 4);
  out->mv_y = (int16_t) (my * 4);
  out->sad_cost = (uint32_t) best;
  out->satd_cost = (uint32_t) best;                  /* MeEndIntepelSearch (:67-72) */
  out->ref_off = (int32_t) (best_ref - ref);
  if (j->calc_satd)                                  /* CalculateSatdCost (:286-291) */
    out->satd_cost = (uint32_t) (orc_satd (j->blk, enc, cs, best_ref, rs) + mvd[out->mv_x - px] + mvd[out->mv_y - py]);
}

/* ------------------------------------------------------------------------------------------
 * VPP bilinear down-sampler (SURVEY.md 8f rank 3): codec/processing/src/downsample/downsamplefuncs.cpp
 *   mode 0 DyadicBilinearDownsampler_c :47      dst = src / 2
 *   mode 1 DyadicBilinearQuarterDownsampler_c :73   dst = src / 4 (top-left 2x2 of every 4x4)
 *   mode 2 DyadicBilinearOneThirdDownsampler_c :99  dst = src / 3 (top-left 2x2 of every 3x3)
 *   mode 3 GeneralBilinearFastDownsampler_c :118    (luma, 16.15 fixed point, 32-bit products)
 *   mode 4 GeneralBilinearAccurateDownsampler_c :189 (chroma, 15.15 fixed point, 64-bit products)
 * dst_w / dst_h are the destination dimensions in every mode.
 * ------------------------------------------------------------------------------------------ */
static int orc_round_ratio (int src, int dst, int scale) {       /* WELS_ROUND ((float)src / (float)dst * scale), macros.h:120 */
  return (int) (0.5 + ((float) src / (float) dst * scale));
}
void orc_downsample (int mode, uint8_t* dst, int ds, int dst_w, int dst_h, const uint8_t* src, int ss, int src_w, int src_h) {
  if (mode <= 2) {
    const int step = mode == 0 ? 2 : mode == 1 ? 4 : 3;
    for (int j = 0; j < dst_h; j++)
      for (int i = 0; i < dst_w; i++) {
        const uint8_t* p = src + (size_t) j * step * ss + i * step;
        const int r1 = (p[0] + p[1] + 1) >> 1, r2 = (p[ss] + p[ss + 1] + 1) >> 1;
        dst[(size_t) j * ds + i] = (uint8_t) ((r1 + r2 + 1) >> 1);
      }
    return;
  }
  const int bw = mode == 3 ? 16 : 15, bh = 15;
  const int sx = orc_round_ratio (src_w, dst_w, 1 << bw), sy = orc_round_ratio (src_h, dst_h, 1 << bh);
  for (int i = 0; i < dst_h; i++) {
    const int yinv = (1 << (bh - 1)) + i * sy;
    const int yy = yinv >> bh, fv = yinv & ((1 << bh) - 1);
    const uint8_t* row = src + (size_t) yy * ss;
    for (int j = 0; j < dst_w; j++) {
      const int xinv = (1 << (bw - 1)) + j * sx;
      const int xx = xinv >> bw, fu = xinv & ((1 << bw) - 1);
      uint8_t v;
      if (i == dst_h - 1 || j == dst_w - 1) v = row[xx];          /* last row / last column: nearest sample */
      else {
        const uint32_t a = row[xx], b = row[xx + 1], c = row[xx + ss], d = row[xx + ss + 1];
        if (mode == 3) {
          const uint32_t W = 1u << bw, Hh = 1u << bh;
          uint32_t x = (((uint32_t) (W - 1 - fu)) * (Hh - 1 - fv) >> bw) * a;
          x += (((uint32_t) fu) * (Hh - 1 - fv) >> bw) * b;
          x += (((uint32_t) (W - 1 - fu)) * (uint32_t) fv >> bw) * c;
          x += (((uint32_t) fu) * (uint32_t) fv >> bw) * d;
          x >>= (bh - 1);
          x += 1;
          x >>= 1;
          v = (uint8_t) (x > 255 ? 255 : x);
        } else {
          const int64_t S = 1 << 15;
          int64_t x = ((S - 1 - fu) * (S - 1 - fv) * a + (int64_t) fu * (S - 1 - fv) * b + (S - 1 - fu) * fv * c + (int64_t) fu * fv * d +
                       ((int64_t) 1 << 29)) >> 30;
          v = (uint8_t) (x < 0 ? 0 : x > 255 ? 255 : x);
        }
      }
      dst[(size_t) i * ds + j] = v;
    }
  }
}

/* ---- WelsMotionCrossSearch / LineFullSearch_c (svc_motion_estimate.cpp:568-643) ------------------------------------------ */
static void orc_line_search (const uint8_t* enc, int cs, const uint8_t* colo, const uint8_t* ref_plane, int rs, const orc_cross_job* j,
                             const uint16_t* mvd, int min_mv, int max_mv, int vertical, orc_me_result* io) {
  /* iFixedMvd: the cost of the component that stays at 0; pMvdCost walks the other one in integer-pel steps (:585-598) */
  const int fixed = vertical ? mvd[-j->mvp_x] : mvd[-j->mvp_y];
  const uint16_t* c = mvd + min_mv * 4 - (vertical ? j->mvp_y : j->mvp_x);
  const int stride = vertical ? rs : 1;
  const uint8_t* r = colo + min_mv * stride;
  uint32_t best = 0xFFFFFFFFu;
  int best_mv = 0;
  for (int mv = min_mv; mv < max_mv; mv++) {                 /* iTargetPos < iMaxPos: the maximum is exclusive */
    const uint32_t cost = (uint32_t) orc_sad (j->blk, enc, cs, r, rs) + (uint32_t) (fixed + *c);
    if (cost < best) { best = cost; best_mv = mv; }
    r += stride; c += 4;
  }
  if (best < io->sad_cost) {                                 /* UpdateMeResults (:60) */
    io->mv_x = (int16_t) (vertical ? 0 : best_mv);
    io->mv_y = (int16_t) (vertical ? best_mv : 0);
    io->sad_cost = best;
    io->ref_off = (int32_t) (colo + io->mv_y * rs + io->mv_x - ref_plane);
  }
}
void orc_me_cross_search (const uint8_t* cur, int cs, const uint8_t* ref, int rs, const orc_cross_job* j, orc_me_result* io) {
  static uint16_t cost_tbl[52][2 * ORC_MVD_SZ + 1];
  static uint8_t cost_ready[52];
  if (!cost_ready[j->qp]) { orc_mvd_cost_init (cost_tbl[j->qp] + ORC_MVD_SZ, ORC_MVD_SZ, j->qp); cost_ready[j->qp] = 1; }
  const uint16_t* mvd = cost_tbl[j->qp] + ORC_MVD_SZ;
  const uint8_t* enc = cur + j->cur_off;
  const uint8_t* colo = ref + j->ref_off;
  orc_line_search (enc, cs, colo, ref, rs, j, mvd, j->mv_min_y, j->mv_max_y, 1, io);
  if (io->sad_cost >= j->sad_cost_threshold)
    orc_line_search (enc, cs, colo, ref, rs, j, mvd, j->mv_min_x, j->mv_max_x, 0, io);
}

/* ---- rec_mb.cpp:298-460: weighted / bi-directional prediction of one plane ------------------------------------------------ */
static uint8_t orc_clip255 (int v) { return (uint8_t) (v < 0 ? 0 : v > 255 ? 255 : v); }
void orc_weight_pred (uint8_t* dst, int stride, int w, int h, int log2_denom, int weight, int offset) {
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) {
      const int p = dst[y * stride + x];
      const int v = log2_denom >= 1 ? ((p * weight + (1 << (log2_denom - 1))) >> log2_denom) + offset : p * weight + offset;
      dst[y * stride + x] = orc_clip255 (v);
    }
}
void orc_biweight_pred (uint8_t* dst, const uint8_t* tmp, int stride, int w, int h, int log2_denom, int w1, int o1, int w2, int o2) {
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) {
      const int v = ((dst[y * stride + x] * w1 + tmp[y * stride + x] * w2 + (1 << log2_denom)) >> (log2_denom + 1)) + ((o1 + o2 + 1) >> 1);
      dst[y * stride + x] = orc_clip255 (v);
    }
}
void orc_bi_pred (uint8_t* dst, const uint8_t* tmp, int stride, int w, int h) {
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) dst[y * stride + x] = (uint8_t) ((dst[y * stride + x] + tmp[y * stride + x] + 1) >> 1);
}
