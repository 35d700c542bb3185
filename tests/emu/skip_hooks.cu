// tests/emu/skip_hooks.cu — test hooks of the P-skip test for the host emulation build (TEST INFRASTRUCTURE ONLY).  The counters
// are the host build's (enc_inter.cuh: g_skip_outcome, g_skip_phase_luma / g_skip_phase_chroma), filled by every emu_encode.
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../../openh264_b200/csrc/stage_hooks.cuh"

using namespace mbk;

extern "C" void b2h264_build_host_tables();

extern "C" void emu_reset_skip_outcomes() {
  memset(g_skip_outcome, 0, sizeof(g_skip_outcome));
  g_skip_phase_luma = g_skip_phase_chroma = 0;
}
// counts of each outcome of the skip test since the last reset (SKIP_RANGE .. SKIP_DCT_OK), then the masks of the luma
// quarter-sample and chroma eighth-sample phases it predicted with
extern "C" int emu_skip_outcomes(uint64_t* out, int n) {
  if (n < SKIP_OUTCOMES + 2) return -1;
  memcpy(out, g_skip_outcome, sizeof(g_skip_outcome));
  out[SKIP_OUTCOMES] = g_skip_phase_luma;
  out[SKIP_OUTCOMES + 1] = g_skip_phase_chroma;
  return SKIP_OUTCOMES + 2;
}
// The host build of the device hook b2h264_debug_skip_test (enc_kernels.cu), same arguments and refusals; planes: HOST memory,
// the one set every job reads.  Each job's outcome is counted like an encode's (emu_skip_outcomes).
extern "C" int emu_skip_test(int n, const uint8_t* planes, long long set_bytes, const uint8_t* jobs, uint8_t* out) {
  if (!skip_test_args_ok(n, planes, set_bytes, jobs, out)) return -1;
  b2h264_build_host_tables();
  static MbScratch s;
  for (int i = 0; i < n; i++) {
    memset(&s, 0, sizeof(s));
    int32_t sad = kSkipSadUnset;
    skip_test_case(jobs + (size_t)kSkipJobIn * i, planes, &sad, out + (size_t)kSkipJobOut * i, s);
  }
  return 0;
}
// warp_mc_chroma_pair against warp_mc_chroma: every eighth-sample phase, widths 2 / 4 / 8, heights 2 / 4 / 8 and every
// source alignment; returns the number of differing samples
extern "C" long emu_check_chroma_pair() {
  const int ss = 40;
  std::vector<uint8_t> src(ss * 20);
  uint32_t x = 12345;
  for (auto& v : src) { x = x * 1664525u + 1013904223u; v = (uint8_t)(x >> 24); }
  long bad = 0;
  for (int ph = 0; ph < 64; ph++)
    for (int w = 2; w <= 8; w *= 2)
      for (int h = 2; h <= 8; h *= 2)
        for (int al = 0; al < 4; al++) {
          alignas(4) uint8_t got[128], want[128];
          memset(got, 0, sizeof(got)); memset(want, 0, sizeof(want));
          const uint8_t* p0 = src.data() + ss + 4 + al;
          const uint8_t* p1 = src.data() + 9 * ss + 12 + al;
          warp_mc_chroma_pair(p0, p1, ss, got, 8, ph & 7, ph >> 3, w, h);
          warp_mc_chroma(p0, ss, want, 8, ph & 7, ph >> 3, w, h);
          warp_mc_chroma(p1, ss, want + 64, 8, ph & 7, ph >> 3, w, h);
          for (int i = 0; i < 128; i++) bad += got[i] != want[i];
        }
  return bad;
}
