// tests/emu/intra_tail_hooks.cu — test hooks of the intra tail for the host emulation build (TEST INFRASTRUCTURE ONLY).
// emu_intra_tail is the host build of the device hook b2h264_debug_intra_tail (enc_kernels.cu), same layout and refusals; the
// I4x4 outcome counters (enc_mb.cuh: g_i4_end) are filled by every intra tail the host build runs.
#include <stdint.h>
#include <string.h>

#include "../../openh264_b200/csrc/stage_hooks.cuh"

using namespace mbk;

extern "C" void b2h264_build_host_tables();

extern "C" int emu_intra_tail(int n, const uint8_t* in, uint8_t* out) {
  if (!intra_tail_args_ok(n, in, out)) return -1;
  b2h264_build_host_tables();
  static MbScratch s;
  for (int i = 0; i < n; i++) {
    memset(&s, 0, sizeof(s));
    int32_t sad = 0;
    intra_tail_case(in + (size_t)kIntraTailIn * i, &sad, out + (size_t)kIntraTailOut * i, s);
  }
  return 0;
}

extern "C" void emu_reset_i4_ends() { memset(g_i4_end, 0, sizeof(g_i4_end)); }
// counts of each end of the I4x4 try since the last reset (I4_END_BREAK, I4_END_COMPLETE, I4_END_WON)
extern "C" int emu_i4_ends(uint64_t* out, int n) {
  if (n < I4_END_OUTCOMES) return -1;
  memcpy(out, g_i4_end, sizeof(g_i4_end));
  return I4_END_OUTCOMES;
}
