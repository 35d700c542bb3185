// tests/emu/inter_residual_hooks.cu — test hooks of stage B's residual step for the host emulation build (TEST INFRASTRUCTURE
// ONLY).  emu_inter_residual is the host build of the device hook b2h264_debug_inter_residual (enc_kernels.cu), same layout
// and refusals; the outcome counters (enc_inter.cuh: g_res_outcome) are filled by every emu_encode.
#include <stdint.h>
#include <string.h>

#include "../../openh264_b200/csrc/stage_hooks.cuh"

using namespace mbk;

extern "C" void b2h264_build_host_tables();

extern "C" int emu_inter_residual(int n, const uint8_t* src_pred, const int* qp, uint8_t* out) {
  if (!inter_residual_args_ok(n, src_pred, qp, out)) return -1;
  b2h264_build_host_tables();
  static MbScratch s;
  for (int i = 0; i < n; i++) {
    memset(&s, 0, sizeof(s));
    inter_residual_case(src_pred + 768 * i, qp[i], out + (size_t)kInterResOut * i, s);
  }
  return 0;
}

extern "C" void emu_reset_res_outcomes() { memset(g_res_outcome, 0, sizeof(g_res_outcome)); }
// counts of each stage-B outcome since the last reset (RES_LUMA_ZEROED .. RES_PSKIP_CODED)
extern "C" int emu_res_outcomes(uint64_t* out, int n) {
  if (n < RES_OUTCOMES) return -1;
  memcpy(out, g_res_outcome, sizeof(g_res_outcome));
  return RES_OUTCOMES;
}
