// tests/emu/me_hooks.cu — test hook of stage B's motion search for the host emulation build (TEST INFRASTRUCTURE ONLY).
// emu_me_partitions is the host build of the device hook b2h264_debug_me_partitions (enc_kernels.cu), with its layout and the
// refusals both builds share.  The host build has no search window (win_issue leaves win_ok 0): every search and refinement
// reads the planes.
#include <stdint.h>
#include <string.h>

#include "../../openh264_b200/csrc/stage_hooks.cuh"

using namespace mbk;

extern "C" void b2h264_build_host_tables();

// planes: HOST memory, job i's set at planes + i * set_bytes (layout as the device hook)
extern "C" int emu_me_partitions(int n, const uint8_t* planes, long long set_bytes, const uint8_t* jobs, uint8_t* out) {
  if (!me_partitions_args_ok(n, planes, set_bytes, jobs, out)) return -1;
  b2h264_build_host_tables();
  static MbScratch s;
  for (int i = 0; i < n; i++) {
    memset(&s, 0, sizeof(s));
    me_partitions_case(i, planes + (size_t)set_bytes * i, jobs + (size_t)kMeJobIn * i, out + (size_t)kMeJobOut * i, s, nullptr, nullptr);
  }
  return 0;
}
