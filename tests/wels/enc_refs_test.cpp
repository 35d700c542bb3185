// enc_refs_test.cpp — TEST INFRASTRUCTURE.  Plays a receiver script (the format of wels_ltr_driver.cpp) against the encoder's
// reference state machine alone (openh264_b200/csrc/enc_refs.h, no CUDA) and prints, per picture, the decisions that reach the
// slice header: IDR, frame_num, list modification, MMCOs, long_term_reference_flag; or that the picture is not coded.  tests/test_enc_refs_cpu.py compares them
// with the slice headers of the reference encoder's bitstreams (tests/golden/ltr.json).
//   enc_refs_test <num_ref_frames> <ltr> <ltr_mark_period> <pictures> <script>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "enc_refs.h"

int main(int argc, char** argv) {
  if (argc < 6) { fprintf(stderr, "usage: see source\n"); return 2; }
  b2h264::RefConfig cfg;
  if (!b2h264::RefConfig::resolve(atoi(argv[1]), atoi(argv[2]) != 0, atoi(argv[3]), 0, &cfg)) return 3;
  b2h264::StreamRefs refs;
  refs.cfg = cfg;
  refs.reset();
  const int n = atoi(argv[4]);
  FILE* f = fopen(argv[5], "r");
  if (!f) return 3;
  std::vector<std::vector<std::string>> ev;
  char line[512];
  while (fgets(line, sizeof(line), f)) {
    std::vector<std::string> t;
    for (char* tok = strtok(line, " \t\r\n"); tok; tok = strtok(NULL, " \t\r\n")) t.push_back(tok);
    if (t.size() >= 2) ev.push_back(t);
  }
  fclose(f);
  printf("sps_num_ref %d slots %d\n", cfg.sps_num_ref_frames, cfg.slots());
  std::vector<int> fn;
  bool force = true;
  auto frame_no = [&](const std::string& t) {
    if (t[0] == 'p') { const int k = atoi(t.c_str() + 1); return k >= 1 && k <= (int)fn.size() ? fn[fn.size() - k] : -1; }
    return atoi(t.c_str());
  };
  auto idr_no = [&](const std::string& t) { return t == "cur" ? refs.idr_pic_id() : t == "old" ? refs.idr_pic_id() - 1 : atoi(t.c_str()); };
  for (int i = 0; i < n; i++) {
    for (const auto& e : ev) {
      if (atoi(e[0].c_str()) != i) continue;
      if (e[1] == "idr") force = true;
      else if (e[1] == "period") refs.set_mark_period(atoi(e[2].c_str()));
      else if (e[1] == "rr") refs.recovery_request(atoi(e[2].c_str()), idr_no(e[3]), frame_no(e[4]), frame_no(e[5]));
      else if (e[1] == "mf") refs.marking_feedback(atoi(e[2].c_str()), idr_no(e[3]), frame_no(e[4]));
    }
    const b2h264::RefDecision d = refs.code_picture(force || refs.idr_wanted());
    force = false;
    if (d.not_coded) { printf("pic %d failed\n", i); continue; }
    fn.push_back(d.frame_num);
    printf("pic %d %d %d", i, (int)d.idr, d.frame_num);
    if (!d.idr) printf(" mod %d %d", d.mod_idc, d.mod_val);
    for (int k = 0; k < d.n_mmco; k++) {
      printf(" mmco %d %d", d.mmco[k][0], d.mmco[k][1]);
      if (d.mmco[k][0] == 3) printf(" %d", d.mmco[k][2]);
    }
    printf(" lt %d rec %d ref %d src %d %d\n", (int)d.long_term_reference_flag, d.rec_slot, d.ref_slot, d.cur_src, d.vaa_src);
  }
  return 0;
}
