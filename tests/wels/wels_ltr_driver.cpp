// wels_ltr_driver.cpp — TEST INFRASTRUCTURE.  An application written against the reference's public API (codec/api/wels/codec_api.h)
// that loads "some libopenh264" with dlopen and encodes a clip through InitializeExt / EncodeFrame with long-term references and
// iNumRefFrame as given, while it plays a receiver's part from a script: loss-recovery requests, LTR marking feedback, marking
// period changes and ForceIntraFrame, each before a given picture.  It writes the bitstream and a log of what InitializeExt
// returned, the resolved reference parameters GetOption reports, every scripted call's return code and the frame layout of every
// EncodeFrame call.  tests/golden/make_ltr_golden.py runs it with the compiled reference, tests/test_wels_api_ltr.py with
// openh264_b200/libopenh264_b200_wels.so.  The input clip is read in a loop when it has fewer pictures than asked for.
//   wels_ltr_driver <lib.so> <in.yuv> <w> <h> <frames> <qp> <out.264> <out.log> <entropy_cabac> <complexity>
//                   <num_ref_frames> <ltr> <ltr_mark_period> <script>
// Script lines: "<picture> rr <type> <idr> <cur_fn> <last_fn>"  ENCODER_LTR_RECOVERY_REQUEST
//               "<picture> mf <type> <idr> <ltr_fn>"            ENCODER_LTR_MARKING_FEEDBACK
//               "<picture> period <n>"                          ENCODER_LTR_MARKING_PERIOD
//               "<picture> idr"                                 ForceIntraFrame(true)
//               "<picture> ltropt <0|1>"                        ENCODER_OPTION_LTR (iLTRRefNum 2)
// <idr> is "cur" (the idr_pic_id of the last IDR), "old" (one less) or a number; a frame number is a number or "pK", the
// frame_num of the picture coded K pictures before the one the line precedes.
#include <dlfcn.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "codec_api.h"

typedef int (*create_fn)(ISVCEncoder**);
typedef void (*destroy_fn)(ISVCEncoder*);

struct Event { int at; std::string op; std::vector<std::string> a; };

int main(int argc, char** argv) {
  if (argc < 15) { fprintf(stderr, "usage: see source\n"); return 2; }
  void* lib = dlopen(argv[1], RTLD_NOW | RTLD_LOCAL);
  if (!lib) { fprintf(stderr, "dlopen: %s\n", dlerror()); return 3; }
  create_fn create = (create_fn)dlsym(lib, "WelsCreateSVCEncoder");
  destroy_fn destroy = (destroy_fn)dlsym(lib, "WelsDestroySVCEncoder");
  if (!create || !destroy) { fprintf(stderr, "missing entry points\n"); return 3; }
  const int w = atoi(argv[3]), h = atoi(argv[4]), n = atoi(argv[5]), qp = atoi(argv[6]);
  FILE* fin = fopen(argv[2], "rb");
  FILE* fout = fopen(argv[7], "wb");
  FILE* flog = fopen(argv[8], "w");
  FILE* fscr = fopen(argv[14], "r");
  if (!fin || !fout || !flog || !fscr) { fprintf(stderr, "cannot open files\n"); return 3; }
  std::vector<Event> ev;
  char line[512];
  while (fgets(line, sizeof(line), fscr)) {
    Event e;
    char* tok = strtok(line, " \t\r\n");
    if (!tok) continue;
    e.at = atoi(tok);
    if (!(tok = strtok(NULL, " \t\r\n"))) continue;
    e.op = tok;
    while ((tok = strtok(NULL, " \t\r\n"))) e.a.push_back(tok);
    ev.push_back(e);
  }
  fclose(fscr);
  ISVCEncoder* enc = NULL;
  if (create(&enc) || !enc) { fprintf(stderr, "WelsCreateSVCEncoder failed\n"); return 4; }
  SEncParamExt p;
  enc->GetDefaultParams(&p);
  p.iUsageType = CAMERA_VIDEO_REAL_TIME;
  p.iPicWidth = w; p.iPicHeight = h;
  p.iTargetBitrate = 5000000;
  p.iRCMode = RC_OFF_MODE;
  p.fMaxFrameRate = 30.0f;
  p.iComplexityMode = (ECOMPLEXITY_MODE)atoi(argv[10]);
  p.iNumRefFrame = atoi(argv[11]);
  p.bEnableLongTermReference = atoi(argv[12]) != 0;
  p.iLtrMarkPeriod = atoi(argv[13]);
  p.bEnableFrameSkip = false;
  p.bEnableDenoise = p.bEnableBackgroundDetection = p.bEnableSceneChangeDetect = p.bEnableAdaptiveQuant = false;
  p.iEntropyCodingModeFlag = atoi(argv[9]);
  p.uiIntraPeriod = 0;
  p.sSpatialLayers[0].iVideoWidth = w; p.sSpatialLayers[0].iVideoHeight = h;
  p.sSpatialLayers[0].fFrameRate = 30.0f;
  p.sSpatialLayers[0].iSpatialBitrate = 5000000;
  p.sSpatialLayers[0].iDLayerQp = qp;
  p.sSpatialLayers[0].sSliceArgument.uiSliceMode = SM_SINGLE_SLICE;
  int rc = enc->InitializeExt(&p);
  fprintf(flog, "InitializeExt -> %d\n", rc);
  if (rc) { fclose(flog); fclose(fout); return 5; }
  int lvl = WELS_LOG_QUIET;
  enc->SetOption(ENCODER_OPTION_TRACE_LEVEL, &lvl);
  SEncParamExt r;
  memset(&r, 0, sizeof(r));
  enc->GetOption(ENCODER_OPTION_SVC_ENCODE_PARAM_EXT, &r);
  fprintf(flog, "resolved ltr=%d ltr_ref_num=%d num_ref=%d period=%d\n", (int)r.bEnableLongTermReference, r.iLTRRefNum,
          r.iNumRefFrame, r.iLtrMarkPeriod);
  const size_t fsz = (size_t)w * h * 3 / 2;
  std::vector<unsigned char> buf(fsz);
  std::vector<int> fn;                        // frame_num of every picture coded so far
  int idr_id = 0, next_fn = 0;                // uiIdrPicId after the IDRs so far; frame_num of the next P picture
  auto frame_no = [&](const std::string& t) {
    if (t[0] == 'p') { const int k = atoi(t.c_str() + 1); return k >= 1 && k <= (int)fn.size() ? fn[fn.size() - k] : -1; }
    return atoi(t.c_str());
  };
  auto idr_no = [&](const std::string& t) { return t == "cur" ? idr_id : t == "old" ? idr_id - 1 : atoi(t.c_str()); };
  for (int i = 0; i < n; i++) {
    if (fread(buf.data(), 1, fsz, fin) != fsz) {
      rewind(fin);
      if (fread(buf.data(), 1, fsz, fin) != fsz) break;
    }
    for (const Event& e : ev) {
      if (e.at != i) continue;
      if (e.op == "idr") {
        fprintf(flog, "%d idr -> %d\n", i, enc->ForceIntraFrame(true));
      } else if (e.op == "period" && e.a.size() == 1) {
        unsigned int v = (unsigned int)atoi(e.a[0].c_str());
        fprintf(flog, "%d period %u -> %d\n", i, v, enc->SetOption(ENCODER_LTR_MARKING_PERIOD, &v));
      } else if (e.op == "ltropt" && e.a.size() == 1) {
        SLTRConfig c;
        c.bEnableLongTermReference = atoi(e.a[0].c_str()) != 0;
        c.iLTRRefNum = 2;
        fprintf(flog, "%d ltropt %d -> %d\n", i, (int)c.bEnableLongTermReference, enc->SetOption(ENCODER_OPTION_LTR, &c));
      } else if (e.op == "rr" && e.a.size() == 4) {
        SLTRRecoverRequest q;
        memset(&q, 0, sizeof(q));
        q.uiFeedbackType = (unsigned int)atoi(e.a[0].c_str());
        q.uiIDRPicId = (unsigned int)idr_no(e.a[1]);
        q.iCurrentFrameNum = frame_no(e.a[2]);
        q.iLastCorrectFrameNum = frame_no(e.a[3]);
        q.iLayerId = 0;
        const int c = enc->SetOption(ENCODER_LTR_RECOVERY_REQUEST, &q);
        fprintf(flog, "%d rr %u %u %d %d -> %d\n", i, q.uiFeedbackType, q.uiIDRPicId, q.iCurrentFrameNum, q.iLastCorrectFrameNum, c);
      } else if (e.op == "mf" && e.a.size() == 3) {
        SLTRMarkingFeedback q;
        memset(&q, 0, sizeof(q));
        q.uiFeedbackType = (unsigned int)atoi(e.a[0].c_str());
        q.uiIDRPicId = (unsigned int)idr_no(e.a[1]);
        q.iLTRFrameNum = frame_no(e.a[2]);
        q.iLayerId = 0;
        const int c = enc->SetOption(ENCODER_LTR_MARKING_FEEDBACK, &q);
        fprintf(flog, "%d mf %u %u %d -> %d\n", i, q.uiFeedbackType, q.uiIDRPicId, q.iLTRFrameNum, c);
      } else {
        fprintf(stderr, "bad script line at picture %d: %s\n", e.at, e.op.c_str());
        return 7;
      }
    }
    SSourcePicture pic;
    memset(&pic, 0, sizeof(pic));
    pic.iColorFormat = videoFormatI420;
    pic.iPicWidth = w; pic.iPicHeight = h;
    pic.iStride[0] = w; pic.iStride[1] = pic.iStride[2] = w / 2;
    pic.pData[0] = buf.data();
    pic.pData[1] = pic.pData[0] + (size_t)w * h;
    pic.pData[2] = pic.pData[1] + (size_t)w * h / 4;
    pic.uiTimeStamp = (long long)(i * 1000.0 / 30.0);
    SFrameBSInfo info;
    memset(&info, 0, sizeof(info));
    rc = enc->EncodeFrame(&pic, &info);
    if (rc) { fprintf(flog, "frame %d failed %d\n", i, rc); continue; }
    const bool idr = info.eFrameType == videoFrameTypeIDR;
    if (idr) { idr_id = idr_id < 65535 ? idr_id + 1 : 0; next_fn = 0; }
    fn.push_back(next_fn);
    next_fn = next_fn < 32767 ? next_fn + 1 : 0;
    fprintf(flog, "frame %d type %d layers %d bytes %d:", i, (int)info.eFrameType, info.iLayerNum, info.iFrameSizeInBytes);
    for (int l = 0; l < info.iLayerNum; l++) {
      const SLayerBSInfo& L = info.sLayerInfo[l];
      int sz = 0;
      for (int k = 0; k < L.iNalCount; k++) { fprintf(flog, " %d", L.pNalLengthInByte[k]); sz += L.pNalLengthInByte[k]; }
      fwrite(L.pBsBuf, 1, sz, fout);
    }
    fprintf(flog, "\n");
  }
  enc->Uninitialize();
  destroy(enc);
  fclose(fin); fclose(fout); fclose(flog);
  return 0;
}
