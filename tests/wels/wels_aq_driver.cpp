// wels_aq_driver.cpp — TEST INFRASTRUCTURE.  An application written against the reference's public API (codec/api/wels/codec_api.h)
// that loads "some libopenh264" with dlopen and encodes a clip through InitializeExt / EncodeFrame with bEnableAdaptiveQuant and
// [iMinQp, iMaxQp] as given.  It writes the bitstream, and a log of what InitializeExt returned, what GetOption reports the
// encoder resolved adaptive quantisation to, and the frame layout of every EncodeFrame call.  tests/test_wels_api_aq.py runs the
// same binary with the compiled reference and with openh264_b200/libopenh264_b200_wels.so.
//   wels_aq_driver <lib.so> <in.yuv> <w> <h> <frames> <qp> <force_idr_at|-1> <out.264> <out.log>
//                  <entropy_cabac> <profile_idc> <intra_period> <aq> <min_qp> <max_qp>
#include <dlfcn.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "codec_api.h"

typedef int (*create_fn)(ISVCEncoder**);
typedef void (*destroy_fn)(ISVCEncoder*);

int main(int argc, char** argv) {
  if (argc < 16) { fprintf(stderr, "usage: see source\n"); return 2; }
  void* lib = dlopen(argv[1], RTLD_NOW | RTLD_LOCAL);
  if (!lib) { fprintf(stderr, "dlopen: %s\n", dlerror()); return 3; }
  create_fn create = (create_fn)dlsym(lib, "WelsCreateSVCEncoder");
  destroy_fn destroy = (destroy_fn)dlsym(lib, "WelsDestroySVCEncoder");
  if (!create || !destroy) { fprintf(stderr, "missing entry points\n"); return 3; }
  const int w = atoi(argv[3]), h = atoi(argv[4]), n = atoi(argv[5]), qp = atoi(argv[6]), idr_at = atoi(argv[7]);
  FILE* fin = fopen(argv[2], "rb");
  FILE* fout = fopen(argv[8], "wb");
  FILE* flog = fopen(argv[9], "w");
  if (!fin || !fout || !flog) { fprintf(stderr, "cannot open files\n"); return 3; }
  ISVCEncoder* enc = NULL;
  if (create(&enc) || !enc) { fprintf(stderr, "WelsCreateSVCEncoder failed\n"); return 4; }
  SEncParamExt p;
  enc->GetDefaultParams(&p);
  p.iUsageType = CAMERA_VIDEO_REAL_TIME;
  p.iPicWidth = w; p.iPicHeight = h;
  p.iTargetBitrate = 5000000;
  p.iRCMode = RC_OFF_MODE;
  p.fMaxFrameRate = 30.0f;
  p.iComplexityMode = HIGH_COMPLEXITY;
  p.iNumRefFrame = 1;
  p.bEnableFrameSkip = false;
  p.bEnableDenoise = p.bEnableBackgroundDetection = p.bEnableSceneChangeDetect = false;
  p.iEntropyCodingModeFlag = atoi(argv[10]);
  p.uiIntraPeriod = (unsigned int)atoi(argv[12]);
  p.bEnableAdaptiveQuant = atoi(argv[13]) != 0;
  p.iMinQp = atoi(argv[14]); p.iMaxQp = atoi(argv[15]);
  p.sSpatialLayers[0].iVideoWidth = w; p.sSpatialLayers[0].iVideoHeight = h;
  p.sSpatialLayers[0].fFrameRate = 30.0f;
  p.sSpatialLayers[0].iSpatialBitrate = 5000000;
  p.sSpatialLayers[0].iDLayerQp = qp;
  p.sSpatialLayers[0].uiProfileIdc = (EProfileIdc)atoi(argv[11]);
  p.sSpatialLayers[0].sSliceArgument.uiSliceMode = SM_SINGLE_SLICE;
  int rc = enc->InitializeExt(&p);
  fprintf(flog, "InitializeExt -> %d\n", rc);
  if (rc) { fclose(flog); fclose(fout); return 5; }
  int lvl = WELS_LOG_QUIET;
  enc->SetOption(ENCODER_OPTION_TRACE_LEVEL, &lvl);
  SEncParamExt r;
  memset(&r, 0, sizeof(r));
  enc->GetOption(ENCODER_OPTION_SVC_ENCODE_PARAM_EXT, &r);
  fprintf(flog, "resolved aq=%d\n", (int)r.bEnableAdaptiveQuant);
  const size_t fsz = (size_t)w * h * 3 / 2;
  std::vector<unsigned char> buf(fsz);
  for (int i = 0; i < n; i++) {
    if (fread(buf.data(), 1, fsz, fin) != fsz) break;
    if (i == idr_at) fprintf(flog, "force_idr -> %d\n", enc->ForceIntraFrame(true));
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
    if (rc) { fprintf(stderr, "EncodeFrame -> %d\n", rc); return 6; }
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
