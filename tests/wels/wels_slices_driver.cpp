// wels_slices_driver.cpp — TEST INFRASTRUCTURE.  An application written against the reference's public API (codec/api/wels/codec_api.h)
// that loads "some libopenh264" with dlopen and encodes a clip through InitializeExt / EncodeFrame with an SSliceArgument, a thread
// count and a load-balancing flag as given.  It writes the bitstream, and a log of whether InitializeExt accepted the
// configuration, the slice argument GetOption reports the encoder resolved, and the NAL layout of every EncodeFrame call.
// tests/golden/make_slices_golden.py runs it with the compiled reference, tests/test_wels_api_slices.py with both libraries.
//   wels_slices_driver <lib.so> <in.yuv> <w> <h> <frames> <qp> <out.264> <out.log> <entropy_cabac> <profile_idc> <complexity>
//                      <intra_period> <lf_idc> <lf_alpha> <lf_beta> <slice_mode> <slice_num> <threads> <load_balancing> [run ...]
#include <dlfcn.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "codec_api.h"

typedef int (*create_fn)(ISVCEncoder**);
typedef void (*destroy_fn)(ISVCEncoder*);

int main(int argc, char** argv) {
  if (argc < 20) { fprintf(stderr, "usage: see source\n"); return 2; }
  void* lib = dlopen(argv[1], RTLD_NOW | RTLD_LOCAL);
  if (!lib) { fprintf(stderr, "dlopen: %s\n", dlerror()); return 3; }
  create_fn create = (create_fn)dlsym(lib, "WelsCreateSVCEncoder");
  destroy_fn destroy = (destroy_fn)dlsym(lib, "WelsDestroySVCEncoder");
  if (!create || !destroy) { fprintf(stderr, "missing entry points\n"); return 3; }
  const int w = atoi(argv[3]), h = atoi(argv[4]), n = atoi(argv[5]), qp = atoi(argv[6]);
  FILE* fin = fopen(argv[2], "rb");
  FILE* fout = fopen(argv[7], "wb");
  FILE* flog = fopen(argv[8], "w");
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
  p.iNumRefFrame = 1;
  p.bEnableFrameSkip = false;
  p.bEnableDenoise = p.bEnableBackgroundDetection = p.bEnableSceneChangeDetect = p.bEnableAdaptiveQuant = false;
  p.iEntropyCodingModeFlag = atoi(argv[9]);
  p.iComplexityMode = (ECOMPLEXITY_MODE)atoi(argv[11]);
  p.uiIntraPeriod = (unsigned int)atoi(argv[12]);
  p.iLoopFilterDisableIdc = atoi(argv[13]);
  p.iLoopFilterAlphaC0Offset = atoi(argv[14]);
  p.iLoopFilterBetaOffset = atoi(argv[15]);
  p.iMultipleThreadIdc = (unsigned short)atoi(argv[18]);
  p.bUseLoadBalancing = atoi(argv[19]) != 0;
  SSpatialLayerConfig& l = p.sSpatialLayers[0];
  l.iVideoWidth = w; l.iVideoHeight = h;
  l.fFrameRate = 30.0f;
  l.iSpatialBitrate = 5000000;
  l.iDLayerQp = qp;
  l.uiProfileIdc = (EProfileIdc)atoi(argv[10]);
  l.sSliceArgument.uiSliceMode = (SliceModeEnum)atoi(argv[16]);
  l.sSliceArgument.uiSliceNum = (unsigned int)atoi(argv[17]);
  for (int i = 20; i < argc && i - 20 < MAX_SLICES_NUM_TMP; i++) l.sSliceArgument.uiSliceMbNum[i - 20] = (unsigned int)atoi(argv[i]);
  int lvl = WELS_LOG_QUIET;
  enc->SetOption(ENCODER_OPTION_TRACE_LEVEL, &lvl);
  int rc = enc->InitializeExt(&p);
  fprintf(flog, "InitializeExt %s\n", rc ? "refused" : "accepted");
  if (rc) { fclose(flog); fclose(fout); destroy(enc); return 0; }
  SEncParamExt r;
  memset(&r, 0, sizeof(r));
  enc->GetOption(ENCODER_OPTION_SVC_ENCODE_PARAM_EXT, &r);
  const SSliceArgument& a = r.sSpatialLayers[0].sSliceArgument;
  fprintf(flog, "resolved mode %d num %u runs", (int)a.uiSliceMode, a.uiSliceNum);
  for (int i = 0; i < MAX_SLICES_NUM_TMP; i++) fprintf(flog, " %u", a.uiSliceMbNum[i]);
  fprintf(flog, "\n");
  const size_t fsz = (size_t)w * h * 3 / 2;
  std::vector<unsigned char> buf(fsz);
  for (int i = 0; i < n; i++) {
    if (fread(buf.data(), 1, fsz, fin) != fsz) break;
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
    for (int k = 0; k < info.iLayerNum; k++) {
      const SLayerBSInfo& L = info.sLayerInfo[k];
      int sz = 0;
      fprintf(flog, " [%d]", (int)L.uiLayerType);
      for (int j = 0; j < L.iNalCount; j++) { fprintf(flog, " %d", L.pNalLengthInByte[j]); sz += L.pNalLengthInByte[j]; }
      fwrite(L.pBsBuf, 1, sz, fout);
    }
    fprintf(flog, "\n");
  }
  enc->Uninitialize();
  destroy(enc);
  fclose(fin); fclose(fout); fclose(flog);
  return 0;
}
