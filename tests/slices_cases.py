"""Slice cases shared by tests/golden/make_slices_golden.py and the tests that read tests/golden/slices.json: the clips, the
configurations, and how to run the ISVCEncoder driver (tests/wels/wels_slices_driver.cpp) on either library.

A case: clip, pictures, QP, (iEntropyCodingModeFlag, uiProfileIdc), iComplexityMode, uiIntraPeriod, (iLoopFilterDisableIdc,
alpha offset, beta offset), (uiSliceMode, uiSliceNum, uiSliceMbNum runs), (iMultipleThreadIdc, bUseLoadBalancing)."""
import os
import subprocess

import numpy as np

import h264lib

ROOT = h264lib.ROOT
API_INC = os.path.join(ROOT, "oracle", "_ref", "include")
REFLIB = os.path.join(ROOT, "oracle", "_ref", "libopenh264_ref.so")
OURLIB = os.path.join(ROOT, "openh264_b200", "libopenh264_b200_wels.so")
DRIVER_SRC = os.path.join(ROOT, "tests", "wels", "wels_slices_driver.cpp")
LOW, HIGH = 0, 2                      # ECOMPLEXITY_MODE
SINGLE, FIXED, RASTER, SIZELIMITED = 0, 1, 2, 3

# name: (w, h, pictures)
CLIPS = {"CiscoVT2people_320x192": (320, 192, 6), "Static_152_100": (152, 100, 6), "synth_96x64": (96, 64, 4)}


def clip(name):
    w, h, n = CLIPS[name]
    if name == "CiscoVT2people_320x192":
        data = np.fromfile(os.path.join(ROOT, "tests", "golden", "CiscoVT2people_320x192_12fps.yuv"), np.uint8)
        return data[:w * h * 3 // 2 * n]
    if name == "Static_152_100":
        return h264lib.reference_clip("Static_152_100.yuv", w, h, n)
    return h264lib.synth_clip(w, h, n)


C = "CiscoVT2people_320x192"
CASES = {
    # the 240-macroblock clip: one slice per row (12 slices), runs that start mid-row, fixed 2 / 3 / 4 / 7 slices
    "rows_cavlc_high": (C, 28, (0, 66), HIGH, 0, (0, 0, 0), (RASTER, 0, []), (1, 1)),
    "rows_cabac_low_period3": (C, 30, (1, 0), LOW, 3, (2, 1, -1), (RASTER, 0, []), (1, 1)),
    "runs_17_100_cavlc_low": (C, 26, (0, 66), LOW, 3, (0, 0, 0), (RASTER, 0, [17, 100]), (1, 1)),
    "runs_17_100_cabac_main_high": (C, 28, (1, 77), HIGH, 0, (2, -2, 3), (RASTER, 0, [17, 100]), (1, 1)),
    "runs_cut_cavlc_high": (C, 32, (0, 66), HIGH, 0, (1, 0, 0), (RASTER, 0, [50, 50, 50, 500]), (1, 1)),
    "fixed2_cabac_high_low": (C, 28, (1, 100), LOW, 0, (0, 2, 2), (FIXED, 2, []), (1, 1)),
    "fixed3_cavlc_low_period2": (C, 24, (0, 66), LOW, 2, (2, 0, 0), (FIXED, 3, []), (1, 1)),
    "fixed4_cabac_high": (C, 28, (1, 0), HIGH, 3, (0, 0, 0), (FIXED, 4, []), (1, 1)),
    "fixed7_cavlc_high": (C, 28, (0, 66), HIGH, 0, (2, 3, -3), (FIXED, 7, []), (1, 1)),
    "fixed7_cabac_low_idc1": (C, 34, (1, 0), LOW, 0, (1, 0, 0), (FIXED, 7, []), (1, 1)),
    # more than one thread without load balancing: the same slices, loop filter idc 0 coded as 2
    "fixed4_threads4_cavlc_low": (C, 28, (0, 66), LOW, 0, (0, 0, 0), (FIXED, 4, []), (4, 0)),
    "rows_threads2_cabac_high": (C, 28, (1, 0), HIGH, 3, (0, 1, 1), (RASTER, 0, []), (2, 1)),
    # edges: a picture with a partial macroblock row and column, and one of at most 48 macroblocks (one slice)
    "static_rows_cavlc_low": ("Static_152_100", 28, (0, 66), LOW, 0, (0, 0, 0), (RASTER, 0, []), (1, 1)),
    "static_fixed3_cabac_high": ("Static_152_100", 26, (1, 0), HIGH, 3, (2, 0, 0), (FIXED, 3, []), (1, 1)),
    "small_fixed4_single": ("synth_96x64", 28, (0, 66), HIGH, 0, (0, 0, 0), (FIXED, 4, []), (1, 1)),
    "small_runs_single": ("synth_96x64", 28, (1, 0), LOW, 0, (2, 0, 0), (RASTER, 0, [10, 14]), (1, 1)),
    "small_rows": ("synth_96x64", 28, (0, 66), LOW, 0, (2, 0, 0), (RASTER, 0, []), (1, 1)),
}

# refused by both libraries: one slice per row with more rows than MAX_SLICES_NUM (35)
REFUSED_BOTH = {"rows_1280x720": (1280, 720, (RASTER, 0, []), (1, 1))}
# accepted by the reference, refused here: bytes that depend on the machine or on the bits spent
REFUSED_OURS = {"fixed0_cores": (320, 192, (FIXED, 0, []), (1, 1)),
                "fixed3_load_balanced": (320, 192, (FIXED, 3, []), (4, 1)),
                "rows_auto_threads": (320, 192, (RASTER, 0, []), (0, 0)),
                "size_limited": (320, 192, (SIZELIMITED, 0, []), (1, 1))}


def effective_idc(case):
    """iLoopFilterDisableIdc as the reference codes it (InitSliceSettings): idc 0 becomes 2 when more than one thread codes slices"""
    threads = min(max(case[7][0], 1), 4)
    return 2 if case[5][0] == 0 and min(threads, slice_count(case)) > 1 else case[5][0]


def slice_count(case):
    w, h, _ = CLIPS[case[0]]
    mode, num, runs = case[6]
    n_mb = ((w + 15) // 16) * ((h + 15) // 16)
    if mode == RASTER and not runs:
        return (h + 15) // 16
    if n_mb <= 48:
        return 1
    if mode == FIXED:
        return min(num, 35)
    total, count = 0, 0
    for r in runs:
        total += r
        count += 1
        if total >= n_mb:
            break
    return count + (1 if total < n_mb else 0)


def build_driver(out_dir):
    exe = os.path.join(out_dir, "wels_slices_driver")
    subprocess.check_call(["g++", "-O1", "-std=c++11", "-I" + API_INC, DRIVER_SRC, "-o", exe, "-ldl"])
    return exe


def run(exe, lib, yuv, w, h, n, qp, entropy, cx, period, lf, slices, threads, tmp, tag):
    """returns (process, bitstream, log)"""
    src, out, log = (os.path.join(tmp, tag + s) for s in (".yuv", ".264", ".log"))
    with open(src, "wb") as f:
        f.write(yuv.tobytes())
    args = [exe, lib, src, w, h, n, qp, out, log, entropy[0], entropy[1], cx, period, *lf, slices[0], slices[1], *threads, *slices[2]]
    r = subprocess.run([str(a) for a in args], capture_output=True, text=True, timeout=600)
    return r, (open(out, "rb").read() if os.path.exists(out) else b""), (open(log).read() if os.path.exists(log) else "")


def run_case(exe, lib, name, tmp):
    c = CASES[name]
    w, h, n = CLIPS[c[0]]
    return run(exe, lib, clip(c[0]), w, h, n, c[1], c[2], c[3], c[4], c[5], c[6], c[7], tmp, name)
