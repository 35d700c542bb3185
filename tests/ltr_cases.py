"""Long-term reference cases shared by tests/golden/make_ltr_golden.py and the tests that read tests/golden/ltr.json: the driver
(tests/wels/wels_ltr_driver.cpp), how to run it, and how to read the reference syntax of each picture out of a bitstream."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import h264_dump  # noqa: E402

API_INC = os.path.join(ROOT, "oracle", "_ref", "include")
REFLIB = os.path.join(ROOT, "oracle", "_ref", "libopenh264_ref.so")
REFDEC = os.path.join(ROOT, "oracle", "_ref", "h264dec_ref")
OURLIB = os.path.join(ROOT, "openh264_b200", "libopenh264_b200_wels.so")
DRIVER_SRC = os.path.join(ROOT, "tests", "wels", "wels_ltr_driver.cpp")
CLIP = os.path.join(ROOT, "tests", "golden", "CiscoVT2people_320x192_12fps.yuv")
W, H, QP = 320, 192, 28
LOW, HIGH = 0, 2                      # ECOMPLEXITY_MODE

# a receiver's calls, each before the picture it names: valid, stale (old idr_pic_id) and -1 recovery requests, marking
# success and failure, period changes and a forced IDR
RECEIVER = [
    "8 rr 1 cur p1 p4", "10 rr 1 old p1 p2", "14 rr 1 cur -1 p3", "17 mf 5 cur p2", "19 period 2", "20 rr 1 cur p1 p2",
    "24 idr", "29 rr 1 cur p1 p3", "33 rr 1 cur p1 -1", "38 rr 1 cur p1 p2", "41 mf 4 old p3", "44 rr 1 cur p2 p5",
]

# name: (entropy_cabac, complexity, iNumRefFrame, bEnableLongTermReference, iLtrMarkPeriod, pictures, script)
CASES = {
    "off_ref1_cavlc_high": (0, HIGH, 1, 0, 30, 12, []),
    "off_ref2_cabac_low": (1, LOW, 2, 0, 30, 12, []),
    "off_ref3_cavlc_low": (0, LOW, 3, 0, 30, 12, []),
    "off_ref4_cabac_high": (1, HIGH, 4, 0, 30, 12, ["5 rr 1 cur p1 p2"]),
    "off_auto_cavlc_low": (0, LOW, -1, 0, 30, 8, []),
    "ltr_p1_cavlc_low": (0, LOW, -1, 1, 1, 48, RECEIVER),
    "ltr_p3_cabac_high": (1, HIGH, 2, 1, 3, 48, RECEIVER),
    "ltr_p30_cavlc_high": (0, HIGH, 4, 1, 30, 48, RECEIVER),
    "ltr_p3_cabac_low": (1, LOW, -1, 1, 3, 48, RECEIVER),
    "ltr_p0_cavlc_high": (0, HIGH, -1, 1, 0, 48, RECEIVER),     # iLtrMarkPeriod 0 resolves to 30
}

# frame_num wraps at 32,768: a long LTR case for the CPU test of the state machine (tests/golden/ltr.json "wrap")
WRAP_FROM = 32740
WRAP = (0, HIGH, -1, 1, 1, 32800, [
    "32745 mf 5 cur 0", "32750 mf 4 cur p5", "32756 mf 4 cur p4", "32760 mf 4 cur p3", "32763 rr 1 cur p1 p6",
    "32766 mf 4 cur p2", "32769 mf 4 cur p3", "32771 rr 1 cur p1 p5", "32773 mf 5 cur p2", "32776 rr 1 cur p1 p3",
    "32779 mf 4 cur p4", "32783 rr 1 cur p2 p4", "32786 mf 4 cur p2", "32790 rr 1 cur p1 p3",
])


def build_driver(out_dir):
    exe = os.path.join(out_dir, "wels_ltr_driver")
    subprocess.check_call(["g++", "-O1", "-std=c++11", "-I" + API_INC, DRIVER_SRC, "-o", exe, "-ldl"])
    return exe


def run(exe, lib, case, script, tmp, tag):
    """returns (process, bitstream, log)"""
    cabac, cx, nref, ltr, period, n, _ = case
    scr, out, log = (os.path.join(tmp, tag + s) for s in (".txt", ".264", ".log"))
    with open(scr, "w") as f:
        f.write("\n".join(script) + "\n")
    args = [exe, lib, CLIP, str(W), str(H), str(n), str(QP), out, log, str(cabac), str(cx), str(nref), str(ltr), str(period), scr]
    r = subprocess.run(args, capture_output=True, text=True, timeout=600)
    return r, (open(out, "rb").read() if os.path.exists(out) else b""), (open(log).read() if os.path.exists(log) else "")


def ref_syntax(bs):
    """per picture: [idr, frame_num, list modification commands, MMCOs, long_term_reference_flag] from the slice headers"""
    out = []
    for info in h264_dump.dump(bs, verbose=False):
        if info["type"] not in (1, 5):
            continue
        idr = info["type"] == 5
        out.append([int(idr), info["frame_num"], [list(c) for c in info.get("reorder_cmds", [])],
                    [list(m) for m in info.get("mmco", [])], int(info.get("long_term", 0))])
    return out


def coded_pictures(log):
    """picture index of every coded picture, from a driver log (a picture that failed is not in the bitstream)"""
    return [int(ln.split()[1]) for ln in log.splitlines() if ln.startswith("frame ") and " type " in ln]


def sps_num_ref(bs):
    return [i["num_ref"] for i in h264_dump.dump(bs, verbose=False) if i["type"] == 7]

