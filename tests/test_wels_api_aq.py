"""bEnableAdaptiveQuant through layer 3.  The reference's ParamValidation switches adaptive quantisation off for every
configuration (codec/encoder/core/src/encoder_ext.cpp:300-301), so a caller who asks for it gets the constant-QP bitstream, and
the resolved parameters report it off.  InitializeExt accepts the flag and does the same.  One driver binary
(tests/wels/wels_aq_driver.cpp, compiled here against the reference's public headers staged under oracle/_ref/include) runs the
compiled reference and our library side by side."""
import os
import subprocess

import pytest

import h264lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
API_INC = os.path.join(ROOT, "oracle", "_ref", "include")
REFLIB = os.path.join(ROOT, "oracle", "_ref", "libopenh264_ref.so")
OURLIB = os.path.join(ROOT, "openh264_b200", "libopenh264_b200_wels.so")
SRC = os.path.join(ROOT, "tests", "wels", "wels_aq_driver.cpp")
need_ref = pytest.mark.skipif(not (os.path.isdir(API_INC) and os.path.exists(REFLIB)),
                              reason="the reference build (library and public headers) is not present")
need_ours = pytest.mark.skipif(not os.path.exists(OURLIB), reason="layer 3 is built where the reference headers exist (build())")


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("aq_driver") / "wels_aq_driver")
    subprocess.check_call(["g++", "-O1", "-std=c++11", "-I" + API_INC, SRC, "-o", exe, "-ldl"])
    return exe


def drive(exe, lib, clip, w, h, n, qp, tmp, tag, aq, entropy=(0, 66), intra_period=0, idr_at=-1):
    """aq = (bEnableAdaptiveQuant, iMinQp, iMaxQp); returns (process, bitstream, log)"""
    yuv = os.path.join(tmp, "in.yuv")
    with open(yuv, "wb") as f:
        f.write(clip.tobytes())
    out, log = os.path.join(tmp, tag + ".264"), os.path.join(tmp, tag + ".log")
    args = [exe, lib, yuv, str(w), str(h), str(n), str(qp), str(idr_at), out, log, str(entropy[0]), str(entropy[1]), str(intra_period)]
    r = subprocess.run(args + [str(v) for v in aq], capture_output=True, text=True, timeout=300)
    return r, (open(out, "rb").read() if os.path.exists(out) else b""), (open(log).read() if os.path.exists(log) else "")


@need_ref
@pytest.mark.parametrize("aq,entropy", [((1, 0, 51), (0, 66)), ((1, 22, 30), (1, 0)), ((1, 30, 20), (1, 77)), ((0, 0, 51), (0, 66))],
                         ids=["default_range", "narrow_cabac_high", "crossed_cabac_main", "off"])
def test_reference_ignores_adaptive_quant(tmp_path, driver, aq, entropy):
    """the reference's own output with AQ requested equals its constant-QP output, and it reports AQ off"""
    w, h, n, qp = 176, 144, 5, 26
    clip = h264lib.synth_clip(w, h, n, seed=4, noise=6)
    r0, bs0, log0 = drive(driver, REFLIB, clip, w, h, n, qp, str(tmp_path), "off", (0, 0, 51), entropy=entropy)
    r1, bs1, log1 = drive(driver, REFLIB, clip, w, h, n, qp, str(tmp_path), "aq", aq, entropy=entropy)
    assert r0.returncode == 0 and r1.returncode == 0, r0.stderr + r1.stderr
    assert len(bs1) > 0 and bs1 == bs0 and log1 == log0
    assert "resolved aq=0" in log1


@pytest.mark.gpu
@need_ref
@need_ours
@pytest.mark.parametrize("aq,entropy,period,idr_at", [((1, 0, 51), (0, 66), 0, -1), ((1, 22, 30), (1, 0), 3, -1),
                                                      ((1, 30, 20), (1, 77), 0, 2), ((1, 0, 51), (0, 66), 0, 3)],
                         ids=["cavlc", "cabac_high_period3", "cabac_main_crossed_idr2", "cavlc_idr3"])
def test_drop_in_with_adaptive_quant(tmp_path, driver, aq, entropy, period, idr_at):
    """ISVCEncoder with bEnableAdaptiveQuant: accepted, and the same bitstream and call log as the reference library"""
    w, h, n, qp = 176, 144, 6, 28
    clip = h264lib.synth_clip(w, h, n, seed=6, noise=6)
    r1, bs1, log1 = drive(driver, OURLIB, clip, w, h, n, qp, str(tmp_path), "b2", aq, entropy=entropy, intra_period=period, idr_at=idr_at)
    r2, bs2, log2 = drive(driver, REFLIB, clip, w, h, n, qp, str(tmp_path), "ref", aq, entropy=entropy, intra_period=period, idr_at=idr_at)
    assert r1.returncode == 0, r1.stderr
    assert r2.returncode == 0, r2.stderr
    assert len(bs1) > 0 and bs1 == bs2
    assert log1 == log2 and "resolved aq=0" in log1
