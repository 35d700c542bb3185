"""Several slices per picture in the host build (tests/emu/slices_hooks.cu: the macroblock code, the deblocking filter and both
slice writers, with the partition resolved as layer 2 resolves it) against the reference's bitstreams in tests/golden/slices.json
(tests/golden/make_slices_golden.py).  Every picture is also read back by the decoder's parser, and with CAVLC the macroblock
code's own bit count must equal what the writer spent.  The GPU build of the same source: tests/test_gpu_encoder_slices.py."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest

import h264lib
import slices_cases as S

GOLD = json.load(open(os.path.join(h264lib.ROOT, "tests", "golden", "slices.json")))


@pytest.fixture(scope="module")
def emu():
    E = h264lib.emu()
    vp, i = C.c_void_p, C.c_int
    E.emu_encode_slices.restype = C.c_long
    E.emu_encode_slices.argtypes = [vp, i, i, i, i, vp, vp, vp, C.c_long, vp, vp]
    return E


def encode_case(E, name, recon=False):
    c = S.CASES[name]
    w, h, n = S.CLIPS[c[0]]
    yuv = S.clip(c[0])
    assert hashlib.sha1(yuv.tobytes()).hexdigest() == GOLD["clips"][c[0]]
    mode, num, runs = c[6]
    cfg = np.array([c[2][0], c[2][1], 1 if c[3] == S.LOW else 0, c[4], S.effective_idc(c), c[5][1], c[5][2], mode, num], np.int32)
    mb = np.zeros(35, np.uint32)
    mb[:len(runs)] = runs
    out, fb = np.zeros(8 << 20, np.uint8), np.zeros(n, np.int32)
    rec = np.zeros(n * w * h * 3 // 2, np.uint8) if recon else None
    tot = E.emu_encode_slices(yuv.ctypes.data, w, h, n, c[1], cfg.ctypes.data, mb.ctypes.data, out.ctypes.data, out.size,
                              fb.ctypes.data, rec.ctypes.data if recon else None)
    assert tot > 0, (name, tot)
    return out[:tot].tobytes(), fb.tolist(), rec


def nal_lengths(bs):
    """lengths of the NAL units of an Annex-B stream written with 4-byte start codes, each with its start code"""
    starts = [i for i in range(len(bs) - 3) if bs[i:i + 4] == b"\0\0\0\1"]
    return [b - a for a, b in zip(starts, starts[1:] + [len(bs)])]


def nal_sizes(log):
    """per picture: the NAL sizes of its layers, from a driver log"""
    return [ln.split(":", 1)[1].split() for ln in log.splitlines() if ln.startswith("frame ")]


@pytest.mark.parametrize("name", sorted(S.CASES))
def test_emu_slices_match_reference(emu, name):
    bs, fb, _ = encode_case(emu, name)
    g = GOLD["cases"][name]
    frames = [ln for ln in g["log"].splitlines() if ln.startswith("frame ")]
    assert fb == [int(ln.split("bytes ")[1].split(":")[0]) for ln in frames]
    assert hashlib.sha1(bs).hexdigest() == g["sha1"]
    # one NAL unit per slice, in the sizes the reference wrote (start codes included)
    assert nal_lengths(bs) == [int(v) for f in nal_sizes(g["log"]) for v in f if not v.startswith("[")]


def test_emu_slices_cover_the_cases():
    """the cases reach every mode, both entropy coders, idc 2 across slices, and the fall-back to one slice"""
    counts = {name: S.slice_count(c) for name, c in S.CASES.items()}
    assert counts["rows_cavlc_high"] == 12 and counts["fixed7_cavlc_high"] == 7 and counts["small_fixed4_single"] == 1
    assert any(S.effective_idc(c) == 2 and counts[k] > 1 and c[2][0] for k, c in S.CASES.items())
    assert any(S.effective_idc(c) == 2 and counts[k] > 1 and not c[2][0] for k, c in S.CASES.items())
    for name, c in S.CASES.items():
        resolved = GOLD["cases"][name]["log"].splitlines()[1].split()
        assert int(resolved[4]) == counts[name] or resolved[2] == "0", name


def test_emu_refuses_too_many_rows(emu):
    """one slice per macroblock row with 45 rows is refused, as by the reference (tests/golden/slices.json: refused_both)"""
    assert "refused" in GOLD["refused_both"]["rows_1280x720"]
    yuv = np.zeros(1280 * 720 * 3 // 2, np.uint8)
    cfg = np.array([0, 66, 0, 0, 0, 0, 0, S.RASTER, 0], np.int32)
    mb = np.zeros(35, np.uint32)
    out = np.zeros(1 << 20, np.uint8)
    assert emu.emu_encode_slices(yuv.ctypes.data, 1280, 720, 1, 28, cfg.ctypes.data, mb.ctypes.data, out.ctypes.data, out.size,
                                 None, None) == -2
