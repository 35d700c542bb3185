"""Fractional motion refinement and the intra 16x16 check of P macroblocks on clips whose motion is at half- and
quarter-sample offsets (tests/golden/make_refine_intra_golden.py): the host emulation build and the GPU encoder, with
batches of sms // 2 + 1 streams, must reproduce the reference encoder's bitstream in complexity HIGH and LOW at QP 12,
26 and 40 (golden = the unmodified reference, tests/golden/refine_intra.json)."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

import h264lib

ROOT = h264lib.ROOT
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_refine_intra_golden import subsample_clip  # noqa: E402

GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "refine_intra.json")))


def parse(key):
    w, h = map(int, key.split("_")[0].split("x"))
    n, seed, qp = (int(key.split(t)[1].split("_")[0]) for t in ("_n", "_seed", "_qp"))
    return w, h, n, seed, qp, key.endswith("_low")


def clip(key):
    w, h, n, seed, _, _ = parse(key)
    yuv = subsample_clip(w, h, n, seed)
    assert hashlib.sha1(yuv.tobytes()).hexdigest() == GOLD[key]["yuv_sha1"]
    return yuv


@pytest.fixture(scope="module")
def emu():
    return h264lib.emu()


@pytest.mark.parametrize("key", sorted(GOLD))
def test_host_build_matches_reference(emu, key):
    w, h, n, _, qp, low = parse(key)
    yuv = clip(key)
    emu.emu_set_complexity_low(1 if low else 0)
    emu.emu_set_entropy(0, 66)
    emu.emu_set_intra_period(0)
    emu.emu_set_loop_filter(0, 0, 0)
    cap = 8 << 20
    out, fb = np.zeros(cap, np.uint8), np.zeros(n, np.int32)
    tot = emu.emu_encode(yuv.ctypes.data, w, h, n, qp, 30.0, out.ctypes.data, cap, fb.ctypes.data, None)
    assert tot > 0
    assert fb.tolist() == GOLD[key]["frame_bytes"]
    assert hashlib.sha1(out[:tot].tobytes()).hexdigest() == GOLD[key]["sha1"]


@pytest.mark.gpu
@pytest.mark.parametrize("key", sorted(GOLD))
def test_gpu_matches_reference(key):
    import torch
    from openh264_b200.binding import BatchEncoder
    w, h, n, _, qp, low = parse(key)
    yuv = clip(key)
    S = torch.cuda.get_device_properties(0).multi_processor_count // 2 + 1
    enc = BatchEncoder(w, h, qp=qp, fps=30.0, n_streams=S, complexity_low=low)
    fsz = w * h * 3 // 2
    out = [[] for _ in range(S)]
    for f in range(n):
        bs, _ = enc.encode([yuv[f * fsz:(f + 1) * fsz]] * S)
        for s in range(S):
            out[s].append(bytes(bs[s]))
    enc.close()
    assert [len(b) for b in out[0]] == GOLD[key]["frame_bytes"]
    assert hashlib.sha1(b"".join(out[0])).hexdigest() == GOLD[key]["sha1"]
    assert all(o == out[0] for o in out[1:])
