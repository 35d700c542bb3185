"""The P-skip test of stage A (WelsMdPSkipEnc) on clips built to reach its branches (tests/golden/make_skip_stage_golden.py):
an integer pan, quarter-sample pans over all 16 luma phases, moving content at the picture border, and residues that make
each test decide.  The host emulation build and the GPU encoder, with batches of sms // 2 + 1 streams, must reproduce the
reference encoder's bitstream in complexity HIGH and LOW at QP 12, 26 and 40 (golden = the unmodified reference,
tests/golden/skip_stage.json); the host build also counts which outcome each skip test had.  The packed chroma
prediction is checked against the per-sample one for every phase and block size."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

import h264lib

ROOT = h264lib.ROOT
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_skip_stage_golden import H, N, W, skip_clip  # noqa: E402

GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "skip_stage.json")))
# enc_inter.cuh: SKIP_RANGE .. SKIP_DCT_OK
OUTCOMES = ["range guard", "accepted by SAD", "luma level > 1", "luma ctr >= 6", "chroma DC", "chroma AC level > 1",
            "Cb AC ctr >= 7", "Cr AC ctr >= 7", "accepted after the DCT tests"]


def parse(key):
    parts = key.split("_")
    return parts[2], int(parts[3][2:]), parts[4] == "low"


def clip(key):
    kind, _, _ = parse(key)
    yuv = skip_clip(kind)
    assert hashlib.sha1(yuv.tobytes()).hexdigest() == GOLD[key]["yuv_sha1"]
    return yuv


@pytest.fixture(scope="module")
def emu():
    return h264lib.emu()


def emu_encode(emu, key):
    _, qp, low = parse(key)
    yuv = clip(key)
    emu.emu_set_complexity_low(1 if low else 0)
    emu.emu_set_entropy(0, 66)
    emu.emu_set_intra_period(0)
    emu.emu_set_loop_filter(0, 0, 0)
    cap = 8 << 20
    out, fb = np.zeros(cap, np.uint8), np.zeros(N, np.int32)
    emu.emu_reset_skip_outcomes()
    tot = emu.emu_encode(yuv.ctypes.data, W, H, N, qp, 30.0, out.ctypes.data, cap, fb.ctypes.data, None)
    assert tot > 0
    cnt = np.zeros(len(OUTCOMES) + 2, np.uint64)
    assert emu.emu_skip_outcomes(cnt.ctypes.data, len(cnt)) == len(cnt)
    return out[:tot].tobytes(), fb.tolist(), cnt


@pytest.mark.parametrize("key", sorted(GOLD))
def test_host_build_matches_reference(emu, key):
    bs, fb, _ = emu_encode(emu, key)
    assert fb == GOLD[key]["frame_bytes"]
    assert hashlib.sha1(bs).hexdigest() == GOLD[key]["sha1"]


def test_clips_reach_every_skip_outcome(emu):
    total = np.zeros(len(OUTCOMES), np.uint64)
    luma_phases = chroma_phases = 0
    for key in sorted(GOLD):
        _, _, cnt = emu_encode(emu, key)
        total += cnt[:len(OUTCOMES)]
        luma_phases |= int(cnt[-2])
        chroma_phases |= int(cnt[-1])
    # the range guard cannot trip here: pred_skip_mv takes its vector from neighbours whose searches were clipped to the
    # picture (me_partition's window), which keeps a skip vector within 16 + 3 samples of it
    reached = {name: int(n) for name, n in zip(OUTCOMES, total)}
    assert all(reached[name] > 0 for name in OUTCOMES[1:]), reached
    assert luma_phases == 0xffff, hex(luma_phases)
    assert bin(chroma_phases).count("1") >= 16, hex(chroma_phases)


def test_packed_chroma_matches_per_sample(emu):
    assert emu.emu_check_chroma_pair() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("key", sorted(GOLD))
def test_gpu_matches_reference(key):
    import torch
    from openh264_b200.binding import BatchEncoder
    _, qp, low = parse(key)
    yuv = clip(key)
    S = torch.cuda.get_device_properties(0).multi_processor_count // 2 + 1
    enc = BatchEncoder(W, H, qp=qp, fps=30.0, n_streams=S, complexity_low=low)
    fsz = W * H * 3 // 2
    out = [[] for _ in range(S)]
    for f in range(N):
        bs, _ = enc.encode([yuv[f * fsz:(f + 1) * fsz]] * S)
        for s in range(S):
            out[s].append(bytes(bs[s]))
    enc.close()
    assert [len(b) for b in out[0]] == GOLD[key]["frame_bytes"]
    assert hashlib.sha1(b"".join(out[0])).hexdigest() == GOLD[key]["sha1"]
    assert all(o == out[0] for o in out[1:])
