"""Several slices per picture on the GPU, through layer 2 (b2h264_enc_set_slices): every case of tests/golden/slices.json
(generated from the reference by tests/golden/make_slices_golden.py) coded by three streams of one batched encoder, with the
sources on the host and on the device; the device's per-macroblock CAVLC count against the host writer's on multi-slice pictures;
and the round trip through the batched decoder, which must decode each picture to the encoder's own reconstruction (loop filter
idc 2 leaves the edges between slices unfiltered on both sides)."""
import hashlib
import json
import os

import numpy as np
import pytest

import h264lib
import slices_cases as S

GOLD = json.load(open(os.path.join(h264lib.ROOT, "tests", "golden", "slices.json")))
pytestmark = pytest.mark.gpu
STREAMS = 3


def make_encoder(name, n_streams=STREAMS):
    from openh264_b200.binding import BatchEncoder
    c = S.CASES[name]
    w, h, _ = S.CLIPS[c[0]]
    enc = BatchEncoder(w, h, qp=c[1], fps=30.0, n_streams=n_streams, entropy_cabac=bool(c[2][0]), profile_idc=c[2][1],
                       complexity_low=c[3] == S.LOW, intra_period=c[4], loop_filter=(S.effective_idc(c),) + tuple(c[5][1:]))
    resolved = enc.set_slices(*c[6])
    return enc, resolved


@pytest.mark.parametrize("on_device", [False, True], ids=["host_sources", "device_sources"])
@pytest.mark.parametrize("name", sorted(S.CASES))
def test_gpu_slices_match_reference(name, on_device):
    import openh264_b200 as m
    c = S.CASES[name]
    w, h, n = S.CLIPS[c[0]]
    yuv = S.clip(c[0])
    assert hashlib.sha1(yuv.tobytes()).hexdigest() == GOLD["clips"][c[0]]
    fsz = w * h * 3 // 2
    enc, resolved = make_encoder(name)
    # the partition the reference reports through GetOption
    want = GOLD["cases"][name]["log"].splitlines()[1].split()
    assert resolved[0] == int(want[2]) and (resolved[0] == 0 or resolved[1] == int(want[4]))
    if resolved[0]:
        assert resolved[2] == [int(v) for v in want[6:6 + resolved[1]]]
    bs = [b""] * STREAMS
    for f in range(n):
        pic = yuv[f * fsz:(f + 1) * fsz]
        if on_device:
            d = m.DeviceArray(np.ascontiguousarray(pic))
            enc.submit([d.ptr] * STREAMS, on_device=True)
            out, _ = enc.collect()
        else:
            out, _ = enc.encode([pic] * STREAMS)
        bs = [bs[i] + out[i] for i in range(STREAMS)]
    enc.close()
    assert all(b == bs[0] for b in bs)
    assert hashlib.sha1(bs[0]).hexdigest() == GOLD["cases"][name]["sha1"]


@pytest.mark.parametrize("name", ["rows_cavlc_high", "runs_17_100_cavlc_low", "fixed7_cavlc_high", "static_rows_cavlc_low"])
def test_gpu_slices_device_bit_count(name):
    """set_mb_bits: the device's CAVLC count per macroblock equals the host writer's on multi-slice pictures"""
    c = S.CASES[name]
    w, h, n = S.CLIPS[c[0]]
    yuv = S.clip(c[0])
    fsz = w * h * 3 // 2
    enc, _ = make_encoder(name, n_streams=2)
    enc.set_mb_bits(True)
    for f in range(n):
        enc.encode([yuv[f * fsz:(f + 1) * fsz]] * 2)
        for s in range(2):
            dev, host = enc.mb_bits(s)
            assert np.array_equal(dev, host), (name, f, s)
    enc.close()


@pytest.mark.parametrize("name", ["rows_cabac_low_period3", "runs_17_100_cabac_main_high", "fixed3_cavlc_low_period2",
                                  "fixed4_threads4_cavlc_low", "static_fixed3_cabac_high", "fixed7_cavlc_high"])
def test_gpu_slices_round_trip(name):
    """each picture decodes through BatchDecoder to the encoder's reconstruction"""
    from openh264_b200.binding import BatchDecoder
    c = S.CASES[name]
    w, h, n = S.CLIPS[c[0]]
    yuv = S.clip(c[0])
    fsz = w * h * 3 // 2
    enc, _ = make_encoder(name, n_streams=2)
    dec = BatchDecoder(w, h, n_streams=2)
    for f in range(n):
        out, _ = enc.encode([yuv[f * fsz:(f + 1) * fsz]] * 2)
        pics = dec.decode(out)
        for s in range(2):
            assert np.array_equal(pics[s], enc.recon(s)), (name, f, s)
    enc.close()
    dec.close()


def test_gpu_slices_refusals():
    """refused partitions leave the encoder as it was; a partition cannot change once a picture was submitted"""
    from openh264_b200.binding import BatchEncoder, B2H264Error
    enc = BatchEncoder(1280, 720, qp=28, n_streams=1)
    for mode, num in [(S.RASTER, 0), (S.FIXED, 0), (S.SIZELIMITED, 0)]:
        with pytest.raises(B2H264Error):
            enc.set_slices(mode, num)
    assert enc.set_slices(S.FIXED, 8) == (S.FIXED, 8, [450] * 7 + [450])
    enc.encode([np.zeros(1280 * 720 * 3 // 2, np.uint8)])
    with pytest.raises(B2H264Error):
        enc.set_slices(S.FIXED, 4)
    enc.close()
