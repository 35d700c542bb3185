"""Explicit weighted prediction in B slices (weighted_bipred_idc 1) through the GPU decoder (include/b2h264_codec.h b2h264_dec_*; host:
h264_parse.cpp + h264_motion.h resolve every 8x8's weighting formula and weights, device: dec_mb.cuh dec_b_mb applies it with the
formulas of wp_formula.h) and through ISVCDecoder.  The streams are the committed B-frame vectors rewritten with seeded
pred_weight_tables (tests/wp_rewrite.py); the hashes are the reference decoder's, committed in tests/golden/explicit_bipred.json.
(File name: runs after the other GPU tests.)"""
import hashlib
import json
import os

import numpy as np
import pytest

import h264lib
import wp_rewrite

pytestmark = pytest.mark.gpu
ROOT = h264lib.ROOT
CONF_B_DIR = os.path.join(ROOT, "tests", "golden", "conformance_b")
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "explicit_bipred.json")))["jobs"]


def source(name):
    return open(os.path.join(CONF_B_DIR, name), "rb").read()


def output_order(pics):
    """(sequence, picture order count, decoding position, picture) -> pictures in output order"""
    return [t[3] for t in sorted(pics, key=lambda t: t[:3])]


def decode_alone(aus, w, h):
    from openh264_b200.binding import BatchDecoder
    dec = BatchDecoder(w, h)
    pics, seq = [], 0
    for au in aus:
        p = dec.decode2([au])[0]
        assert p is not None
        poc, idr, _ = dec.picture_order(0)
        seq += idr & 1
        pics.append((seq, poc, len(pics), p.copy()))
    dec.close()
    return pics


@pytest.mark.parametrize("job", GOLD, ids=lambda j: "%s-seed%d" % (j["source"][:24], j["seed"]))
def test_gpu_decoder_explicit_b_weights(job):
    aus = h264lib.split_access_units(wp_rewrite.rewrite(source(job["source"]), job["seed"]))
    assert len(aus) == job["pictures"]
    pics = output_order(decode_alone(aus, job["width"], job["height"]))
    assert hashlib.sha1(b"".join(p.tobytes() for p in pics)).hexdigest() == job["sha1"]


def test_gpu_decoder_explicit_implicit_and_baseline_streams_in_one_batch():
    """an explicit-weight B stream, an implicit-weight B stream (the unmodified prefix) and a Baseline stream of the same size in one
    batch: each decodes exactly as it does alone"""
    from openh264_b200.binding import BatchDecoder, BatchEncoder
    name = "VID_1280x544_cabac_temporal_direct_first14.264"
    job = [j for j in GOLD if j["source"] == name][0]
    w, h = job["width"], job["height"]
    aus_x = h264lib.split_access_units(wp_rewrite.rewrite(source(name), job["seed"]))
    aus_i = h264lib.split_access_units(source(name))
    n = len(aus_x)
    yuv = h264lib.synth_clip(w, h, n, seed=11, noise=4)
    fsz = w * h * 3 // 2
    enc = BatchEncoder(w, h, qp=27, fps=30.0, n_streams=1)
    aus_p = [enc.encode([yuv[f * fsz:(f + 1) * fsz]])[0][0] for f in range(n)]
    enc.close()
    streams = [aus_x, aus_i, aus_p]
    alone = [decode_alone(s, w, h) for s in streams]
    dec = BatchDecoder(w, h, n_streams=3)
    together, seq = [[], [], []], [0, 0, 0]
    for k in range(n):
        got = dec.decode2([s[k] for s in streams])
        for i in range(3):
            assert got[i] is not None
            poc, idr, _ = dec.picture_order(i)
            seq[i] += idr & 1
            together[i].append((seq[i], poc, k, got[i].copy()))
    dec.close()
    for i in range(3):
        for a, b in zip(alone[i], together[i]):
            assert a[:3] == b[:3] and np.array_equal(a[3], b[3]), (i, a[:3])
    assert hashlib.sha1(b"".join(p.tobytes() for p in output_order(together[0]))).hexdigest() == job["sha1"]


def test_gpu_decoder_rejects_a_bad_table():
    """a luma weight of 128 in a B slice: that stream's call fails, no picture"""
    from openh264_b200.binding import BatchDecoder

    def table(n_ref):
        t = wp_rewrite.neutral_table(n_ref)
        t["lists"][1][0] = ((128, 0), None)
        return t
    aus = h264lib.split_access_units(wp_rewrite.rewrite(source("Cisco_Men_whisper_640x320_CAVLC_Bframe_9.264"), make_table=table))
    dec = BatchDecoder(640, 320)
    statuses = [dec.decode3([au])[1][0] for au in aus]
    dec.close()
    assert statuses[0] == 1 and min(statuses) < 0


@pytest.mark.parametrize("name,seed", [("Cisco_Men_whisper_640x320_CAVLC_Bframe_9.264", 2), ("VID_1280x544_cabac_temporal_direct_first14.264", 3)])
def test_isvcdecoder_explicit_b_weights_same_driver_two_libraries(tmp_path, name, seed):
    """ISVCDecoder NAL by NAL (tests/wels/wels_dec_driver.cpp through DecodeFrameNoDelay) with the compiled reference and with our
    library on a rewritten CAVLC and a rewritten CABAC stream: identical pictures in identical calls, identical call log"""
    import subprocess
    driver = os.path.join(ROOT, "oracle", "_ref", "wels_dec_driver")
    reflib = os.path.join(ROOT, "oracle", "_ref", "libopenh264_ref.so")
    ourlib = os.path.join(ROOT, "openh264_b200", "libopenh264_b200_wels.so")
    assert os.path.exists(driver) and os.path.exists(ourlib) and os.path.exists(reflib), "prebuilt layer-3 artefacts missing on the GPU box"
    src = os.path.join(str(tmp_path), "explicit.264")
    open(src, "wb").write(wp_rewrite.rewrite(source(name), seed))
    res = {}
    for tag, lib in (("ref", reflib), ("b2", ourlib)):
        out, log = os.path.join(str(tmp_path), tag + ".yuv"), os.path.join(str(tmp_path), tag + ".log")
        r = subprocess.run([driver, lib, src, out, log], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        res[tag] = (open(out, "rb").read(), open(log).read())
    assert len(res["ref"][0]) > 0 and res["ref"][0] == res["b2"][0], "pictures through ISVCDecoder differ from the reference"
    assert res["ref"][1] == res["b2"][1], "call log differs:\n" + res["ref"][1][:3000] + "\n---\n" + res["b2"][1][:3000]
