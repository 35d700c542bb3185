"""Explicit weighted prediction in B slices (weighted_bipred_idc 1), CPU side: the host build of the parser + construct path
(tests/emu, the same h264_parse.cpp / h264_motion.h / dec_mb.cuh the GPU decoder runs) on the committed B-frame vectors rewritten
with seeded pred_weight_tables (tests/wp_rewrite.py), against the reference decoder's output recorded in
tests/golden/explicit_bipred.json (tests/golden/make_explicit_bipred_golden.py) and, where oracle/_ref exists, against the reference
itself."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest

import h264lib
import wp_rewrite

ROOT = h264lib.ROOT
CONF_B_DIR = os.path.join(ROOT, "tests", "golden", "conformance_b")
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "explicit_bipred.json")))["jobs"]
MAIN = ["Cisco_Men_whisper_640x320_CAVLC_Bframe_9.264", "Cisco_Men_whisper_640x320_CABAC_Bframe_9.264",
        "Cisco_Adobe_PDF_sample_a_1024x768_CAVLC_Bframe_9.264"]
# the counters of b2h264_dec_wp_stats, in the order of WPS_* (openh264_b200/csrc/wp_formula.h)
STATS = ["one list L0", "one list L1", "two lists 16x16", "two lists 16x8", "two lists 8x16", "two lists B_8x8 sub-macroblock",
         "16x8/8x16 first partition, w0+w1 != 2^(ld+1), offsets", "16x8/8x16 second partition, w0+w1 != 2^(ld+1), offsets",
         "spatial direct", "temporal direct", "B_Skip", "refIdxL0 > 0", "refIdxL1 > 0", "luma denominator 0", "luma denominator 7",
         "chroma denominator 0", "chroma denominator 7", "weight -128", "weight 127", "offset -128", "offset 127", "defaulted entry",
         "one-list 8x4 / 4x8 (second half weighted)", "clipped at 0", "clipped at 255"]


@pytest.fixture(scope="module")
def emu():
    return h264lib.emu()


def source(name):
    return open(os.path.join(CONF_B_DIR, name), "rb").read()


def emu_decode(E, bs):
    a = np.frombuffer(bs, np.uint8)
    out = np.zeros(64 << 20, np.uint8)
    W, H = C.c_int(), C.c_int()
    n = E.emu_decode(a.ctypes.data, len(a), out.ctypes.data, out.size, C.byref(W), C.byref(H))
    return n, W.value, H.value, hashlib.sha1(out[:max(n, 0) * W.value * H.value * 3 // 2].tobytes()).hexdigest()


def ref_decode(bs):
    from golden.make_explicit_bipred_golden import ref_decode as rd
    return rd(bs)


def published(name):
    tab = dict((p.split("/")[-1], s) for p, s in json.load(open(os.path.join(ROOT, "tests", "golden", "reference_decoder_hashes.json")))["pairs"])
    return tab[name]


@pytest.mark.parametrize("name", MAIN)
def test_neutral_rewrite_decodes_to_the_published_hash(emu, name):
    """denominators 5 and every flag off: weights 32, offsets 0 reproduce default prediction for every partition shape, the quirky
    16x8 / 8x16 partitions included, so the rewritten stream must decode to the vector's PUBLISHED SHA-1 — this pins the rewriter
    without trusting either decoder"""
    bs = wp_rewrite.rewrite(source(name))
    assert bs != source(name)
    n, _, _, sha = emu_decode(emu, bs)
    assert n == 9 and sha == published(name)
    if h264lib.have_ref():
        assert ref_decode(bs)[3] == published(name)


@pytest.mark.parametrize("job", GOLD, ids=lambda j: "%s-seed%d" % (j["source"][:24], j["seed"]))
def test_seeded_rewrite_host_build_matches_reference(emu, job):
    bs = wp_rewrite.rewrite(source(job["source"]), job["seed"])
    got = emu_decode(emu, bs)
    assert got == (job["pictures"], job["width"], job["height"], job["sha1"])
    if h264lib.have_ref():                                        # the committed hashes are still what the reference makes
        assert ref_decode(bs) == got


def test_the_jobs_reach_every_case_of_the_weighting(emu):
    """counted by the host build itself (b2h264_dec_wp_stats), not by this test"""
    st = (C.c_longlong * 64)()
    n = emu.b2h264_dec_wp_stats(st, 64, 1)
    assert n == len(STATS)
    for job in GOLD:
        assert emu_decode(emu, wp_rewrite.rewrite(source(job["source"]), job["seed"]))[0] == job["pictures"]
    emu.b2h264_dec_wp_stats(st, 64, 1)
    counts = dict(zip(STATS, st[:n]))
    print(counts)
    missing = [k for k, v in counts.items() if v == 0]
    assert not missing, counts


def test_neutral_rewrite_keeps_implicit_streams_decodable(emu):
    """a High-profile prefix with implicit weights (wbi 2) rewritten to neutral explicit weights: default prediction instead of
    implicit, so a different picture than the source, but one the reference agrees with"""
    name = "VID_1280x544_cavlc_temporal_direct_first14.264"
    bs = wp_rewrite.rewrite(source(name))
    got = emu_decode(emu, bs)
    assert got[0] == 14
    if h264lib.have_ref():
        assert ref_decode(bs) == got


@pytest.mark.parametrize("bad", ["weight 128", "offset -129", "chroma weight -129", "truncated"])
def test_bad_pred_weight_table_in_a_b_slice_is_rejected(emu, bad):
    """a value outside [-128, 127] or a slice that ends inside its table: an error, never pictures"""
    def table(n_ref):
        t = wp_rewrite.neutral_table(n_ref)
        luma, chroma = (None, None)
        if bad == "weight 128":
            luma = (128, 0)
        elif bad == "offset -129":
            luma = (3, -129)
        elif bad == "chroma weight -129":
            chroma = ((-129, 0), (1, 0))
        t["lists"][1][0] = (luma, chroma)
        return t
    bs = wp_rewrite.rewrite(source(MAIN[0]), make_table=table, cut=bad == "truncated")
    assert emu_decode(emu, bs)[0] < 0
