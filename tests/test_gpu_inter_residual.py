"""Stage B's residual step (inter_residual_pass, enc_inter.cuh): the device codes the luma and chroma residual of an inter
macroblock, its JVT-O079 decisions and its reconstruction in one warp pass; the host emulation build keeps the serial
sequence (WelsEncInterY / WelsEncRecUV restated block by block), which is the specification.  The device pass must leave
byte for byte the same levels (kept or dropped), chroma DC levels, nnz, cbp and reconstruction as the host build, on random
macroblocks at every QP and on sparse residues built to land on the decision thresholds.  The host build also counts which
decisions the encoder reached on the reference-pinned skip-stage clips (tests/golden/skip_stage.json)."""
import ctypes as C
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

OUT_BYTES = 896 + 32 + 384          # MbOut, nnz[24] + cbp + pad, reconstruction (b2h264_debug_inter_residual)
# enc_inter.cuh: RES_LUMA_ZEROED .. RES_PSKIP_CODED
OUTCOMES = ["luma levels dropped by ctr_mb < 6", "kept and dropped 8x8 in one macroblock", "chroma cbp 0", "chroma cbp 1",
            "chroma cbp 2", "P16x16 coded", "P16x8 coded", "P8x16 coded", "P8x8 coded", "16x16 became P_SKIP after coding"]


@pytest.fixture(scope="module")
def emu():
    return h264lib.emu()


def make_cases():
    """(src_pred [n, 768] uint8, qp [n] int32): random macroblocks at every QP, then sparse residues around the thresholds."""
    rng = np.random.RandomState(7)
    srcs, qps = [], []
    for qp in range(52):                                   # random content, random prediction
        for _ in range(4):
            srcs.append(rng.randint(0, 256, 768).astype(np.uint8)); qps.append(qp)
    for qp in range(52):                                   # prediction = source + small noise
        for amp in (1, 2, 4, 8):
            s = rng.randint(16, 240, 384)
            srcs.append(np.concatenate([s, np.clip(s + rng.randint(-amp, amp + 1, 384), 0, 255)]).astype(np.uint8)); qps.append(qp)
    # sparse residues: a few samples differ by +-d in chosen 4x4 blocks, so that single +-1 levels (and the odd level > 1)
    # land in chosen 8x8s / planes: ctr8 / ctr_mb / chroma ctr around 4, 6 and 7, and DC-only chroma planes
    for qp in (12, 18, 24, 26, 30, 36):
        for _ in range(160):
            s = rng.randint(32, 224, 384)
            p = s.copy()
            for _ in range(rng.randint(1, 12)):
                pos = rng.randint(0, 384)
                p[pos] += rng.choice([-1, 1]) * rng.randint(1, 4 + qp // 3)
            if rng.rand() < 0.25:                          # a flat offset over one chroma block: DC only
                b, pl = rng.randint(0, 4), rng.randint(0, 2)
                for y in range(4):
                    o = 256 + 64 * pl + ((b >> 1) * 4 + y) * 8 + (b & 1) * 4
                    p[o:o + 4] += rng.choice([-1, 1]) * rng.randint(2, 6 + qp // 4)
            srcs.append(np.concatenate([s, np.clip(p, 0, 255)]).astype(np.uint8)); qps.append(qp)
    # flat offsets over a few luma 4x4 blocks: a lone DC level (score 3) per block, so that ctr8 and ctr_mb land on 3 / 6
    for qp in (12, 18, 24, 30):
        for _ in range(60):
            s = rng.randint(64, 192, 384)
            p = s.copy()
            for b in rng.choice(16, rng.randint(1, 4), replace=False):
                bx, by = (b & 1) | ((b >> 1) & 2), ((b >> 1) & 1) | ((b >> 2) & 2)
                for y in range(4):
                    o = (4 * by + y) * 16 + 4 * bx
                    p[o:o + 4] += rng.choice([-1, 1]) * rng.randint(1, 3 + qp // 2)
            srcs.append(np.concatenate([s, np.clip(p, 0, 255)]).astype(np.uint8)); qps.append(qp)
    return np.stack(srcs), np.array(qps, np.int32)


def run_emu(emu, src, qp):
    out = np.zeros((len(qp), OUT_BYTES), np.uint8)
    assert emu.emu_inter_residual(len(qp), src.ctypes.data, qp.ctypes.data, out.ctypes.data) == 0
    return out


def decisions(out):
    """per case: luma cbp bits, chroma cbp, whether luma / each chroma plane carries levels"""
    lv = out[:, 112:112 + 512].view(np.int16).reshape(-1, 16, 16)
    ac = out[:, 640:640 + 256].view(np.int16).reshape(-1, 8, 16)
    dc = out[:, 624:624 + 16].view(np.int16).reshape(-1, 2, 4)
    cbp = out[:, 896 + 24].astype(int)
    return cbp & 15, cbp >> 4, (lv != 0).reshape(-1, 4, 64).any(2), (ac != 0).reshape(-1, 2, 64).any(2), (dc != 0).any(2)


def single_ctr(lv):
    """WelsCalculateSingleCtr4x4_c over the last axis: every non-zero level costs T[zero levels directly before it]"""
    T = np.array([3, 2, 2, 1, 1, 1] + [0] * 10)
    run = np.zeros(lv.shape[:-1], int)
    tot = np.zeros(lv.shape[:-1], int)
    for i in range(lv.shape[-1]):
        nz = lv[..., i] != 0
        tot += np.where(nz, T[np.minimum(run, 15)], 0)
        run = np.where(nz, 0, run + 1)
    return tot


def walk(mx, ctr, thr):
    """the reference's serial JVT-O079 walk over the last axis (4 blocks): skip mx == 0, add 9 for mx > 1, else add ctr
    while the running total is below thr"""
    s = np.zeros(mx.shape[:-1], int)
    for j in range(4):
        s = np.where(mx[..., j] == 0, s, np.where(mx[..., j] > 1, s + 9, np.where(s < thr, s + ctr[..., j], s)))
    return s


def test_cases_reach_the_thresholds(emu):
    src, qp = make_cases()
    out = run_emu(emu, src, qp)
    # the scores of every case, recomputed here from the levels the host build returns (kept or dropped)
    lv = out[:, 112:112 + 512].view(np.int16).reshape(-1, 4, 4, 16).astype(int)        # [case, 8x8, block, level]
    ac = out[:, 640:640 + 256].view(np.int16).reshape(-1, 2, 4, 16).astype(int)        # [case, plane, block, level]
    ctr8 = walk(np.abs(lv).max(3), single_ctr(lv), 6)
    ctr_mb = ctr8.sum(1)
    ctr_c = walk(np.abs(ac).max(3), single_ctr(ac), 7)
    cbp = out[:, 896 + 24].astype(int)
    # the decisions follow from them
    keep8 = (ctr_mb[:, None] >= 6) & (ctr8 >= 4)
    assert ((cbp & 15) == (keep8 * (1 << np.arange(4))).sum(1)).all()
    assert (((cbp >> 4) == 2) == (ctr_c >= 7).any(1)).all()
    # every boundary is landed on: ctr8 3 / 4 / 5 / 6, ctr_mb 5 / 6, chroma 6 / 7, a level > 1 in an otherwise low 8x8
    for v in (3, 4, 5, 6):
        assert (ctr8 == v).any(), v
    for v in (5, 6):
        assert (ctr_mb == v).any(), v
    for v in (6, 7):
        assert (ctr_c == v).any(), v
    big = np.abs(lv).max(3) > 1
    rest = np.where(big, 0, single_ctr(lv)).sum(2)
    assert ((big.sum(2) == 1) & (rest < 4) & (rest > 0)).any()
    cl, cc, l8, acp, dcp = decisions(out)
    lev = l8.any(1)
    assert (lev & (cl == 0)).any()                                        # levels present, luma zeroed (ctr_mb < 6)
    dropped = (l8 & ~((cl[:, None] >> np.arange(4)) & 1).astype(bool)).any(1)
    assert ((cl != 0) & dropped).any()                                    # kept and dropped 8x8s in one macroblock
    assert (cl == 15).any()
    assert (acp.any(1) & (cc < 2)).any()                                  # chroma AC levels dropped (ctr < 7)
    assert ((cc == 1) & dcp.any(1)).any()                                 # a DC-only chroma plane
    for v in (0, 1, 2):
        assert (cc == v).any()


def test_host_build_reaches_every_outcome(emu):
    # The skip-stage clips in HIGH and LOW complexity at QP 12 / 26 / 40: their bitstreams are pinned to the unmodified
    # reference (tests/golden/skip_stage.json, tests/golden/make_skip_stage_golden.py) and checked here too, and between them
    # they reach every residual outcome of stage B, every partition shape and a 16x16 that becomes P_SKIP after coding.  The
    # GPU encoder's bitstreams on the same clips are checked by tests/test_gpu_skip_stage.py.
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "skip_stage.json")))
    total = np.zeros(len(OUTCOMES), np.uint64)
    for key in sorted(gold):
        parts = key.split("_")
        yuv = skip_clip(parts[2])
        assert hashlib.sha1(yuv.tobytes()).hexdigest() == gold[key]["yuv_sha1"]
        emu.emu_set_complexity_low(1 if parts[4] == "low" else 0)
        emu.emu_set_entropy(0, 66)
        emu.emu_set_intra_period(0)
        emu.emu_set_loop_filter(0, 0, 0)
        cap = 8 << 20
        out, fb = np.zeros(cap, np.uint8), np.zeros(N, np.int32)
        emu.emu_reset_res_outcomes()
        tot = emu.emu_encode(yuv.ctypes.data, W, H, N, int(parts[3][2:]), 30.0, out.ctypes.data, cap, fb.ctypes.data, None)
        assert tot > 0
        assert hashlib.sha1(out[:tot].tobytes()).hexdigest() == gold[key]["sha1"], key
        cnt = np.zeros(len(OUTCOMES), np.uint64)
        assert emu.emu_res_outcomes(cnt.ctypes.data, len(cnt)) == len(cnt)
        total += cnt
    reached = {name: int(n) for name, n in zip(OUTCOMES, total)}
    assert all(n > 0 for n in reached.values()), reached


@pytest.mark.gpu
def test_device_pass_matches_host_build(emu):
    import openh264_b200 as m
    L = m.lib(0)
    L.b2h264_debug_inter_residual.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    src, qp = make_cases()
    want = run_emu(emu, src, qp)
    got = np.zeros_like(want)
    assert L.b2h264_debug_inter_residual(len(qp), src.ctypes.data, qp.ctypes.data, got.ctypes.data) == 0
    bad = np.nonzero((got != want).any(1))[0]
    assert len(bad) == 0, f"{len(bad)} of {len(qp)} cases differ, first: case {bad[0]} qp {qp[bad[0]]}"
    _refusals(L.b2h264_debug_inter_residual)


def test_host_build_refuses_bad_arguments(emu):
    """the host build refuses what the device hook refuses (stage_hooks.cuh: inter_residual_args_ok)"""
    _refusals(emu.emu_inter_residual)


def _refusals(fn):
    # bad arguments are refused before anything runs
    src, qp = make_cases()
    got = np.zeros((1, OUT_BYTES), np.uint8)
    q = np.array([52], np.int32)
    assert fn(1, src.ctypes.data, q.ctypes.data, got.ctypes.data) == -1
    assert fn(0, src.ctypes.data, qp.ctypes.data, got.ctypes.data) == -1
