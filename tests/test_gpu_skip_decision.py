"""Stage A's P-skip test of a P macroblock (enc_inter.cuh: fill_inter_cache, predict_sad_skip, pskip_enc), one macroblock job
at a time, against the CPU oracle orc_pskip (PredictSadSkip, PredSkipMv and WelsMdPSkipEnc with WelsTryPYskip / WelsTryPUVskip,
pinned to the reference by the `pskip` kernel case of test_oracle_vs_ref.py).

The device builds the skip prediction in one memory round trip (skip_predict): integer vectors as unaligned words, fractional
vectors from a 21 x 21 window staged as aligned words at an offset `wsh` (the window's start address & 3) and filtered eight
samples per lane, chroma at the alignment of its row address; the luma and chroma SADs come back packed in one warp sum.  Its
residual tests run one block per lane and replace the reference's serial early exits by one packed sum.  The host emulation
build does none of that, so the device is compared with the oracle and with the host build, byte for byte.

The reference planes hold random samples everywhere, padding included, and are not border-expanded: a read from a wrong
address gives a wrong sample rather than a copy of the right one.  The jobs reach, and test_cases_reach_every_path asserts:
every outcome of the skip test in the reference's order, every quarter-sample phase at every window alignment, every
eighth-sample chroma phase at every chroma alignment, the range guard's limits from both sides, every branch of the skip
vector's derivation, the early accepts exactly at their boundaries, the largest packed SAD, the residual scores exactly at
their thresholds, and every QP in both complexity modes."""
import ctypes as C

import numpy as np
import pytest

import h264lib
from h264lib import PskipJob, PskipResult, ptr

ROOT = h264lib.ROOT
IN_BYTES = 32 * 4 + 384             # b2h264_debug_skip_test's job record
OUT_BYTES = 8 * 4 + 384             # its output record
UNSET = 0x5a5a5a5a                  # the sad_cost slot before the call
PSKIP, P16, I16 = 6, 2, 1           # enc_types.h: MBT_PSKIP, MBT_P16x16, MBT_I16x16
NB_L, NB_T, NB_TL, NB_TR = 1, 2, 4, 8
O = {name: k for k, name in enumerate(h264lib.PSKIP_OUTCOMES)}


@pytest.fixture(scope="module")
def emu():
    return h264lib.emu()


# ---- pictures ------------------------------------------------------------------------------------------------------
class Pic:
    """the reference planes (Y, Cb, Cr) of one picture as the hook reads them, random everywhere, padding included"""

    def __init__(self, rng, mb_w, mb_h):
        self.mb_w, self.mb_h = mb_w, mb_h
        self.sy, self.sc = 16 * mb_w + 64, 8 * mb_w + 32              # the encoder's padded strides (enc_host.h)
        self.cb = self.sy * (16 * mb_h + 64)
        self.cr = self.cb + self.sc * (8 * mb_h + 32)
        self.set = rng.randint(0, 256, self.cr + self.sc * (8 * mb_h + 32)).astype(np.uint8)

    def ref_off(self, mbx, mby):
        return [(32 + 16 * mby) * self.sy + 32 + 16 * mbx, self.cb + (16 + 8 * mby) * self.sc + 16 + 8 * mbx,
                self.cr + (16 + 8 * mby) * self.sc + 16 + 8 * mbx]

    def fill(self, mbx, mby, v, margin=6):
        """set the luma and chroma reference samples around macroblock (mbx, mby) to v"""
        y0, c0 = self.ref_off(mbx, mby)[0], self.ref_off(mbx, mby)[1:]
        for r in range(-margin, 16 + margin):
            self.set[y0 + r * self.sy - margin:y0 + r * self.sy + 16 + margin] = v
        for o in c0:
            for r in range(-margin, 8 + margin):
                self.set[o + r * self.sc - margin:o + r * self.sc + 8 + margin] = v


def wsh(pic, j):
    """skip_predict's window alignment: the address of luma sample (-2, -2) of the predicted block & 3 (the set starts aligned)"""
    ix, iy = j["mv"][0] >> 2, j["mv"][1] >> 2
    return ((32 + 16 * j["mby"] + iy - 2) * pic.sy + 32 + 16 * j["mbx"] + ix - 2) & 3


def chroma_align(pic, j):
    """the alignment of skip_predict's chroma row address (every row and half row shares it: the strides are multiples of 4)"""
    ix, iy = j["mv"][0] >> 2, j["mv"][1] >> 2
    return (pic.cb + (16 + 8 * j["mby"] + (iy >> 1)) * pic.sc + 16 + 8 * j["mbx"] + (ix >> 1)) & 3


# ---- jobs ------------------------------------------------------------------------------------------------------------
def nbr(t=P16, mv=(0, 0), sad=0, skip_sad=0):
    return {"type": t, "mv": mv, "sad": sad, "skip_sad": skip_sad}


def job(pic, mbx, mby, cur, qp=26, fast=0, nb=15, nbrs=None, ref_is_p=0, col=(P16, 0), mv=None):
    """a job; mv = the skip vector wanted: all four neighbours inter with that vector (the median of three equal vectors)"""
    if nbrs is None:
        v = mv if mv is not None else (0, 0)
        nbrs = [nbr(P16, v) for _ in range(4)]
    return {"mbx": mbx, "mby": mby, "cur": cur, "qp": qp, "fast": fast, "nb": nb, "nbrs": nbrs, "ref_is_p": ref_is_p,
            "col": col}


def oracle_job(pic, j):
    oj = PskipJob()
    oj.cur_off[:] = [0, 256, 320]
    oj.ref_off[:] = pic.ref_off(j["mbx"], j["mby"])
    oj.mb_x, oj.mb_y, oj.mb_w, oj.mb_h = j["mbx"], j["mby"], pic.mb_w, pic.mb_h
    oj.qp, oj.md_using_sad = j["qp"], j["fast"]
    bits = [NB_TL, NB_T, NB_TR, NB_L]
    for cell, k in enumerate((3, 1, 2, 0)):                           # cells A, B, C, D = neighbours left, top, top-right, top-left
        n, avail = j["nbrs"][k], j["nb"] & bits[k]
        inter = avail and n["type"] >= P16
        oj.ref[cell] = -2 if not avail else 0 if inter else -1
        oj.mv[cell][0], oj.mv[cell][1] = n["mv"] if inter else (0, 0)
    for k in range(4):
        oj.skip[k] = int(bool(j["nb"] & bits[k]) and j["nbrs"][k]["type"] == PSKIP)
        oj.skip_sad[k] = j["nbrs"][k]["skip_sad"]
    oj.ref_is_p, oj.col_type, oj.col_skip_sad = j["ref_is_p"], j["col"][0], j["col"][1]
    return oj


def run_oracle(pic, j):
    r, pred = PskipResult(), np.zeros(384, np.uint8)
    h264lib.oracle().pskip(ptr(j["cur"]), 16, 8, ptr(pic.set), pic.sy, pic.sc, C.byref(oracle_job(pic, j)), C.byref(r), ptr(pred))
    j["mv"] = (r.mv_x, r.mv_y)
    return r, pred


def record(pic, j):
    w = np.zeros(32, np.int32)
    w[:12] = [pic.mb_w, pic.mb_h, pic.sy, pic.sc, j["mbx"], j["mby"], j["qp"], j["fast"], j["nb"], j["ref_is_p"], j["col"][0], j["col"][1]]
    for k, n in enumerate(j["nbrs"]):
        w[12 + 5 * k:17 + 5 * k] = [n["type"], n["mv"][0], n["mv"][1], n["sad"], n["skip_sad"]]
    return np.concatenate([w.view(np.uint8), j["cur"]])


def with_pred(rng, pic, j, delta=None):
    """j with its source replaced by the oracle's skip prediction (plus `delta`, int, 384)"""
    _, pred = run_oracle(pic, dict(j, cur=rng.randint(0, 256, 384).astype(np.uint8)))
    d = 0 if delta is None else delta
    return dict(j, cur=np.clip(pred.astype(int) + d, 0, 255).astype(np.uint8))


def sparse_delta(rng, qp):
    d = np.zeros(384, int)
    for _ in range(rng.randint(1, 10)):
        d[rng.randint(0, 384)] += rng.choice([-1, 1]) * rng.randint(1, 4 + qp // 3)
    if rng.rand() < 0.5:                                               # a flat offset over one 4x4 block: a lone DC
        b = rng.randint(0, 24)
        for y in range(4):
            o = ((b >> 2) * 4 + y) * 16 + (b & 3) * 4 if b < 16 else 256 + 64 * ((b - 16) >> 2) + (((b - 16) >> 1 & 1) * 4 + y) * 8 + (b & 1) * 4
            d[o:o + 4] += rng.choice([-1, 1]) * rng.randint(1, 3 + qp // 2)
    return d


def small_mv(rng, r=20):
    return (int(rng.randint(-r, r + 1)), int(rng.randint(-r, r + 1)))


def phase_jobs(rng, pic):
    """every luma quarter-sample phase at every window alignment (and integer vectors at every ix & 3), every chroma
    eighth-sample phase at every chroma alignment; the source is the prediction plus sparse noise or random"""
    jobs = []
    for fy in range(4):
        for fx in range(4):
            for a in range(4):
                ix, iy = 4 * int(rng.randint(-3, 4)) + a, int(rng.randint(-8, 9))
                jobs.append((4 * ix + fx, 4 * iy + fy))
    for py in range(8):
        for px in range(8):
            for a in range(4):
                jobs.append((8 * (4 * int(rng.randint(-2, 3)) + a) + px, 8 * int(rng.randint(-4, 5)) + py))
    out = []
    for mv in jobs:
        mbx, mby, qp = int(rng.randint(0, pic.mb_w)), int(rng.randint(0, pic.mb_h)), int(rng.randint(0, 52))
        j = job(pic, mbx, mby, None, qp=qp, fast=int(rng.randint(0, 2)), mv=mv)
        if rng.rand() < 0.3:
            out.append(dict(j, cur=rng.randint(0, 256, 384).astype(np.uint8)))
        else:
            out.append(with_pred(rng, pic, j, sparse_delta(rng, qp) if rng.rand() < 0.8 else None))
    return out


def guard_jobs(rng, pic):
    """skip vectors exactly at the range guard's limits (n = -29, n = 16 mb_w + 12 and likewise vertically), with fractional
    parts so that the staged window reaches the farthest padding samples it may read, and one sample beyond them"""
    out = []
    for side in range(4):
        for beyond in (0, 1):
            for frac in ((1, 1), (3, 3), (2, 1), (0, 0), (3, 2)):
                mbx, mby = int(rng.randint(0, pic.mb_w)), int(rng.randint(0, pic.mb_h))
                ix, iy = small_mv(rng, 4)
                if side == 0:
                    ix = -29 - beyond - 16 * mbx
                elif side == 1:
                    ix = 16 * pic.mb_w + 12 + beyond - 16 * mbx
                elif side == 2:
                    iy = -29 - beyond - 16 * mby
                else:
                    iy = 16 * pic.mb_h + 12 + beyond - 16 * mby
                if beyond == 0 and rng.rand() < 0.5:                   # a corner: both limits at once
                    ix = -29 - 16 * mbx if side >= 2 else ix
                    iy = 16 * pic.mb_h + 12 - 16 * mby if side < 2 else iy
                j = job(pic, mbx, mby, None, qp=int(rng.randint(0, 52)), fast=int(rng.randint(0, 2)), mv=(4 * ix + frac[0], 4 * iy + frac[1]))
                out.append(dict(j, cur=rng.randint(0, 256, 384).astype(np.uint8)) if beyond else with_pred(rng, pic, j, sparse_delta(rng, 20)))
    return out


def derivation_jobs(rng, pic):
    """neighbour cells that derive the skip vector through each branch of PredSkipMv, with varied skip flags and skip SADs for
    PredictSadSkip"""
    out = []
    a, b, c, d = small_mv(rng), small_mv(rng), small_mv(rng), small_mv(rng)
    cases = [
        (15 & ~NB_L, [P16, P16, P16, P16]),                           # A missing
        (15 & ~NB_T, [P16, P16, P16, P16]),                           # B missing
        (15, [P16, P16, P16, P16], "A zero"),
        (15, [P16, P16, P16, P16], "B zero"),
        (15, [P16, P16, P16, P16]),                                   # median of A, B, C
        (15 & ~NB_TR, [P16, P16, P16, P16]),                          # median of A, B, D
        (15, [I16, I16, I16, P16]),                                   # only A is reference 0
        (15, [I16, P16, I16, I16]),                                   # only B
        (15, [I16, I16, P16, I16]),                                   # only C
        (15 & ~NB_TR, [P16, I16, I16, I16]),                          # only D
        (15, [PSKIP, PSKIP, PSKIP, PSKIP]),
        (15 & ~NB_TR, [PSKIP, PSKIP, P16, PSKIP]),
        (NB_L, [P16, P16, P16, PSKIP]),                               # left only
        (0, [P16, P16, P16, P16]),
    ]
    for rep in range(6):
        for case in cases:
            nb, types = case[0], case[1]
            mvs = [d, b, c, a]                                        # neighbours top-left, top, top-right, left
            if len(case) > 2:
                mvs = [d, b if case[2] == "A zero" else (0, 0), c, (0, 0) if case[2] == "A zero" else a]
            ns = [nbr(types[k], mvs[k], int(rng.randint(0, 3000)), int(rng.randint(0, 3000))) for k in range(4)]
            mbx, mby = int(rng.randint(0, pic.mb_w)), int(rng.randint(0, pic.mb_h))
            j = job(pic, mbx, mby, None, qp=int(rng.randint(0, 52)), fast=rep & 1, nb=nb, nbrs=ns)
            out.append(with_pred(rng, pic, j, sparse_delta(rng, 26)) if rep < 4 else dict(j, cur=rng.randint(0, 256, 384).astype(np.uint8)))
        a, b, c, d = small_mv(rng), small_mv(rng), small_mv(rng), small_mv(rng)
    return out


def boundary_jobs(rng, pic):
    """the early accepts exactly at their boundaries: SAD 0, SAD == iSadPredSkip and iSadPredSkip - 1 (the left neighbour is the
    only skipped one: the predictor is its skip SAD), the co-located rule with ref_is_p 0 / 1 and a skipped or coded co-located
    macroblock, at its SAD and one above"""
    out = []
    for rep in range(8):
        mbx, mby, mv = int(rng.randint(0, pic.mb_w)), int(rng.randint(0, pic.mb_h)), small_mv(rng)
        qp, fast = int(rng.randint(0, 52)), rep & 1
        base = with_pred(rng, pic, job(pic, mbx, mby, None, qp=qp, fast=fast, mv=mv))
        out.append(base)                                               # SAD 0
        j = with_pred(rng, pic, job(pic, mbx, mby, None, qp=qp, fast=fast, mv=mv), sparse_delta(rng, qp))
        r, _ = run_oracle(pic, j)
        sad = r.sad_luma + r.sad_chroma
        for p in (sad, sad + 1):
            ns = [nbr(P16, mv), nbr(P16, mv), nbr(P16, mv), nbr(PSKIP, mv, skip_sad=p)]
            out.append(dict(j, nbrs=ns))
        for ref_is_p in (0, 1):
            for t in (PSKIP, P16):
                for p in (sad, sad + 1):
                    out.append(dict(j, ref_is_p=ref_is_p, col=(t, p)))
    return out


def extreme_jobs(rng, pic):
    """the largest packed SAD: a source of 255 against a prediction of 0 (luma 65,280, chroma 32,640), and the reverse, with an
    integer and a fractional vector"""
    out = []
    for mbx, mby, v, mv in ((0, 0, 0, (0, 0)), (pic.mb_w - 1, pic.mb_h - 1, 255, (0, 0)), (0, 0, 0, (2, 5)), (pic.mb_w - 1, pic.mb_h - 1, 255, (6, 1))):
        pic.fill(mbx, mby, v)
        for fast in (0, 1):
            out.append(job(pic, mbx, mby, np.full(384, 255 - v, np.uint8), qp=int(rng.randint(0, 52)), fast=fast, mv=mv))
    return out


def threshold_jobs(rng, pic, per=6):
    """sources = prediction + sparse deltas, kept where the oracle lands on a threshold: luma score exactly 5 and 6, a lone
    level 1 against a level 2, the chroma DC test just passing and just failing, chroma score 6 and 7 on Cb and on Cr, Cb
    passing while Cr fails"""
    want = {"luma score 5": [], "luma score 6": [], "luma level 2": [], "luma lone level 1": [], "Cb score 6": [], "Cb score 7": [],
            "Cr score 6": [], "Cr score 7": [], "Cb passes, Cr fails": []}
    tries = 0
    while any(len(v) < per for v in want.values()) and tries < 40000:
        tries += 1
        qp = int(rng.choice([12, 18, 24, 26, 30, 36]))
        mbx, mby = int(rng.randint(0, pic.mb_w)), int(rng.randint(0, pic.mb_h))
        j = job(pic, mbx, mby, None, qp=qp, fast=int(rng.randint(0, 2)), mv=small_mv(rng))
        j = with_pred(rng, pic, j, sparse_delta(rng, qp))
        r, _ = run_oracle(pic, j)
        keys = []
        if r.score[0] == 5:
            keys.append("luma score 5")
        if r.outcome == O["luma score >= 6"] and r.score[0] == 6:
            keys.append("luma score 6")
        if r.outcome == O["luma level > 1"]:
            keys.append("luma level 2")
        if r.score[0] == 3 and r.outcome > O["luma score >= 6"]:
            keys.append("luma lone level 1")
        for pl, name in ((1, "Cb"), (2, "Cr")):
            if r.score[pl] == 6:
                keys.append(f"{name} score 6")
            if r.score[pl] == 7 and r.outcome == O[f"{name} score >= 7"]:
                keys.append(f"{name} score 7")
        if r.outcome in (O["Cr DC"], O["Cr level > 1"], O["Cr score >= 7"]):
            keys.append("Cb passes, Cr fails")
        for k in keys:
            if len(want[k]) < per:
                want[k].append(j)
                break
    assert all(want.values()), {k: len(v) for k, v in want.items()}
    out = [j for v in want.values() for j in v]
    # the chroma 2x2 DC test just passing and just failing: a flat offset over one chroma plane, grown until the test fails
    for pl in (0, 1):
        for qp in (10, 26, 40):
            j = job(pic, 0, 0, None, qp=qp, mv=small_mv(rng))
            last = None
            for m in range(1, 64):
                d = np.zeros(384, int)
                d[256 + 64 * pl:320 + 64 * pl] = m
                jm = with_pred(rng, pic, j, d)
                r, _ = run_oracle(pic, jm)
                if r.outcome == O["Cb DC"] + pl:
                    out += [jm] if last is None else [last, jm]
                    break
                last = jm
    return out


def qp_jobs(rng, pic):
    """every QP in both complexity modes: a prediction plus noise of a few amplitudes, and a random source"""
    out = []
    for qp in range(52):
        for fast in (0, 1):
            mbx, mby = int(rng.randint(0, pic.mb_w)), int(rng.randint(0, pic.mb_h))
            j = job(pic, mbx, mby, None, qp=qp, fast=fast, mv=small_mv(rng, 40))
            amp = int(rng.choice([1, 2, 4]))
            out.append(with_pred(rng, pic, j, rng.randint(-amp, amp + 1, 384)))
            out.append(with_pred(rng, pic, j, sparse_delta(rng, qp)))
    return out


def build_cases():
    """(picture, jobs) per picture: 1x1, 3x2 and 20x12 macroblocks and a 1920-wide strip"""
    rng = np.random.RandomState(5)
    cases = []
    for mb_w, mb_h in ((1, 1), (3, 2), (20, 12), (120, 1)):
        pic = Pic(rng, mb_w, mb_h)
        jobs = extreme_jobs(rng, pic) + phase_jobs(rng, pic) + guard_jobs(rng, pic) + derivation_jobs(rng, pic) + boundary_jobs(rng, pic)
        if mb_w == 3:
            jobs += threshold_jobs(rng, pic) + qp_jobs(rng, pic)
        for j in jobs:
            run_oracle(pic, j)                                         # fills in the skip vector
        cases.append((pic, jobs))
    return cases


_CASES = None


def cases():
    global _CASES
    if _CASES is None:
        _CASES = build_cases()
    return _CASES


# ---- expected results ------------------------------------------------------------------------------------------------
def expect(pic, jobs):
    """(the hook's output records as the oracle computes them, the oracle's results); the prediction of a job that the range
    guard rejected is left zero, as the scratch was"""
    out = np.zeros((len(jobs), OUT_BYTES), np.uint8)
    res = []
    for i, j in enumerate(jobs):
        r, pred = run_oracle(pic, j)
        o = np.array([r.ok, r.mv_x, r.mv_y, r.sad_pred_skip, r.cost_luma, r.cost_skip, UNSET if r.sad_cost == -1 else r.sad_cost, 0], np.int32)
        out[i, :32] = o.view(np.uint8)
        out[i, 32:] = pred
        res.append(r)
    return out, res


def run_emu(emu, pic, jobs):
    recs = np.stack([record(pic, j) for j in jobs])
    out = np.zeros((len(jobs), OUT_BYTES), np.uint8)
    assert emu.emu_skip_test(len(jobs), pic.set.ctypes.data, len(pic.set), recs.ctypes.data, out.ctypes.data) == 0
    return out


def describe(got, want, jobs, pic, res):
    bad = np.nonzero((got != want).any(1))[0]
    if len(bad) == 0:
        return ""
    i = bad[0]
    g, w = got[i, :32].view(np.int32), want[i, :32].view(np.int32)
    j = {k: v for k, v in jobs[i].items() if k != "cur"}
    pix = np.nonzero(got[i, 32:] != want[i, 32:])[0][:8].tolist()
    return (f"{len(bad)} of {len(jobs)} jobs differ ({pic.mb_w}x{pic.mb_h} MBs); first: job {i} {j} "
            f"(oracle: {h264lib.PSKIP_OUTCOMES[res[i].outcome]}, wsh {wsh(pic, jobs[i])}, chroma alignment {chroma_align(pic, jobs[i])}): "
            f"words got {g.tolist()} want {w.tolist()}, prediction bytes {pix}")


# ---- CPU tests ---------------------------------------------------------------------------------------------------------
def test_host_build_matches_oracle(emu):
    for pic, jobs in cases():
        (want, res), got = expect(pic, jobs), run_emu(emu, pic, jobs)
        assert np.array_equal(got, want), describe(got, want, jobs, pic, res)


def test_host_build_counts_each_outcome(emu):
    """the host build's outcome counters (emu_skip_outcomes: SKIP_RANGE .. SKIP_DCT_OK) see each job's outcome"""
    coarse = [0, 0, 0, 0, 1, 1, 1, 2, 3, 4, 4, 5, 5, 6, 7, 8]         # ORC_PSKIP_* -> enc_inter.cuh SKIP_*
    emu.emu_reset_skip_outcomes()
    want = np.zeros(9, np.uint64)
    for pic, jobs in cases():
        run_emu(emu, pic, jobs)
        for j, r in zip(jobs, expect(pic, jobs)[1]):
            # an early accept in HIGH complexity still takes the luma SATD, but runs no residual test and counts once
            want[coarse[r.outcome]] += 1
    got = np.zeros(11, np.uint64)
    assert emu.emu_skip_outcomes(got.ctypes.data, 11) == 11
    assert got[:9].tolist() == want.tolist(), (got[:9].tolist(), want.tolist())


def test_cases_reach_every_path():
    seen = {k: 0 for k in h264lib.PSKIP_OUTCOMES}
    extra = {k: 0 for k in ("guard at the left limit", "guard at the right limit", "guard at the top limit", "guard at the bottom limit",
                            "left limit - 1", "right limit + 1", "top limit - 1", "bottom limit + 1", "largest packed SAD",
                            "SAD == predictor", "SAD == predictor - 1", "co-located accept", "co-located type not skip",
                            "co-located in an I picture", "SAD == co-located", "luma score 5", "luma score 6", "lone luma level 1",
                            "Cb score 6", "Cb score 7", "Cr score 6", "Cr score 7", "Cb passes, Cr fails", "1920-wide picture")}
    luma, chroma, qps = set(), set(), set()
    for pic, jobs in cases():
        _, res = expect(pic, jobs)
        for j, r in zip(jobs, res):
            seen[h264lib.PSKIP_OUTCOMES[r.outcome]] += 1
            qps.add((j["qp"], j["fast"]))
            extra["1920-wide picture"] += pic.mb_w == 120
            nx, ny = 16 * j["mbx"] + (r.mv_x >> 2), 16 * j["mby"] + (r.mv_y >> 2)
            extra["guard at the left limit"] += nx == -29 and r.outcome >= 4
            extra["guard at the right limit"] += nx == 16 * pic.mb_w + 12 and r.outcome >= 4
            extra["guard at the top limit"] += ny == -29 and r.outcome >= 4
            extra["guard at the bottom limit"] += ny == 16 * pic.mb_h + 12 and r.outcome >= 4
            extra["left limit - 1"] += nx == -30 and r.outcome == 0
            extra["right limit + 1"] += nx == 16 * pic.mb_w + 13 and r.outcome == 1
            extra["top limit - 1"] += ny == -30 and r.outcome == 2
            extra["bottom limit + 1"] += ny == 16 * pic.mb_h + 13 and r.outcome == 3
            if r.outcome < 4:
                continue
            sad = r.sad_luma + r.sad_chroma
            extra["largest packed SAD"] += r.sad_luma == 65280 and r.sad_chroma == 32640
            extra["SAD == predictor"] += sad == r.sad_pred_skip and r.outcome > O["SAD < predictor"]
            extra["SAD == predictor - 1"] += sad == r.sad_pred_skip - 1 and r.outcome == O["SAD < predictor"]
            extra["co-located accept"] += r.outcome == O["SAD < co-located"] and sad == j["col"][1] - 1
            col_rule = sad < j["col"][1] and sad >= r.sad_pred_skip and sad > 0
            extra["co-located type not skip"] += col_rule and j["ref_is_p"] and j["col"][0] != PSKIP and r.outcome > O["SAD < co-located"]
            extra["co-located in an I picture"] += col_rule and not j["ref_is_p"] and j["col"][0] == PSKIP and r.outcome > O["SAD < co-located"]
            extra["SAD == co-located"] += sad == j["col"][1] and j["ref_is_p"] and j["col"][0] == PSKIP and r.outcome > O["SAD < co-located"]
            extra["luma score 5"] += r.score[0] == 5
            extra["luma score 6"] += r.score[0] == 6 and r.outcome == O["luma score >= 6"]
            extra["lone luma level 1"] += r.score[0] == 3 and r.outcome > O["luma score >= 6"]
            extra["Cb score 6"] += r.score[1] == 6
            extra["Cb score 7"] += r.score[1] == 7 and r.outcome == O["Cb score >= 7"]
            extra["Cr score 6"] += r.score[2] == 6
            extra["Cr score 7"] += r.score[2] == 7 and r.outcome == O["Cr score >= 7"]
            extra["Cb passes, Cr fails"] += r.outcome in (O["Cr DC"], O["Cr level > 1"], O["Cr score >= 7"])
            luma.add((r.mv_x & 3, r.mv_y & 3, wsh(pic, j)))
            chroma.add((r.mv_x & 7, r.mv_y & 7, chroma_align(pic, j)))
    assert all(seen.values()), seen
    assert all(extra.values()), extra
    assert len(luma) == 64, sorted({(x, y, a) for x in range(4) for y in range(4) for a in range(4)} - luma)
    assert len(chroma) == 256, sorted({(x, y, a) for x in range(8) for y in range(8) for a in range(4)} - chroma)
    assert len(qps) == 104


def test_derivation_reaches_every_branch():
    """PredSkipMv's branches, from the jobs' neighbour cells: a missing A or B, a zero vector on A or B, the median with C and
    with D, and a single matching reference on A, B, C and D"""
    seen = set()
    for pic, jobs in cases():
        for j in jobs:
            oj = oracle_job(pic, j)
            ra, rb, rc, rd = oj.ref[0], oj.ref[1], oj.ref[2], oj.ref[3]
            if ra == -2 or rb == -2:
                seen.add("A or B missing")
            elif (ra == 0 and tuple(oj.mv[0]) == (0, 0)) or (rb == 0 and tuple(oj.mv[1]) == (0, 0)):
                seen.add("zero vector on A or B")
            else:
                c = "C" if rc != -2 else "D"
                rr = rc if rc != -2 else rd
                m = (ra == 0) | (rb == 0) << 1 | (rr == 0) << 2
                seen.add({1: "only A", 2: "only B", 4: "only " + c}.get(m, "median with " + c))
    assert seen >= {"A or B missing", "zero vector on A or B", "only A", "only B", "only C", "only D", "median with C",
                    "median with D"}, seen


def test_pskip_case_reaches_every_outcome():
    """the oracle's pskip kernel case (kernel_cases.py), which pins it to the reference, reaches every outcome"""
    from kernel_cases import pskip_case_jobs
    rng = np.random.RandomState(1234 + sum(map(ord, "pskip")))          # the seed run_case gives the case
    assert set(r.outcome for _, _, _, r in pskip_case_jobs(rng)) == set(range(len(h264lib.PSKIP_OUTCOMES)))


# ---- GPU tests -------------------------------------------------------------------------------------------------------
def run_device(L, pic, jobs):
    recs = np.stack([record(pic, j) for j in jobs])
    out = np.zeros((len(jobs), OUT_BYTES), np.uint8)
    rc = L.b2h264_debug_skip_test(len(jobs), pic.set.ctypes.data, len(pic.set), recs.ctypes.data, out.ctypes.data)
    assert rc == 0, rc
    return out


@pytest.fixture(scope="module")
def dev():
    import openh264_b200 as m
    L = m.lib(0)
    L.b2h264_debug_skip_test.argtypes = [C.c_int, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p]
    return L


@pytest.mark.gpu
def test_device_matches_oracle(dev):
    for pic, jobs in cases():
        got, (want, res) = run_device(dev, pic, jobs), expect(pic, jobs)
        for i, r in enumerate(res):
            if r.outcome < 4:
                got[i, 32:] = 0                                        # the range guard rejected: no prediction to compare
        assert np.array_equal(got, want), describe(got, want, jobs, pic, res)


@pytest.mark.gpu
def test_device_matches_host_build(dev, emu):
    for pic, jobs in cases():
        got, host = run_device(dev, pic, jobs), run_emu(emu, pic, jobs)
        assert np.array_equal(got, host), describe(got, host, jobs, pic, expect(pic, jobs)[1])


@pytest.mark.gpu
def test_device_refuses_bad_arguments(dev):
    _refusals(dev.b2h264_debug_skip_test)


def test_host_build_refuses_bad_arguments(emu):
    """the host build refuses what the device hook refuses (stage_hooks.cuh: skip_test_args_ok)"""
    _refusals(emu.emu_skip_test)


def _refusals(fn):
    pic, jobs = cases()[1]
    good = np.stack([record(pic, j) for j in jobs[:2]])
    out = np.zeros((2, OUT_BYTES), np.uint8)
    n_set = len(pic.set)
    assert fn(2, pic.set.ctypes.data, n_set, good.ctypes.data, out.ctypes.data) == 0

    def refused(word, value, n=2, set_bytes=n_set):
        bad = good.copy()
        if word is not None:
            bad[1, 4 * word:4 * word + 4] = np.array([value], np.int32).view(np.uint8)
        return fn(n, pic.set.ctypes.data, set_bytes, bad.ctypes.data, out.ctypes.data) == -1
    assert refused(6, 52) and refused(6, -1)                           # QP
    assert refused(4, pic.mb_w) and refused(5, pic.mb_h) and refused(4, -1) and refused(5, -1)   # macroblock outside the picture
    assert refused(2, pic.sy - 1) and refused(3, pic.sc - 1)           # strides narrower than the padded picture
    assert refused(8, 16) and refused(8, -1)                           # availability bits
    assert refused(10, 7) and refused(12, 7) and refused(27, -1)       # macroblock types (co-located, neighbours)
    assert refused(1, pic.mb_h + 1)                                    # the set would be smaller than the planes
    assert refused(None, 0, set_bytes=n_set - 1)
    assert refused(None, 0, n=0)
