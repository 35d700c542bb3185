"""Stage B's motion search of a P macroblock (enc_inter.cuh: me_start_point, win_issue / win_wait, me_partition, me_refine,
mc_chroma_part), one partition shape per macroblock job, against the CPU oracle: every integer search against orc_me_search
(WelsMotionEstimateSearch), every fractional refinement against orc_me_refine (MeRefineFracPixel, its candidates predicted one
by one by orc_mc_luma rather than from the device's averaged half-sample planes) and every partition's chroma prediction
against orc_mc_chroma at the refined vector.

On the device the searches read a 64 x 48 window of the reference staged by one bulk tensor copy wherever it covers the block,
and the plane elsewhere; the first refinement stages its integer samples out of that window too (its last rows share their
bytes with the coefficient buffer the staging writes).  The host emulation build never has a window.  So the device runs every
job with the window and without it, and both runs must equal the oracle and the host build.

The jobs are built so that the window paths are all reached; which ones are is computed here from the clip window, the
window origin and a replay of the integer search's path, and asserted: a search wholly inside the window, a start candidate
outside it, a diamond that leaves it mid-walk, the early stop, the 16-iteration cap, the out-of-range spin, a refinement
staged from the window (also from its rows that alias the coefficient buffer), from the plane because the window does not
cover it (at the edge: exactly covered, one to four columns short: the staging reads up to two bytes per row more than it
uses, so only three or four columns short would a wrong choice show) and from the plane because the window was given up after the first
refinement; all quarter-sample phases the refinement can end on (the centre (2, 2) and the diagonals (1|3, 1|3) are not
among its candidates) and the chroma eighth-sample phases that follow, for 4- and 8-wide chroma blocks."""
import ctypes as C

import numpy as np
import pytest

import h264lib
from h264lib import MeJob, MeResult, RefineJob, RefineResult, ptr

ROOT = h264lib.ROOT
IN_BYTES = 80 * 4 + 256             # b2h264_debug_me_partitions' job record
OUT_BYTES = 64 * 4 + 256 + 128      # its output record
WIN_W, WIN_H = 64, 48               # enc_mb.cuh: the search window
COEF_ROW = (256 + 384 + 3 * 18 * 32) // WIN_W     # first window row that shares its bytes with MbScratch::coef (37)
EARLY = 0x7fffffff                  # sad_pred that every start point beats
PARTS = {0: [(0, 0)], 1: [(0, 0), (0, 8)], 2: [(0, 0), (8, 0)], 3: [(0, 0), (8, 0), (0, 8), (8, 8)]}   # (ox, oy) per shape
DIMS = {0: (16, 16), 1: (16, 8), 2: (8, 16), 3: (8, 8)}                                               # (w, h) per shape
# final quarter-sample phases (x, y) the refinement can reach: the integer point, the four half-sample points, and the
# quarter-sample points around the integer point and around each half-sample point
REFINE_PHASES = {(0, 0), (2, 0), (0, 2), (1, 0), (3, 0), (0, 1), (0, 3), (2, 1), (2, 3), (1, 2), (3, 2)}


@pytest.fixture(scope="module")
def emu():
    return h264lib.emu()


# ---- pictures ------------------------------------------------------------------------------------------------------
def content(rng, kind, h, w):
    """0 textured noise (a few random sinusoids plus noise), 1 smooth gradient, 2 periodic stripes (SAD ties)"""
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    if kind == 0:
        v = 128.0 + rng.randint(-6, 7, (h, w))
        for _ in range(4):
            fx, fy = rng.uniform(-1, 1, 2) * 2 * np.pi / rng.uniform(6, 40)
            v += rng.uniform(10, 30) * np.sin(fx * x + fy * y + rng.uniform(0, 6.3))
    elif kind == 1:
        v = 128 + rng.uniform(-2, 2) * (x - w / 2) + rng.uniform(-2, 2) * (y - h / 2) + rng.randint(-1, 2, (h, w))
    else:
        period = rng.randint(2, 7)
        v = np.where(((x if rng.rand() < 0.5 else y) // period) % 2 == 0, 60, 190) + rng.randint(-1, 2, (h, w))
    return np.clip(v, 0, 255).astype(np.uint8)


class Pic:
    """current luma and the padded, expanded reference planes (Y, Cb, Cr) of one picture, laid out as the hook reads them"""

    def __init__(self, rng, mb_w, mb_h, kind, shift):
        orc = h264lib.oracle()
        W, H = 16 * mb_w, 16 * mb_h
        self.mb_w, self.mb_h = mb_w, mb_h
        self.sy, self.sc = W + 64, W // 2 + 32               # the encoder's padded strides (enc_host.h)
        self.cur = content(rng, kind, H, W)
        # reference: the current picture moved by `shift` quarter samples (interpolated block by block out of the expanded
        # current picture), plus noise
        cp = np.zeros((H + 64, self.sy), np.uint8)
        cp[32:32 + H, 32:32 + W] = self.cur
        orc.expand_plane(ptr(cp, off=32 * self.sy + 32), self.sy, W, H, 32)
        qx, qy = shift
        ref = np.zeros((H, W), np.uint8)
        tmp = np.zeros((16, 16), np.uint8)
        for by in range(0, H, 16):
            for bx in range(0, W, 16):
                orc.mc_luma(ptr(cp, off=(32 + by + (qy >> 2)) * self.sy + 32 + bx + (qx >> 2)), self.sy, ptr(tmp), 16, qx, qy, 16, 16)
                ref[by:by + 16, bx:bx + 16] = tmp
        ref = np.clip(ref.astype(int) + rng.randint(-2, 3, ref.shape), 0, 255).astype(np.uint8)
        self.Y = np.zeros((H + 64, self.sy), np.uint8)
        self.Y[32:32 + H, 32:32 + W] = ref
        orc.expand_plane(ptr(self.Y, off=32 * self.sy + 32), self.sy, W, H, 32)
        self.C = []
        for _ in range(2):
            p = np.zeros((H // 2 + 32, self.sc), np.uint8)
            p[16:16 + H // 2, 16:16 + W // 2] = content(rng, int(rng.randint(0, 3)), H // 2, W // 2)
            orc.expand_plane(ptr(p, off=16 * self.sc + 16), self.sc, W // 2, H // 2, 16)
            self.C.append(p)
        s = np.concatenate([self.Y.ravel(), self.C[0].ravel(), self.C[1].ravel()])
        self.set = np.concatenate([s, np.zeros(-len(s) % 16, np.uint8)])
        self.Yi = self.Y.astype(np.int32)


# ---- the search, as the reference defines it ------------------------------------------------------------------------
def se_bits(v):
    code = 2 * v - 1 if v > 0 else -2 * v
    return 2 * (code + 1).bit_length() - 1


def mvd(lam, dx, dy):
    return ((lam * se_bits(dx)) & 0xffff) + ((lam * se_bits(dy)) & 0xffff)


def clip_window(pic, mbx, mby, r):
    """SetMvWithinIntegerMvRange (svc_motion_estimate.h:345): integer-sample range of the macroblock's searches"""
    lo_x, lo_y = max(-((mbx + 1) << 4) + 3, -r), max(-((mby + 1) << 4) + 3, -r)
    hi_x, hi_y = min(((pic.mb_w - mbx) << 4) - 3, r), min(((pic.mb_h - mby) << 4) - 3, r)
    return lo_x, lo_y, hi_x, hi_y


def clip3(v, lo, hi):
    return lo if v < lo else hi if v > hi else v


def window_origin(pic, j):
    """win_issue: the window starts 16 samples left of and above the 16x16 search's start point, X rounded down to 16 bytes"""
    lo_x, lo_y, hi_x, hi_y = clip_window(pic, j["mbx"], j["mby"], j["range"])
    sx, sy = clip3((2 + j["p16"][0]) >> 2, lo_x, hi_x), clip3((2 + j["p16"][1]) >> 2, lo_y, hi_y)
    X = (32 + j["mbx"] * 16 + sx - 16) & ~15
    return X - 32 - j["mbx"] * 16, sy - 16


def replay_search(pic, j, q):
    """the integer search's path (WelsMotionEstimateSearch), for the coverage: the blocks it reads and what ended it"""
    (ox, oy), (w, h) = PARTS[j["shape"]][q], DIMS[j["shape"]]
    pt = j["parts"][q]
    lam = h264lib.oracle().qp_lambda(j["qp"])
    lo_x, lo_y, hi_x, hi_y = clip_window(pic, j["mbx"], j["mby"], j["range"])
    x0, y0 = 32 + 16 * j["mbx"] + ox, 32 + 16 * j["mby"] + oy
    cur = pic.cur[16 * j["mby"] + oy:16 * j["mby"] + oy + h, 16 * j["mbx"] + ox:16 * j["mbx"] + ox + w].astype(np.int32)

    def sad(mx, my):
        return int(np.abs(cur - pic.Yi[y0 + my:y0 + my + h, x0 + mx:x0 + mx + w]).sum())
    px, py = pt["mvp"]
    mx, my = clip3((2 + px) >> 2, lo_x, hi_x), clip3((2 + py) >> 2, lo_y, hi_y)
    best = sad(mx, my) + mvd(lam, mx * 4 - px, my * 4 - py)
    cands = []
    for cx, cy in pt["cands"]:
        cx, cy = clip3((2 + cx) >> 2, lo_x, hi_x), clip3((2 + cy) >> 2, lo_y, hi_y)
        if (cx, cy) == (mx, my):
            continue
        cands.append((cx, cy))
        c = sad(cx, cy) + mvd(lam, cx * 4 - px, cy * 4 - py)
        if c < best:
            best, mx, my = c, cx, cy
    start = [(clip3((2 + px) >> 2, lo_x, hi_x), clip3((2 + py) >> 2, lo_y, hi_y))]
    r = {"early": best < pt["sad_pred"], "spin": False, "cap": False, "centres": [], "reads": start + cands, "cands": cands}
    if not r["early"]:
        dx, dy = mx * 4 - px, my * 4 - py
        moves = 0
        for _ in range(16):
            tx, ty = (dx + px) >> 2, (dy + py) >> 2
            if not (lo_x <= tx < hi_x and lo_y <= ty < hi_y):
                r["spin"] = True
                continue
            r["centres"].append((tx, ty))
            cs = [sad(tx, ty - 1) + mvd(lam, dx, dy - 4), sad(tx, ty + 1) + mvd(lam, dx, dy + 4),
                  sad(tx - 1, ty) + mvd(lam, dx - 4, dy), sad(tx + 1, ty) + mvd(lam, dx + 4, dy)]
            step = None
            for k, c in enumerate(cs):
                if c < best:
                    best, step = c, k
            if step is None:
                break
            moves += 1
            dx += 4 * (0, 0, -1, 1)[step]
            dy += 4 * (-1, 1, 0, 0)[step]
        r["cap"] = moves == 16
        mx, my = (dx + px) >> 2, (dy + py) >> 2
    r["mv"], r["sad"] = (4 * mx, 4 * my), best
    r["reads"].append((mx, my))
    return r


def in_window(pic, j, q, mx, my, m):
    """me_block: the block at integer offset (mx, my) from partition q's co-located block, with m samples of margin, lies in
    the window"""
    (ox, oy), (w, h) = PARTS[j["shape"]][q], DIMS[j["shape"]]
    wx, wy = window_origin(pic, j)
    x, y = ox + mx - wx, oy + my - wy
    return x >= m and y >= m and x + w + m <= WIN_W and y + h + m <= WIN_H


def refine_staging(pic, j, q, mv):
    """me_refine's source for partition q with integer vector mv when the macroblock has a window: (window covers it,
    window rows it reads up to, x0 + 4 * words per row)"""
    (ox, oy), (w, h) = PARTS[j["shape"]][q], DIMS[j["shape"]]
    wx, wy = window_origin(pic, j)
    x0, y0 = ox + (mv[0] >> 2) - 3 - wx, oy + (mv[1] >> 2) - 3 - wy
    wq, wh = (w + 9) >> 2, h + 6
    return x0 >= 0 and y0 >= 0 and x0 + 4 * wq <= WIN_W and y0 + wh <= WIN_H, y0 + wh - 1, x0 + 4 * wq


# ---- jobs ------------------------------------------------------------------------------------------------------------
def record(pic, j):
    w = np.zeros(80, np.int32)
    w[:12] = [pic.mb_w, pic.mb_h, pic.sy, pic.sc, j["range"], j["mbx"], j["mby"], j["qp"], j["fast"], j["p16"][0], j["p16"][1],
              j["shape"]]
    for q, pt in enumerate(j["parts"]):
        b = 12 + 16 * q
        w[b:b + 4] = [pt["mvp"][0], pt["mvp"][1], len(pt["cands"]), pt["sad_pred"]]
        for k, (cx, cy) in enumerate(pt["cands"]):
            w[b + 4 + 2 * k:b + 6 + 2 * k] = [cx, cy]
        w[b + 14:b + 16] = pt["rmvp"]
    cur = pic.cur[16 * j["mby"]:16 * j["mby"] + 16, 16 * j["mbx"]:16 * j["mbx"] + 16]
    return np.concatenate([w.view(np.uint8), cur.ravel()])


def part(rng, mvp, n_cand=None, sad_pred=None, spread=60):
    n = int(rng.randint(0, 6)) if n_cand is None else n_cand
    cands = [(int(rng.randint(-spread, spread + 1)), int(rng.randint(-spread, spread + 1))) for _ in range(n)]
    sp = int(rng.choice([0, 0, 0, 300, 2000, EARLY])) if sad_pred is None else sad_pred
    return {"mvp": mvp, "cands": cands, "sad_pred": sp, "rmvp": (mvp[0] + int(rng.randint(-9, 10)), mvp[1] + int(rng.randint(-9, 10)))}


def random_jobs(rng, pic, n, true_mv):
    jobs = []
    for _ in range(n):
        shape = int(rng.randint(0, 4))
        mv = lambda s: (true_mv[0] + int(rng.randint(-s, s + 1)), true_mv[1] + int(rng.randint(-s, s + 1)))   # noqa: E731
        p16 = mv(24) if rng.rand() < 0.8 else (int(rng.randint(-400, 401)), int(rng.randint(-400, 401)))
        parts = []
        for _q in PARTS[shape]:
            # far predictors start the search clipped to the range (the spin); |mvd| stays inside the cost tables
            m = mv(40) if rng.rand() < 0.85 else (int(rng.randint(-600, 601)), int(rng.randint(-600, 601)))
            parts.append(part(rng, m, spread=int(rng.choice([20, 80, 200]))))
        jobs.append({"mbx": int(rng.randint(0, pic.mb_w)), "mby": int(rng.randint(0, pic.mb_h)), "qp": int(rng.choice([0, 12, 26, 40, 51])),
                     "fast": int(rng.randint(0, 2)), "range": int(rng.choice([64, 64, 63, 8])), "p16": p16, "shape": shape,
                     "parts": parts})
    return jobs


def edge_jobs(rng, pic):
    """refinements placed against the window's edges: each partition stops at the start point (sad_pred = EARLY, no
    candidates), so its integer vector is the rounded predictor, chosen so that the refinement's staged rows end exactly at the
    window's right edge or one column beyond it, at its bottom edge or one row beyond it, and inside the rows that alias the
    coefficient buffer"""
    jobs = []
    mbx, mby = pic.mb_w // 2, pic.mb_h // 2
    for shape in range(4):
        (ox, oy), (w, h) = PARTS[shape][0], DIMS[shape]
        wq, wh = (w + 9) >> 2, h + 6
        for p16 in ((0, 0), (20, -12), (-36, 28)):
            j0 = {"mbx": mbx, "mby": mby, "qp": int(rng.choice([0, 26, 51])), "fast": int(rng.randint(0, 2)), "range": 64, "p16": p16,
                  "shape": shape}
            wx, wy = window_origin(pic, j0)
            # the staging reads 4 * wq bytes per row but uses w + 6 of them: only 3 or 4 columns beyond the edge would a
            # window read pick up samples of the next row
            targets = [(WIN_W - 4 * wq + k, 10) for k in range(5)] + [(10, WIN_H - wh), (10, WIN_H - wh + 1), (4, COEF_ROW - wh + 3)]
            for x0, y0 in targets:
                ix, iy = x0 + 3 + wx - ox, y0 + 3 + wy - oy
                parts = [part(rng, (4 * ix, 4 * iy), n_cand=0, sad_pred=EARLY)]
                parts += [part(rng, (4 * ix + 8, 4 * iy - 4), n_cand=0, sad_pred=EARLY) for _ in PARTS[shape][1:]]
                jobs.append(dict(j0, parts=parts))
    return jobs


def build_cases():
    """(picture, jobs) per picture: 1x1, 3x2 and 20x12 macroblocks and a 1920-wide strip (1984-byte stride)"""
    rng = np.random.RandomState(11)
    cases = []
    for mb_w, mb_h, kind, shift, n in [(1, 1, 0, (5, -3), 40), (1, 1, 1, (-14, 9), 40), (3, 2, 2, (22, 6), 60), (3, 2, 0, (-7, -2), 60),
                                       (20, 12, 0, (-30, 18), 110), (20, 12, 1, (70, -45), 110), (20, 12, 2, (9, 3), 60),
                                       (120, 1, 0, (13, -6), 60), (120, 1, 1, (-50, 2), 40),
                                       # moved by whole samples of each parity: refinements that end on the integer point, at
                                       # chroma phase 0 or 4 in each direction
                                       (3, 2, 0, (4, 4), 30), (3, 2, 0, (8, -4), 30), (3, 2, 0, (-4, 0), 30), (3, 2, 0, (-16, 8), 30)]:
        pic = Pic(rng, mb_w, mb_h, kind, shift)
        jobs = random_jobs(rng, pic, n, (-shift[0], -shift[1]))
        if mb_w >= 3:
            jobs += edge_jobs(rng, pic)
        # long walks: a gradient moved far, the search started at the co-located block
        if kind == 1:
            for q in range(8):
                jobs.append({"mbx": int(rng.randint(0, pic.mb_w)), "mby": int(rng.randint(0, pic.mb_h)), "qp": 0, "fast": q & 1, "range": 64,
                             "p16": (0, 0), "shape": 0, "parts": [part(rng, (0, 0), n_cand=0, sad_pred=0)]})
        cases.append((pic, jobs))
    return cases


_CASES = None


def cases():
    global _CASES
    if _CASES is None:
        _CASES = build_cases()
    return _CASES


# ---- expected results ------------------------------------------------------------------------------------------------
def expect(pic, jobs, window):
    """the hook's output records as the oracle computes them (window origin and flag as win_issue sets them)"""
    orc = h264lib.oracle()
    out = np.zeros((len(jobs), OUT_BYTES), np.uint8)
    for i, j in enumerate(jobs):
        o = np.zeros(64, np.int32)
        pred_y = np.zeros((16, 16), np.uint8)
        pred_c = np.zeros((2, 8, 8), np.uint8)
        lo_x, lo_y, hi_x, hi_y = clip_window(pic, j["mbx"], j["mby"], j["range"])
        cur = np.ascontiguousarray(pic.cur[16 * j["mby"]:16 * j["mby"] + 16, 16 * j["mbx"]:16 * j["mbx"] + 16])
        lam = orc.qp_lambda(j["qp"])
        (w, h), blk = DIMS[j["shape"]], j["shape"]
        for q, ((ox, oy), pt) in enumerate(zip(PARTS[j["shape"]], j["parts"])):
            mj = MeJob()
            mj.blk, mj.cur_off = blk, oy * 16 + ox
            mj.ref_off = (32 + 16 * j["mby"] + oy) * pic.sy + 32 + 16 * j["mbx"] + ox
            mj.mvp_x, mj.mvp_y = pt["mvp"]
            mj.mv_min_x, mj.mv_min_y, mj.mv_max_x, mj.mv_max_y = lo_x, lo_y, hi_x, hi_y
            mj.n_mvc = len(pt["cands"])
            for k, c in enumerate(pt["cands"]):
                mj.mvc[k][0], mj.mvc[k][1] = c
            mj.sad_pred, mj.qp, mj.calc_satd = pt["sad_pred"], j["qp"], 1 - j["fast"]
            r = MeResult()
            orc.me_search(ptr(cur), 16, ptr(pic.Y), pic.sy, C.byref(mj), C.byref(r))
            satd = r.satd_cost - mvd(lam, r.mv_x - pt["mvp"][0], r.mv_y - pt["mvp"][1])
            o[12 * q:12 * q + 8] = [r.mv_x, r.mv_y, pt["mvp"][0], pt["mvp"][1], r.sad_cost, r.satd_cost, satd,
                                    r.ref_off - (32 * pic.sy + 32)]
            rj = RefineJob()
            rj.w, rj.h, rj.cur_off, rj.ref_off = w, h, oy * 16 + ox, r.ref_off
            rj.mv_x, rj.mv_y = r.mv_x, r.mv_y
            rj.mvp_x, rj.mvp_y = pt["rmvp"]
            rj.qp, rj.satd_in_md, rj.satd = j["qp"], 1 - j["fast"], satd
            rr = RefineResult()
            pr = np.zeros((16, 16), np.uint8)
            orc.me_refine(ptr(cur), 16, ptr(pic.Y), pic.sy, C.byref(rj), C.byref(rr), ptr(pr))
            o[12 * q + 8:12 * q + 11] = [rr.mv_x, rr.mv_y, rr.cost]
            pred_y[oy:oy + h, ox:ox + w] = pr[:h, :w]
            cx, cy = 8 * j["mbx"] + ox // 2 + (rr.mv_x >> 3), 8 * j["mby"] + oy // 2 + (rr.mv_y >> 3)
            for pl in range(2):
                d = np.zeros((8, 8), np.uint8)
                orc.mc_chroma(ptr(pic.C[pl], off=(16 + cy) * pic.sc + 16 + cx), pic.sc, ptr(d), 8, rr.mv_x, rr.mv_y, w // 2, h // 2)
                pred_c[pl, oy // 2:(oy + h) // 2, ox // 2:(ox + w) // 2] = d[:h // 2, :w // 2]
        if window:
            o[48:51] = list(window_origin(pic, j)) + [1]
        out[i, :256] = o.view(np.uint8)
        out[i, 256:512] = pred_y.ravel()
        out[i, 512:] = pred_c.ravel()
    return out


def run_emu(emu, pic, jobs):
    recs = np.stack([record(pic, j) for j in jobs])
    planes = np.tile(pic.set, len(jobs))
    out = np.zeros((len(jobs), OUT_BYTES), np.uint8)
    assert emu.emu_me_partitions(len(jobs), planes.ctypes.data, len(pic.set), recs.ctypes.data, out.ctypes.data) == 0
    return out


def describe(got, want, jobs, pic):
    bad = np.nonzero((got != want).any(1))[0]
    if len(bad) == 0:
        return ""
    i = bad[0]
    g, w = got[i, :256].view(np.int32), want[i, :256].view(np.int32)
    words = np.nonzero(g != w)[0][:8].tolist()
    pix = np.nonzero(got[i, 256:] != want[i, 256:])[0][:8].tolist()
    return (f"{len(bad)} of {len(jobs)} jobs differ ({pic.mb_w}x{pic.mb_h} MBs); first: job {i} {jobs[i]}, words {words} "
            f"got {g[words].tolist()} want {w[words].tolist()}, prediction bytes {pix}")


# ---- CPU tests ---------------------------------------------------------------------------------------------------------
def test_host_build_matches_oracle(emu):
    for pic, jobs in cases():
        got, want = run_emu(emu, pic, jobs), expect(pic, jobs, window=False)
        assert np.array_equal(got, want), describe(got, want, jobs, pic)


def test_cases_reach_every_path():
    seen = {k: 0 for k in ("search inside the window", "start candidate outside the window", "diamond leaves the window mid-walk",
                           "early stop", "16-iteration cap", "out-of-range spin", "refinement from the window",
                           "refinement from window rows aliasing coef", "refinement from the plane: not covered",
                           "refinement at the window's right edge", "refinement one column beyond it",
                           "refinement from the plane: window given up", "1920-wide picture")}
    phases, chroma, beyond = set(), {4: set(), 8: set()}, set()
    for pic, jobs in cases():
        want = expect(pic, jobs, window=True)
        for i, j in enumerate(jobs):
            o = want[i, :256].view(np.int32)
            for q, (ox, oy) in enumerate(PARTS[j["shape"]]):
                r = replay_search(pic, j, q)
                assert r["mv"] == (o[12 * q], o[12 * q + 1]) and r["sad"] == o[12 * q + 4], "the replay is not the search"
                inside = [in_window(pic, j, q, x, y, 0) for x, y in r["reads"]] + [in_window(pic, j, q, x, y, 1) for x, y in r["centres"]]
                seen["search inside the window"] += all(inside)
                seen["start candidate outside the window"] += any(not in_window(pic, j, q, x, y, 0) for x, y in r["cands"])
                ins = [in_window(pic, j, q, x, y, 1) for x, y in r["centres"]]
                seen["diamond leaves the window mid-walk"] += bool(ins) and ins[0] and not all(ins)
                seen["early stop"] += r["early"]
                seen["16-iteration cap"] += r["cap"]
                seen["out-of-range spin"] += r["spin"]
                covered, last_row, right = refine_staging(pic, j, q, r["mv"])
                if q == 0:
                    seen["refinement from the window"] += covered
                    seen["refinement from window rows aliasing coef"] += covered and last_row >= COEF_ROW
                    seen["refinement from the plane: not covered"] += not covered
                    seen["refinement at the window's right edge"] += covered and right == WIN_W
                    seen["refinement one column beyond it"] += right == WIN_W + 1
                    beyond.add(right - WIN_W)
                else:
                    seen["refinement from the plane: window given up"] += covered
                mv = (int(o[12 * q + 8]), int(o[12 * q + 9]))
                phases.add((mv[0] & 3, mv[1] & 3))
                chroma[DIMS[j["shape"]][0] // 2].add((mv[0] & 7, mv[1] & 7))
            seen["1920-wide picture"] += pic.sy == 1984
    assert all(seen.values()), seen
    assert {1, 2, 3, 4} <= beyond, sorted(beyond)                      # first refinements 1..4 columns past the window's edge
    assert phases == REFINE_PHASES, sorted(phases)
    reachable = {(4 * ix + fx, 4 * iy + fy) for fx, fy in REFINE_PHASES for ix in (0, 1) for iy in (0, 1)}
    for w in (4, 8):
        assert chroma[w] == reachable, (w, sorted(reachable - chroma[w]))


def test_refine_case_reaches_every_winner():
    """the oracle's me_refine kernel case (kernel_cases.py) ends on the integer point, a half-sample and a quarter-sample point"""
    from kernel_cases import run_case
    out = run_case("me_refine", h264lib.oracle())
    mv = np.array([out[i][:2] for i in range(0, len(out), 2)])
    frac = (mv[:, 0] & 3) | ((mv[:, 1] & 3) << 2)
    assert (frac == 0).any() and ((frac != 0) & ((mv & 1) == 0).all(1)).any() and ((mv & 1) != 0).any(1).any()


# ---- GPU tests -------------------------------------------------------------------------------------------------------
def run_device(L, m, pic, jobs, window):
    recs = np.stack([record(pic, j) for j in jobs])
    planes = m.DeviceArray(np.tile(pic.set, len(jobs)))
    out = np.zeros((len(jobs), OUT_BYTES), np.uint8)
    rc = L.b2h264_debug_me_partitions(len(jobs), planes.ptr, len(pic.set), recs.ctypes.data, window, out.ctypes.data)
    assert rc == 0, rc
    return out


@pytest.fixture(scope="module")
def dev():
    import openh264_b200 as m
    L = m.lib(0)
    L.b2h264_debug_me_partitions.argtypes = [C.c_int, C.c_void_p, C.c_longlong, C.c_void_p, C.c_int, C.c_void_p]
    return L, m


@pytest.mark.gpu
@pytest.mark.parametrize("window", [1, 0])
def test_device_matches_oracle(dev, window):
    L, m = dev
    for pic, jobs in cases():
        got, want = run_device(L, m, pic, jobs, window), expect(pic, jobs, window=window)
        assert np.array_equal(got, want), describe(got, want, jobs, pic)


@pytest.mark.gpu
def test_device_matches_host_build(dev, emu):
    L, m = dev
    for pic, jobs in cases():
        host = run_emu(emu, pic, jobs)
        for window in (0, 1):
            got = run_device(L, m, pic, jobs, window)
            got[:, 192:204] = 0                                   # win_x0, win_y0, win_ok: the host build has no window
            assert np.array_equal(got, host), describe(got, host, jobs, pic)


@pytest.mark.gpu
def test_device_refuses_bad_arguments(dev):
    L, m = dev
    pic, _ = cases()[2]
    planes = m.DeviceArray(np.tile(pic.set, 2))
    call = _refusals(lambda n, set_bytes, jobs, out: L.b2h264_debug_me_partitions(n, planes.ptr, set_bytes, jobs, 1, out))
    # device only: one tensor map covers every job's planes, and the window copy needs 16- / 8-byte aligned rows
    assert call(2, pic.sy + 8) and call(3, pic.sc + 4)                 # strides: luma not a multiple of 16, chroma of 8
    assert call(None, 0, set_bytes=len(pic.set) + 8)                   # sets not on 16-byte boundaries


def test_host_build_refuses_bad_arguments(emu):
    """the host build refuses what both builds refuse (stage_hooks.cuh: me_partitions_args_ok)"""
    pic, _ = cases()[2]
    planes = np.tile(pic.set, 2)
    _refusals(lambda n, set_bytes, jobs, out: emu.emu_me_partitions(n, planes.ctypes.data, set_bytes, jobs, out))


def _refusals(fn):
    """the refusals both builds share; fn(n, set_bytes, jobs, out) runs one build's hook on two plane sets.  Returns the refused()
    check for the caller's own rules."""
    pic, jobs = cases()[2]
    good = np.stack([record(pic, j) for j in jobs[:2]])
    out = np.zeros((2, OUT_BYTES), np.uint8)
    n_set = len(pic.set)
    assert fn(2, n_set, good.ctypes.data, out.ctypes.data) == 0

    def refused(word, value, n=2, set_bytes=n_set):
        bad = good.copy()
        if word is not None:
            bad[1, 4 * word:4 * word + 4] = np.array([value], np.int32).view(np.uint8)
        return fn(n, set_bytes, bad.ctypes.data, out.ctypes.data) == -1
    assert refused(7, 52) and refused(7, -1)                           # QP
    assert refused(5, pic.mb_w) and refused(6, pic.mb_h) and refused(5, -1)   # macroblock outside the picture
    assert refused(2, pic.sy - 16)                                     # narrower than the padded picture
    assert refused(4, -1)                                              # negative mv_range: blocks could leave the padding
    assert refused(11, 4) and refused(14, 6)                           # shape, candidate count
    assert refused(None, 0, set_bytes=n_set - 16)
    assert refused(None, 0, n=0)
    return refused
