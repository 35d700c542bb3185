"""Seeded macroblock cases for the intra path that stages I and C share (md_i16x16, then intra_mb_finish: enc_mb.cuh,
enc_inter.cuh), in the case record of b2h264_debug_intra_tail (enc_kernels.cu), and the views the tests compare.

Content classes (CLASSES) reach what natural clips rarely do: plane predictions that saturate at 0 and 255 in luma and chroma,
exact cost ties between modes (flat blocks with flat borders), LOW-complexity textures whose block-mean variance is 149, 150 and
151 (the I4x4 gate is >= 150), stripes, edges and noise.  Every class runs under all 16 neighbour-availability nibbles at the QPs
of MAIN_QPS in HIGH and LOW complexity, with the neighbours' I4x4 modes random or absent; a smaller set sweeps all 52 QPs; and
cost limits below, at and above the I4x4 running total (taken from a run without a limit) make the I4x4 try break early,
complete and lose, and complete and win.
"""
import ctypes as C

import numpy as np

import h264lib
import mb_recon_oracle as mr

ROOT = h264lib.ROOT
TILE = 17 * 32 + 2 * 9 * 16         # RecTile: luma rows -1..15 x cols -1..30, Cb / Cr rows -1..7 x cols -1..14
IN_BYTES = TILE + 384 + 32          # the case record
OUT_BYTES = 896 + 120 + 16 + TILE   # MbOut, MbInfo, limit / I4x4 cost / lambda / 0, the tile
INFO = 896                          # MbInfo: nnz at +64, i4_mode at +88, mb_type at +112, cbp at +113
TAIL = INFO + 120
NB_LEFT, NB_TOP, NB_TOPLEFT, NB_TOPRIGHT = 1, 2, 4, 8
INT_MAX = 0x7fffffff
CLASSES = ["noise", "smooth", "steep", "flat", "near-flat", "stripes", "var149", "var150", "var151"]
MAIN_QPS = (0, 1, 12, 26, 40, 50, 51)

_Y, _X = np.mgrid[0:17, 0:25]                                          # luma rows -1..15, cols -1..23 (+1)
_YC, _XC = np.mgrid[0:9, 0:9]


def _variance_texture(rng, target):
    """16 x 16 source whose sixteen 4x4 block means m satisfy sum(m^2) - (sum(m)^2 >> 4) == target (AnalysisVaaInfoIntra):
    each block is its mean plus a zero-sum checkerboard, so the means are exact"""
    while True:
        m = rng.randint(60, 190) + rng.randint(-5, 6, 16)
        if int((m * m).sum()) - (int(m.sum()) ** 2 >> 4) == target:
            break
    a = rng.randint(0, 30)
    chk = np.where((np.arange(4)[:, None] + np.arange(4)[None, :]) % 2 == 0, a, -a)
    src = np.zeros((16, 16), int)
    for k in range(16):
        by, bx = k // 4, k % 4
        src[4 * by:4 * by + 4, 4 * bx:4 * bx + 4] = m[k] + chk
    return src, int(m.mean())


def content(rng, kind, chroma):
    """the (17 x 25) luma or (9 x 9) chroma samples of one case: row 0 / column 0 are the neighbours' samples"""
    y, x = (_YC, _XC) if chroma else (_Y, _X)
    h, w = y.shape
    name = CLASSES[kind]
    if name == "noise":
        v = rng.randint(0, 256, (h, w))
    elif name == "smooth":
        v = rng.randint(40, 200) + rng.uniform(-4, 4) * x + rng.uniform(-4, 4) * y + rng.randint(-2, 3, (h, w))
    elif name == "steep":
        # slopes that carry the plane prediction past 0 and 255 at opposite corners
        s = (2.0 if chroma else 1.0) * rng.uniform(14, 24)
        gx, gy = s * rng.choice([-1, 1]), s * rng.uniform(0.6, 1.0) * rng.choice([-1, 1])
        v = 128 + gx * (x - (w - 1) / 2) + gy * (y - (h - 1) / 2) + rng.randint(-3, 4, (h, w))
    elif name == "flat":
        v = np.full((h, w), rng.randint(0, 256))
    elif name == "near-flat":
        v = np.full((h, w), rng.randint(1, 255))
        v[1:, 1:] += rng.randint(-1, 2, (h - 1, w - 1)) * (rng.rand(h - 1, w - 1) < 0.3)
    elif name == "stripes":
        period, phase = rng.randint(2, 9), rng.randint(0, 8)
        v = np.where(((x if rng.rand() < 0.5 else y) + phase) // period % 2 == 0, rng.randint(0, 256), rng.randint(0, 256))
        v = v + rng.randint(-3, 4, (h, w))
    else:
        target = int(name[3:])
        if chroma:
            v = rng.randint(100, 156) + rng.randint(-6, 7, (h, w))
        else:
            src, mean = _variance_texture(rng, target)
            v = mean + rng.randint(-4, 5, (h, w))
            v[1:17, 1:17] = src
    return np.clip(v, 0, 255).astype(np.uint8)


def make_case(rng, kind, qp, nb, fast, limit=-1):
    """one case record: the tile with the available neighbours' samples (zero where a neighbour is missing, as the encoder
    loads them), the source, QP / availability / LOW complexity / cost limit, the neighbours' I4x4 modes"""
    rec = np.zeros(IN_BYTES, np.uint8)
    ty = np.zeros((17, 32), np.uint8)
    luma = content(rng, kind, False)
    if nb & NB_TOPLEFT:
        ty[0, 0] = luma[0, 0]
    if nb & NB_TOP:
        ty[0, 1:17] = luma[0, 1:17]
    if nb & NB_TOPRIGHT:
        ty[0, 17:25] = luma[0, 17:25]
    if nb & NB_LEFT:
        ty[1:17, 0] = luma[1:17, 0]
    planes, cur_c = [ty.reshape(-1)], []
    for _ in range(2):
        tc = np.zeros((9, 16), np.uint8)
        ch = content(rng, kind, True)
        if nb & NB_TOPLEFT:
            tc[0, 0] = ch[0, 0]
        if nb & NB_TOP:
            tc[0, 1:9] = ch[0, 1:9]
        if nb & NB_LEFT:
            tc[1:9, 0] = ch[1:9, 0]
        planes.append(tc.reshape(-1))
        cur_c.append(ch[1:9, 1:9].reshape(-1))
    rec[:TILE] = np.concatenate(planes)
    rec[TILE:TILE + 256] = luma[1:17, 1:17].reshape(-1)
    rec[TILE + 256:TILE + 384] = np.concatenate(cur_c)
    rec[TILE + 384:TILE + 400] = np.array([qp, nb, fast, limit], np.int32).view(np.uint8)
    nm = np.full(8, -1, np.int8)
    for side in (0, 4):                                               # left column, top row: I4x4 neighbour or not
        if rng.rand() < 0.6:
            nm[side:side + 4] = rng.randint(0, 9, 4)
    rec[TILE + 400:TILE + 408] = nm.view(np.uint8)
    return rec


def base_cases():
    """(records, class, QP): every class x MAIN_QPS x HIGH / LOW x 16 nibbles, then every class x all 52 QPs x HIGH / LOW"""
    rng = np.random.RandomState(2026)
    recs, kinds, qps = [], [], []
    for kind in range(len(CLASSES)):
        for qp in MAIN_QPS:
            for fast in (0, 1):
                for nb in range(16):
                    recs.append(make_case(rng, kind, qp, nb, fast))
                    kinds.append(kind)
                    qps.append(qp)
    for kind in range(len(CLASSES)):
        for qp in range(52):
            for fast in (0, 1):
                recs.append(make_case(rng, kind, qp, rng.randint(16), fast))
                kinds.append(kind)
                qps.append(qp)
    return np.stack(recs), np.array(kinds), np.array(qps)


def with_limits(base, kinds, qps, run):
    """the base cases, then every sixth case whose I4x4 try ran again with cost limits just below, at and above the running
    total after the 16th block, above the I4x4 cost, and somewhere inside; `run(cases) -> result records` of a build that
    implements the path (the limits come from a run without one)"""
    free = base.copy()
    free[:, TILE + 396:TILE + 400] = np.array([1 << 30], np.int32).view(np.uint8)
    t = run(free)[:, TAIL:TAIL + 12].view(np.int32)
    cost4, lam = t[:, 1], t[:, 2]
    total = cost4.astype(np.int64) - 24 * lam
    rng = np.random.RandomState(7)
    extra, ek, eq = [], [], []
    for i in np.nonzero(cost4 != INT_MAX)[0][::6]:
        for lim in (total[i] - 1, total[i], total[i] + 1, cost4[i] + 1, rng.randint(0, total[i] + 1)):
            c = base[i].copy()
            c[TILE + 396:TILE + 400] = np.array([max(int(lim), 0)], np.int32).view(np.uint8)
            extra.append(c)
            ek.append(kinds[i])
            eq.append(qps[i])
    return np.concatenate([base, np.stack(extra)]), np.concatenate([kinds, ek]), np.concatenate([qps, eq])


def run_emu(emu, cases):
    out = np.zeros((len(cases), OUT_BYTES), np.uint8)
    assert emu.emu_intra_tail(len(cases), cases.ctypes.data, out.ctypes.data) == 0
    return out


def run_ref(cases):
    """the reference itself (oracle/_ref: ref_intra_mb in oracle/ref_shim.cpp): result records and (I16x16, I4x4, chroma) costs"""
    lib = h264lib.ref().lib
    lib.ref_intra_mb.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    cases = np.ascontiguousarray(cases)
    out = np.zeros((len(cases), OUT_BYTES), np.uint8)
    costs = np.zeros((len(cases), 3), np.int32)
    assert lib.ref_intra_mb(len(cases), cases.ctypes.data, out.ctypes.data, costs.ctypes.data) == 0
    return out, costs


def fields(out):
    """what the intra path decides and codes, from result records, with the entries that carry no meaning for the chosen type
    cleared: the mode and coded-block fields, levels, counts, the costs of the tail and the reconstructed samples"""
    out = np.ascontiguousarray(out)
    n = len(out)
    i4 = out[:, INFO + 112] == 0
    prev = out[:, 8:24].astype(np.int16) * i4[:, None]
    rem = out[:, 24:40].astype(np.int16) * (i4[:, None] & (prev == 0))
    i4m = out[:, INFO + 88:INFO + 104].astype(np.int16) * i4[:, None]
    i16 = np.where(i4, -1, out[:, 3].astype(np.int16))
    dc = out[:, 80:112].copy().view(np.int16) * ~i4[:, None]
    luma = out[:, 112:624].copy().view(np.int16).reshape(n, 16, 16)
    luma[:, :, 15] *= i4[:, None]                                       # I16x16 AC: 15 levels per block
    cdc = out[:, 624:640].copy().view(np.int16)
    cac = out[:, 640:896].copy().view(np.int16).reshape(n, 8, 16)
    cac[:, :, 15] = 0
    nnz = out[:, INFO + 64:INFO + 88].astype(np.int16)
    head = np.stack([out[:, INFO + 112], out[:, INFO + 113], i16, out[:, 4]], 1).astype(np.int16)
    tail = out[:, TAIL:TAIL + 12].copy().view(np.int32)
    t = out[:, TAIL + 16:TAIL + 16 + TILE]
    rec = np.concatenate([t[:, :17 * 32].reshape(n, 17, 32)[:, 1:, 1:17].reshape(n, -1),
                          t[:, 17 * 32:17 * 32 + 144].reshape(n, 9, 16)[:, 1:, 1:9].reshape(n, -1),
                          t[:, 17 * 32 + 144:].reshape(n, 9, 16)[:, 1:, 1:9].reshape(n, -1)], 1)
    return {"head": head, "prev": prev, "rem": rem, "i4_mode": i4m, "luma_dc": dc, "luma": luma.reshape(n, -1),
            "chroma_dc": cdc, "chroma_ac": cac.reshape(n, -1), "nnz": nnz, "costs": tail, "rec": rec}


def first_difference(a, b):
    """None if two result sets agree on every field, else (case, field name)"""
    fa, fb = fields(a), fields(b)
    for name in fa:
        bad = np.nonzero((fa[name] != fb[name]).reshape(len(a), -1).any(1))[0]
        if len(bad):
            return int(bad[0]), name, len(bad)
    return None


def group_hashes(out, kinds, qps):
    """SHA-1 of the compared fields per (class, QP) group"""
    f = fields(out)
    res = {}
    for k in range(len(CLASSES)):
        for q in range(52):
            sel = (kinds == k) & (qps == q)
            if sel.any():
                res[f"{CLASSES[k]}/{q}"] = h264lib.sha1(*[f[name][sel] for name in sorted(f)])
    return res

def spec_decode(cases, out, sel):
    """a conforming decoder's reconstruction (tests/mb_recon_oracle.py, H.264 8.3 and 8.5) of the selected cases' result
    records, the macroblock at (1, 1) of a 3 x 2 macroblock picture whose neighbours carry the case's samples and I4x4 modes,
    against the reconstruction the records came with.  Returns the indices that match, that the decoder refuses as
    non-conforming (its 16-bit range checks) and that differ."""
    match, refused, differ = [], [], []
    for i in sel:
        c, o = cases[i], out[i]
        qp, nb = (int(v) for v in c[TILE + 384:TILE + 392].view(np.int32))
        nm = c[TILE + 400:TILE + 408].view(np.int8)
        recs = np.zeros(6, mr.MBOUT)
        aux = np.zeros(6, mr.DECAUX)
        recs[:] = np.frombuffer(o[:896].tobytes(), mr.MBOUT)[0]
        for n in range(6):
            recs[n]["mb_type"] = mr.I16x16
        cur = recs[4]
        cur["mb_type"], cur["cbp"], cur["qp"] = o[INFO + 112], o[INFO + 113], qp
        aux[4]["avail"] = nb
        pic = mr.Picture(3, 2, recs, aux, None, 0, [])
        for n, side in ((3, 0), (1, 4)):
            if nm[side] >= 0:
                recs[n]["mb_type"] = mr.I4x4
                modes = [2] * 16
                for j in range(4):
                    modes[4 * j + 3 if side == 0 else 12 + j] = int(nm[side + j])
                pic.modes[n] = modes
        ty = c[:17 * 32].reshape(17, 32).astype(np.int64)
        pic.pl[0][15, 15:40] = ty[0, :25]
        pic.pl[0][16:32, 15] = ty[1:17, 0]
        for p in range(2):
            tc = c[17 * 32 + 144 * p:17 * 32 + 144 * (p + 1)].reshape(9, 16).astype(np.int64)
            pic.pl[1 + p][7, 7:16] = tc[0, :9]
            pic.pl[1 + p][8:16, 7] = tc[1:9, 0]
        try:
            pic.mb(1, 1)
        except mr.NotConforming:
            refused.append(i)
            continue
        t = o[TAIL + 16:TAIL + 16 + TILE]
        want = [t[:17 * 32].reshape(17, 32)[1:, 1:17], t[17 * 32:17 * 32 + 144].reshape(9, 16)[1:, 1:9],
                t[17 * 32 + 144:].reshape(9, 16)[1:, 1:9]]
        got = [pic.pl[0][16:32, 16:32], pic.pl[1][8:16, 8:16], pic.pl[2][8:16, 8:16]]
        (match if all(np.array_equal(g, w) for g, w in zip(got, want)) else differ).append(i)
    return match, refused, differ
