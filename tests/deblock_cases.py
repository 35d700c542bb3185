"""Seeded random pictures for the picture deblocking filter (k_deblock_pictures, enc_deblock.cuh).

One description of a picture yields two views of the same inputs:
- the records the device filter reads: MbInfo (120 bytes) per macroblock and, for pictures with B macroblocks, DecMbAuxB
  (132 bytes), encoded exactly as the decoder (dec_mb.cuh) or the encoder leaves them;
- the plain per-macroblock arrays of oracle/orc_deblock_picture (raster 4x4 blocks, both lists).
The pictures stay inside what the parser and the encoder guarantee: one reference picture in encoder mode, no coefficients and
one vector in a P_Skip macroblock, one vector and coefficient count per 8x8 in a macroblock with the 8x8 transform, list-1
records only for B macroblocks.  Samples are smooth blocks with steps mostly below alpha, some large steps and flat areas,
so that every filter branch runs.
"""
import ctypes as C

import numpy as np

import h264lib

MBINFO = np.dtype([("mv", "<i2", (16, 2)), ("nnz", "i1", 24), ("i4_mode", "i1", 16), ("p16x16_mv", "<i2", 2),
                   ("sad_cost", "<i4"), ("mb_type", "u1"), ("cbp", "u1"), ("qp", "u1"), ("qp_c", "u1"), ("ref_idx", "i1"),
                   ("t8x8", "u1"), ("pad", "u1", 2)])
AUXB = np.dtype([("ref_idx", "i1", 4), ("pred_lists", "u1", 4), ("w1", "<i2", 4), ("mv", "<i2", (16, 2)), ("wp_on", "u1"),
                 ("wp_log2", "u1", 2), ("pad", "u1"), ("wp", "<i2", (4, 3, 2))])
assert MBINFO.itemsize == 120 and AUXB.itemsize == 132

# macroblock types (enc_types.h numbering; oracle/h264_oracle.h ORC_MB_* uses the same)
I4x4, I16x16, P16x16, P16x8, P8x16, P8x8, PSKIP, IPCM, B, BSKIP = range(10)
INTRA = (I4x4, I16x16, IPCM)

# raster 4x4 block -> (8x8 index, 4x4 inside the 8x8): DecMbAuxB vectors are in coding order [4 * k + j]
_BX, _BY = np.arange(16) % 4, np.arange(16) // 4
B8 = (_BY >> 1) * 2 + (_BX >> 1)
CODING = B8 * 4 + (_BY & 1) * 2 + (_BX & 1)

ORC_NSTATS = 17
STAT_NAMES = ["luma bS1", "luma bS2", "luma bS3", "luma bS4", "chroma bS1", "chroma bS2", "chroma bS3", "chroma bS4",
              "strong", "strong ap", "strong aq", "lt4 ap", "lt4 aq", "off idc1", "off idc2", "off t8x8", "off border"]
assert len(STAT_NAMES) == ORC_NSTATS


class OrcDbkPic(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("type", "qp", "qp_c", "nnz", "t8x8", "ref0", "mv0", "ref1", "mv1", "slice", "idc",
                                          "off_a", "off_b")] + [("compare_refs", C.c_int32)]


def strides(mb_w):
    """the product's plane layout (enc_host.h): luma / chroma strides, sample (0, 0) after 32 / 16 samples of padding"""
    return 16 * mb_w + 64, 8 * mb_w + 32


class Picture:
    """one random picture: padded planes (y, cb, cr as flat uint8 arrays), the device records and the oracle's arrays"""

    def plane_shapes(self):
        sy, sc = strides(self.mb_w)
        return [(16 * self.mb_h + 64) * sy, (8 * self.mb_h + 32) * sc, (8 * self.mb_h + 32) * sc]

    def origin(self, pl):
        sy, sc = strides(self.mb_w)
        return 32 * sy + 32 if pl == 0 else 16 * sc + 16


def _fold(v):
    """reflects a random walk into [0, 255]"""
    v = np.mod(v, 510)
    return 255 - np.abs(v - 255)


def _texture(rng, w, h, blk):
    """smooth blocks of blk x blk samples: block levels from two separable random walks plus jitter, mostly small steps,
    some large ones; inside a block a small gradient and +-1 noise, or flat"""
    gw, gh = w // blk, h // blk

    def walk(n):
        kind = rng.rand(n)
        step = np.where(kind < 0.7, rng.normal(0, 5, n), np.where(kind < 0.9, rng.uniform(-30, 30, n), rng.uniform(-110, 110, n)))
        step[kind > 0.96] = 0
        return np.cumsum(step)
    base = 128 + walk(gh)[:, None] + walk(gw)[None, :] + rng.normal(0, 2, (gh, gw))
    base = np.where(rng.rand(gh, gw) < 0.05, rng.uniform(0, 255, (gh, gw)), base)
    base = _fold(base)
    flat = rng.rand(gh, gw) < 0.2
    gx = np.where(flat, 0, rng.randint(-2, 3, (gh, gw)))
    gy = np.where(flat, 0, rng.randint(-2, 3, (gh, gw)))
    yy, xx = np.mgrid[0:h, 0:w]
    by, bx = yy // blk, xx // blk
    off = (xx % blk - (blk - 1) / 2.0) * gx[by, bx] + (yy % blk - (blk - 1) / 2.0) * gy[by, bx]
    noise = np.where(flat[by, bx], 0, rng.randint(-1, 2, (h, w)))
    return np.clip(np.rint(base[by, bx] + off + noise), 0, 255).astype(np.uint8)


def _qp(rng):
    return int(rng.randint(20, 46)) if rng.rand() < 0.85 else int(rng.randint(0, 52))


def random_picture(seed, mb_w, mb_h, mode, t8=False, n_slices=1, skip_frac=0.0, idc=None, enc_ctl=None):
    """mode: "enc" (encoder records, one reference, per-picture control), "dec_p" (decoded P picture, reference pictures
    compared), "dec_b" (decoded B picture: intra, B and B_Skip macroblocks, list-1 records).  t8: macroblocks with the 8x8
    transform (decoder modes).  n_slices: slices of the decoded picture, each with its own idc 0 / 1 / 2 and offsets.
    skip_frac: share of macroblocks that are P_Skip / B_Skip with the picture's common motion and no coefficients (all-zero
    strengths between them).  idc: force one disable_deblocking_filter_idc on every slice.  enc_ctl: the encoder's
    (idc, FilterOffsetA, FilterOffsetB) for the picture (random when None; one launch of the device filter shares it)."""
    rng = np.random.RandomState(seed)
    orc = h264lib.oracle()
    n = mb_w * mb_h
    p = Picture()
    p.mb_w, p.mb_h, p.mode, p.dec_mode = mb_w, mb_h, mode, 0 if mode == "enc" else 1
    sy, sc = strides(mb_w)
    # planes: the padding carries random bytes that must come back untouched
    p.planes = [rng.randint(0, 256, s).astype(np.uint8) for s in p.plane_shapes()]
    for pl, (w, h, st) in enumerate([(16 * mb_w, 16 * mb_h, sy), (8 * mb_w, 8 * mb_h, sc), (8 * mb_w, 8 * mb_h, sc)]):
        view = p.planes[pl][p.origin(pl):p.origin(pl) + h * st].reshape(h, st)
        view[:, :w] = _texture(rng, w, h, 4 if pl == 0 else 2)
    cqp_off = int(rng.randint(-12, 13))
    # slices: contiguous macroblock runs with their own control (encoder: one per picture)
    cuts = np.sort(rng.choice(np.arange(1, n), min(n_slices, n) - 1, replace=False)) if n > 1 and n_slices > 1 else []
    slice_of = np.searchsorted(np.asarray(cuts, np.int64), np.arange(n), side="right").astype(np.int32)
    n_sl = int(slice_of.max()) + 1
    if p.dec_mode:
        s_idc = rng.choice([0, 0, 1, 2, 2], n_sl) if idc is None else np.full(n_sl, idc)
    else:
        s_idc = np.full(n_sl, rng.choice([0, 0, 0, 1]) if idc is None else idc)
    s_a = 2 * rng.randint(-6, 7, n_sl)
    s_b = 2 * rng.randint(-6, 7, n_sl)
    if enc_ctl is not None and not p.dec_mode:
        s_idc, s_a, s_b = (np.full(n_sl, v) for v in enc_ctl)
    p.enc_ctl = (int(s_idc[0]), int(s_a[0]), int(s_b[0])) if not p.dec_mode else (0, 0, 0)
    base_mv = rng.randint(-40, 41, 2)
    n_refs = 1 if mode == "enc" else 3

    typ = np.zeros(n, np.int32)
    qp, qp_c, t8x8 = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.int32)
    nnz = np.zeros((n, 16), np.int32)
    ref0, ref1 = np.full((n, 16), -1, np.int32), np.full((n, 16), -1, np.int32)
    mv0, mv1 = np.zeros((n, 16, 2), np.int32), np.zeros((n, 16, 2), np.int32)
    mbi = np.zeros(n, MBINFO)
    auxb = None
    if mode == "dec_b":
        auxb = np.frombuffer(rng.randint(0, 256, n * AUXB.itemsize).astype(np.uint8).tobytes(), AUXB).copy()   # non-B: never read
    raw = np.frombuffer(rng.randint(0, 256, n * MBINFO.itemsize).astype(np.uint8).tobytes(), MBINFO)
    mbi[:] = raw                                     # fields the filter does not read keep random bytes

    def vec():
        d = rng.choice([0, 0, 1, -1, 2, -3, 3, 4, -4, 5, 7]) if rng.rand() < 0.85 else rng.randint(-64, 65)
        return base_mv + np.array([d if rng.rand() < 0.5 else 0, d if rng.rand() < 0.5 else 0]) + (rng.rand() < 0.1) * rng.randint(-3, 4, 2)

    def per8x8(values):                              # 4 per-8x8 values -> 16 raster blocks
        return np.asarray(values)[B8]

    for i in range(n):
        skip = rng.rand() < skip_frac
        if mode == "enc":
            t = PSKIP if skip else rng.choice([I4x4, I16x16, P16x16, P16x8, P8x16, P8x8, PSKIP, P16x16, P8x8, PSKIP])
        elif mode == "dec_p":
            t = PSKIP if skip else rng.choice([I4x4, I16x16, IPCM, P16x16, P16x8, P8x16, P8x8, P8x8, PSKIP, PSKIP])
        else:
            t = BSKIP if skip else rng.choice([I4x4, I16x16, IPCM, B, B, B, B, BSKIP, BSKIP])
        typ[i] = t
        qp[i] = 0 if t == IPCM else (_qp(rng) if rng.rand() < 0.7 or i == 0 else qp[i - 1])
        qp_c[i] = orc.chroma_qp(min(51, max(0, qp[i] + cqp_off)))
        t8x8[i] = 1 if t8 and t in (I4x4, P16x16, P16x8, P8x16, P8x8, B) and rng.rand() < 0.5 else 0
        if t in (PSKIP, BSKIP) or skip:
            pass                                      # no coefficients
        elif t8x8[i]:
            nnz[i] = per8x8(np.where(rng.rand(4) < 0.35, rng.randint(1, 17, 4), 0))
        else:
            nnz[i] = np.where(rng.rand(16) < 0.3, rng.randint(1, 17, 16), 0)
        if t in INTRA:
            continue
        # motion: a partition pattern, one vector per partition; 4x4 partitions only without the 8x8 transform
        if skip:
            parts = np.zeros(16, np.int64)
        elif t == PSKIP:
            parts = np.zeros(16, np.int64)
        elif t in (BSKIP,) or t8x8[i]:
            parts = [np.zeros(16, np.int64), _BY >> 1, _BX >> 1, B8][rng.randint(4)]
        else:
            parts = [np.zeros(16, np.int64), _BY >> 1, _BX >> 1, B8, np.arange(16)][rng.randint(5)]
        npart = int(parts.max()) + 1
        if skip:
            v0 = np.tile(base_mv, (npart, 1))
        else:
            v0 = np.array([vec() for _ in range(npart)])
        mv0[i] = v0[parts]
        if mode != "dec_b":
            r = 0 if (n_refs == 1 or skip) else int(rng.choice([0, 0, 0, 1, 2]))
            r8 = [r] * 4 if t == PSKIP or skip else [0 if n_refs == 1 else int(rng.choice([0, 0, 0, 1, 2])) for _ in range(4)]
            if npart == 1 or t == PSKIP:
                r8 = [r8[0]] * 4
            ref0[i] = per8x8(r8)
        else:
            # per 8x8: list 0 only, list 1 only or both; pictures from one id space (the same picture may sit in both lists)
            if skip:
                use = [3] * 4
                r0, r1 = [0] * 4, [1] * 4
            else:
                use = rng.choice([1, 2, 3], 4)
                r0 = [int(rng.choice([0, 0, 1, 2])) for _ in range(4)]
                r1 = [int(rng.choice([1, 1, 0, 2])) for _ in range(4)]
                if npart == 1:
                    use, r0, r1 = [use[0]] * 4, [r0[0]] * 4, [r1[0]] * 4
            ref0[i] = per8x8([r0[k] if use[k] & 1 else -1 for k in range(4)])
            ref1[i] = per8x8([r1[k] if use[k] & 2 else -1 for k in range(4)])
            v1 = np.tile(base_mv, (npart, 1)) if skip else np.array([vec() for _ in range(npart)])
            mv1[i] = v1[parts]
            mv1[i][ref1[i] < 0] = 0
            # the device record carries whatever vector an unused list has; the filter must ignore it
            mv0_dev = np.where((ref0[i] < 0)[:, None], rng.randint(-300, 300, (16, 2)), mv0[i])
            mv0[i][ref0[i] < 0] = 0
            auxb["ref_idx"][i] = [ref1[i][[0, 2, 8, 10][k]] for k in range(4)]
            mvc = np.zeros((16, 2), np.int64)
            mvc[CODING] = np.where((ref1[i] < 0)[:, None], rng.randint(-300, 300, (16, 2)), mv1[i])
            auxb["mv"][i] = mvc
            mbi["mv"][i] = mv0_dev
    # the device records
    mbi["mb_type"] = typ
    mbi["qp"], mbi["qp_c"], mbi["t8x8"] = qp, qp_c, t8x8
    mbi["nnz"][:, :16] = nnz
    for i in range(n):
        if typ[i] in INTRA:
            mbi["i4_mode"][i] = rng.randint(0, 9, 16)
            continue
        if mode != "dec_b":
            mbi["mv"][i] = mv0[i]
        if p.dec_mode:
            mbi["i4_mode"][i] = ref0[i]               # decoder: the list-0 reference picture of every 4x4 block
    if p.dec_mode:
        mbi["p16x16_mv"][:, 0] = slice_of
        mbi["p16x16_mv"][:, 1] = (s_idc | (s_a + 16) << 2 | (s_b + 16) << 7)[slice_of].astype(np.int16)
    p.mbi, p.auxb = mbi, auxb
    p.orc = dict(type=typ, qp=qp, qp_c=qp_c, nnz=nnz, t8x8=t8x8, ref0=ref0, mv0=mv0.reshape(n, 32),
                 ref1=ref1 if mode == "dec_b" else None, mv1=mv1.reshape(n, 32) if mode == "dec_b" else None,
                 slice=slice_of if p.dec_mode else np.zeros(n, np.int32),
                 idc=s_idc[slice_of].astype(np.int32), off_a=s_a[slice_of].astype(np.int32), off_b=s_b[slice_of].astype(np.int32))
    p.compare_refs = p.dec_mode
    return p


def oracle_deblock(p, stats=None):
    """the picture's planes after oracle/orc_deblock_picture; stats (int32[ORC_NSTATS]) is added to"""
    orc = h264lib.oracle()
    fn = orc.lib.orc_deblock_picture
    fn.restype = None
    fn.argtypes = [C.c_void_p] * 3 + [C.c_int] * 4 + [C.POINTER(OrcDbkPic), C.c_void_p]
    keep = {k: (None if v is None else np.ascontiguousarray(v, np.int32)) for k, v in p.orc.items()}
    d = OrcDbkPic(*[None if keep[k] is None else keep[k].ctypes.data for k in
                    ("type", "qp", "qp_c", "nnz", "t8x8", "ref0", "mv0", "ref1", "mv1", "slice", "idc", "off_a", "off_b")],
                  p.compare_refs)
    out = [a.copy() for a in p.planes]
    sy, sc = strides(p.mb_w)
    if stats is None:
        stats = np.zeros(ORC_NSTATS, np.int32)
    fn(*[out[pl].ctypes.data + p.origin(pl) for pl in range(3)], sy, sc, p.mb_w, p.mb_h, C.byref(d), stats.ctypes.data)
    return out


def emu_deblock(p):
    """the picture's planes after the host build of the device filter (deblock_frame_host)"""
    out = [a.copy() for a in p.planes]
    mbi = p.mbi.copy()
    auxb = None if p.auxb is None else p.auxb.copy()
    sy, sc = strides(p.mb_w)
    rc = h264lib.emu().emu_deblock_picture(*[out[pl].ctypes.data + p.origin(pl) for pl in range(3)], sy, sc, p.mb_w, p.mb_h,
                                   mbi.ctypes.data, None if auxb is None else auxb.ctypes.data, p.dec_mode, *p.enc_ctl)
    assert rc == 0
    return out
