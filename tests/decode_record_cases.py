"""Seeded, conforming records for the decoder's construct stage (dec_mb.cuh), for tests/test_decode_records_emu.py and
tests/test_gpu_decode_records.py.  A case is one picture: its macroblock records in the decoder's formats (enc_types.h),
its chroma QP offset and its reference pictures.  The records are drawn in raster order, and each macroblock is run through
the oracle (mb_recon_oracle) as soon as it is drawn, so that the next one can ask what its neighbours left:

- intra modes are drawn among those whose samples exist, and coded as prev / rem flags against the predicted mode;
- levels are drawn small, then one block per macroblock is pushed to the largest level the 16-bit constraints of 8.5.10 to
  8.5.13 allow (binary search on the oracle's checks), so every class reaches the bound;
- vectors are drawn up to +-2048 horizontal and +-512 vertical quarter samples, far beyond the 32-sample pad at every edge.

Classes (CLASSES): Intra_8x8, Intra_4x4 DDL / VL without a top-right neighbour, Intra_16x16 and chroma, QP sweeps, I_PCM,
P partitions and sub-partitions with 1..4 reference slots, P and B with the 8x8 transform, B / weighted records, a
1920x1088 picture (the coded size of a 1080-line stream; nothing is cropped here) whose vectors point past its edges, and
Intra_8x8 blocks placed behind constrained-intra neighbours so that every availability pattern that can occur does, with
every mode it allows.

Weights follow 7.4.3.2 (each in -128..127, and w0 + w1 in -128..128, ..127 at logWD 7), so every record is conforming."""
import numpy as np

import mb_recon_oracle as orc

CLASSES = ["i8x8", "i4x4_tr", "i16", "qp", "ipcm", "p", "p_t8", "b_t8", "b", "hd", "i8x8_nb"]
# Availability patterns of an Intra_8x8 block (L 1, T 2, TL 4, TR 8) that can occur.  Block 0 takes its top-right samples from
# the top macroblock (TR = T): 0, 1, 4, 5, 10, 11, 14, 15; block 1 always has its left, its top-left comes with its top: 1, 7,
# 9, 15; block 2 has top and top-right, its top-left comes with its left: 10, 15; block 3 has no top-right: 7.  The other six
# of the 16 combinations cannot occur.
I8X8_PATTERNS = [0, 1, 4, 5, 7, 9, 10, 11, 14, 15]
# (pattern, a mode it allows) for the class i8x8_nb, one per case
I8X8_COMBOS = [(pat, mode) for pat in I8X8_PATTERNS for mode in range(9)
               if mode == 2 or (mode in (0, 3, 7) and pat & 2) or (mode in (1, 8) and pat & 1) or (mode in (4, 5, 6) and pat & 7 == 7)]
SIZES = [(1, 1), (1, 4), (4, 1), (4, 3), (3, 2), (2, 3)]


class Case:
    def __init__(self, cls, seed, mb_w, mb_h, n_refs, cqp_off):
        self.cls, self.seed, self.mb_w, self.mb_h, self.n_refs, self.cqp_off = cls, seed, mb_w, mb_h, n_refs, cqp_off
        n = mb_w * mb_h
        self.recs = np.zeros(n, orc.MBOUT)
        self.aux = np.zeros(n, orc.DECAUX)
        self.aux_b = np.zeros(n, orc.DECAUXB)
        self.refs = []
        self.stats = {"bound": 0, "i8x8": set()}

    @property
    def has_b(self):
        return bool(np.isin(self.recs["mb_type"], (orc.B, orc.BSKIP)).any())

    def dense_refs(self):
        """the reference pictures as the hooks take them: per slot Y, Cb, Cr back to back"""
        return np.concatenate([np.concatenate([p.reshape(-1) for p in r]) for r in self.refs]).astype(np.uint8)

    def oracle(self):
        return orc.reconstruct(self.mb_w, self.mb_h, self.recs, self.aux, self.aux_b, self.cqp_off, self.refs)


def _texture(rng, h, w):
    y, x = np.mgrid[0:h, 0:w]
    v = rng.randint(30, 220) + rng.uniform(-3, 3) * x + rng.uniform(-3, 3) * y + rng.randint(-20, 21, (h, w))
    if rng.rand() < 0.5:
        v = np.where(((x // rng.randint(2, 9)) + (y // rng.randint(2, 9))) % 2 == 0, v, v + rng.randint(-90, 90))
    return np.clip(v, 0, 255).astype(np.int64)


def _push(rng, lv, positions, ok):
    """set one level at a random position of `positions` to the largest magnitude (up to 2^15 - 1) that ok() accepts; returns
    True when the bound was reached below the level syntax's own limit"""
    pos = positions[rng.randint(len(positions))]
    sign = 1 if rng.rand() < 0.5 else -1
    lo, hi = 0, 32767
    lv[pos] = 0
    if not ok():
        return False
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lv[pos] = sign * mid
        if ok():
            lo = mid
        else:
            hi = mid - 1
    lv[pos] = sign * lo
    return lo < 32767


def _ok(f):
    try:
        f()
        return True
    except orc.NotConforming:
        return False


def _small_levels(rng, n, density):
    lv = np.zeros(n, np.int64)
    on = rng.rand(n) < density
    lv[on] = rng.choice([-3, -2, -1, 1, 1, 2, 3, 5, -7, 12], on.sum())
    return lv


class Gen:
    def __init__(self, case, rng, cip=False, slices=1):
        self.c, self.rng = case, rng
        c = case
        for _ in range(c.n_refs):
            c.refs.append([_texture(rng, 16 * c.mb_h, 16 * c.mb_w), _texture(rng, 8 * c.mb_h, 8 * c.mb_w), _texture(rng, 8 * c.mb_h, 8 * c.mb_w)])
        n = c.mb_w * c.mb_h
        starts = sorted(set([0] + list(rng.choice(np.arange(1, n), min(slices - 1, n - 1), replace=False)) if n > 1 else [0]))
        self.slice = np.searchsorted(starts, np.arange(n), side="right") - 1
        for i in range(n):
            x, y = i % c.mb_w, i // c.mb_w
            av = 0
            for bit, ok, j in ((orc.NB_LEFT, x > 0, i - 1), (orc.NB_TOP, y > 0, i - c.mb_w), (orc.NB_TOPLEFT, x > 0 and y > 0, i - c.mb_w - 1),
                               (orc.NB_TOPRIGHT, y > 0 and x < c.mb_w - 1, i - c.mb_w + 1)):
                if ok and self.slice[j] == self.slice[i]:
                    av |= bit
            a = c.aux[i]
            a["avail"], a["slice"], a["flags"] = av, self.slice[i], orc.DECAUX_CIP if cip else 0
            a["dbk_idc"], a["alpha_off"], a["beta_off"] = rng.randint(3), 2 * rng.randint(-6, 7), 2 * rng.randint(-6, 7)
        self.pic = orc.Picture(c.mb_w, c.mb_h, c.recs, c.aux, c.aux_b, c.cqp_off, c.refs)

    # ---- helpers ----------------------------------------------------------------------------------------------------------
    def avail(self, mbx, mby, x, y):
        """intra sample availability at (x, y) relative to the macroblock, for a block whose earlier blocks are decoded"""
        if 0 <= x < 16 and 0 <= y < 16:
            return True
        return self.pic.nb_mb(mbx, mby, x, y, True) is not None

    def intra_modes(self, mbx, mby, bx, by, size):
        x, y = 4 * bx, 4 * by
        L, T, TL = self.avail(mbx, mby, x - 1, y), self.avail(mbx, mby, x, y - 1), self.avail(mbx, mby, x - 1, y - 1)
        TR = self.avail(mbx, mby, x + size, y - 1) and not (0 <= x + size < 16 and 0 <= y - 1 < 16 and not _done_before(bx, by, size))
        modes = [2] + ([0, 3, 7] if T else []) + ([1, 8] if L else []) + ([4, 5, 6] if T and L and TL else [])
        return modes, (1 if L else 0) | (2 if T else 0) | (4 if TL else 0) | (8 if TR else 0)

    def code_mode(self, m, k, mode, pm):
        m["prev_i4_flag"][k] = 1 if mode == pm else 0
        m["rem_i4_mode"][k] = 0 if mode == pm else (mode if mode < pm else mode - 1)

    def commit(self, mbx, mby, redraw):
        """reconstruct the macroblock with the oracle; while it breaks a constraint, halve its levels and try again"""
        i = mby * self.c.mb_w + mbx
        for _ in range(20):
            try:
                self.pic.mb(mbx, mby)
                return
            except orc.NotConforming:
                m = self.c.recs[i]
                if m["mb_type"] == orc.IPCM:
                    raise
                for f in ("luma", "luma_dc", "chroma_dc", "chroma_ac"):
                    m[f] = m[f] // 2
                redraw()
        raise AssertionError("no conforming levels found")

    # ---- residual ---------------------------------------------------------------------------------------------------------
    def residual(self, m, qp, t8, i16, density=0.15):
        rng = self.rng
        cbp_l = 15 if i16 and rng.rand() < 0.7 else (0 if i16 else rng.randint(16))
        cbp_c = rng.randint(3)
        m["cbp"] = cbp_l | (cbp_c << 4)
        qpc = orc.chroma_qp(qp, self.c.cqp_off)
        for k in range(16):
            if cbp_l & (1 << (k >> 2)):
                m["luma"][k] = _small_levels(rng, 16, density) * (np.arange(16) < (15 if i16 else 16))
        if i16:
            m["luma_dc"] = _small_levels(rng, 16, density)
        if cbp_c:
            m["chroma_dc"] = _small_levels(rng, 8, 0.5).reshape(2, 4)
        if cbp_c == 2:
            for j in range(8):
                m["chroma_ac"][j] = _small_levels(rng, 16, density) * (np.arange(16) < 15)
        # one block pushed to the 16-bit bound
        choice = rng.randint(3)
        pushed = False
        if choice == 0 and i16:
            lv = m["luma_dc"].astype(np.int64)
            pushed = _push(rng, lv, list(range(16)), lambda: _ok(lambda: orc.luma_dc(lv, qp)))
            m["luma_dc"] = lv
        elif choice == 1 and cbp_c:
            uv = rng.randint(2)
            lv = m["chroma_dc"][uv].astype(np.int64)
            pushed = _push(rng, lv, list(range(4)), lambda: _ok(lambda: orc.chroma_dc(lv, qpc)))
            m["chroma_dc"][uv] = lv
        elif cbp_l and not i16:
            k8 = [k for k in range(4) if cbp_l & (1 << k)][rng.randint(bin(cbp_l).count("1"))]
            if t8:
                lv = m["luma"][4 * k8:4 * k8 + 4].reshape(-1).astype(np.int64)
                pushed = _push(rng, lv, list(range(64)), lambda: _ok(lambda: orc.residual8(lv, qp)))
                m["luma"][4 * k8:4 * k8 + 4] = lv.reshape(4, 16)
            else:
                k = 4 * k8 + rng.randint(4)
                lv = m["luma"][k].astype(np.int64)
                pushed = _push(rng, lv, list(range(16)), lambda: _ok(lambda: orc.residual4(lv, qp)))
                m["luma"][k] = lv
        self.c.stats["bound"] += int(pushed)
        for k in range(16):                                  # nnz as the parser leaves it (raster), per 4x4 block of levels
            bx, by = orc.blk_xy(k)
            m["nnz"][by * 4 + bx] = int((m["luma"][k] != 0).sum()) if cbp_l & (1 << (k >> 2)) else 0
        for j in range(8):
            m["nnz"][16 + j] = int((m["chroma_ac"][j] != 0).sum()) if cbp_c == 2 else 0

    # ---- macroblock kinds -------------------------------------------------------------------------------------------------
    def intra_nxn(self, mbx, mby, qp, t8, prefer=None, force=None):
        i = mby * self.c.mb_w + mbx
        m, a = self.c.recs[i], self.c.aux[i]

        def draw():
            own = [None] * 16
            if t8:
                a["flags"] |= orc.DECAUX_T8
                for k in range(4):
                    bx, by = (k & 1) * 2, (k >> 1) * 2
                    modes, pat = self.intra_modes(mbx, mby, bx, by, 8)
                    fresh = [md for md in modes if (md, pat) not in self.c.stats["i8x8"]]     # modes this pattern has not had yet
                    pool = fresh if fresh and self.rng.rand() < 0.8 else modes
                    mode = pool[self.rng.randint(len(pool))]
                    if force is not None and force[0] == k:      # (block, mode): the block must see force[2] as its pattern
                        assert force[1] in modes and force[2] == pat, (force, pat)
                        mode = force[1]
                    self.code_mode(m, k, mode, self.pic.pred_mode(mbx, mby, bx, by, own))
                    for cc in (0, 1, 4, 5):
                        own[by * 4 + bx + cc] = mode
                    self.c.stats["i8x8"].add((mode, pat))
                    self.c.stats.setdefault("i8x8_blocks", []).append(pat)
            else:
                for k in range(16):
                    bx, by = orc.blk_xy(k)
                    modes, pat = self.intra_modes(mbx, mby, bx, by, 4)
                    pick = [md for md in modes if md in (3, 7)] if prefer == "ddl_vl" and not pat & 8 else []
                    pool = pick or modes
                    mode = pool[self.rng.randint(len(pool))]
                    self.code_mode(m, k, mode, self.pic.pred_mode(mbx, mby, bx, by, own))
                    own[by * 4 + bx] = mode
                    if prefer == "ddl_vl" and mode in (3, 7) and not pat & 8:
                        self.c.stats.setdefault("tr_blocks", set()).add(k)
        m["mb_type"], m["qp"] = orc.I4x4, qp
        self.chroma_mode(mbx, mby, m)
        self.residual(m, qp, t8, False)
        draw()
        self.commit(mbx, mby, lambda: None)

    def chroma_mode(self, mbx, mby, m):
        L, T, TL = self.avail(mbx, mby, -1, 0), self.avail(mbx, mby, 0, -1), self.avail(mbx, mby, -1, -1)
        modes = [0] + ([1] if L else []) + ([2] if T else []) + ([3] if L and T and TL else [])
        m["chroma_mode"] = modes[self.rng.randint(len(modes))]

    def intra16(self, mbx, mby, qp):
        i = mby * self.c.mb_w + mbx
        m = self.c.recs[i]
        L, T, TL = self.avail(mbx, mby, -1, 0), self.avail(mbx, mby, 0, -1), self.avail(mbx, mby, -1, -1)
        modes = [2] + ([0] if T else []) + ([1] if L else []) + ([3] if L and T and TL else [])
        m["mb_type"], m["qp"], m["i16_mode"] = orc.I16x16, qp, modes[self.rng.randint(len(modes))]
        self.chroma_mode(mbx, mby, m)
        self.residual(m, qp, False, True)
        self.commit(mbx, mby, lambda: None)

    def ipcm(self, mbx, mby):
        i = mby * self.c.mb_w + mbx
        m = self.c.recs[i]
        m["mb_type"], m["cbp"], m["qp"] = orc.IPCM, 0x2F, 0
        m["nnz"] = 16
        raw = self.rng.randint(0, 256, 512).astype(np.uint8)
        m["luma"] = np.frombuffer(np.concatenate([raw[:256], np.zeros(256, np.uint8)]).tobytes(), np.int16).reshape(16, 16)
        m["chroma_ac"] = np.frombuffer(np.concatenate([raw[256:384], np.zeros(128, np.uint8)]).tobytes(), np.int16).reshape(8, 16)
        self.commit(mbx, mby, lambda: None)

    def vector(self, mbx, mby, x, y, far):
        """a target vector: mostly near, sometimes up to the level limits, pointing out of the picture where it can"""
        rng = self.rng
        if not far or rng.rand() < 0.4:
            return rng.randint(-64, 65), rng.randint(-48, 49)
        W, H = 16 * self.c.mb_w, 16 * self.c.mb_h
        X, Y = 16 * mbx + x, 16 * mby + y
        vx = rng.choice([-2048, 2047, rng.randint(-4 * (X + 40), -4 * X + 1), rng.randint(4 * (W - X), 4 * (W - X + 40) + 1)])
        vy = rng.choice([-512, 511, rng.randint(-4 * (Y + 40), -4 * Y + 1), rng.randint(4 * (H - Y), 4 * (H - Y + 40) + 1)])
        return int(np.clip(vx, -2048, 2047)), int(np.clip(vy, -512, 511))

    def p_mb(self, mbx, mby, qp, t8, kinds=(orc.P16x16, orc.P16x8, orc.P8x16, orc.P8x8, orc.PSKIP), far=True):
        rng, c = self.rng, self.c
        i = mby * c.mb_w + mbx
        m, a = c.recs[i], c.aux[i]
        t = kinds[rng.randint(len(kinds))]
        m["mb_type"], m["qp"] = t, qp
        sub = t == orc.P8x8 and rng.rand() < 0.7 and not t8
        if sub:
            a["flags"] |= orc.DECAUX_SUB
            a["sub_type"] = rng.randint(0, 4, 4)
        if t8 and t != orc.PSKIP:
            a["flags"] |= orc.DECAUX_T8
        refs = rng.randint(0, c.n_refs, 4)
        if t == orc.PSKIP:
            refs[:] = rng.randint(0, c.n_refs)
        elif t == orc.P16x16:
            refs[:] = refs[0]
        elif t == orc.P16x8:
            refs[1], refs[3] = refs[0], refs[2]
        elif t == orc.P8x16:
            refs[2], refs[3] = refs[0], refs[1]
        a["ref_idx"] = refs
        # differences against the predictor the oracle derives: draw target vectors, decode once with zero differences to
        # learn the predictors partition by partition (each prediction depends on the previous partitions' final vectors)
        if t != orc.PSKIP:
            self._p_vectors(mbx, mby, m, a, t, sub, far)
            self.residual(m, qp, t8, False)
        self.commit(mbx, mby, lambda: None)

    def _p_vectors(self, mbx, mby, m, a, t, sub, far):
        parts = []
        if sub:
            for k in range(4):
                st = int(a["sub_type"][k])
                w, h = (8, 8) if st == 0 else (8, 4) if st == 1 else (4, 8) if st == 2 else (4, 4)
                for j in range(1 if st == 0 else 4 if st == 3 else 2):
                    x = (k & 1) * 8 + (0 if st in (0, 1) else (j & 1) * 4)
                    y = (k >> 1) * 8 + (j * 4 if st == 1 else (j >> 1) * 4 if st == 3 else 0)
                    parts.append(("aux", 4 * k + j, x, y))
        else:
            geo = {orc.P16x16: [(0, 0)], orc.P16x8: [(0, 0), (0, 8)], orc.P8x16: [(0, 0), (8, 0)], orc.P8x8: [(0, 0), (8, 0), (0, 8), (8, 8)]}[t]
            parts = [("rec", n, x, y) for n, (x, y) in enumerate(geo)]
        for n, (where, idx, x, y) in enumerate(parts):
            tgt = self.vector(mbx, mby, x, y, far)
            # the predictor of this partition: decode with this difference zero, read the final vector of its first cell
            if where == "aux":
                a["mvd"][idx] = (0, 0)
            else:
                m["mvd"][idx] = (0, 0)
            self.pic.mb(mbx, mby)
            p = self.pic.mbi[mby * self.c.mb_w + mbx]["mv"][(y // 4) * 4 + x // 4]
            d = (int(np.clip(tgt[0] - int(p[0]), -4096, 4095)), int(np.clip(tgt[1] - int(p[1]), -1024, 1023)))
            if where == "aux":
                a["mvd"][idx] = d
            else:
                m["mvd"][idx] = d

    def b_mb(self, mbx, mby, qp, t8, halves=True):
        rng, c = self.rng, self.c
        i = mby * c.mb_w + mbx
        m, a, ab = c.recs[i], c.aux[i], c.aux_b[i]
        m["mb_type"], m["qp"] = (orc.BSKIP if rng.rand() < 0.2 else orc.B), qp
        if t8:
            a["flags"] |= orc.DECAUX_T8
        ld_y, ld_c = rng.randint(0, 8), rng.randint(0, 8)
        a["wp_log2"] = ld_y | (ld_c << 4)
        for k in range(4):
            pred = [orc.DECB_L0, orc.DECB_L1, orc.DECB_L0 | orc.DECB_L1][rng.randint(3)]
            two = pred == orc.DECB_L0 | orc.DECB_L1
            style = rng.randint(3)
            if two:
                pred |= orc.DECB_BI
            elif style == 1:
                pred |= orc.DECB_WEIGHT
                if halves and rng.rand() < 0.4:
                    pred |= [orc.DECB_LOWER, orc.DECB_RIGHT][rng.randint(2)]
            elif style == 2:
                pred |= orc.DECB_BI                       # one list through the two-list formula (buffer 0 twice)
            ab["pred"][k] = pred
            a["ref_idx"][k] = rng.randint(c.n_refs) if pred & orc.DECB_L0 else -1
            ab["ref_idx"][k] = rng.randint(c.n_refs) if pred & orc.DECB_L1 else -1
            same = rng.rand() < 0.5
            v0, v1 = self.vector(mbx, mby, (k & 1) * 8, (k >> 1) * 8, True), self.vector(mbx, mby, (k & 1) * 8, (k >> 1) * 8, True)
            for j in range(4):
                if not same:
                    v0, v1 = self.vector(mbx, mby, (k & 1) * 8, (k >> 1) * 8, True), self.vector(mbx, mby, (k & 1) * 8, (k >> 1) * 8, True)
                a["mvd"][4 * k + j] = v0 if pred & orc.DECB_L0 else (0, 0)
                ab["mv"][4 * k + j] = v1 if pred & orc.DECB_L1 else (0, 0)
        for e in range(12):
            ld = ld_c if e >= 4 else ld_y
            if rng.rand() < 0.3:                        # default: ld 0 with 1 / 1, or the implicit form
                ab["w0"][e], ab["w1"][e], ab["o"][e] = 1, 1, 0
            else:                                       # 7.4.3.2: -128 <= w0 + w1 <= (logWD == 7 ? 127 : 128)
                w0 = rng.randint(-128, 128)
                w1 = rng.randint(max(-128, -128 - w0), min(127, (127 if ld == 7 else 128) - w0) + 1)
                ab["w0"][e], ab["w1"][e] = w0, w1
                ab["o"][e] = rng.randint(-128, 128)
        if m["mb_type"] == orc.B:
            self.residual(m, qp, t8, False)
        self.commit(mbx, mby, lambda: None)


def _done_before(bx, by, size):
    """is the block at the top-right of the size x size block at (bx, by) (4x4 units) decoded before it"""
    if size == 8:
        return (bx, by) == (0, 2)
    k = [kk for kk in range(16) if orc.blk_xy(kk) == (bx, by)][0]
    tx, ty = bx + 1, by - 1
    kt = [kk for kk in range(16) if orc.blk_xy(kk) == (tx, ty)]
    return bool(kt) and kt[0] < k


def make(cls, seed):
    """one case of class `cls`"""
    rng = np.random.RandomState(seed)
    mb_w, mb_h = SIZES[seed % len(SIZES)]
    cqp = [-12, 0, 12][rng.randint(3)]
    n_refs = 1 + rng.randint(4) if cls in ("p", "p_t8", "b", "b_t8") else 1
    if cls == "hd":
        mb_w, mb_h = 120, 68
    if cls == "i8x8_nb":
        return _i8x8_behind(rng, seed, cqp)
    c = Case(cls, seed, mb_w, mb_h, n_refs, cqp)
    g = Gen(c, rng, cip=cls in ("i8x8", "i4x4_tr", "i16") and rng.rand() < 0.5, slices=1 + rng.randint(3) if cls != "hd" else 1)
    qp_list = [0, 5, 6, 11, 12, 35, 36, 51]
    for mby in range(mb_h):
        for mbx in range(mb_w):
            i = mby * mb_w + mbx
            qp = int(rng.randint(0, 52))
            if cls == "i8x8":
                r = rng.rand()
                if r < 0.7:
                    g.intra_nxn(mbx, mby, qp, True)
                elif r < 0.8:
                    g.intra_nxn(mbx, mby, qp, False)
                else:
                    g.p_mb(mbx, mby, qp, False, far=False)
            elif cls == "i4x4_tr":
                if rng.rand() < 0.85:
                    g.intra_nxn(mbx, mby, qp, False, prefer="ddl_vl")
                else:
                    g.p_mb(mbx, mby, qp, False, far=False)
            elif cls == "i16":
                if rng.rand() < 0.75:
                    g.intra16(mbx, mby, [0, 5, 6, 11, 12, 13, 26, 51][rng.randint(8)])
                else:
                    g.p_mb(mbx, mby, qp, False, far=False)
            elif cls == "qp":
                qp = int(qp_list[(seed + i) % len(qp_list)] if rng.rand() < 0.5 else (seed * 7 + i * 3) % 52)
                r = rng.randint(4)
                if r == 0:
                    g.intra16(mbx, mby, qp)
                elif r == 1:
                    g.intra_nxn(mbx, mby, qp, rng.rand() < 0.5)
                else:
                    g.p_mb(mbx, mby, qp, rng.rand() < 0.5, kinds=(orc.P16x16, orc.P8x8), far=False)
            elif cls == "ipcm":
                if rng.rand() < 0.5:
                    g.ipcm(mbx, mby)
                else:
                    [lambda: g.intra16(mbx, mby, qp), lambda: g.intra_nxn(mbx, mby, qp, rng.rand() < 0.5),
                     lambda: g.p_mb(mbx, mby, qp, False, far=False)][rng.randint(3)]()
            elif cls == "p":
                g.p_mb(mbx, mby, qp, False)
            elif cls == "p_t8":
                g.p_mb(mbx, mby, qp, rng.rand() < 0.8, kinds=(orc.P16x16, orc.P16x8, orc.P8x16, orc.P8x8))
            elif cls in ("b", "b_t8"):
                if rng.rand() < 0.85:
                    g.b_mb(mbx, mby, qp, cls == "b_t8" and rng.rand() < 0.8)
                else:
                    g.intra_nxn(mbx, mby, qp, cls == "b_t8")
            else:                                            # hd: cheap inter macroblocks, vectors past the edges near them
                edge = mbx in (0, mb_w - 1) or mby in (0, mb_h - 1)
                g.p_mb(mbx, mby, 26, False, kinds=(orc.P16x16, orc.PSKIP) if not edge else (orc.P16x16, orc.P8x8), far=edge)
    return c


def _i8x8_behind(rng, seed, cqp):
    """3 x 2 macroblocks under constrained intra prediction: each neighbour of macroblock (1, 1) is intra or P as the pattern of
    I8X8_COMBOS[seed % 1000] needs, so that its block 0 (patterns with TR = T) or its block 1 (patterns 7 and 9) sees exactly
    that pattern and is predicted with the combination's mode"""
    pat, mode = I8X8_COMBOS[seed % 1000]
    c = Case("i8x8_nb", seed, 3, 2, 1, cqp)
    g = Gen(c, rng, cip=True, slices=1)
    if pat in (7, 9):                           # block 1: top-left and top from the top macroblock, top-right from its own
        k, intra = 1, {orc.NB_TOP: pat == 7, orc.NB_TOPRIGHT: pat == 9, orc.NB_TOPLEFT: rng.rand() < 0.5, orc.NB_LEFT: rng.rand() < 0.5}
    else:                                       # block 0: top-right from the top macroblock
        k, intra = 0, {orc.NB_TOP: bool(pat & 2), orc.NB_TOPRIGHT: rng.rand() < 0.5, orc.NB_TOPLEFT: bool(pat & 4), orc.NB_LEFT: bool(pat & 1)}
    for (mbx, mby), bit in (((0, 0), orc.NB_TOPLEFT), ((1, 0), orc.NB_TOP), ((2, 0), orc.NB_TOPRIGHT), ((0, 1), orc.NB_LEFT)):
        qp = int(rng.randint(0, 52))
        if not intra[bit]:
            g.p_mb(mbx, mby, qp, False, far=False)
        elif rng.rand() < 0.5:
            g.intra16(mbx, mby, qp)
        else:
            g.intra_nxn(mbx, mby, qp, rng.rand() < 0.5)
    g.intra_nxn(1, 1, int(rng.randint(0, 52)), True, force=(k, mode, pat))
    g.intra_nxn(2, 1, int(rng.randint(0, 52)), True)
    return c


def cases(per_class=None):
    """(class, seed) of the standard set"""
    n = {"i8x8": 96, "i4x4_tr": 10, "i16": 10, "qp": 32, "ipcm": 6, "p": 16, "p_t8": 10, "b_t8": 8, "b": 12, "hd": 1,
         "i8x8_nb": len(I8X8_COMBOS)}
    if per_class:
        n = dict((k, min(v, per_class)) for k, v in n.items())
    return [(cls, 1000 * (CLASSES.index(cls) + 1) + s) for cls in CLASSES for s in range(n[cls])]
