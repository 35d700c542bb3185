"""Plain oracle of one picture's macroblock reconstruction, written from Rec. ITU-T H.264 (8.3 intra prediction, 8.4 inter
prediction, 8.5 scaling and transforms; 8-bit 4:2:0 frames, flat scaling lists).  Python integers throughout, no 16-bit
wrap: every intermediate value that 8.5.10 to 8.5.13 bound ("the bitstream shall not contain data that result in ...
exceeds the range -2^15 .. 2^15 - 1") is asserted, so a record outside that range is refused here instead of being
reconstructed.  Slower than the kernel by orders of magnitude, and meant to be read.

The input is the decoder's own record formats (enc_types.h): per macroblock an MbOut, a DecMbAux and, for B macroblocks, a
DecMbAuxB, plus the chroma QP offset and the reference pictures (unpadded planes, indexed by picture slot).  Neighbour
availability comes from DecMbAux.avail, so slice boundaries are whatever the records say.  Reference indices are picture
slots (the parser resolves RefPicList0 to slots); vector prediction compares them as 8.4.1.3 compares refIdxL0.

The output is the unfiltered picture and, per macroblock, the MbInfo record that deblocking and the neighbours read."""
import numpy as np

# ---- record layouts (enc_types.h) ---------------------------------------------------------------------------------------
MBOUT = np.dtype([("mb_type", "u1"), ("cbp", "u1"), ("qp", "u1"), ("i16_mode", "u1"), ("chroma_mode", "u1"), ("pad0", "u1", 3),
                  ("prev_i4_flag", "i1", 16), ("rem_i4_mode", "i1", 16), ("mvd", "<i2", (4, 2)), ("nnz", "i1", 24),
                  ("luma_dc", "<i2", 16), ("luma", "<i2", (16, 16)), ("chroma_dc", "<i2", (2, 4)), ("chroma_ac", "<i2", (8, 16))])
DECAUX = np.dtype([("avail", "u1"), ("flags", "u1"), ("dbk_idc", "u1"), ("alpha_off", "i1"), ("beta_off", "i1"), ("wp_log2", "u1"),
                   ("slice", "<u2"), ("sub_type", "u1", 4), ("ref_idx", "i1", 4), ("mvd", "<i2", (16, 2))])
DECAUXB = np.dtype([("ref_idx", "i1", 4), ("o", "i1", 12), ("mv", "<i2", (16, 2)), ("w0", "<i2", 12), ("w1", "<i2", 12), ("pred", "u1", 4)])
MBINFO = np.dtype([("mv", "<i2", (16, 2)), ("nnz", "i1", 24), ("i4_mode", "i1", 16), ("p16x16_mv", "<i2", 2), ("sad_cost", "<i4"),
                   ("mb_type", "u1"), ("cbp", "u1"), ("qp", "u1"), ("qp_c", "u1"), ("ref_idx", "i1"), ("t8x8", "u1"), ("pad", "u1", 2)])
assert (MBOUT.itemsize, DECAUX.itemsize, DECAUXB.itemsize, MBINFO.itemsize) == (896, 80, 132, 120)

I4x4, I16x16, P16x16, P16x8, P8x16, P8x8, PSKIP, IPCM, B, BSKIP = range(10)     # MbOut.mb_type (MBT_*)
NB_LEFT, NB_TOP, NB_TOPLEFT, NB_TOPRIGHT = 1, 2, 4, 8
DECAUX_SUB, DECAUX_CIP, DECAUX_T8 = 1, 2, 4
DECB_L0, DECB_L1, DECB_WEIGHT, DECB_BI, DECB_LOWER, DECB_RIGHT = 1, 2, 4, 8, 16, 32


def is_intra(t):
    return t in (I4x4, I16x16, IPCM)


def is_inter(t):
    return not is_intra(t)


class NotConforming(AssertionError):
    """the record breaks a constraint the standard puts on conforming bitstreams"""


def chk(v, what):
    if not -32768 <= v <= 32767:
        raise NotConforming(f"{what} = {v} outside the 16-bit range")
    return v


def clip1(v):
    return 0 if v < 0 else 255 if v > 255 else v


def clip3(lo, hi, v):
    return lo if v < lo else hi if v > hi else v


# ---- 8.5.6 / 8.5.7: inverse scans (frame macroblocks) --------------------------------------------------------------------
ZIGZAG4 = [0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15]            # Table 8-13: scan index -> raster position
ZIGZAG8 = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
           35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63]


def blk_xy(k):
    """4x4 block k in decoding order (6.4.3) -> (x, y) in 4-sample units"""
    return (k & 1) | ((k >> 1) & 2), ((k >> 1) & 1) | ((k >> 2) & 2)


# ---- 8.5.8 / 8.5.9: quantisation parameters and level scales -------------------------------------------------------------
QPC = list(range(30)) + [29, 30, 31, 32, 32, 33, 34, 34, 35, 35, 36, 36, 37, 37, 37, 38, 38, 38, 39, 39, 39, 39]   # Table 8-15
V4 = [[10, 16, 13], [11, 18, 14], [13, 20, 16], [14, 23, 18], [16, 25, 20], [18, 29, 23]]
V8 = [[20, 18, 32, 19, 25, 24], [22, 19, 35, 21, 28, 26], [26, 23, 42, 24, 33, 31], [28, 25, 45, 26, 35, 33], [32, 28, 51, 30, 40, 38],
      [36, 32, 58, 34, 46, 43]]


def chroma_qp(qp, off):
    return QPC[clip3(0, 51, qp + off)]


def level_scale4(m, i, j):          # flat weightScale4x4 (16) x normAdjust4x4 (8-315)
    return 16 * (V4[m][0] if i % 2 == 0 and j % 2 == 0 else V4[m][1] if i % 2 == 1 and j % 2 == 1 else V4[m][2])


def level_scale8(m, i, j):          # flat weightScale8x8 (16) x normAdjust8x8 (8-318)
    if i % 4 == 0 and j % 4 == 0:
        k = 0
    elif i % 2 == 1 and j % 2 == 1:
        k = 1
    elif i % 4 == 2 and j % 4 == 2:
        k = 2
    elif (i % 4 == 0 and j % 2 == 1) or (i % 2 == 1 and j % 4 == 0):
        k = 3
    elif (i % 4 == 0 and j % 4 == 2) or (i % 4 == 2 and j % 4 == 0):
        k = 4
    else:
        k = 5
    return 16 * V8[m][k]


def scale4(c, qp, skip_dc=False):
    """8.5.12.1: c[i][j] (i row) -> d; skip_dc leaves d00 to the caller (Intra16x16 / chroma: already scaled DC)"""
    d = [[0] * 4 for _ in range(4)]
    for i in range(4):
        for j in range(4):
            if skip_dc and i == 0 and j == 0:
                d[i][j] = c[i][j]
            elif qp >= 24:
                d[i][j] = (c[i][j] * level_scale4(qp % 6, i, j)) << (qp // 6 - 4)
            else:
                d[i][j] = (c[i][j] * level_scale4(qp % 6, i, j) + (1 << (3 - qp // 6))) >> (4 - qp // 6)
            chk(d[i][j], "8.5.12.1 d")
    return d


def scale8(c, qp):
    """8.5.13.1"""
    d = [[0] * 8 for _ in range(8)]
    for i in range(8):
        for j in range(8):
            if qp >= 36:
                d[i][j] = (c[i][j] * level_scale8(qp % 6, i, j)) << (qp // 6 - 6)
            else:
                d[i][j] = (c[i][j] * level_scale8(qp % 6, i, j) + (1 << (5 - qp // 6))) >> (6 - qp // 6)
            chk(d[i][j], "8.5.13.1 d")
    return d


def idct4(d):
    """8.5.12.2: residual r[i][j] (row i) of scaled coefficients d"""
    def one(v, what):
        e0, e1 = chk(v[0] + v[2], what), chk(v[0] - v[2], what)
        e2, e3 = chk((v[1] >> 1) - v[3], what), chk(v[1] + (v[3] >> 1), what)
        return [chk(e0 + e3, what), chk(e1 + e2, what), chk(e1 - e2, what), chk(e0 - e3, what)]
    f = [one(d[i], "8.5.12.2 e/f") for i in range(4)]
    h = [one([f[i][j] for i in range(4)], "8.5.12.2 g/h") for j in range(4)]     # h[j][i]: column j
    return [[(h[j][i] + 32) >> 6 for j in range(4)] for i in range(4)]


def idct8(d):
    """8.5.13.2"""
    def one(v, what):
        a0, a4 = v[0] + v[4], v[0] - v[4]
        a2, a6 = (v[2] >> 1) - v[6], v[2] + (v[6] >> 1)
        b0, b2, b4, b6 = a0 + a6, a4 + a2, a4 - a2, a0 - a6
        a1 = -v[3] + v[5] - v[7] - (v[7] >> 1)
        a3 = v[1] + v[7] - v[3] - (v[3] >> 1)
        a5 = -v[1] + v[7] + v[5] + (v[5] >> 1)
        a7 = v[3] + v[5] + v[1] + (v[1] >> 1)
        b1, b7 = a1 + (a7 >> 2), a7 - (a1 >> 2)
        b3, b5 = a3 + (a5 >> 2), (a3 >> 2) - a5
        for x in (a0, a4, a2, a6, b0, b2, b4, b6, a1, a3, a5, a7, b1, b7, b3, b5):
            chk(x, what)
        return [chk(x, what) for x in (b0 + b7, b2 + b5, b4 + b3, b6 + b1, b6 - b1, b4 - b3, b2 - b5, b0 - b7)]
    g = [one(d[i], "8.5.13.2 rows") for i in range(8)]
    m = [one([g[i][j] for i in range(8)], "8.5.13.2 columns") for j in range(8)]
    return [[(m[j][i] + 32) >> 6 for j in range(8)] for i in range(8)]


def luma_dc(levels, qp):
    """8.5.10: Intra16x16 DC levels (scan order) -> dcY[i][j] of the 4x4 array of blocks"""
    c = [[0] * 4 for _ in range(4)]
    for k in range(16):
        c[ZIGZAG4[k] // 4][ZIGZAG4[k] % 4] = int(levels[k])
    H = [[1, 1, 1, 1], [1, 1, -1, -1], [1, -1, -1, 1], [1, -1, 1, -1]]
    t = [[sum(H[i][k] * c[k][j] for k in range(4)) for j in range(4)] for i in range(4)]
    f = [[chk(sum(t[i][k] * H[k][j] for k in range(4)), "8.5.10 f") for j in range(4)] for i in range(4)]
    ls = level_scale4(qp % 6, 0, 0)
    if qp >= 36:
        return [[chk((f[i][j] * ls) << (qp // 6 - 6), "8.5.10 dcY") for j in range(4)] for i in range(4)]
    return [[chk((f[i][j] * ls + (1 << (5 - qp // 6))) >> (6 - qp // 6), "8.5.10 dcY") for j in range(4)] for i in range(4)]


def chroma_dc(levels, qpc):
    """8.5.11 (4:2:0): chroma DC levels c0..c3 (raster of the 2x2) -> dcC per 4x4 block (raster)"""
    c = [[int(levels[0]), int(levels[1])], [int(levels[2]), int(levels[3])]]
    f = [[chk(c[0][0] + c[0][1] + c[1][0] + c[1][1], "8.5.11.1 f"), chk(c[0][0] - c[0][1] + c[1][0] - c[1][1], "8.5.11.1 f")],
         [chk(c[0][0] + c[0][1] - c[1][0] - c[1][1], "8.5.11.1 f"), chk(c[0][0] - c[0][1] - c[1][0] + c[1][1], "8.5.11.1 f")]]
    ls = level_scale4(qpc % 6, 0, 0)
    return [chk(((f[i][j] * ls) << (qpc // 6)) >> 5, "8.5.11.2 dcC") for i in range(2) for j in range(2)]


def residual4(levels, qp, first=0, dc=None):
    """one 4x4 block: levels in scan order (first = 1: AC only, levels[0] is scan position 1), dc = scaled DC or None"""
    c = [[0] * 4 for _ in range(4)]
    for k in range(16 - first):
        pos = ZIGZAG4[k + first]
        c[pos // 4][pos % 4] = int(levels[k])
    if dc is not None:
        c[0][0] = dc
    return idct4(scale4(c, qp, skip_dc=dc is not None))


def residual8(levels, qp):
    c = [[0] * 8 for _ in range(8)]
    for k in range(64):
        c[ZIGZAG8[k] // 8][ZIGZAG8[k] % 8] = int(levels[k])
    return idct8(scale8(c, qp))


# ---- the picture ---------------------------------------------------------------------------------------------------------
class Picture:
    def __init__(self, mb_w, mb_h, recs, aux, aux_b, cqp_off, refs):
        self.mb_w, self.mb_h = mb_w, mb_h
        self.recs, self.aux, self.aux_b, self.cqp_off = recs, aux, aux_b, cqp_off
        self.refs = [[np.asarray(p, np.int64) for p in r] for r in refs]
        self.pl = [np.zeros((16 * mb_h, 16 * mb_w), np.int64), np.zeros((8 * mb_h, 8 * mb_w), np.int64),
                   np.zeros((8 * mb_h, 8 * mb_w), np.int64)]
        self.mbi = np.zeros(mb_w * mb_h, MBINFO)
        self.modes = {}            # mb index -> 16 intra prediction modes (raster 4x4 cells; an Intra_8x8 mode fills its four)
        self.mvs = {}              # mb index -> (16 (mvx, mvy) raster, 16 ref slots raster) of list 0, inter macroblocks

    # 6.4.12: the macroblock holding luma location (x, y) relative to the current one, and whether it is available
    def nb_mb(self, mbx, mby, x, y, for_intra):
        a = self.aux[mby * self.mb_w + mbx]
        if 0 <= x < 16 and 0 <= y < 16:
            return mby * self.mb_w + mbx
        if x < 0 and y < 0:
            bit, n = NB_TOPLEFT, (mby - 1) * self.mb_w + mbx - 1
        elif x < 0 and 0 <= y < 16:
            bit, n = NB_LEFT, mby * self.mb_w + mbx - 1
        elif 0 <= x < 16 and y < 0:
            bit, n = NB_TOP, (mby - 1) * self.mb_w + mbx
        elif x > 15 and y < 0:
            bit, n = NB_TOPRIGHT, (mby - 1) * self.mb_w + mbx + 1
        else:
            return None
        if not (a["avail"] & bit):
            return None
        # constrained_intra_pred_flag: Inter macroblocks do not count for intra prediction (8.3.1.2, 8.3.1.1, 8.3.2, 8.3.3, 8.3.4)
        if for_intra and (a["flags"] & DECAUX_CIP) and is_inter(int(self.recs[n]["mb_type"])):
            return None
        return n

    def intra_sample(self, mbx, mby, done, x, y, chroma=False):
        """neighbouring sample for intra prediction or None.  (x, y) relative to the macroblock in the plane's units; `done`:
        the 4x4 (luma) cells of the current macroblock reconstructed so far"""
        s = 2 if chroma else 1
        n = self.nb_mb(mbx, mby, x * s, y * s, True)
        if n is None:
            return None
        if n == mby * self.mb_w + mbx and not chroma and not done[(y // 4) * 4 + x // 4]:
            return None                           # inside the macroblock, not yet decoded (luma4x4BlkIdx 3, 11, ...)
        w = 8 if chroma else 16
        return int(self.cur_plane[(mby * w) + y, (mbx * w) + x])

    # 8.3.1.1 / 8.3.2.1: predicted Intra4x4 / Intra8x8 mode of the cell at 4x4 position (bx, by)
    def pred_mode(self, mbx, mby, bx, by, own):
        res = []
        for dx, dy in ((-1, 0), (0, -1)):
            x, y = bx * 4 + dx, by * 4 + dy
            n = self.nb_mb(mbx, mby, x, y, True)
            if n is None:
                return 2                          # dcPredModePredictedFlag
            cur = mby * self.mb_w + mbx
            if n == cur:
                res.append(own[(y // 4) * 4 + x // 4])
            elif int(self.recs[n]["mb_type"]) == I4x4:
                res.append(self.modes[n][((y % 16) // 4) * 4 + (x % 16) // 4])
            else:
                res.append(2)
        return min(res)

    def run(self):
        for mby in range(self.mb_h):
            for mbx in range(self.mb_w):
                self.mb(mbx, mby)
        return [p.astype(np.uint8) for p in self.pl], self.mbi

    def put(self, pl, x0, y0, block):
        for y, row in enumerate(block):
            for x, v in enumerate(row):
                self.pl[pl][y0 + y, x0 + x] = v

    def mb(self, mbx, mby):
        i = mby * self.mb_w + mbx
        m, a = self.recs[i], self.aux[i]
        t, qp = int(m["mb_type"]), int(m["qp"])
        off = int(self.cqp_off)
        info = self.mbi[i]
        info["mb_type"], info["cbp"] = t, m["cbp"]
        info["nnz"] = m["nnz"]
        info["ref_idx"] = 0 if is_inter(t) else -1
        info["p16x16_mv"] = (int(a["slice"]), int(a["dbk_idc"]) | ((int(a["alpha_off"]) + 16) << 2) | ((int(a["beta_off"]) + 16) << 7))
        X, Y = 16 * mbx, 16 * mby
        if t == IPCM:                              # 8.3.5: the samples as they are; QP'Y 0 for the filter
            raw = m["luma"].reshape(-1).view(np.uint8)
            self.pl[0][Y:Y + 16, X:X + 16] = raw[:256].reshape(16, 16)
            rc = m["chroma_ac"].reshape(-1).view(np.uint8)
            self.pl[1][Y // 2:Y // 2 + 8, X // 2:X // 2 + 8] = rc[:64].reshape(8, 8)
            self.pl[2][Y // 2:Y // 2 + 8, X // 2:X // 2 + 8] = rc[64:128].reshape(8, 8)
            info["qp"], info["qp_c"] = 0, chroma_qp(0, off)
            return
        qpc = chroma_qp(qp, off)
        info["qp"], info["qp_c"] = qp, qpc
        t8 = bool(a["flags"] & DECAUX_T8)
        cbp = int(m["cbp"])
        if t == I4x4 and t8:
            self.intra8x8(mbx, mby, m, qp)
        elif t == I4x4:
            self.intra4x4(mbx, mby, m, qp)
        elif t == I16x16:
            self.intra16x16(mbx, mby, m, qp)
        else:
            pred_y, pred_c = self.inter_pred(mbx, mby, m, a, info)
            if t8:
                for k in range(4):
                    ox, oy = (k & 1) * 8, (k >> 1) * 8
                    r = residual8(m["luma"][4 * k:4 * k + 4].reshape(-1), qp) if cbp & (1 << k) else [[0] * 8 for _ in range(8)]
                    self.put(0, X + ox, Y + oy, [[clip1(int(pred_y[oy + y, ox + x]) + r[y][x]) for x in range(8)] for y in range(8)])
            else:
                for k in range(16):
                    bx, by = blk_xy(k)
                    r = residual4(m["luma"][k], qp) if cbp & (1 << (k >> 2)) else [[0] * 4 for _ in range(4)]
                    self.put(0, X + 4 * bx, Y + 4 * by,
                             [[clip1(int(pred_y[4 * by + y, 4 * bx + x]) + r[y][x]) for x in range(4)] for y in range(4)])
        if t8:                                     # MbInfo: the filter asks per 8x8 transform block (nnz summed, capped at 64)
            info["t8x8"] = 1
            for k in range(4):
                b0 = (k >> 1) * 8 + (k & 1) * 2
                tot = sum(int(info["nnz"][b]) for b in (b0, b0 + 1, b0 + 4, b0 + 5))
                for b in (b0, b0 + 1, b0 + 4, b0 + 5):
                    info["nnz"][b] = min(tot, 64)
        if is_intra(t):
            pred_c = self.intra_chroma(mbx, mby, m)
        # chroma residual (8.5.11), both planes
        cbp_c = cbp >> 4
        for uv in range(2):
            dcc = chroma_dc(m["chroma_dc"][uv], qpc) if cbp_c else [0, 0, 0, 0]
            for j in range(4):
                ox, oy = (j & 1) * 4, (j >> 1) * 4
                if cbp_c == 2:
                    r = residual4(m["chroma_ac"][4 * uv + j], qpc, first=1, dc=dcc[j])
                else:
                    r = residual4([0] * 16, qpc, dc=dcc[j])
                self.put(1 + uv, X // 2 + ox, Y // 2 + oy,
                         [[clip1(int(pred_c[uv][oy + y, ox + x]) + r[y][x]) for x in range(4)] for y in range(4)])

    # ---- intra ------------------------------------------------------------------------------------------------------------
    @property
    def cur_plane(self):
        return self._cur

    def samples(self, mbx, mby, done, pl=0):
        self._cur = self.pl[pl]
        return lambda x, y: self.intra_sample(mbx, mby, done, x, y, chroma=pl > 0)

    def intra4x4(self, mbx, mby, m, qp):
        i = mby * self.mb_w + mbx
        own, done = [None] * 16, [False] * 16
        self.modes[i] = own
        cbp = int(m["cbp"])
        for k in range(16):
            bx, by = blk_xy(k)
            pm = self.pred_mode(mbx, mby, bx, by, own)
            rem = int(m["rem_i4_mode"][k])
            mode = pm if m["prev_i4_flag"][k] else (rem if rem < pm else rem + 1)
            own[by * 4 + bx] = mode
            S = self.samples(mbx, mby, done)
            p = {}
            for x in range(-1, 8):
                p[(x, -1)] = S(4 * bx + x, 4 * by - 1)
            for y in range(4):
                p[(-1, y)] = S(4 * bx - 1, 4 * by + y)
            if all(p[(x, -1)] is None for x in range(4, 8)) and p[(3, -1)] is not None:   # 8.3.1.2
                for x in range(4, 8):
                    p[(x, -1)] = p[(3, -1)]
            pred = pred4x4(p, mode)
            r = residual4(m["luma"][k], qp) if cbp & (1 << (k >> 2)) else [[0] * 4 for _ in range(4)]
            self.put(0, 16 * mbx + 4 * bx, 16 * mby + 4 * by, [[clip1(pred[y][x] + r[y][x]) for x in range(4)] for y in range(4)])
            done[by * 4 + bx] = True
        self.mbi[i]["i4_mode"] = own

    def intra8x8(self, mbx, mby, m, qp):
        i = mby * self.mb_w + mbx
        own, done = [None] * 16, [False] * 16
        self.modes[i] = own
        cbp = int(m["cbp"])
        for k in range(4):
            bx, by = (k & 1) * 2, (k >> 1) * 2
            pm = self.pred_mode(mbx, mby, bx, by, own)
            rem = int(m["rem_i4_mode"][k])
            mode = pm if m["prev_i4_flag"][k] else (rem if rem < pm else rem + 1)
            for c in (0, 1, 4, 5):
                own[by * 4 + bx + c] = mode
            S = self.samples(mbx, mby, done)
            p = {}
            for x in range(-1, 16):
                p[(x, -1)] = S(4 * bx + x, 4 * by - 1)
            for y in range(8):
                p[(-1, y)] = S(4 * bx - 1, 4 * by + y)
            if all(p[(x, -1)] is None for x in range(8, 16)) and p[(7, -1)] is not None:   # 8.3.2.2
                for x in range(8, 16):
                    p[(x, -1)] = p[(7, -1)]
            pred = pred8x8(filter8x8(p), mode)
            r = residual8(m["luma"][4 * k:4 * k + 4].reshape(-1), qp) if cbp & (1 << k) else [[0] * 8 for _ in range(8)]
            self.put(0, 16 * mbx + 4 * bx, 16 * mby + 4 * by, [[clip1(pred[y][x] + r[y][x]) for x in range(8)] for y in range(8)])
            for c in (0, 1, 4, 5):
                done[by * 4 + bx + c] = True
        self.mbi[i]["i4_mode"] = own

    def intra16x16(self, mbx, mby, m, qp):
        S = self.samples(mbx, mby, [False] * 16)
        top = [S(x, -1) for x in range(16)]
        left = [S(-1, y) for y in range(16)]
        tl = S(-1, -1)
        mode = int(m["i16_mode"])
        T, L = top[0] is not None, left[0] is not None
        if mode == 0:
            assert T, "Intra_16x16 vertical without the top samples"
            pred = [[top[x] for x in range(16)] for y in range(16)]
        elif mode == 1:
            assert L, "Intra_16x16 horizontal without the left samples"
            pred = [[left[y]] * 16 for y in range(16)]
        elif mode == 2:
            dc = (sum(top) + sum(left) + 16) >> 5 if T and L else (sum(left) + 8) >> 4 if L else (sum(top) + 8) >> 4 if T else 128
            pred = [[dc] * 16 for _ in range(16)]
        else:
            assert T and L and tl is not None, "Intra_16x16 plane without all neighbours"
            pt = lambda x: tl if x < 0 else top[x]
            plft = lambda y: tl if y < 0 else left[y]
            H = sum((x + 1) * (pt(8 + x) - pt(6 - x)) for x in range(8))
            V = sum((y + 1) * (plft(8 + y) - plft(6 - y)) for y in range(8))
            a, b, c = 16 * (left[15] + top[15]), (5 * H + 32) >> 6, (5 * V + 32) >> 6
            pred = [[clip1((a + b * (x - 7) + c * (y - 7) + 16) >> 5) for x in range(16)] for y in range(16)]
        dcy = luma_dc(m["luma_dc"], qp)
        cbp = int(m["cbp"])
        for k in range(16):
            bx, by = blk_xy(k)
            lv = m["luma"][k] if cbp & 15 else np.zeros(16, np.int16)
            r = residual4(lv, qp, first=1, dc=dcy[by][bx])
            self.put(0, 16 * mbx + 4 * bx, 16 * mby + 4 * by,
                     [[clip1(pred[4 * by + y][4 * bx + x] + r[y][x]) for x in range(4)] for y in range(4)])

    def intra_chroma(self, mbx, mby, m):
        out = []
        mode = int(m["chroma_mode"])
        for uv in range(2):
            S = self.samples(mbx, mby, None, 1 + uv)
            top = [S(x, -1) for x in range(8)]
            left = [S(-1, y) for y in range(8)]
            tl = S(-1, -1)
            T, L = top[0] is not None, left[0] is not None
            pred = np.zeros((8, 8), np.int64)
            if mode == 0:                        # 8.3.4.1-3: DC per 4x4 chroma block
                for yo in (0, 4):
                    for xo in (0, 4):
                        st, sl = sum(top[xo:xo + 4]) if T else None, sum(left[yo:yo + 4]) if L else None
                        if (xo, yo) == (0, 0) or (xo > 0 and yo > 0):
                            v = (st + sl + 4) >> 3 if T and L else (sl + 2) >> 2 if L else (st + 2) >> 2 if T else 128
                        elif xo > 0:
                            v = (st + 2) >> 2 if T else (sl + 2) >> 2 if L else 128
                        else:
                            v = (sl + 2) >> 2 if L else (st + 2) >> 2 if T else 128
                        pred[yo:yo + 4, xo:xo + 4] = v
            elif mode == 1:
                assert L, "chroma horizontal without the left samples"
                for y in range(8):
                    pred[y, :] = left[y]
            elif mode == 2:
                assert T, "chroma vertical without the top samples"
                for y in range(8):
                    pred[y, :] = top
            else:
                assert T and L and tl is not None, "chroma plane without all neighbours"
                pt = lambda x: tl if x < 0 else top[x]
                plft = lambda y: tl if y < 0 else left[y]
                H = sum((x + 1) * (pt(4 + x) - pt(2 - x)) for x in range(4))
                V = sum((y + 1) * (plft(4 + y) - plft(2 - y)) for y in range(4))
                a, b, c = 16 * (left[7] + top[7]), (34 * H + 32) >> 6, (34 * V + 32) >> 6
                for y in range(8):
                    for x in range(8):
                        pred[y, x] = clip1((a + b * (x - 3) + c * (y - 3) + 16) >> 5)
            out.append(pred)
        return out

    # ---- inter --------------------------------------------------------------------------------------------------------------
    def nb_motion(self, mbx, mby, x, y, own_mv, own_ref):
        """8.4.1.3.2 for the luma location (x, y) relative to the macroblock: None if the partition is not available, else
        (mv, ref) with ref -1 for an intra neighbour.  own_*: the current macroblock's cells decoded so far (None: not yet)"""
        n = self.nb_mb(mbx, mby, x, y, False)
        if n is None:
            return None
        cell = ((y % 16) // 4) * 4 + (x % 16) // 4
        if n == mby * self.mb_w + mbx:
            return None if own_ref[cell] is None else (own_mv[cell], own_ref[cell])
        if n not in self.mvs:
            return ((0, 0), -1)
        mv, ref = self.mvs[n]
        return (mv[cell], ref[cell]) if ref[cell] >= 0 else ((0, 0), -1)

    def mvp(self, mbx, mby, x, y, w, h, ref, shape, own_mv, own_ref):
        A = self.nb_motion(mbx, mby, x - 1, y, own_mv, own_ref)
        B = self.nb_motion(mbx, mby, x, y - 1, own_mv, own_ref)
        Cn = self.nb_motion(mbx, mby, x + w, y - 1, own_mv, own_ref)
        if Cn is None:
            Cn = self.nb_motion(mbx, mby, x - 1, y - 1, own_mv, own_ref)
        un = ((0, 0), -1)
        a, b, c = A or un, B or un, Cn or un
        if shape == "16x8":
            if y == 0 and b[1] == ref:
                return b[0]
            if y == 8 and a[1] == ref:
                return a[0]
        if shape == "8x16":
            if x == 0 and a[1] == ref:
                return a[0]
            if x == 8 and c[1] == ref:
                return c[0]
        if B is None and Cn is None and A is not None:          # 8.4.1.3.1
            b = c = a
        match = [n for n in (a, b, c) if n[1] == ref]
        if len(match) == 1:
            return match[0][0]
        return (sorted([a[0][0], b[0][0], c[0][0]])[1], sorted([a[0][1], b[0][1], c[0][1]])[1])

    def inter_pred(self, mbx, mby, m, a, info):
        t = int(m["mb_type"])
        i = mby * self.mb_w + mbx
        pred_y = np.zeros((16, 16), np.int64)
        pred_c = [np.zeros((8, 8), np.int64), np.zeros((8, 8), np.int64)]
        own_mv, own_ref = [None] * 16, [None] * 16

        def part(x, y, w, h, mv, ref, dst_y=pred_y, dst_c=pred_c):
            dst_y[y:y + h, x:x + w] = luma_mc(self.refs[ref][0], 16 * mbx + x, 16 * mby + y, w, h, mv[0], mv[1])
            for uv in range(2):
                dst_c[uv][y // 2:(y + h) // 2, x // 2:(x + w) // 2] = chroma_mc(self.refs[ref][1 + uv], (16 * mbx + x) // 2, (16 * mby + y) // 2,
                                                                                 w // 2, h // 2, mv[0], mv[1])
            for yy in range(y // 4, (y + h) // 4):
                for xx in range(x // 4, (x + w) // 4):
                    own_mv[yy * 4 + xx], own_ref[yy * 4 + xx] = mv, ref

        if t in (B, BSKIP):
            ab = self.aux_b[i]
            p1y = np.zeros((16, 16), np.int64)
            p1c = [np.zeros((8, 8), np.int64), np.zeros((8, 8), np.int64)]
            for k in range(4):
                pr = int(ab["pred"][k])
                r0 = int(a["ref_idx"][k]) if pr & DECB_L0 else -1
                r1 = int(ab["ref_idx"][k]) if pr & DECB_L1 else -1
                qx, qy = (k & 1) * 8, (k >> 1) * 8
                for j in range(4):
                    x, y = qx + (j & 1) * 4, qy + (j >> 1) * 4
                    if r0 >= 0:
                        part(x, y, 4, 4, tuple(int(v) for v in a["mvd"][4 * k + j]), r0)
                    if r1 >= 0:
                        mv1 = tuple(int(v) for v in ab["mv"][4 * k + j])
                        if r0 >= 0:
                            part(x, y, 4, 4, mv1, r1, p1y, p1c)
                        else:
                            part(x, y, 4, 4, mv1, r1)
                # 8.4.2.3 with the weights the record carries
                if pr & (DECB_WEIGHT | DECB_BI):
                    two = r0 >= 0 and r1 >= 0
                    x0, y0 = (4 if pr & DECB_RIGHT else 0), (4 if pr & DECB_LOWER else 0)
                    for plane in range(3):
                        e = 4 * plane + k
                        ld = (int(a["wp_log2"]) >> (4 if plane else 0)) & 15
                        w0, w1, o = int(ab["w0"][e]), int(ab["w1"][e]), int(ab["o"][e])
                        s = 2 if plane else 1
                        P0 = pred_y if plane == 0 else pred_c[plane - 1]
                        P1 = (p1y if plane == 0 else p1c[plane - 1]) if two else P0
                        for y in range(qy // s, (qy + 8) // s):
                            for x in range(qx // s, (qx + 8) // s):
                                if x * s - qx < x0 or y * s - qy < y0:
                                    continue
                                p0, p1 = int(P0[y, x]), int(P1[y, x])
                                if pr & DECB_BI:
                                    v = ((p0 * w0 + p1 * w1 + (1 << ld)) >> (ld + 1)) + o
                                else:
                                    v = ((p0 * w0 + (1 << (ld - 1))) >> ld) + o if ld >= 1 else p0 * w0 + o
                                P0[y, x] = clip1(v)
            mv_out = [tuple(int(v) for v in a["mvd"][4 * (((b >> 3) << 1) | ((b >> 1) & 1)) + ((b >> 2) & 1) * 2 + (b & 1)])
                      if a["ref_idx"][((b >> 3) << 1) | ((b >> 1) & 1)] >= 0 else (0, 0) for b in range(16)]
        else:
            ref_of = lambda x, y: int(a["ref_idx"][(y // 8) * 2 + x // 8])
            if t == PSKIP:                         # 8.4.1.1
                ref = ref_of(0, 0)
                A = self.nb_motion(mbx, mby, -1, 0, own_mv, own_ref)
                Bn = self.nb_motion(mbx, mby, 0, -1, own_mv, own_ref)
                if A is None or Bn is None or (A[1] == ref and A[0] == (0, 0)) or (Bn[1] == ref and Bn[0] == (0, 0)):
                    mv = (0, 0)
                else:
                    mv = self.mvp(mbx, mby, 0, 0, 16, 16, ref, "16x16", own_mv, own_ref)
                part(0, 0, 16, 16, mv, ref)
            elif t == P8x8 and (a["flags"] & DECAUX_SUB):
                for k in range(4):
                    st = int(a["sub_type"][k])
                    w, h = (8, 8) if st == 0 else (8, 4) if st == 1 else (4, 8) if st == 2 else (4, 4)
                    np_ = 1 if st == 0 else 4 if st == 3 else 2
                    for j in range(np_):
                        x = (k & 1) * 8 + (0 if st == 1 else (j & 1) * 4 if st != 0 else 0)
                        y = (k >> 1) * 8 + (j * 4 if st == 1 else (j >> 1) * 4 if st == 3 else 0)
                        ref = ref_of(x, y)
                        p = self.mvp(mbx, mby, x, y, w, h, ref, "sub", own_mv, own_ref)
                        part(x, y, w, h, (p[0] + int(a["mvd"][4 * k + j][0]), p[1] + int(a["mvd"][4 * k + j][1])), ref)
            else:
                parts = {P16x16: [(0, 0, 16, 16)], P16x8: [(0, 0, 16, 8), (0, 8, 16, 8)], P8x16: [(0, 0, 8, 16), (8, 0, 8, 16)],
                         P8x8: [(0, 0, 8, 8), (8, 0, 8, 8), (0, 8, 8, 8), (8, 8, 8, 8)]}[t]
                shape = {P16x16: "16x16", P16x8: "16x8", P8x16: "8x16", P8x8: "8x8"}[t]
                for n, (x, y, w, h) in enumerate(parts):
                    ref = ref_of(x, y)
                    p = self.mvp(mbx, mby, x, y, w, h, ref, shape, own_mv, own_ref)
                    part(x, y, w, h, (p[0] + int(m["mvd"][n][0]), p[1] + int(m["mvd"][n][1])), ref)
            mv_out = own_mv
        refs = [int(a["ref_idx"][(b >> 3) * 2 + ((b >> 1) & 1)]) for b in range(16)]
        self.mvs[i] = (mv_out, refs)
        info["mv"] = mv_out
        info["i4_mode"] = refs
        return pred_y, pred_c


# ---- 8.3.1.2.x / 8.3.2.2.x: the directional predictors ------------------------------------------------------------------
def pred4x4(p, mode):
    P = lambda x, y: _need(p, x, y, mode, "Intra_4x4")
    out = [[0] * 4 for _ in range(4)]
    T, L = p[(0, -1)] is not None, p[(-1, 0)] is not None
    for y in range(4):
        for x in range(4):
            if mode == 0:
                v = P(x, -1)
            elif mode == 1:
                v = P(-1, y)
            elif mode == 2:
                st, sl = (sum(P(i, -1) for i in range(4)) if T else 0), (sum(P(-1, i) for i in range(4)) if L else 0)
                v = (st + sl + 4) >> 3 if T and L else (sl + 2) >> 2 if L else (st + 2) >> 2 if T else 128
            elif mode == 3:
                v = (P(6, -1) + 3 * P(7, -1) + 2) >> 2 if x == 3 and y == 3 else (P(x + y, -1) + 2 * P(x + y + 1, -1) + P(x + y + 2, -1) + 2) >> 2
            elif mode == 4:
                if x > y:
                    v = (P(x - y - 2, -1) + 2 * P(x - y - 1, -1) + P(x - y, -1) + 2) >> 2
                elif x < y:
                    v = (P(-1, y - x - 2) + 2 * P(-1, y - x - 1) + P(-1, y - x) + 2) >> 2
                else:
                    v = (P(0, -1) + 2 * P(-1, -1) + P(-1, 0) + 2) >> 2
            elif mode == 5:
                z = 2 * x - y
                if z >= 0 and z % 2 == 0:
                    v = (P(x - (y >> 1) - 1, -1) + P(x - (y >> 1), -1) + 1) >> 1
                elif z >= 0:
                    v = (P(x - (y >> 1) - 2, -1) + 2 * P(x - (y >> 1) - 1, -1) + P(x - (y >> 1), -1) + 2) >> 2
                elif z == -1:
                    v = (P(-1, 0) + 2 * P(-1, -1) + P(0, -1) + 2) >> 2
                else:
                    v = (P(-1, y - 1) + 2 * P(-1, y - 2) + P(-1, y - 3) + 2) >> 2
            elif mode == 6:
                z = 2 * y - x
                if z >= 0 and z % 2 == 0:
                    v = (P(-1, y - (x >> 1) - 1) + P(-1, y - (x >> 1)) + 1) >> 1
                elif z >= 0:
                    v = (P(-1, y - (x >> 1) - 2) + 2 * P(-1, y - (x >> 1) - 1) + P(-1, y - (x >> 1)) + 2) >> 2
                elif z == -1:
                    v = (P(-1, 0) + 2 * P(-1, -1) + P(0, -1) + 2) >> 2
                else:
                    v = (P(x - 1, -1) + 2 * P(x - 2, -1) + P(x - 3, -1) + 2) >> 2
            elif mode == 7:
                if y % 2 == 0:
                    v = (P(x + (y >> 1), -1) + P(x + (y >> 1) + 1, -1) + 1) >> 1
                else:
                    v = (P(x + (y >> 1), -1) + 2 * P(x + (y >> 1) + 1, -1) + P(x + (y >> 1) + 2, -1) + 2) >> 2
            else:
                z = x + 2 * y
                if z > 5:
                    v = P(-1, 3)
                elif z == 5:
                    v = (P(-1, 2) + 3 * P(-1, 3) + 2) >> 2
                elif z % 2 == 0:
                    v = (P(-1, y + (x >> 1)) + P(-1, y + (x >> 1) + 1) + 1) >> 1
                else:
                    v = (P(-1, y + (x >> 1)) + 2 * P(-1, y + (x >> 1) + 1) + P(-1, y + (x >> 1) + 2) + 2) >> 2
            out[y][x] = v
    return out


def _need(p, x, y, mode, what):
    v = p[(x, y)]
    if v is None:
        raise NotConforming(f"{what} mode {mode} reads p[{x},{y}], which is not available")
    return v


def filter8x8(p):
    """8.3.2.2.1: reference sample filtering; unavailable samples stay None"""
    q = dict((k, None) for k in p)
    top = all(p[(x, -1)] is not None for x in range(16))
    left = all(p[(-1, y)] is not None for y in range(8))
    c = p[(-1, -1)]
    if top:
        q[(0, -1)] = (c + 2 * p[(0, -1)] + p[(1, -1)] + 2) >> 2 if c is not None else (3 * p[(0, -1)] + p[(1, -1)] + 2) >> 2
        for x in range(1, 15):
            q[(x, -1)] = (p[(x - 1, -1)] + 2 * p[(x, -1)] + p[(x + 1, -1)] + 2) >> 2
        q[(15, -1)] = (p[(14, -1)] + 3 * p[(15, -1)] + 2) >> 2
    if c is not None:
        t0, l0 = p[(0, -1)], p[(-1, 0)]
        if t0 is None or l0 is None:
            q[(-1, -1)] = (3 * c + t0 + 2) >> 2 if t0 is not None else (3 * c + l0 + 2) >> 2 if l0 is not None else c
        else:
            q[(-1, -1)] = (t0 + 2 * c + l0 + 2) >> 2
    if left:
        q[(-1, 0)] = (c + 2 * p[(-1, 0)] + p[(-1, 1)] + 2) >> 2 if c is not None else (3 * p[(-1, 0)] + p[(-1, 1)] + 2) >> 2
        for y in range(1, 7):
            q[(-1, y)] = (p[(-1, y - 1)] + 2 * p[(-1, y)] + p[(-1, y + 1)] + 2) >> 2
        q[(-1, 7)] = (p[(-1, 6)] + 3 * p[(-1, 7)] + 2) >> 2
    return q


def pred8x8(p, mode):
    P = lambda x, y: _need(p, x, y, mode, "Intra_8x8")
    out = [[0] * 8 for _ in range(8)]
    T, L = p[(0, -1)] is not None, p[(-1, 0)] is not None
    for y in range(8):
        for x in range(8):
            if mode == 0:
                v = P(x, -1)
            elif mode == 1:
                v = P(-1, y)
            elif mode == 2:
                st, sl = (sum(P(i, -1) for i in range(8)) if T else 0), (sum(P(-1, i) for i in range(8)) if L else 0)
                v = (st + sl + 8) >> 4 if T and L else (sl + 4) >> 3 if L else (st + 4) >> 3 if T else 128
            elif mode == 3:
                v = (P(14, -1) + 3 * P(15, -1) + 2) >> 2 if x == 7 and y == 7 else (P(x + y, -1) + 2 * P(x + y + 1, -1) + P(x + y + 2, -1) + 2) >> 2
            elif mode == 4:
                if x > y:
                    v = (P(x - y - 2, -1) + 2 * P(x - y - 1, -1) + P(x - y, -1) + 2) >> 2
                elif x < y:
                    v = (P(-1, y - x - 2) + 2 * P(-1, y - x - 1) + P(-1, y - x) + 2) >> 2
                else:
                    v = (P(0, -1) + 2 * P(-1, -1) + P(-1, 0) + 2) >> 2
            elif mode == 5:
                z = 2 * x - y
                if z >= 0 and z % 2 == 0:
                    v = (P(x - (y >> 1) - 1, -1) + P(x - (y >> 1), -1) + 1) >> 1
                elif z >= 0:
                    v = (P(x - (y >> 1) - 2, -1) + 2 * P(x - (y >> 1) - 1, -1) + P(x - (y >> 1), -1) + 2) >> 2
                elif z == -1:
                    v = (P(-1, 0) + 2 * P(-1, -1) + P(0, -1) + 2) >> 2
                else:
                    v = (P(-1, y - 2 * x - 1) + 2 * P(-1, y - 2 * x - 2) + P(-1, y - 2 * x - 3) + 2) >> 2
            elif mode == 6:
                z = 2 * y - x
                if z >= 0 and z % 2 == 0:
                    v = (P(-1, y - (x >> 1) - 1) + P(-1, y - (x >> 1)) + 1) >> 1
                elif z >= 0:
                    v = (P(-1, y - (x >> 1) - 2) + 2 * P(-1, y - (x >> 1) - 1) + P(-1, y - (x >> 1)) + 2) >> 2
                elif z == -1:
                    v = (P(-1, 0) + 2 * P(-1, -1) + P(0, -1) + 2) >> 2
                else:
                    v = (P(x - 2 * y - 1, -1) + 2 * P(x - 2 * y - 2, -1) + P(x - 2 * y - 3, -1) + 2) >> 2
            elif mode == 7:
                if y % 2 == 0:
                    v = (P(x + (y >> 1), -1) + P(x + (y >> 1) + 1, -1) + 1) >> 1
                else:
                    v = (P(x + (y >> 1), -1) + 2 * P(x + (y >> 1) + 1, -1) + P(x + (y >> 1) + 2, -1) + 2) >> 2
            else:
                z = x + 2 * y
                if z > 13:
                    v = P(-1, 7)
                elif z == 13:
                    v = (P(-1, 6) + 3 * P(-1, 7) + 2) >> 2
                elif z % 2 == 0:
                    v = (P(-1, y + (x >> 1)) + P(-1, y + (x >> 1) + 1) + 1) >> 1
                else:
                    v = (P(-1, y + (x >> 1)) + 2 * P(-1, y + (x >> 1) + 1) + P(-1, y + (x >> 1) + 2) + 2) >> 2
            out[y][x] = v
    return out


# ---- 8.4.2.2: fractional sample interpolation, Clip3 on every coordinate ------------------------------------------------
def _taps(a, axis, n):
    s = [slice(None)] * a.ndim
    def at(k):
        s2 = list(s)
        s2[axis] = slice(k, k + n)
        return a[tuple(s2)]
    return at(0) - 5 * at(1) + 20 * at(2) + 20 * at(3) - 5 * at(4) + at(5)


def luma_mc(ref, X, Y, w, h, mvx, mvy):
    """8.4.2.2.1: the w x h prediction of the block at (X, Y) moved by (mvx, mvy) quarter samples"""
    H_, W_ = ref.shape
    xi, yi, xf, yf = X + (mvx >> 2), Y + (mvy >> 2), mvx & 3, mvy & 3
    cols = np.clip(np.arange(xi - 2, xi + w + 4), 0, W_ - 1)
    rows = np.clip(np.arange(yi - 2, yi + h + 4), 0, H_ - 1)
    win = ref[np.ix_(rows, cols)]                     # G(x, y) = win[y + 2, x + 2]
    c1 = lambda v: np.clip(v, 0, 255)
    B1 = _taps(win, 1, w + 1)                         # b1 of (x, row) at [row + 2, x]
    H1 = _taps(win, 0, h + 1)                         # h1 of (col, y) at [y, col + 2]
    J1 = _taps(B1, 0, h)                              # j1 at [y, x]
    G = win[2:2 + h, 2:2 + w]
    b = c1((B1[2:2 + h, 0:w] + 16) >> 5)
    hh = c1((H1[0:h, 2:2 + w] + 16) >> 5)
    j = c1((J1[0:h, 0:w] + 512) >> 10)
    s = c1((B1[3:3 + h, 0:w] + 16) >> 5)
    m = c1((H1[0:h, 3:3 + w] + 16) >> 5)
    avg = lambda p, q: (p + q + 1) >> 1
    table = {(0, 0): G, (0, 1): lambda: avg(G, hh), (0, 2): hh, (0, 3): lambda: avg(win[3:3 + h, 2:2 + w], hh),
             (1, 0): lambda: avg(G, b), (1, 1): lambda: avg(b, hh), (1, 2): lambda: avg(hh, j), (1, 3): lambda: avg(hh, s),
             (2, 0): b, (2, 1): lambda: avg(b, j), (2, 2): j, (2, 3): lambda: avg(j, s),
             (3, 0): lambda: avg(win[2:2 + h, 3:3 + w], b), (3, 1): lambda: avg(b, m), (3, 2): lambda: avg(j, m), (3, 3): lambda: avg(m, s)}
    v = table[(xf, yf)]
    return v() if callable(v) else v


def chroma_mc(ref, Xc, Yc, w, h, mvx, mvy):
    """8.4.2.2.2 (4:2:0 frames: the chroma vector is the luma vector in eighth samples)"""
    H_, W_ = ref.shape
    xi, yi, xf, yf = Xc + (mvx >> 3), Yc + (mvy >> 3), mvx & 7, mvy & 7
    cols = np.clip(np.arange(xi, xi + w + 1), 0, W_ - 1)
    rows = np.clip(np.arange(yi, yi + h + 1), 0, H_ - 1)
    win = ref[np.ix_(rows, cols)]
    A, B_, C_, D = win[:h, :w], win[:h, 1:], win[1:, :w], win[1:, 1:]
    return ((8 - xf) * (8 - yf) * A + xf * (8 - yf) * B_ + (8 - xf) * yf * C_ + xf * yf * D + 32) >> 6


def reconstruct(mb_w, mb_h, recs, aux, aux_b, cqp_off, refs):
    """the unfiltered picture (Y, Cb, Cr as uint8 arrays) and the MbInfo records (MBINFO array) of one picture"""
    return Picture(mb_w, mb_h, recs, aux, aux_b, cqp_off, refs).run()
