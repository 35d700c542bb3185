"""CPU: the decoder's construct stage (dec_one_mb, dec_mb.cuh / dec_t8x8.cuh) in the host build, run in raster order by
emu_decode_records (tests/emu/decode_records_hooks.cu), against the spec oracle (tests/mb_recon_oracle.py) on the seeded
record classes of tests/decode_record_cases.py: Intra_8x8 in every mode at every neighbour pattern that can occur,
Intra_4x4 DDL / VL without a top-right neighbour, Intra_16x16 and chroma, every QP with both transform sizes and chroma
offsets -12 / 0 / 12, I_PCM, P partitions and sub-partitions with 1..4 reference slots, P and B with the 8x8 transform,
weighted B records, and a 1920x1088 picture with vectors past its edges.  Every sample of the padded picture and every MbInfo record must match.
tests/test_gpu_decode_records.py holds the device kernel to the same oracle.  The oracle itself is anchored to the reference
decoder: on seeded random Baseline streams written with the loop filter off it must reproduce the reference's pictures
(skipped where the reference build, oracle/_ref, is absent)."""
import ctypes as C

import numpy as np
import pytest

import decode_record_cases as drc
import h264lib
import mb_recon_oracle as orc

ROOT = h264lib.ROOT
CASES = drc.cases()


@pytest.fixture(scope="module")
def emu():
    return h264lib.emu()


def padded_bytes(mb_w, mb_h):
    sty, stc = 16 * mb_w + 64, 8 * mb_w + 32
    return sty, stc, sty * (16 * mb_h + 64), stc * (8 * mb_h + 32)


def run_hook(fn, cases):
    """one call of emu_decode_records / b2h264_debug_decode_records on the cases (all of one geometry and reference count):
    the padded planes (Y, Cb, Cr) and MbInfo records of each"""
    c0 = cases[0]
    n, n_mb = len(cases), c0.mb_w * c0.mb_h
    sty, stc, yb, cb = padded_bytes(c0.mb_w, c0.mb_h)
    recs = np.concatenate([c.recs for c in cases])
    aux = np.concatenate([c.aux for c in cases])
    aux_b = np.concatenate([c.aux_b for c in cases])
    cq = np.array([c.cqp_off for c in cases], np.int32)
    refs = np.concatenate([c.dense_refs() for c in cases])
    planes = np.zeros(n * (yb + 2 * cb), np.uint8)
    mbi = np.zeros(n * n_mb, orc.MBINFO)
    rc = fn(n, c0.mb_w, c0.mb_h, cq.ctypes.data, recs.ctypes.data, aux.ctypes.data,
            aux_b.ctypes.data if any(c.has_b for c in cases) else None, c0.n_refs, refs.ctypes.data, planes.ctypes.data, mbi.ctypes.data)
    assert rc == 0, rc
    out = []
    for s in range(n):
        p = planes[s * (yb + 2 * cb):(s + 1) * (yb + 2 * cb)]
        out.append(([p[:yb].reshape(-1, sty), p[yb:yb + cb].reshape(-1, stc), p[yb + cb:].reshape(-1, stc)], mbi[s * n_mb:(s + 1) * n_mb]))
    return out


def compare(case, got, want):
    """padded planes against the oracle's picture (interior) and edge replication (border); MbInfo byte for byte"""
    planes, mbi = got
    wp, wmbi = want
    for pl, name in enumerate(("Y", "Cb", "Cr")):
        pad = 16 if pl else 32
        inner = planes[pl][pad:-pad, pad:-pad]
        bad = np.argwhere(inner != wp[pl])
        assert bad.size == 0, (f"{name}: {len(bad)} samples differ, first at (x {bad[0][1]}, y {bad[0][0]}) = macroblock "
                               f"({bad[0][1] // (8 if pl else 16)}, {bad[0][0] // (8 if pl else 16)}): got {inner[tuple(bad[0])]}, "
                               f"want {wp[pl][tuple(bad[0])]}")
        assert np.array_equal(planes[pl], np.pad(wp[pl], pad, mode="edge")), f"{name}: the border is not the edge replicated"
    for i in range(len(wmbi)):
        if mbi[i].tobytes() != wmbi[i].tobytes():
            diff = [f for f in orc.MBINFO.names if not np.array_equal(mbi[i][f], wmbi[i][f])]
            raise AssertionError(f"MbInfo of macroblock {i} (type {case.recs[i]['mb_type']}): fields {diff} differ: "
                                 + "; ".join(f"{f} got {mbi[i][f].tolist()} want {wmbi[i][f].tolist()}" for f in diff))


_made = {}


def make(cls, seed):
    if (cls, seed) not in _made:
        _made[(cls, seed)] = drc.make(cls, seed)
    return _made[(cls, seed)]


@pytest.mark.parametrize("cls,seed", CASES, ids=[f"{c}-{s}" for c, s in CASES])
def test_oracle_matches_host_build(emu, cls, seed):
    case = make(cls, seed)
    compare(case, run_hook(emu.emu_decode_records, [case])[0], case.oracle())


def test_coverage():
    """the set reaches what it is for; the figures are printed (pytest -s) for the record"""
    cs = [make(c, s) for c, s in CASES]
    per_class = dict((cls, sum(1 for c in cs if c.cls == cls)) for cls in drc.CLASSES)
    i8 = set().union(*(c.stats["i8x8"] for c in cs))
    pats = sorted(set(p for _, p in i8))
    q4, q8 = set(), set()                     # QPs that dequantised coded luma levels, per transform size
    for c in cs:
        for m, a in zip(c.recs, c.aux):
            t = int(m["mb_type"])
            if t in (orc.IPCM, orc.PSKIP, orc.BSKIP):
                continue
            coded = any(m["cbp"] & (1 << (k >> 2)) and m["luma"][k].any() for k in range(16))
            if t == orc.I16x16:
                coded = bool(m["luma_dc"].any()) or (bool(m["cbp"] & 15) and bool(m["luma"].any()))
            if coded:
                (q8 if a["flags"] & orc.DECAUX_T8 else q4).add(int(m["qp"]))
    tr = set().union(*(c.stats.get("tr_blocks", set()) for c in cs))
    bound = dict((cls, sum(c.stats["bound"] for c in cs if c.cls == cls)) for cls in drc.CLASSES)
    sides = set()
    for c in cs:
        _, mbi = c.oracle() if c.cls == "hd" or c.mb_w * c.mb_h <= 12 else (None, None)
        if mbi is None:
            continue
        W, H = 16 * c.mb_w, 16 * c.mb_h
        for i in range(c.mb_w * c.mb_h):
            if not orc.is_inter(int(c.recs[i]["mb_type"])):
                continue
            for b in range(16):
                x = 16 * (i % c.mb_w) + 4 * (b & 3) + (int(mbi[i]["mv"][b][0]) >> 2)
                y = 16 * (i // c.mb_w) + 4 * (b >> 2) + (int(mbi[i]["mv"][b][1]) >> 2)
                sides |= {s for s, hit in (("left", x + 4 < -32), ("right", x > W + 32), ("top", y + 4 < -32), ("bottom", y > H + 32)) if hit}
    print(f"\ncases per class: {per_class}\nlevels pushed to the 16-bit bound per class: {bound}\n"
          f"Intra_8x8 availability patterns (L1 T2 TL4 TR8): {pats}; (mode, pattern) pairs {len(i8)} of the {len(drc.I8X8_COMBOS)} that can occur\n"
          f"QPs with 4x4: {len(q4)}, with 8x8: {len(q8)}\nIntra_4x4 DDL/VL blocks without top-right: {sorted(tr)}\n"
          f"vectors beyond the pad: {sorted(sides)}")
    blocks = [p for c in cs for p in c.stats.get("i8x8_blocks", [])]
    print(f"Intra_8x8 blocks per pattern: {dict((p, blocks.count(p)) for p in pats)}")
    missing = [(md, p) for p in drc.I8X8_PATTERNS for md in range(9) if (md, p) not in i8 and _mode_possible(md, p)]
    assert pats == drc.I8X8_PATTERNS, pats
    assert not missing, f"Intra_8x8 (mode, pattern) never drawn: {missing}"
    assert q4 == set(range(52)) and q8 == set(range(52)), (sorted(set(range(52)) - q4), sorted(set(range(52)) - q8))
    assert tr >= {3, 7, 11, 13, 15}
    assert all(bound[c] > 0 for c in drc.CLASSES if c not in ("ipcm", "hd")), bound
    assert sides == {"left", "right", "top", "bottom"}, sides


def test_anchor_oracle_reproduces_reference_decoder(emu):
    """the oracle is tied to the reference decoder, not only to the code it checks: seeded random Baseline streams
    (emu_random_stream_records: every Intra_4x4 mode with its prediction, Intra_16x16 and chroma modes, every P partition with
    vectors that leave the picture, P_Skip, per-macroblock QP changes), written with the loop filter off, are decoded by the
    reference decoder; the oracle reconstructs every picture from the parser's records, each P picture from the oracle's own
    earlier pictures in their slots, and must give the same samples"""
    if not h264lib.have_ref():
        pytest.skip("reference build not on this machine")
    from test_decoder_emu import ref_decode
    emu.emu_random_stream_records.restype = C.c_long
    emu.emu_random_stream_records.argtypes = [C.c_uint, C.c_int, C.c_void_p, C.c_long, C.c_void_p, C.c_void_p, C.c_void_p]
    n_pic, kinds = 6, set()
    buf = np.zeros(4 << 20, np.uint8)
    for seed in range(24):
        recs, aux, info = np.zeros(20 * n_pic, orc.MBOUT), np.zeros(20 * n_pic, orc.DECAUX), np.zeros(3 * n_pic, np.int32)
        n = emu.emu_random_stream_records(seed, n_pic, buf.ctypes.data, buf.size, recs.ctypes.data, aux.ctypes.data, info.ctypes.data)
        assert n > 0, (seed, n)
        nr, w, h, want = ref_decode(buf[:n].tobytes())
        assert (nr, w, h) == (n_pic, 80, 64), (seed, nr, w, h)
        slots = {}
        for p in range(n_pic):
            cur, n_slots, cq = info[3 * p:3 * p + 3]
            blank = [np.zeros((64, 80), np.int64), np.zeros((32, 40), np.int64), np.zeros((32, 40), np.int64)]
            refs = [slots.get(k, blank) for k in range(n_slots)]
            r, a = recs[20 * p:20 * p + 20], aux[20 * p:20 * p + 20]
            got, _ = orc.reconstruct(5, 4, r, a, np.zeros(20, orc.DECAUXB), int(cq), refs)
            slots[int(cur)] = got
            ref_pic = want[p * 7680:(p + 1) * 7680]
            for pl, (o, sh) in enumerate(((0, (64, 80)), (5120, (32, 40)), (6400, (32, 40)))):
                exp = ref_pic[o:o + sh[0] * sh[1]].reshape(sh)
                bad = np.argwhere(got[pl] != exp)
                assert bad.size == 0, (f"seed {seed} picture {p} plane {pl}: {len(bad)} samples differ, first at (x {bad[0][1]}, "
                                       f"y {bad[0][0]}): oracle {got[pl][tuple(bad[0])]}, reference {exp[tuple(bad[0])]}")
            kinds |= set(int(t) for t in r["mb_type"])
    assert kinds >= {orc.I4x4, orc.I16x16, orc.P16x16, orc.P16x8, orc.P8x16, orc.P8x8, orc.PSKIP}, kinds


def _mode_possible(mode, pat):
    L, T, TL = pat & 1, pat & 2, pat & 4
    return mode == 2 or (mode in (0, 3, 7) and T) or (mode in (1, 8) and L) or (mode in (4, 5, 6) and L and T and TL)


def test_refusals(emu):
    """bad arguments are refused before anything runs, as the device hook refuses them"""
    _refusals(emu.emu_decode_records)


def _refusals(fn):
    c = make("p", CASES[[k for k, (cl, _) in enumerate(CASES) if cl == "p"][0]][1])
    n_mb = c.mb_w * c.mb_h
    sty, stc, yb, cb = padded_bytes(c.mb_w, c.mb_h)
    planes = np.zeros(yb + 2 * cb, np.uint8)
    mbi = np.zeros(n_mb, orc.MBINFO)
    refs = c.dense_refs()

    def call(recs=None, aux=None, cq=0, n_refs=None, mb_w=None, mb_h=None):
        recs = c.recs if recs is None else recs
        aux = c.aux if aux is None else aux
        cqa = np.array([cq], np.int32)
        return fn(1, c.mb_w if mb_w is None else mb_w, c.mb_h if mb_h is None else mb_h, cqa.ctypes.data, recs.ctypes.data, aux.ctypes.data,
                  None, c.n_refs if n_refs is None else n_refs, refs.ctypes.data, planes.ctypes.data, mbi.ctypes.data)

    assert call() == 0
    assert call(cq=13) == -1 and call(cq=-13) == -1
    assert call(n_refs=0) == -1 and call(n_refs=17) == -1
    assert call(mb_w=0) == -1 and call(mb_h=513) == -1
    r = c.recs.copy(); r[0]["qp"] = 52
    assert call(recs=r) == -1
    r = c.recs.copy(); r[0]["mb_type"] = 10
    assert call(recs=r) == -1
    r = c.recs.copy(); r[0]["mb_type"] = orc.B                  # a B record without list-1 records
    assert call(recs=r) == -1
    a = c.aux.copy(); a[0]["avail"] = orc.NB_LEFT               # the first macroblock has no left neighbour
    assert call(aux=a) == -1
    a = c.aux.copy(); r = c.recs.copy(); r[0]["mb_type"] = orc.P16x16; a[0]["ref_idx"] = c.n_refs
    assert call(recs=r, aux=a) == -1
    a = c.aux.copy(); a[0]["sub_type"][1] = 4
    assert call(aux=a) == -1
