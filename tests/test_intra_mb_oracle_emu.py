"""The intra path of stages I and C (md_i16x16, then intra_mb_finish) per macroblock against the reference's own mode decision
and coding.  The host emulation build of the path (emu_intra_tail, tests/emu/intra_tail_hooks.cu) must equal, on every case of
tests/intra_mb_cases.py, the reference driven through WelsMdI16x16 and WelsMdIntraSecondaryModesEnc (ref_intra_mb in
oracle/ref_shim.cpp, where oracle/_ref is built) and the SHA-1s that driver left in tests/golden/intra_mb.json (everywhere).
Compared: mb_type, cbp, the I16x16 and chroma modes as coded, the I4x4 modes and their prev / rem flags, every level, nnz, the
reconstruction, the cost limit (the I16x16 cost when no limit is given), the I4x4 cost and lambda.  The cases must reach what
natural clips rarely do; the coverage test names each thing and requires it."""
import json
import os

import numpy as np
import pytest

import h264lib
import intra_mb_cases as ic

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "intra_mb.json")
I4_END = ["broke early", "completed and lost", "completed and won"]


@pytest.fixture(scope="module")
def emu():
    return h264lib.emu()


@pytest.fixture(scope="module")
def cases(emu):
    base, kinds, qps = ic.base_cases()
    return ic.with_limits(base, kinds, qps, lambda c: ic.run_emu(emu, c))


@pytest.fixture(scope="module")
def emu_out(emu, cases):
    return ic.run_emu(emu, cases[0])


def test_host_build_matches_reference(cases, emu_out):
    if not h264lib.have_ref():
        pytest.skip("oracle/_ref not built on this machine")
    if "intra_mb" in h264lib.ref().missing or not hasattr(h264lib.ref().lib, "ref_intra_mb"):
        pytest.skip("oracle/_ref was built before ref_intra_mb was added to the shim (the golden test still pins the path)")
    ref, costs = ic.run_ref(cases[0])
    d = ic.first_difference(emu_out, ref)
    assert d is None, f"{d[2]} cases differ in {d[1]}, first: case {d[0]} ({ic.CLASSES[cases[1][d[0]]]}, QP {cases[2][d[0]]})"
    # the I16x16 cost is the limit used where the case gives none
    free = cases[0][:, ic.TILE + 396:ic.TILE + 400].copy().view(np.int32)[:, 0] < 0
    assert np.array_equal(costs[free, 0], emu_out[free, ic.TAIL:ic.TAIL + 4].copy().view(np.int32)[:, 0])


def test_host_build_matches_golden(cases, emu_out):
    with open(GOLDEN) as f:
        golden = json.load(f)
    assert len(cases[0]) == golden["cases"]
    got = ic.group_hashes(emu_out, cases[1], cases[2])
    assert sorted(got) == sorted(golden["groups"])
    bad = [g for g in sorted(got) if got[g] != golden["groups"][g]]
    assert not bad, f"{len(bad)} of {len(got)} (class / QP) groups differ from the reference: {bad[:8]}"


def _plane_range(tile, chroma):
    """min and max of the unclipped plane prediction (H.264 8.3.3.4 / 8.3.4.4) of each case from its tile's border"""
    n = 8 if chroma else 16
    h = n // 2
    top, left = tile[:, 0, 1:n + 1].astype(np.int64), tile[:, 1:n + 1, 0].astype(np.int64)
    corner = tile[:, 0, 0].astype(np.int64)
    ext_t = np.concatenate([corner[:, None], top], 1)               # index 0 = p[-1, -1]
    ext_l = np.concatenate([corner[:, None], left], 1)
    H = sum((i + 1) * (ext_t[:, h + 1 + i] - ext_t[:, h - 1 - i]) for i in range(h))
    V = sum((i + 1) * (ext_l[:, h + 1 + i] - ext_l[:, h - 1 - i]) for i in range(h))
    a = 16 * (left[:, n - 1] + top[:, n - 1])
    b, c = ((5 * H + 32) >> 6, (5 * V + 32) >> 6) if not chroma else ((34 * H + 32) >> 6, (34 * V + 32) >> 6)
    corners = [(a + b * (x - h + 1) + c * (y - h + 1) + 16) >> 5 for x in (0, n - 1) for y in (0, n - 1)]
    return np.min(corners, 0), np.max(corners, 0)


def test_cases_reach_every_path(emu, cases):
    recs, kinds, qps = cases
    prm = recs[:, ic.TILE + 384:ic.TILE + 400].copy().view(np.int32)
    nb, fast, limit = prm[:, 1], prm[:, 2], prm[:, 3]
    ends = {}
    for f in (0, 1):
        emu.emu_reset_i4_ends()
        ic.run_emu(emu, recs[fast == f])
        e = np.zeros(3, np.uint64)
        assert emu.emu_i4_ends(e.ctypes.data, 3) == 3
        ends[f] = [int(e[0]), int(e[1] - e[2]), int(e[2])]
    emu.emu_reset_i4_ends()
    out = ic.run_emu(emu, recs)
    reached = {}
    for f in (0, 1):
        for j, name in enumerate(I4_END):
            reached[f"I4x4 try {name}, {'LOW' if f else 'HIGH'}"] = ends[f][j]
    i4 = out[:, ic.INFO + 112] == 0
    i16 = ~i4
    cbp = out[:, ic.INFO + 113].astype(int)
    cost4 = out[:, ic.TAIL + 4:ic.TAIL + 8].copy().view(np.int32)[:, 0]
    # every entry of the I16x16 and chroma lists, as coded, under each (left, top, top-left) pattern that allows it
    for p in range(8):
        l, t, tl = p & 1, p & 2, p & 4
        sel = (nb & 7) == p
        allowed16 = [2] + ([0] if t else []) + ([1] if l else []) + ([3] if l and t and tl else [])
        allowed_c = [0] + ([1] if l else []) + ([2] if t else []) + ([3] if l and t and tl else [])
        for m in allowed16:
            reached[f"I16x16 mode {m} with neighbours {p}"] = int((sel & i16 & (out[:, 3] == m)).sum())
        for m in allowed_c:
            reached[f"chroma mode {m} with neighbours {p}"] = int((sel & (out[:, 4] == m)).sum())
    # every I4x4 mode; DDL and VL in blocks without (3, 5, 7, 11, 13, 15) and with a top-right neighbour
    modes = out[:, ic.INFO + 88:ic.INFO + 104].astype(int)            # raster
    no_tr = np.zeros(16, bool)
    no_tr[[5, 7, 13, 15, 11, 3]] = True                              # the raster positions of coding blocks 3, 5, 7, 11, 13, 15
    for m in range(9):
        reached[f"I4x4 mode {m}"] = int((modes[i4] == m).sum())
    for m in (3, 7):
        reached[f"I4x4 mode {m} without top-right"] = int((modes[i4][:, no_tr] == m).sum())
        reached[f"I4x4 mode {m} with top-right"] = int((modes[i4][:, ~no_tr] == m).sum())
    # the LOW texture gate both ways, at exactly 150 and on either side of it
    tried = cost4 != ic.INT_MAX
    for k, want in (("var149", False), ("var150", True), ("var151", True)):
        sel = (kinds == ic.CLASSES.index(k)) & (fast == 1)
        reached[f"LOW gate at variance {k[3:]}"] = int((sel & (tried == want)).sum())
        reached[f"LOW gate at variance {k[3:]}, other side"] = int((sel & (tried != want)).sum()) == 0
    reached["I16x16 cbp 15"] = int((i16 & ((cbp & 15) == 15)).sum())
    reached["I16x16 cbp 0"] = int((i16 & ((cbp & 15) == 0)).sum())
    for v in (0, 1, 2):
        reached[f"chroma cbp {v}"] = int(((cbp >> 4) == v).sum())
    # plane predictions that saturate at both ends where the plane mode was chosen, in luma and in chroma
    tile = recs[:, :ic.TILE]
    lo, hi = _plane_range(tile[:, :17 * 32].reshape(-1, 17, 32), False)
    p16 = i16 & (out[:, 3] == 3)
    reached["luma plane below 0"] = int((p16 & (lo < 0)).sum())
    reached["luma plane above 255"] = int((p16 & (hi > 255)).sum())
    pc = out[:, 4] == 3
    for name, off in (("Cb", 17 * 32), ("Cr", 17 * 32 + 144)):
        lo, hi = _plane_range(tile[:, off:off + 144].reshape(-1, 9, 16), True)
        reached[f"{name} plane below 0"] = int((pc & (lo < 0)).sum())
        reached[f"{name} plane above 255"] = int((pc & (hi > 255)).sum())
    # cost limits given by the case, and the QPs
    reached["cases with a cost limit"] = int((limit >= 0).sum())
    for q in range(52):
        reached[f"QP {q}"] = int((qps == q).sum())
    print("\n" + "\n".join(f"  {k}: {v}" for k, v in reached.items()))
    missing = [k for k, v in reached.items() if not v]
    assert not missing, missing


# cases whose records a conforming decoder refuses (its 16-bit range checks), by (class, QP); the reference encoder emits the
# same levels (test_host_build_matches_reference), so such a case is not a failure, but the set must not change unnoticed
REFUSED = set()


def test_spec_decode_of_host_build_records(cases, emu_out):
    recs, kinds, qps = cases
    match, refused, differ = ic.spec_decode(recs, emu_out, range(len(recs)))
    assert not differ, f"{len(differ)} cases decode to other samples than the host build keeps, first: case {differ[0]} " \
                       f"({ic.CLASSES[kinds[differ[0]]]}, QP {qps[differ[0]]})"
    assert {(ic.CLASSES[kinds[i]], int(qps[i])) for i in refused} == REFUSED
    assert len(match) + len(refused) == len(recs)
