"""The intra tail that stages I and C share (intra_mb_finish, enc_mb.cuh): the I4x4 try with its in-loop coding, the I16x16
residual and the chroma.  On the device the I4x4 candidates are costed one lane each and the lane that holds the winner codes
the block from its registers; the host emulation build keeps the serial sequence (re-predict the winner, code it through the
helpers), which is the specification.  The device tail must leave byte for byte the same records (levels, nnz, cbp, mb_type,
I4x4 modes and their prev / rem flags, I16x16 and chroma modes), reconstruction and I4x4 cost as the host build, on random and
structured macroblocks at QP 0 / 12 / 26 / 40 / 51, every neighbour-availability nibble, HIGH and LOW complexity, and cost
limits placed around the I4x4 running total so that the loop breaks early, completes and loses, or completes and wins."""
import ctypes as C

import numpy as np
import pytest

import h264lib

ROOT = h264lib.ROOT
TILE = 17 * 32 + 2 * 9 * 16         # RecTile: luma rows -1..15 x cols -1..30, Cb / Cr rows -1..7 x cols -1..14
IN_BYTES = TILE + 384 + 32          # b2h264_debug_intra_tail's case record
OUT_BYTES = 896 + 120 + 16 + TILE   # MbOut, MbInfo, limit / I4x4 cost / lambda / 0, the tile
INFO = 896                          # MbInfo: nnz at +64, i4_mode at +88, mb_type at +112, cbp at +113
MBT_I4x4, MBT_I16x16 = 0, 1
NB_LEFT, NB_TOP, NB_TOPLEFT, NB_TOPRIGHT = 1, 2, 4, 8
I4_END = ["I4x4 loop broke early", "I4x4 loop completed", "I4x4 won"]   # enc_mb.cuh: I4_END_BREAK .. I4_END_WON


@pytest.fixture(scope="module")
def emu():
    return h264lib.emu()


def content(rng, kind, h, w):
    """an h x w block of samples: 0 noise, 1 smooth gradient, 2 flat with faint noise, 3 stripes / edges"""
    y, x = np.mgrid[0:h, 0:w]
    if kind == 0:
        v = rng.randint(0, 256, (h, w))
    elif kind == 1:
        v = rng.randint(40, 200) + rng.uniform(-4, 4) * x + rng.uniform(-4, 4) * y + rng.randint(-2, 3, (h, w))
    elif kind == 2:
        v = rng.randint(16, 240) + rng.randint(-rng.randint(0, 3), rng.randint(0, 3) + 1, (h, w))
    else:
        period, phase = rng.randint(2, 9), rng.randint(0, 8)
        v = np.where(((x if rng.rand() < 0.5 else y) + phase) // period % 2 == 0, rng.randint(0, 256), rng.randint(0, 256))
        v = v + rng.randint(-3, 4, (h, w))
    return np.clip(v, 0, 255).astype(np.uint8)


def make_case(rng, qp, nb, fast, kind, limit=-1):
    """one case record: the tile's neighbour samples (zero where the neighbour is missing, as the encoder loads them), the
    source, the parameters and the neighbours' I4x4 modes"""
    rec = np.zeros(IN_BYTES, np.uint8)
    ty = np.zeros((17, 32), np.uint8)
    luma = content(rng, kind, 17, 25)                                  # rows -1..15, cols -1..23
    if nb & NB_TOPLEFT:
        ty[0, 0] = luma[0, 0]
    if nb & NB_TOP:
        ty[0, 1:17] = luma[0, 1:17]
    if nb & NB_TOPRIGHT:
        ty[0, 17:25] = luma[0, 17:25]
    if nb & NB_LEFT:
        ty[1:17, 0] = luma[1:17, 0]
    planes = [ty.reshape(-1)]
    cur_c = []
    for _ in range(2):
        tc = np.zeros((9, 16), np.uint8)
        ch = content(rng, kind, 9, 9)
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
    rng = np.random.RandomState(5)
    return np.stack([make_case(rng, qp, nb, fast, kind) for qp in (0, 12, 26, 40, 51) for fast in (0, 1) for nb in range(16)
                     for kind in range(4) for _ in range(2)])


def run_emu(emu, cases):
    out = np.zeros((len(cases), OUT_BYTES), np.uint8)
    assert emu.emu_intra_tail(len(cases), cases.ctypes.data, out.ctypes.data) == 0
    return out


def tails(out):
    """per case: cost limit used, I4x4 cost (INT_MAX: not tried), lambda"""
    t = out[:, INFO + 120:INFO + 136].view(np.int32)
    return t[:, 0], t[:, 1], t[:, 2]


def make_cases(emu):
    """the base cases with the I16x16 cost as the limit, then again with limits just below, at and above the I4x4 running total
    (taken from a host run without a limit) and somewhere inside it"""
    base = base_cases()
    free = base.copy()
    free[:, TILE + 396:TILE + 400] = np.array([1 << 30], np.int32).view(np.uint8)
    _, cost4, lam = tails(run_emu(emu, free))
    tried = cost4 != 0x7fffffff
    total = cost4 - 24 * lam                                          # the running total after the 16th block
    rng = np.random.RandomState(6)
    extra = []
    for i in np.nonzero(tried)[0]:
        for lim in (total[i] - 1, total[i], total[i] + 1, cost4[i] + 1, rng.randint(0, total[i] + 1)):
            c = base[i].copy()
            c[TILE + 396:TILE + 400] = np.array([max(int(lim), 0)], np.int32).view(np.uint8)
            extra.append(c)
    return np.concatenate([base, np.stack(extra)])


def test_cases_reach_every_outcome(emu):
    cases = make_cases(emu)
    emu.emu_reset_i4_ends()
    out = run_emu(emu, cases)
    ends = np.zeros(3, np.uint64)
    assert emu.emu_i4_ends(ends.ctypes.data, 3) == 3
    reached = {name: int(n) for name, n in zip(I4_END, ends)}
    assert all(n > 0 for n in reached.values()) and ends[1] > ends[2], reached  # broke, completed and lost, completed and won
    mbt = out[:, INFO + 112]
    cbp = out[:, INFO + 113].astype(int)
    i4 = mbt == MBT_I4x4
    i16 = mbt == MBT_I16x16
    assert i4.any() and i16.any()
    modes4 = out[i4, INFO + 88:INFO + 104]
    for m in range(9):
        assert (modes4 == m).any(), f"I4x4 mode {m}"
    for m in range(4):
        assert (out[i16, 3] == m).any(), f"I16x16 mode {m}"
        assert (out[:, 4] == m).any(), f"chroma mode {m}"
    dc = out[:, 80:112].view(np.int16)
    has_dc = (dc != 0).any(1)
    assert (i16 & has_dc & ((cbp & 15) == 0)).any()                  # I16x16 with DC levels only
    assert (i16 & ((cbp & 15) == 15)).any()                           # ... with AC levels
    assert (i16 & ~has_dc & ((cbp & 15) == 0)).any()                  # ... empty
    for v in (0, 1, 2):
        assert ((cbp >> 4) == v).any(), f"chroma cbp {v}"
    lim, cost4, _ = tails(out)
    assert ((cost4 == 0x7fffffff) & (out[:, INFO + 112] == MBT_I16x16)).any()   # LOW complexity: I4x4 not tried (flat source)


@pytest.mark.gpu
def test_device_tail_matches_host_build(emu):
    import openh264_b200 as m
    L = m.lib(0)
    L.b2h264_debug_intra_tail.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
    cases = make_cases(emu)
    want = run_emu(emu, cases)
    got = np.zeros_like(want)
    assert L.b2h264_debug_intra_tail(len(cases), cases.ctypes.data, got.ctypes.data) == 0
    bad = np.nonzero((got != want).any(1))[0]
    assert len(bad) == 0, f"{len(bad)} of {len(cases)} cases differ, first: case {bad[0]}, bytes " \
                          f"{np.nonzero(got[bad[0]] != want[bad[0]])[0][:16].tolist()}"
    _refusals(L.b2h264_debug_intra_tail)


def test_host_build_refuses_bad_arguments(emu):
    """the host build refuses what the device hook refuses (stage_hooks.cuh: intra_tail_args_ok)"""
    _refusals(emu.emu_intra_tail)


def _refusals(fn):
    # bad arguments are refused before anything runs
    c = base_cases()[:1].copy()
    got = np.zeros((1, OUT_BYTES), np.uint8)
    assert fn(1, c.ctypes.data, got.ctypes.data) == 0
    assert fn(0, c.ctypes.data, got.ctypes.data) == -1
    c[0, TILE + 384:TILE + 388] = np.array([52], np.int32).view(np.uint8)
    assert fn(1, c.ctypes.data, got.ctypes.data) == -1
