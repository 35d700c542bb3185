"""CPU: the plain raster-order picture deblocking oracle (oracle/orc_deblock_picture) against the host build of the device
filter (enc_deblock.cuh through tests/emu: deblock_one_mb in encoder mode, deblock_one_mb_b in decoder mode), on seeded
random pictures (tests/deblock_cases.py).  The host build is tied to the reference by test_encoder_emu / test_decoder_emu;
this pins the oracle that tests/test_gpu_deblock_pictures.py holds the device kernel to.  Every plane is compared over its
whole padded allocation, and the oracle's branch counters must show that every strength, filter branch and suppression
rule ran somewhere in the set."""
import numpy as np
import pytest

import deblock_cases as dc

# (seed, mb_w, mb_h, mode, 8x8 transform, slices, share of skipped macroblocks)
CASES = []
_SIZES = [(1, 1), (1, 5), (5, 1), (2, 2), (3, 7), (23, 17), (11, 4), (4, 11), (16, 9), (7, 3)]
for _k in range(40):
    _w, _h = _SIZES[_k % len(_SIZES)]
    _mode = ["enc", "dec_p", "dec_b", "dec_p"][_k % 4]
    _t8 = _mode != "enc" and _k % 3 != 0
    _slices = 1 if _mode == "enc" else 1 + _k % 4
    _skip = [0.0, 0.0, 0.6, 1.0][(_k // 4) % 4] if _k % 5 == 4 else 0.0
    CASES.append((1000 + _k, _w, _h, _mode, _t8, _slices, _skip))


def _name(c):
    return f"s{c[0]}-{c[1]}x{c[2]}-{c[3]}{'-t8' if c[4] else ''}-sl{c[5]}{'-skip%g' % c[6] if c[6] else ''}"


@pytest.mark.parametrize("case", CASES, ids=_name)
def test_oracle_matches_host_filter(case):
    seed, w, h, mode, t8, slices, skip = case
    p = dc.random_picture(seed, w, h, mode, t8=t8, n_slices=slices, skip_frac=skip)
    want = dc.oracle_deblock(p)
    got = dc.emu_deblock(p)
    for pl, name in enumerate("Y Cb Cr".split()):
        bad = np.flatnonzero(got[pl] != want[pl])
        assert bad.size == 0, f"{name}: {bad.size} samples differ, first at byte {bad[0]} (stride {dc.strides(w)[pl > 0]})"


def test_every_branch_ran():
    """the set above is not vacuous: over all its pictures the oracle filtered lines of every bS in luma and chroma, took the
    strong branch and the ap / aq branches, and left edges alone for each of idc 1, idc 2, the 8x8 transform and the border"""
    stats = np.zeros(dc.ORC_NSTATS, np.int32)
    for seed, w, h, mode, t8, slices, skip in CASES:
        dc.oracle_deblock(dc.random_picture(seed, w, h, mode, t8=t8, n_slices=slices, skip_frac=skip), stats)
    missing = [n for n, v in zip(dc.STAT_NAMES, stats) if v == 0]
    assert not missing, f"never exercised: {missing} (counters {dict(zip(dc.STAT_NAMES, stats.tolist()))})"


def test_filter_changes_pictures():
    """a picture with smooth content and strong edges must actually change (the comparison above is not of two no-ops)"""
    p = dc.random_picture(7, 6, 5, "dec_p", n_slices=1, idc=0)
    want = dc.oracle_deblock(p)
    assert sum(int((a != b).sum()) for a, b in zip(want, p.planes)) > 100
