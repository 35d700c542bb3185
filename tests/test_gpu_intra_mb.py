"""The device intra path of stage I (b2h264_debug_intra_tail: md_i16x16, then intra_mb_finish) per macroblock on the cases of
tests/intra_mb_cases.py: it must code what the reference codes, through the SHA-1s ref_intra_mb (oracle/ref_shim.cpp) left in
tests/golden/intra_mb.json, and leave byte for byte the records, reconstruction and costs of the host emulation build; a
conforming decoder (tests/mb_recon_oracle.py) must rebuild the device's reconstruction from the device's records."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import h264lib
import intra_mb_cases as ic

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "intra_mb.json")


@pytest.fixture(scope="module")
def emu():
    return h264lib.emu()


@pytest.mark.gpu
def test_device_intra_mb_matches_reference_and_host_build(emu):
    import openh264_b200 as m
    L = m.lib(0)
    L.b2h264_debug_intra_tail.argtypes = [C.c_int, C.c_void_p, C.c_void_p]

    def run_dev(cases):
        out = np.zeros((len(cases), ic.OUT_BYTES), np.uint8)
        assert L.b2h264_debug_intra_tail(len(cases), np.ascontiguousarray(cases).ctypes.data, out.ctypes.data) == 0
        return out

    base, kinds, qps = ic.base_cases()
    cases, kinds, qps = ic.with_limits(base, kinds, qps, run_dev)     # the limits from the device's own run
    got = run_dev(cases)
    with open(GOLDEN) as f:
        golden = json.load(f)
    assert len(cases) == golden["cases"]
    hashes = ic.group_hashes(got, kinds, qps)
    bad = [g for g in sorted(hashes) if hashes[g] != golden["groups"].get(g)]
    assert not bad, f"{len(bad)} of {len(hashes)} (class / QP) groups differ from the reference: {bad[:8]}"
    match, refused, differ = ic.spec_decode(cases, got, range(len(cases)))
    assert not differ and not refused, (len(differ), len(refused))
    want = ic.run_emu(emu, cases)
    bad = np.nonzero((got != want).any(1))[0]
    assert len(bad) == 0, f"{len(bad)} of {len(cases)} cases differ from the host build, first: case {bad[0]} " \
                          f"({ic.CLASSES[kinds[bad[0]]]}, QP {qps[bad[0]]}), bytes {np.nonzero(got[bad[0]] != want[bad[0]])[0][:16].tolist()}"
