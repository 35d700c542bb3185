"""GPU: the decoder's construct stage on the device, through the test hook b2h264_debug_decode_records (enc_kernels.cu), which
runs the production path (pack_records_compact, dec_launch_unpack, the border replication of the reference pictures,
dec_launch_frame without deblocking) on given records.  On the record classes of tests/decode_record_cases.py every padded
picture and every MbInfo record must equal the spec oracle's (tests/mb_recon_oracle.py, the border as edge replication)
and, byte for byte, the host build's (tests/emu/decode_records_hooks.cu); classes are also mixed across the streams of one
launch, and the hook's refusals are checked."""
import ctypes as C

import pytest

import decode_record_cases as drc
import test_decode_records_emu as T

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    from openh264_b200.binding import lib
    L = lib()
    fn = L.b2h264_debug_decode_records
    fn.restype = C.c_int
    fn.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return fn


emu = T.emu


def _same(a, b):
    (pa, ma), (pb, mb) = a, b
    return all(x.tobytes() == y.tobytes() for x, y in zip(pa, pb)) and ma.tobytes() == mb.tobytes()


@pytest.mark.parametrize("cls", drc.CLASSES)
def test_device_matches_oracle_and_host_build(dev, emu, cls):
    cs = [T.make(c, s) for c, s in T.CASES if c == cls]
    for case in cs:
        got = T.run_hook(dev, [case])[0]
        T.compare(case, got, case.oracle())
        assert _same(got, T.run_hook(emu.emu_decode_records, [case])[0]), f"{cls} seed {case.seed}: device and host build differ"


def test_classes_mixed_across_streams(dev, emu):
    """one launch of many streams of one geometry, each a different class (and reference count 1: the hook takes one count)"""
    groups = {}
    for c, s in T.CASES:
        case = T.make(c, s)
        if case.n_refs == 1 and c != "hd":
            groups.setdefault((case.mb_w, case.mb_h), []).append(case)
    launched = 0
    for (w, h), cs in sorted(groups.items()):
        if len(set(c.cls for c in cs)) < 3:
            continue
        got = T.run_hook(dev, cs)
        want = T.run_hook(emu.emu_decode_records, cs)
        for case, g, e in zip(cs, got, want):
            T.compare(case, g, case.oracle())
            assert _same(g, e)
        launched += 1
    assert launched >= 3


def test_refusals(dev):
    T._refusals(dev)
