"""GPU: the picture deblocking kernel (k_deblock_pictures, enc_kernels.cu / enc_deblock.cuh) against the raster-order oracle
(oracle/orc_deblock_picture), through the test hook b2h264_debug_deblock_pictures, which launches it through the same launcher
as the encoder and the decoder.

Every launch is compared with the oracle over the whole allocation, byte for byte: every picture, its padding, and a random
canary gap between pictures must come back exactly as the oracle leaves them.  The cases force every warp count the wavefront
has to get right (1, 2, 3, 16, 17, 31, 32, with heights that end one row after a multiple of it), narrow and wide shapes, the
launcher's own choice of 17 and 32 warps, both instantiations (one list; two lists with B records, with and without them in
one launch), and pictures whose macroblocks have no edge to filter.  The large-batch tests at the end run the public encoder
and decoder at more than half the SM count, where the launcher picks 17 warps, on pictures whose height is not a multiple
of 17.  Pictures: tests/deblock_cases.py (pinned to the host build by tests/test_deblock_oracle_emu.py)."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest

import deblock_cases as dc
import h264lib

pytestmark = pytest.mark.gpu
ROOT = h264lib.ROOT
GAP = 64                      # canary bytes before every plane (keeps every plane 16-byte aligned)


def _lib():
    from openh264_b200.binding import lib
    L = lib()
    fn = L.b2h264_debug_deblock_pictures
    fn.restype = C.c_int
    fn.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                   C.POINTER(C.c_int)]
    return L


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _layout(pics, rng):
    """one host buffer for all planes of all pictures, each plane behind a canary gap; returns (buffer, plane offsets)"""
    parts, offs, pos = [], [], 0
    for p in pics:
        for pl in range(3):
            parts.append(rng.randint(0, 256, GAP).astype(np.uint8))
            pos += GAP
            offs.append(pos)
            parts.append(p.planes[pl])
            pad = -len(p.planes[pl]) % 16
            parts.append(rng.randint(0, 256, pad).astype(np.uint8))
            pos += len(p.planes[pl]) + pad
    parts.append(rng.randint(0, 256, GAP).astype(np.uint8))
    return np.concatenate(parts), offs


def _launch(pics, dec_mode, bsl, n_warps=0, geo_fix=None, plane_shift=0):
    """runs the hook on the pictures (encoder mode: with their common control); returns (rc, warps used, device buffer after, host buffer before, plane offsets)"""
    from openh264_b200.binding import DeviceArray
    L = _lib()
    rng = np.random.RandomState(len(pics) * 7 + n_warps)
    buf, offs = _layout(pics, rng)
    dbuf = DeviceArray(buf)
    dmbi = [DeviceArray(np.frombuffer(p.mbi.tobytes(), np.uint8)) for p in pics]
    daux = [None if p.auxb is None else DeviceArray(np.frombuffer(p.auxb.tobytes(), np.uint8)) for p in pics]
    n = len(pics)
    planes = (C.c_void_p * (3 * n))(*[dbuf.ptr + offs[3 * i + pl] + pics[i].origin(pl) + plane_shift for i in range(n) for pl in range(3)])
    geo = np.array([[*dc.strides(p.mb_w), p.mb_w, p.mb_h] for p in pics], np.int32)
    if geo_fix:
        geo_fix(geo)
    mbi = (C.c_void_p * n)(*[d.ptr for d in dmbi])
    aux = (C.c_void_p * n)(*[None if d is None else d.ptr for d in daux]) if any(d is not None for d in daux) else None
    enc_ctl = pics[0].enc_ctl
    assert dec_mode or all(p.enc_ctl == enc_ctl for p in pics)
    used = C.c_int(-7)
    rc = L.b2h264_debug_deblock_pictures(n, planes, geo.ctypes.data, mbi, aux, dec_mode, *enc_ctl, bsl, n_warps, C.byref(used))
    got = dbuf.get()
    for d in [dbuf] + dmbi + [d for d in daux if d is not None]:
        d.free()
    return rc, used.value, got, buf, offs


def _expect(pics, buf, offs):
    want = buf.copy()
    for i, p in enumerate(pics):
        out = dc.oracle_deblock(p)
        for pl in range(3):
            want[offs[3 * i + pl]:offs[3 * i + pl] + len(out[pl])] = out[pl]
    return want


def _check(pics, dec_mode, bsl, n_warps=0):
    """one launch of the pictures (a DecMbAuxB* is NULL for those without B records); returns the warp count used"""
    rc, used, got, buf, offs = _launch(pics, dec_mode, bsl, n_warps)
    assert rc == 0, f"hook returned {rc}"
    want = _expect(pics, buf, offs)
    bad = np.flatnonzero(got != want)
    if bad.size:
        k = int(np.searchsorted(np.asarray(offs), bad[0], side="right")) - 1
        i, pl = max(k, 0) // 3, max(k, 0) % 3
        p = pics[i]
        st = dc.strides(p.mb_w)[pl > 0]
        r = int(bad[0]) - offs[max(k, 0)] - p.origin(pl)
        pytest.fail(f"{bad.size} bytes differ; first in picture {i} plane {pl} at row {r // st} col {r % st} (relative to sample "
                    f"(0,0); {p.mb_w}x{p.mb_h} MBs, {used} warps)")
    return used


def _pictures(seed, shapes, mode, **kw):
    return [dc.random_picture(seed + k, w, h, mode, **kw) for k, (w, h) in enumerate(shapes)]


# (mode, bsl): the encoder, a decoded P picture (reference pictures compared, one list), and decoded pictures with the 8x8
# transform and B macroblocks (two-list instantiation)
MODES = [("enc", 0), ("dec_p", 0), ("dec_b", 1), ("dec_p_t8", 1)]


def _mode_pictures(seed, shapes, mode):
    if mode == "enc":           # one control per launch: idc 0, offsets from the seed
        return _pictures(seed, shapes, "enc", enc_ctl=(0, 2 * (seed % 13 - 6), 2 * (seed // 13 % 13 - 6))), 0
    if mode == "dec_p":
        return _pictures(seed, shapes, "dec_p", n_slices=3), 1
    if mode == "dec_b":
        return _pictures(seed, shapes, "dec_b", t8=True, n_slices=2), 1
    return _pictures(seed, shapes, "dec_p", t8=True, n_slices=4), 1


@pytest.mark.parametrize("nw", [1, 2, 3, 16, 17, 31, 32])
def test_forced_warp_counts(nw):
    """a warp count forced on the launcher, with heights 1, nw, nw + 1 (warp 0 takes a second row and waits on warp nw - 1)
    and 2 nw + 1; one launch of two pictures per height, the instantiation rotating over the modes"""
    for k, mb_h in enumerate(sorted({1, nw, nw + 1, 2 * nw + 1})):
        mode, bsl = MODES[(nw + k) % len(MODES)]
        mb_w = 3 if mb_h > 20 else 11
        pics, dec_mode = _mode_pictures(100 * nw + 10 * k, [(mb_w, mb_h)] * 2, mode)
        used = _check(pics, dec_mode, bsl, n_warps=nw)
        assert used == min(nw, mb_h)


# narrow, flat and full-size pictures (one 1080p picture per instantiation)
SHAPES = [(s, m) for s in [(1, 40), (120, 1), (2, 2), (3, 5), (11, 9), (120, 68)] for m, _ in MODES if s != (120, 68) or m in ("enc", "dec_b")]


@pytest.mark.parametrize("shape,mode", SHAPES, ids=[f"{s[0]}x{s[1]}-{m}" for s, m in SHAPES])
def test_shapes(shape, mode):
    """one picture: the launcher's own choice is 32 warps, or mb_h when smaller"""
    pics, dec_mode = _mode_pictures(100 * shape[0] + shape[1], [shape], mode)
    bsl = dict(MODES)[mode]
    used = _check(pics, dec_mode, bsl)
    assert used == min(32, shape[1])
    print(f"[deblock] {shape[0]}x{shape[1]} {mode}: launcher chose {used} warps")


def test_launcher_choice_for_a_large_batch():
    """more pictures than half the SMs: the launcher gives each CTA 17 warps; 23 rows do not divide evenly over them"""
    sms = _sms()
    n = sms // 2 + 1
    pics = [dc.random_picture(5000 + k, 40, 23, "dec_b" if k % 2 else "dec_p", t8=k % 3 == 0, n_slices=1 + k % 4,
                              skip_frac=0.3 if k % 5 == 0 else 0.0) for k in range(n)]
    # the decoder's mixed batch: pictures with B records next to pictures without (their DecMbAuxB* is NULL)
    used = _check(pics, 1, 1)
    print(f"[deblock] {n} pictures of 40x23 on {sms} SMs: launcher chose {used} warps")
    assert used == 17


def test_one_picture_gets_32_warps():
    pics = [dc.random_picture(77, 20, 45, "enc", enc_ctl=(0, -2, 4))]
    used = _check(pics, 0, 0)
    assert used == 32


def test_two_list_instantiation_with_and_without_b_records():
    """bsl = 1 with pictures that carry B records and Baseline-like pictures whose DecMbAuxB* is NULL, in one launch"""
    pics = [dc.random_picture(900 + k, 9, 13, "dec_b" if k % 2 == 0 else "dec_p", t8=k % 2 == 0, n_slices=2) for k in range(4)]
    _check(pics, 1, 1)


@pytest.mark.parametrize("mode", ["enc", "dec_p", "dec_b"])
def test_pictures_without_edges_to_filter(mode):
    """every macroblock skipped with one vector and no coefficients (every strength 0: nothing is written back), next to
    pictures where most macroblocks are, and a picture whose slices all have idc 1"""
    bsl = 1 if mode == "dec_b" else 0
    dec_mode = 0 if mode == "enc" else 1
    ctl = (0, 0, 0)
    pics = [dc.random_picture(300, 7, 6, mode, skip_frac=1.0, enc_ctl=ctl), dc.random_picture(301, 7, 6, mode, skip_frac=0.9, enc_ctl=ctl),
            dc.random_picture(302, 7, 6, mode, skip_frac=0.9, enc_ctl=ctl)]
    if mode != "enc":
        pics.append(dc.random_picture(303, 7, 6, mode, n_slices=3, idc=1))
    _check(pics, dec_mode, bsl, n_warps=3)
    if mode == "enc":          # encoder mode: idc 1 is the picture's control
        _check([dc.random_picture(304, 7, 6, "enc", enc_ctl=(1, 0, 0))], 0, 0)


def test_hook_rejects_bad_arguments_without_launching():
    L = _lib()
    pics = [dc.random_picture(11, 3, 4, "dec_p")]
    before = L.b2h264_launch_count()

    def bad(**kw):
        rc, _, got, buf, _ = _launch(pics, 1, 0, **kw)
        assert rc == -1
        assert np.array_equal(got, buf)           # nothing written

    def fix_y(g):
        g[0, 0] += 8                               # luma rows no longer 16-byte aligned

    def fix_c(g):
        g[0, 1] += 4                               # chroma rows no longer 8-byte aligned
    bad(geo_fix=fix_y)
    bad(geo_fix=fix_c)
    bad(plane_shift=8)                             # plane origins not 16-byte aligned
    bad(n_warps=-1)
    bad(n_warps=33)
    assert L.b2h264_launch_count() == before
    assert L.b2h264_debug_deblock_pictures(0, None, None, None, None, 1, 0, 0, 0, 0, 0, None) == -1


# ---- large batches through the public encoder and decoder: more than SMs / 2 streams, so the deblocking launch uses 17 warps --
def _free_bytes():
    import torch
    return torch.cuda.mem_get_info(0)[0]


@pytest.mark.parametrize("key", ["640x360_n5_qp30_fps30", "1280x720_n4_qp32_fps30"])
def test_encoder_large_batch_matches_golden(key):
    """mb_h 23 and 45: uneven over 17 warps; every stream's bitstream equals the reference's"""
    from openh264_b200.binding import BatchEncoder
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "encoder.json")))[key]
    w, h = map(int, key.split("_")[0].split("x"))
    n, qp = int(key.split("_n")[1].split("_")[0]), int(key.split("_qp")[1].split("_")[0])
    S = _sms() // 2 + 1
    yuv = h264lib.synth_clip(w, h, n)
    assert hashlib.sha1(yuv.tobytes()).hexdigest() == gold["yuv_sha1"]
    fsz = w * h * 3 // 2
    enc = BatchEncoder(w, h, qp=qp, fps=30.0, n_streams=S)
    outs = [[] for _ in range(S)]
    for f in range(n):
        bs, _ = enc.encode([np.ascontiguousarray(yuv[f * fsz:(f + 1) * fsz])] * S)
        for s in range(S):
            outs[s].append(bs[s])
    enc.close()
    bad = [s for s in range(S) if hashlib.sha1(b"".join(outs[s])).hexdigest() != gold["sha1"]]
    assert not bad, f"streams {bad} of {S} differ from the reference"


def _output_order(items):
    items.sort(key=lambda t: t[:3])
    hs = hashlib.sha1()
    for t in items:
        hs.update(t[3].tobytes())
    return hs.hexdigest()


def test_decoder_large_batch_b_and_baseline():
    """S > SMs / 2 streams of 640x320 (mb_h 20): the CAVLC and CABAC B-frame vectors alternate with a Baseline stream of our
    encoder, so the two-list kernel runs at 17 warps with and without B records per picture"""
    from openh264_b200.binding import BatchDecoder, BatchEncoder
    conf = os.path.join(ROOT, "tests", "golden", "conformance_b")
    tab = dict((p.split("/")[-1], s) for p, s in json.load(open(os.path.join(ROOT, "tests", "golden", "reference_decoder_hashes.json")))["pairs"])
    names = ["Cisco_Men_whisper_640x320_CAVLC_Bframe_9.264", "Cisco_Men_whisper_640x320_CABAC_Bframe_9.264"]
    aus_b = {nm: h264lib.split_access_units(open(os.path.join(conf, nm), "rb").read()) for nm in names}
    w, h, n = 640, 320, len(aus_b[names[0]])
    assert all(len(a) == n for a in aus_b.values())
    yuv = h264lib.synth_clip(w, h, n, seed=5, noise=4)
    fsz = w * h * 3 // 2
    enc = BatchEncoder(w, h, qp=27, fps=30.0, n_streams=1)
    aus_p = [enc.encode([yuv[f * fsz:(f + 1) * fsz]])[0][0] for f in range(n)]
    enc.close()
    alone = BatchDecoder(w, h)
    want_p = [alone.decode([au])[0].copy() for au in aus_p]
    alone.close()
    S = _sms() // 2 + 1
    kind = [("p" if s % 3 == 2 else names[(s // 3 + s) % 2]) for s in range(S)]
    free0 = _free_bytes()
    dec = BatchDecoder(w, h, n_streams=S)
    got = [[] for _ in range(S)]
    seq = [0] * S
    for k in range(n):
        pics = dec.decode2([aus_p[k] if kind[s] == "p" else aus_b[kind[s]][k] for s in range(S)])
        if k == 0:
            print(f"[deblock] decoder batch of {S} 640x320 streams allocated {(free0 - _free_bytes()) / 2**20:.0f} MiB")
        for s in range(S):
            assert pics[s] is not None
            poc, idr, _ = dec.picture_order(s)
            seq[s] += idr & 1
            got[s].append((seq[s], poc, k, pics[s].copy()))
    dec.close()
    for s in range(S):
        if kind[s] == "p":
            assert all(np.array_equal(got[s][k][3], want_p[k]) for k in range(n)), f"Baseline stream {s}"
        else:
            assert _output_order(got[s]) == tab[kind[s]], f"stream {s} ({kind[s]})"


def test_decoder_large_batch_1080p_high_profile():
    """S > SMs / 2 streams of a 1920x1080 High-profile vector (8x8 transform, B slices, mb_h 68) in one batch"""
    from openh264_b200.binding import BatchDecoder
    name = "VID_1920x1080_cabac_temporal_direct_first10.264"
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "high_profile_prefix.json")))[name]
    aus = h264lib.split_access_units(open(os.path.join(ROOT, "tests", "golden", "conformance_b", name), "rb").read())
    assert len(aus) == gold["pictures"]
    S = _sms() // 2 + 1
    free0 = _free_bytes()
    dec = BatchDecoder(gold["width"], gold["height"], n_streams=S)
    got = [[] for _ in range(S)]
    seq = [0] * S
    for k, au in enumerate(aus):
        pics = dec.decode2([au] * S)
        if k == 0:
            print(f"[deblock] decoder batch of {S} 1080p streams allocated {(free0 - _free_bytes()) / 2**20:.0f} MiB")
        for s in range(S):
            assert pics[s] is not None
            poc, idr, _ = dec.picture_order(s)
            seq[s] += idr & 1
            got[s].append((seq[s], poc, k, pics[s].copy()))
    dec.close()
    bad = [s for s in range(S) if _output_order(got[s]) != gold["sha1"]]
    assert not bad, f"streams {bad} of {S} differ from the reference decoder"
