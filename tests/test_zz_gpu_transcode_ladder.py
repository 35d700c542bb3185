"""The transcoding ladder on the GPU: b2h264_k_downsample_ladder against the oracle's down-sampler plane by plane, and
openh264_b200.transcode.Transcoder with rungs, where every rung must give the bytes of the reference chain for that rung (reference
decoder, pictures in output order -> the oracle's down-sampler on the full-size decoded picture, with the function
CDownsampling::Process picks per plane -> reference encoder with the rung's configuration) and of a single-output Transcoder.
(File name: runs after the other GPU tests.)"""
import ctypes as C
import os

import numpy as np
import pytest

import h264lib
from h264lib import ptr
from test_zz_gpu_transcode import B_VECTORS, GOLDEN, _need_ref, _ref_chain, _transcode

pytestmark = pytest.mark.gpu
SENTINEL = 0xA5


def _orc(mode, plane, ss, sw, sh, dw, dh):
    """the oracle's down-sampler on one plane given as a host array with stride ss (one spare row and column of reads allowed)"""
    O = h264lib.oracle().lib
    O.orc_downsample.argtypes = [C.c_int, h264lib.u8p, C.c_int, C.c_int, C.c_int, h264lib.u8p, C.c_int, C.c_int, C.c_int]
    O.orc_downsample.restype = None
    src = np.zeros((sh + 1, ss + 3), np.uint8)
    src[:sh, :sw] = plane.reshape(-1)[:sh * ss].reshape(sh, ss)[:, :sw]
    dst = np.zeros((dh, dw), np.uint8)
    O.orc_downsample(mode, ptr(dst), dw, dw, dh, ptr(src), ss + 3, sw, sh)
    return dst


def _run_ladder(planes, src, dst, src_pitch, dst_pitch, lo, cnt):
    """one b2h264_k_downsample_ladder launch over host arrays src / dst (one picture per row); returns the device's dst"""
    import openh264_b200 as m
    from openh264_b200.binding import DsPlane, check
    L = m.lib(0)
    tab = (DsPlane * len(planes))(*[DsPlane(*p) for p in planes])
    ddst = m.DeviceArray(dst)
    dsrc = ddst if src is dst else m.DeviceArray(src)
    check(L.b2h264_k_downsample_ladder(C.addressof(tab), len(planes), ddst.ptr, dst_pitch, dsrc.ptr, src_pitch, lo, cnt, None))
    return ddst.get()


def _check_planes(planes, got, before, src, lo, cnt):
    """every plane of the pictures lo .. lo + cnt - 1 equals the oracle; every byte outside those planes' samples is unchanged"""
    untouched = np.ones(got.shape, bool)
    for s in range(lo, lo + cnt):
        for mode, sx, sy, sw, sh, ss, dw, dh, ds, row0, so, do in planes:
            want = _orc(mode, src[s, so:so + ss * sh], ss, sw, sh, dw, dh)
            rows = got[s, do:do + ds * (dh - 1) + dw]
            have = np.stack([rows[y * ds:y * ds + dw] for y in range(dh)])
            assert np.array_equal(have, want), (s, mode, dw, dh)
            for y in range(dh):
                untouched[s, do + y * ds:do + y * ds + dw] = False
    assert np.array_equal(got[untouched], before[untouched]), "bytes outside the planes (or of sit-out pictures) were written"


def test_ladder_kernel_every_mode_unaligned_offsets_and_sit_outs():
    """eight planes in one launch: all five modes, widths that are not multiples of 4, odd strides and plane offsets, a half-mode
    plane with an 8-aligned source and a destination that is not 4-aligned, and one plane on the half mode's aligned-word path.
    Pictures 0 and 4 lie outside the launch's range [lo, lo + cnt) and keep their sentinel bytes.  (The kernel down-samples every
    picture inside the range; a stream inside it that got no picture is scaled from stale bytes into a row Transcoder never reads.)"""
    from openh264_b200.transcode import round_ratio
    from openh264_b200.binding import load
    L = load()
    # source planes of one picture: (offset, width, height, stride)
    a, b, c, d, e = (1, 1280, 720, 1283), (1283 * 721 + 1, 99, 51, 101), (1283 * 721 + 1 + 101 * 52, 167, 109, 170), \
        (1283 * 721 + 1 + 101 * 52 + 170 * 110, 34, 18, 37), (1024 * 1024, 64, 36, 64)
    src_pitch = ((1024 * 1024 + 64 * 37 + 255) & ~255) + 256    # a multiple of 256, with slack after the last plane
    want_modes = [0, 1, 2, 3, 4, 0, 0, 0]
    jobs = [(a, 640, 360, 0, 1), (a, 320, 180, 0, 3), (b, 33, 17, 0, 2), (a, 854, 480, 0, 5), (c, 50, 39, 1, 1), (d, 17, 9, 0, 0),
            (e, 32, 18, 0, 1), (e, 32, 18, 0, None)]
    planes, off, row = [], 3, 0
    for (so, sw, sh, ss), dw, dh, chroma, pad in jobs:
        mode = L.b2h264_downsample_mode(sw, sh, dw, dh, chroma)
        sx = round_ratio(sw, dw, 1 << (16 if mode == 3 else 15)) if mode >= 3 else 0
        sy = round_ratio(sh, dh, 1 << 15) if mode >= 3 else 0
        if pad is None:                                   # aligned offsets and stride: the 8-byte loads and the word stores
            off, ds = (off + 3) & ~3, dw
        else:
            off, ds = off + (off % 4 == 0), dw + pad
        planes.append((mode, sx, sy, sw, sh, ss, dw, dh, ds, row, so, off))
        off += ds * dh + 1
        row += dh
    assert [p[0] for p in planes] == want_modes
    assert planes[-1][11] % 4 == 0 and all(p[11] % 4 for p in planes[:-1])
    dst_pitch = (off + 255) & ~255
    rng = np.random.RandomState(11)
    S, lo, cnt = 5, 1, 3
    src = rng.randint(0, 256, size=(S, src_pitch)).astype(np.uint8)
    dst = np.full((S, dst_pitch), SENTINEL, np.uint8)
    got = _run_ladder(planes, src, dst, src_pitch, dst_pitch, lo, cnt)
    _check_planes(planes, got, dst, src, lo, cnt)


def test_ladder_kernel_baseline_config4_ladder():
    """BASELINE.json configs[4] (1280x720 -> 640x360 / 320x180 / 160x90) with Transcoder's own table, reading the decoded picture at
    offset 0 of the same step buffer it writes the rungs into; pictures 0 and 3 sit out"""
    from openh264_b200.transcode import ladder_layout
    offsets, pitch, planes = ladder_layout(1280, 720, [(1280, 720), (640, 360), (320, 180), (160, 90)])
    assert [p[0] for p in planes] == [0, 0, 0, 1, 1, 1, 3, 4, 4]
    S, lo, cnt = 4, 1, 2
    rng = np.random.RandomState(12)
    buf = np.full((S, pitch + 256), SENTINEL, np.uint8)
    buf[:, :1280 * 720 * 3 // 2] = rng.randint(0, 256, size=(S, 1280 * 720 * 3 // 2))
    got = _run_ladder(planes, buf, buf, pitch + 256, pitch + 256, lo, cnt)
    _check_planes(planes, got, buf, buf, lo, cnt)


def _ladder(streams, w, h, rungs):
    """per rung, per stream: the bytes of Transcoder(rungs=...) over all pushes and the flush; and the transcoder"""
    from openh264_b200.transcode import Transcoder
    t = Transcoder(w, h, len(streams), rungs=rungs)
    got = [[b""] * len(rungs) for _ in streams]
    outs = [t.push([a[k] if k < len(a) else None for a in streams]) for k in range(max(len(a) for a in streams))] + [t.flush()]
    for out in outs:
        assert len(out) == len(streams) and all(len(o) == len(rungs) for o in out)
        got = [[g + o for g, o in zip(gs, os_)] for gs, os_ in zip(got, out)]
    t.close()
    return [[got[s][r] for s in range(len(streams))] for r in range(len(rungs))], t


def _chain_args(rung, w, h):
    dst = (rung["width"], rung["height"])
    cabac = rung.get("entropy_cabac", False)
    return dict(dst=None if dst == (w, h) else dst, qp=rung.get("qp", 26), intra_period=rung.get("intra_period", 0),
                entropy=(1 if cabac else 0, rung.get("profile_idc", 0) or 66))


RUNGS_640 = [dict(width=640, height=320, qp=26, entropy_cabac=True, profile_idc=100, intra_period=4), dict(width=320, height=160, qp=28),
             dict(width=480, height=240, qp=30)]


def test_ladder_source_size_rung_not_first():
    """the input size as the last rung: the decoded picture still sits at offset 0 of the step buffer, where the decoder writes it
    and the down-sampler reads it"""
    _need_ref()
    data = open(os.path.join(GOLDEN, "conformance_b", B_VECTORS[2]), "rb").read()
    rungs = [dict(width=320, height=160, qp=28), dict(width=480, height=240, qp=30), dict(width=640, height=320, qp=28)]
    got, _ = _ladder([h264lib.split_access_units(data)], 640, 320, rungs)
    for rung, g in zip(rungs, got):
        assert g[0] == _ref_chain(data, **_chain_args(rung, 640, 320)), rung


@pytest.mark.parametrize("name", B_VECTORS[1:])
def test_ladder_b_vectors_640x320(name):
    """CABAC and CAVLC B pyramids, each twice back to back (a second IDR period), to a full-size CABAC High rung with an intra
    period, a half-size rung and a general-ratio rung: each equals the reference chain and a single-output Transcoder"""
    _need_ref()
    data = open(os.path.join(GOLDEN, "conformance_b", name), "rb").read() * 2
    aus = h264lib.split_access_units(data)
    got, _ = _ladder([aus], 640, 320, RUNGS_640)
    for rung, g in zip(RUNGS_640, got):
        kw = {k: v for k, v in rung.items() if k not in ("width", "height")}
        assert g[0] == _transcode([aus], 640, 320, dst_w=rung["width"], dst_h=rung["height"], **kw)[0], rung
        assert g[0] == _ref_chain(data, **_chain_args(rung, 640, 320)), rung


def test_ladder_b_vector_1024x768():
    _need_ref()
    data = open(os.path.join(GOLDEN, "conformance_b", B_VECTORS[0]), "rb").read()
    rungs = [dict(width=w, height=h, qp=28) for w, h in ((1024, 768), (512, 384), (256, 192), (640, 480))]
    got, _ = _ladder([h264lib.split_access_units(data)], 1024, 768, rungs)
    for rung, g in zip(rungs, got):
        assert g[0] == _ref_chain(data, **_chain_args(rung, 1024, 768)), rung


def test_ladder_qcif_conformance_batch():
    """the QCIF Baseline conformance vectors as one batch of different lengths (sit-outs in the encoders' batches) to 176x144 and
    88x72"""
    _need_ref()
    import wp_rewrite as W
    from openh264_b200.binding import probe_access_unit
    cdir = os.path.join(GOLDEN, "conformance")
    files, streams = [], []
    for f in sorted(os.listdir(cdir)):
        data = open(os.path.join(cdir, f), "rb").read()
        aus = h264lib.split_access_units(data)
        sps = [W.parse_sps(W.unescape(nal[1:]))[1] for _, nal in W.nal_units(aus[0]) if nal[0] & 0x1f == 7]
        if probe_access_unit(aus[0])[:2] == (176, 144) and sps[0]["profile"] == 66:
            files.append((f, data)); streams.append(aus)
    assert len(files) >= 10 and len(set(len(a) for a in streams)) > 1
    rungs = [dict(width=176, height=144, qp=30), dict(width=88, height=72, qp=30)]
    got, _ = _ladder(streams, 176, 144, rungs)
    for rung, g in zip(rungs, got):
        bad = [f for (f, data), b in zip(files, g) if b != _ref_chain(data, **_chain_args(rung, 176, 144))]
        assert not bad, (rung, bad)


def test_ladder_reuses_step_buffers_like_a_single_output():
    """over the doubled B vector the ladder makes no more step buffers than a single-output Transcoder, and all of them are free
    after flush()"""
    from openh264_b200.transcode import Transcoder
    data = open(os.path.join(GOLDEN, "conformance_b", B_VECTORS[2]), "rb").read() * 2
    aus = h264lib.split_access_units(data)
    counts = []
    for kw in (dict(dst_w=320, dst_h=160, qp=28), dict(rungs=RUNGS_640)):
        t = Transcoder(640, 320, 1, **kw)
        for au in aus:
            t.push([au])
        t.flush()
        assert t.allocated >= 1 and len(t.free) == t.allocated and not t.refs, kw
        counts.append(t.allocated)
        t.close()
    assert counts[1] <= counts[0], counts
