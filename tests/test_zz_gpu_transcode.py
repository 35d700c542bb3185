"""Transcoding on the GPU (openh264_b200.transcode.Transcoder): device decode -> [down-sampling] -> device-input encode must give, per
stream, the Annex-B bytes of the reference chain: the reference decoder (pictures in output order) -> [the oracle's down-sampler with
the function CDownsampling::Process picks per plane] -> the reference encoder with the same configuration.
(File name: runs after the other GPU tests.)"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import h264lib
import wp_rewrite as W
from h264lib import ptr

pytestmark = pytest.mark.gpu
ROOT = h264lib.ROOT
GOLDEN = os.path.join(ROOT, "tests", "golden")
B_VECTORS = ["Cisco_Adobe_PDF_sample_a_1024x768_CAVLC_Bframe_9.264", "Cisco_Men_whisper_640x320_CABAC_Bframe_9.264",
             "Cisco_Men_whisper_640x320_CAVLC_Bframe_9.264"]


def _ref_decode(bs):
    """the reference decoder's pictures in output order: (frames, w, h, uint8 array)"""
    R = C.CDLL(h264lib.REFSHIM_SO)
    R.ref_decode.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_double)]
    out = np.zeros(64 << 20, np.uint8)
    w, h, s = C.c_int(), C.c_int(), C.c_double()
    a = np.frombuffer(bs, np.uint8)
    n = R.ref_decode(a.ctypes.data, len(a), out.ctypes.data, out.size, C.byref(w), C.byref(h), C.byref(s))
    assert n > 0
    return n, w.value, h.value, out[:n * w.value * h.value * 3 // 2]


def _orc_scale(yuv, n, sw, sh, dw, dh):
    from openh264_b200.binding import load
    O = h264lib.oracle().lib
    O.orc_downsample.argtypes = [C.c_int, h264lib.u8p, C.c_int, C.c_int, C.c_int, h264lib.u8p, C.c_int, C.c_int, C.c_int]
    O.orc_downsample.restype = None
    out = []
    for f in range(n):
        pic = yuv[f * sw * sh * 3 // 2:(f + 1) * sw * sh * 3 // 2]
        off = 0
        for pl in range(3):
            c = 1 if pl else 0
            pw, ph, qw, qh = sw >> c, sh >> c, dw >> c, dh >> c
            src = np.zeros((ph + 1, pw + 3), np.uint8)          # the 2x2 reads at the last row / column stay inside
            src[:ph, :pw] = pic[off:off + pw * ph].reshape(ph, pw)
            off += pw * ph
            dst = np.zeros((qh, qw), np.uint8)
            O.orc_downsample(load().b2h264_downsample_mode(pw, ph, qw, qh, c), ptr(dst), qw, qw, qh, ptr(src), pw + 3, pw, ph)
            out.append(dst.ravel())
    return np.concatenate(out)


def _ref_chain(bs, dst=None, qp=28, entropy=(0, 66), intra_period=0):
    sys.path.insert(0, GOLDEN)
    from make_encoder_golden import ref_encode
    n, w, h, yuv = _ref_decode(bs)
    dw, dh = dst or (w, h)
    if (dw, dh) != (w, h):
        yuv = _orc_scale(yuv, n, w, h, dw, dh)
    return ref_encode(yuv, dw, dh, n, qp, 30.0, entropy=entropy, intra_period=intra_period)[0]


def _transcode(streams, w, h, **kw):
    from openh264_b200.transcode import Transcoder
    t = Transcoder(w, h, len(streams), **kw)
    got = [b""] * len(streams)
    for k in range(max(len(a) for a in streams)):
        out = t.push([a[k] if k < len(a) else None for a in streams])
        got = [g + o for g, o in zip(got, out)]
    got = [g + o for g, o in zip(got, t.flush())]
    t.close()
    return got


def _need_ref():
    if not h264lib.have_ref():
        pytest.skip("oracle/_ref not present")


def test_transcode_qcif_conformance_batch_baseline():
    """the QCIF Baseline conformance vectors as one batch of different lengths (the encoder sees sit-outs), re-encoded as Baseline
    CAVLC at QP 30"""
    _need_ref()
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
    got = _transcode(streams, 176, 144, qp=30)
    bad = [f for (f, data), g in zip(files, got) if g != _ref_chain(data, qp=30)]
    assert not bad, bad


@pytest.mark.parametrize("names", [B_VECTORS[:1], B_VECTORS[1:]])
def test_transcode_b_frame_vectors_cabac_high(names):
    """B pyramids (output order differs from decoding order), each vector twice back to back (a second IDR period whose counts
    start over while pictures of the first are held), re-encoded as CABAC High with an intra period"""
    _need_ref()
    datas = [open(os.path.join(GOLDEN, "conformance_b", n), "rb").read() * 2 for n in names]
    w, h = (1024, 768) if "1024x768" in names[0] else (640, 320)
    kw = dict(qp=26, entropy_cabac=True, profile_idc=100, intra_period=4)
    got = _transcode([h264lib.split_access_units(d) for d in datas], w, h, **kw)
    for name, d, g in zip(names, datas, got):
        assert g == _ref_chain(d, qp=26, entropy=(1, 100), intra_period=4), name


@pytest.mark.parametrize("name,src,dst", [(B_VECTORS[2], (640, 320), (320, 160)), (B_VECTORS[0], (1024, 768), (640, 480))])
def test_transcode_down_scaled(name, src, dst):
    """a dyadic (half: mode 0 for every plane) and a non-dyadic down-scale (general ratio: mode 3 for luma, 4 for chroma)"""
    _need_ref()
    data = open(os.path.join(GOLDEN, "conformance_b", name), "rb").read()
    got = _transcode([h264lib.split_access_units(data)], *src, dst_w=dst[0], dst_h=dst[1], qp=28)
    assert got[0] == _ref_chain(data, dst=dst, qp=28)
