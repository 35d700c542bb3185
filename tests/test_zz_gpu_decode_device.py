"""Decoder output into device memory (include/b2h264_codec.h b2h264_dec_decode_device, BatchDecoder.decode_device): the pictures
k_dec_output writes into HBM must be byte for byte those the host output path gives (b2h264_dec_decode2 / decode3) and the reference's
published SHA-1 in output order, at any destination alignment and crop window, with decode3's per-stream status; the call is
asynchronous and ordered on the caller's stream.  (File name: runs after the other GPU tests.)"""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest

import h264lib
import wp_rewrite as W

pytestmark = pytest.mark.gpu
ROOT = h264lib.ROOT
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _hashes():
    return dict((p.split("/")[-1], s) for p, s in json.load(open(os.path.join(GOLDEN, "reference_decoder_hashes.json")))["pairs"])


def _units(d, name):
    return h264lib.split_access_units(open(os.path.join(GOLDEN, d, name), "rb").read())


def _vectors():
    """(directory, file, published SHA-1 of the pictures in output order) of every committed vector the decoder takes"""
    tab = _hashes()
    out = [("conformance", f, tab[f]) for f in sorted(os.listdir(os.path.join(GOLDEN, "conformance"))) if f in tab]
    out += [("conformance_b", f, tab[f]) for f in sorted(os.listdir(os.path.join(GOLDEN, "conformance_b"))) if f in tab]
    out += [("conformance_b", f, g["sha1"]) for f, g in sorted(json.load(open(os.path.join(GOLDEN, "high_profile_prefix.json"))).items())]
    return out


def _size(aus):
    from openh264_b200.binding import probe_access_unit
    return probe_access_unit(aus[0])[:2]


def _output_order_sha(pics_with_order):
    """pictures with (picture order count, flags, reorder depth) in decoding order -> SHA-1 in output order (bumping per IDR period)"""
    from openh264_b200.transcode import OutputOrder
    q, hs = OutputOrder(), hashlib.sha1()
    for p, (poc, flags, depth) in pics_with_order:
        for o in q.push(p, poc, flags, depth):
            hs.update(o)
    for o in q.drain():
        hs.update(o)
    return hs.hexdigest()


def test_decode_device_qcif_conformance_batch():
    """the QCIF vectors as ONE batch (the slot array widens mid-run): every picture equals the host path's, every stream its SHA-1"""
    import torch
    from openh264_b200.binding import BatchDecoder
    items = [(f, sha, _units(d, f)) for d, f, sha in _vectors() if d == "conformance"]
    items = [t for t in items if _size(t[2]) == (176, 144)]
    assert len(items) >= 17
    n = len(items)
    host, dev = BatchDecoder(176, 144, n_streams=n), BatchDecoder(176, 144, n_streams=n)
    out = torch.full((n, dev.frame_bytes), 0x5a, dtype=torch.uint8, device="cuda")
    hashes = [hashlib.sha1() for _ in items]
    for k in range(max(len(t[2]) for t in items)):
        units = [t[2][k] if k < len(t[2]) else None for t in items]
        want = [None if p is None else p.copy() for p in host.decode2(units)]
        _, st = dev.decode_device(units, out)
        got = out.cpu().numpy()
        for i in range(n):
            assert st[i] == (1 if want[i] is not None else 0), (items[i][0], k)
            if want[i] is not None:
                assert np.array_equal(got[i], want[i]), (items[i][0], k)
                hashes[i].update(got[i].tobytes())
    host.close(); dev.close()
    bad = [items[i][0] for i in range(n) if hashes[i].hexdigest() != items[i][1]]
    assert not bad, bad


def test_decode_device_other_vectors():
    """the other sizes, the B-frame vectors, the High-profile prefixes and the 1080p prefix: device pictures equal the host path's,
    and give the published SHA-1 in output order"""
    import torch
    from openh264_b200.binding import BatchDecoder
    ran, bad = 0, []
    for d, name, sha in _vectors():
        aus = _units(d, name)
        w, h = _size(aus)
        if d == "conformance" and (w, h) == (176, 144):
            continue
        host, dev = BatchDecoder(w, h), BatchDecoder(w, h)
        out = torch.empty((1, dev.frame_bytes), dtype=torch.uint8, device="cuda")
        seq = []
        for au in aus:
            want = host.decode2([au])[0]
            _, st = dev.decode_device([au], out)
            assert st == [1], name
            got = out[0].cpu().numpy()
            assert np.array_equal(got, want), name
            seq.append((got.tobytes(), dev.picture_order(0)))
        host.close(); dev.close()
        if d == "conformance":                              # no reordering in these: decoding order is output order
            ok = hashlib.sha1(b"".join(p for p, _ in seq)).hexdigest() == sha
        else:
            ok = _output_order_sha(seq) == sha
        if not ok:
            bad.append(name)
        ran += 1
    assert not bad, bad
    assert ran >= 8


# ---- crop windows: a stream whose SPS crops on all four sides ------------------------------------------------------------

def _recrop(bs, left, right, top, bottom):
    """rewrites every SPS of a 4:2:0 frame stream to crop (left, right, top, bottom) chroma samples (2 luma samples each)"""
    out = []
    for sc, nal in W.nal_units(bs):
        if nal[0] & 0x1f != 7:
            out.append(sc + nal)
            continue
        r = W.Reader(W.unescape(nal[1:]))
        W.parse_sps(W.unescape(nal[1:]))                    # refuses what it cannot rewrite
        profile = r.u(8)
        r.u(16)
        r.ue()
        assert profile in (66, 77, 88)
        r.ue()
        poc_type = r.ue()
        if poc_type == 0:
            r.ue()
        elif poc_type == 1:
            r.u(1); r.se(); r.se()
            for _ in range(r.ue()):
                r.se()
        r.ue(); r.u(1); r.ue(); r.ue()
        assert r.u(1) == 1                                 # frame_mbs_only_flag
        r.u(1)                                             # direct_8x8_inference_flag
        head = r.bits[:r.pos]
        if r.u(1):
            for _ in range(4):
                r.ue()
        rest = r.bits[r.pos:].rstrip("0")[:-1]            # VUI and the rest, without the stop bit
        bits = head + "1" + "".join(W.ue_bits(v) for v in (left, right, top, bottom)) + rest + "1"
        bits += "0" * (-len(bits) % 8)
        out.append(sc + nal[:1] + W.escape(W.to_bytes(bits)))
    return b"".join(out)


def _cropped_stream():
    """a 176x144 stream of the GPU encoder re-cropped to 172x134 at an odd offset: (units, uncropped units, window)"""
    from openh264_b200.binding import BatchEncoder
    w, h, n = 176, 144, 4
    yuv = h264lib.synth_clip(w, h, n, seed=31, noise=6)
    fsz = w * h * 3 // 2
    enc = BatchEncoder(w, h, qp=24, fps=30.0)
    aus = [enc.encode([yuv[f * fsz:(f + 1) * fsz]])[0][0] for f in range(n)]
    enc.close()
    win = (1, 1, 3, 2)                                     # left, right, top, bottom in chroma samples
    return [_recrop(a, *win) for a in aus], aus, win


def _crop(pic, w, h, win):
    l, r, t, b = win
    y = pic[:w * h].reshape(h, w)[2 * t:h - 2 * b, 2 * l:w - 2 * r]
    u = pic[w * h:w * h * 5 // 4].reshape(h // 2, w // 2)[t:h // 2 - b, l:w // 2 - r]
    v = pic[w * h * 5 // 4:].reshape(h // 2, w // 2)[t:h // 2 - b, l:w // 2 - r]
    return np.concatenate([y.ravel(), u.ravel(), v.ravel()])


def test_decode_device_alignment_crop_and_guards():
    """destinations at byte offsets 1..15 (and 0) inside one tensor, guard bytes around every picture: the pictures are exact and
    the guards untouched, for a QCIF vector (rows of 176 and 88 bytes; chroma stride 120), a stream cropped on all four sides and
    the 1080p prefix (cropped at the bottom)"""
    import torch
    from openh264_b200.binding import BatchDecoder
    cropped, plain, win = _cropped_stream()
    cases = [(_units("conformance", "BA_MW_D.264")[:6], None), (cropped, (plain, win)),
             (_units("conformance_b", "VID_1920x1080_cabac_temporal_direct_first10.264")[:3], None)]
    for aus, crop in cases:
        w, h = _size(aus)
        n = 16
        host = BatchDecoder(176, 144) if crop else BatchDecoder(w, h)
        dev = BatchDecoder(w, h, n_streams=n)
        fsz = dev.frame_bytes
        slot = (fsz + 64 + 15) // 16 * 16                     # each picture at 32 + its offset inside a 16-aligned slot
        big = torch.full((n * slot + 64,), 0xa5, dtype=torch.uint8, device="cuda")
        offs = [32 + k for k in range(n)]                     # k = 0..15: every alignment
        rows = [big[i * slot + offs[i]:i * slot + offs[i] + fsz] for i in range(n)]
        for k, au in enumerate(aus):
            ref = host.decode2([crop[0][k] if crop else au])[0]
            want = _crop(ref, 176, 144, crop[1]) if crop else ref
            _, st = dev.decode_device([au] * n, rows)
            assert st == [1] * n
            whole = big.cpu().numpy()
            for i in range(n):
                assert np.array_equal(whole[i * slot + offs[i]:i * slot + offs[i] + fsz], want), (w, h, k, "offset", offs[i] % 16)
            mask = np.ones(whole.size, bool)
            for i in range(n):
                mask[i * slot + offs[i]:i * slot + offs[i] + fsz] = False
            assert (whole[mask] == 0xa5).all(), (w, h, k, "guard bytes written")
        host.close(); dev.close()


def test_decode_device_status_sentinels_and_refusals():
    """the scenario of test_gpu_decoder_per_stream_status_and_slot_reuse through decode_device: status equals decode3's, the
    destinations of streams that sat out or failed keep their sentinel fill; host destinations are refused with -1"""
    if not h264lib.have_ref():
        pytest.skip("oracle/_ref not present")
    import torch
    from openh264_b200.binding import BatchDecoder, vp
    from test_gpu_decoder import ref_streams
    w, h, n = 176, 144, 5
    streams = ref_streams(w, h, n, 28, (11, 12))
    high_sps = b"\x00\x00\x00\x01\x67\x6e\x00\x1f\xac\xd9\x40\x50\x05\xbb\x01\x10"
    host, dev = BatchDecoder(w, h, n_streams=4), BatchDecoder(w, h, n_streams=4)

    def step(units):
        pics, want_st = host.decode3(units)
        pics = [None if p is None else p.copy() for p in pics]
        out = torch.full((4, dev.frame_bytes), 0x3c, dtype=torch.uint8, device="cuda")
        _, st = dev.decode_device(units, out)
        assert st == want_st
        got = out.cpu().numpy()
        for s in range(4):
            if st[s] == 1:
                assert np.array_equal(got[s], pics[s])
            else:
                assert (got[s] == 0x3c).all(), ("destination of a stream without a picture was written", s, st)
        return st

    for f in range(n):
        a1 = streams[1][1][f] if f != 2 else streams[1][1][f][:len(streams[1][1][f]) // 2]
        st = step([streams[0][1][f], a1, high_sps if f == 0 else None, None])
        assert st[0] == 1 and (st[1] == 1) == (f < 2)
    host.reset_stream(1); dev.reset_stream(1)
    for f in range(n):
        assert step([None, streams[0][1][f], None, None]) == [0, 1, 0, 0]
    # host memory (pageable and page-locked) is refused before anything runs; so is a NULL destination of a stream with a unit
    L = dev.L
    au = np.frombuffer(streams[0][1][0], np.uint8)
    aus = (vp * 4)(au.ctypes.data, None, None, None)
    nb = (C.c_int32 * 4)(len(au), 0, 0, 0)
    st = (C.c_int32 * 4)()
    pageable = np.zeros(dev.frame_bytes, np.uint8)
    pinned = torch.zeros(dev.frame_bytes, dtype=torch.uint8).pin_memory()
    for p in (pageable.ctypes.data, pinned.data_ptr(), None):
        assert L.b2h264_dec_decode_device(dev.h, aus, nb, (vp * 4)(p, None, None, None), st) == -1
    assert not pageable.any() and not pinned.any()
    host.close(); dev.close()


def test_decode_device_asynchronous_and_ordered():
    """eight calls back to back into eight tensors with one synchronize at the end equal the synchronous pictures; a host-output
    call between device calls is still exact; a torch op issued right after a call on the same stream reads finished pictures"""
    import torch
    from openh264_b200.binding import BatchDecoder
    name = "VID_1920x1080_cabac_temporal_direct_first10.264"
    aus = _units("conformance_b", name)
    w, h = _size(aus)
    host = BatchDecoder(w, h, n_streams=2)
    want = [[p.copy() for p in host.decode2([au, au])] for au in aus]
    host.close()
    dev = BatchDecoder(w, h, n_streams=2)
    outs = [torch.empty((2, dev.frame_bytes), dtype=torch.uint8, device="cuda") for _ in range(8)]
    for k in range(8):
        dev.decode_device([aus[k], aus[k]], outs[k])
    torch.cuda.synchronize()
    for k in range(8):
        for s in range(2):
            assert np.array_equal(outs[k][s].cpu().numpy(), want[k][s]), (k, s)
    # picture 8 through the host path right after nothing was synchronized, picture 9 on the device again
    out9 = torch.empty((2, dev.frame_bytes), dtype=torch.uint8, device="cuda")
    dev.decode_device([aus[0], None], out9)                 # stream 0 restarts at its IDR: queued work ahead of the host call
    pics = dev.decode2([aus[1], aus[8]])
    assert np.array_equal(pics[0], want[1][0]) and np.array_equal(pics[1], want[8][1])
    _, st = dev.decode_device([aus[2], aus[9]], out9)
    # a reduction queued right behind the call, on the same stream, without a synchronize in between
    sums = out9.to(torch.int64).sum(dim=1).cpu().numpy()
    assert st == [1, 1]
    assert sums[1] == int(want[9][1].astype(np.int64).sum())
    assert np.array_equal(out9[1].cpu().numpy(), want[9][1])
    assert np.array_equal(out9[0].cpu().numpy(), want[2][0])
    # the caller's stream: the decoder follows torch.cuda.current_stream()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        dev.reset_stream(0)
        o = torch.empty((2, dev.frame_bytes), dtype=torch.uint8, device="cuda")
        dev.decode_device([aus[0], None], o)
        first = o[0].clone()
    side.synchronize()
    assert np.array_equal(first.cpu().numpy(), want[0][0])
    dev.close()


def test_encoder_device_input_equals_host_input():
    """b2h264_enc_submit with src_on_device = 1: the same pictures from HBM and from host memory give the same bitstreams"""
    import torch
    from openh264_b200.binding import BatchEncoder
    w, h, n = 320, 192, 6
    fsz = w * h * 3 // 2
    clips = [h264lib.synth_clip(w, h, n, seed=s, noise=5) for s in (41, 42)]
    dclips = [torch.from_numpy(c).cuda() for c in clips]
    torch.cuda.synchronize()
    for kw in ({}, {"entropy_cabac": True, "intra_period": 3}):
        a = BatchEncoder(w, h, qp=27, n_streams=2, **kw)
        b = BatchEncoder(w, h, qp=27, n_streams=2, **kw)
        for f in range(n):
            host = a.encode([c[f * fsz:(f + 1) * fsz] for c in clips])
            b.submit([dc[f * fsz:(f + 1) * fsz].data_ptr() for dc in dclips], on_device=True)
            assert b.collect() == host, (kw, f)
        a.close(); b.close()
