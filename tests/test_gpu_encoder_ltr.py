"""Long-term references through layer 2 (BatchEncoder / b2h264_enc_*): several streams of one batched encoder play the receiver
scripts of tests/golden/ltr.json, with feedback for some streams only and streams that sit calls out.  Every stream's bitstream
equals the reference encoder's; decoded by the GPU decoder it equals b2h264_enc_get_recon picture by picture and the reference
decoder's pictures (CAVLC streams; see test_batch_with_partial_feedback); and a recovery picture's slice header names a
long-term picture."""
import hashlib
import json
import os

import numpy as np
import pytest

import ltr_cases as L
from openh264_b200.binding import BatchDecoder, BatchEncoder

GOLD = json.load(open(os.path.join(L.ROOT, "tests", "golden", "ltr.json")))
FSZ = L.W * L.H * 3 // 2


def clip_pictures(n):
    data = np.fromfile(L.CLIP, np.uint8)
    k = len(data) // FSZ
    return [data[(i % k) * FSZ:(i % k + 1) * FSZ].copy() for i in range(n)]


class Receiver:
    """one stream's script, with the driver's idr / frame-number tokens resolved from what the stream produced so far"""

    def __init__(self, script):
        self.ev = [s.split() for s in script]
        self.fn, self.idr_id, self.next_fn = [], 0, 0

    def frame_no(self, t):
        if t[0] == "p":
            k = int(t[1:])
            return self.fn[-k] if 1 <= k <= len(self.fn) else -1
        return int(t)

    def idr_no(self, t):
        return self.idr_id if t == "cur" else self.idr_id - 1 if t == "old" else int(t)

    def before(self, enc, s, i):
        for e in self.ev:
            if int(e[0]) != i:
                continue
            if e[1] == "idr":
                enc.force_idr(s)
            elif e[1] == "period":
                enc.ltr_mark_period(s, int(e[2]))
            elif e[1] == "rr":
                enc.ltr_recovery_request(s, self.idr_no(e[3]), self.frame_no(e[4]), self.frame_no(e[5]), int(e[2]))
            elif e[1] == "mf":
                enc.ltr_marking_feedback(s, self.idr_no(e[3]), self.frame_no(e[4]), int(e[2]) == 4)

    def after(self, idr):
        if idr:
            self.idr_id, self.next_fn = (self.idr_id + 1) % 65536, 0
        self.fn.append(self.next_fn)
        self.next_fn = self.next_fn + 1 if self.next_fn < 32767 else 0


def encoder_for(cfg, n_streams):
    cabac, cx, nref, ltr, period, _ = cfg
    return BatchEncoder(L.W, L.H, qp=L.QP, fps=30.0, n_streams=n_streams, complexity_low=cx == L.LOW, entropy_cabac=bool(cabac),
                        num_ref_frames=nref, ltr=bool(ltr), ltr_mark_period=period)


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in sorted(GOLD["cases"]) if n.startswith("ltr_")])
def test_batch_with_partial_feedback(name):
    """stream 0 plays the script on every call; stream 1 plays it too but sits out every third call; stream 2 gets the same
    pictures and no feedback at all (it has no golden: it is checked against the decoder only)"""
    gold = GOLD["cases"][name]
    n = gold["config"][5]
    pics = clip_pictures(n)
    enc = encoder_for(gold["config"], 3)
    assert enc.references()[2:] == (2, 4)
    rx = [Receiver(gold["script"]), Receiver(gold["script"]), Receiver([])]
    nxt = [0, 0, 0]
    out = [[], [], []]
    recon = [[], [], []]
    call = 0
    while min(nxt) < n:
        take = [nxt[0] < n, nxt[1] < n and (call % 3 != 2 or nxt[0] == n), nxt[2] < n]
        for s in range(3):
            if take[s]:
                rx[s].before(enc, s, nxt[s])
        aus, ft = enc.encode([pics[nxt[s]] if take[s] else None for s in range(3)])
        for s in range(3):
            if take[s]:
                assert ft[s] in (1, 2, -1)
                if ft[s] > 0:                 # -1: the picture was dropped (no confirmed long-term picture to recover from)
                    out[s].append(bytes(aus[s]))
                    rx[s].after(ft[s] == 1)
                    recon[s].append(enc.recon(s))
                else:
                    assert aus[s] == b""
                nxt[s] += 1
            else:
                assert aus[s] == b"" and ft[s] == 0
        call += 1
    enc.close()
    for s in (0, 1):
        bs = b"".join(out[s])
        assert hashlib.sha1(bs).hexdigest() == gold["sha1"], f"stream {s}"
        assert L.ref_syntax(bs) == gold["syntax"]
    # decoded by the GPU decoder: the encoder's reconstruction, and (streams 0, 1) the reference decoder's pictures
    decoded = [[], [], []]
    for s in range(3):
        dec = BatchDecoder(L.W, L.H, n_streams=1)
        for i, au in enumerate(out[s]):
            got = dec.decode([au])[0]
            assert np.array_equal(got, recon[s][i]), f"stream {s} picture {i}"
            decoded[s].append(hashlib.sha1(got.tobytes()).hexdigest())
        dec.close()
    # The two CABAC (High profile) LTR streams: the reference decoder's pictures differ from the reference ENCODER's own
    # reconstruction (a frame-dump build of the reference shows it from picture 6 on, the first P picture that predicts from a
    # long-term picture marked by MMCO 6), so they cannot serve as an independent check there.  The GPU decoder agrees with the
    # encoders' reconstruction; that it disagrees with the reference decoder on these streams is a decoder parity gap
    # (DESIGN.md §6).  The CAVLC streams agree with the reference decoder picture for picture.
    if not gold["config"][0]:
        for s in (0, 1):
            assert decoded[s] == gold["decoded_sha1"]


@pytest.mark.gpu
def test_recovery_picture_names_long_term_picture():
    """after a valid recovery request the next P picture's ref_pic_list_modification is idc 2 (long_term_pic_num)"""
    gold = GOLD["cases"]["ltr_p1_cavlc_low"]
    n = gold["config"][5]
    pics = clip_pictures(n)
    enc = encoder_for(gold["config"], 1)
    rx = Receiver(gold["script"])
    out, requested, dropped = [], [], 0
    for i in range(n):
        rx.before(enc, 0, i)
        req = any(e[0] == str(i) and e[1] == "rr" and e[3] == "cur" and e[4] != "-1" and e[5] != "-1" for e in rx.ev)
        aus, ft = enc.encode([pics[i]])
        if ft[0] < 0:                         # dropped: no confirmed long-term picture, and the next picture is an IDR
            dropped += 1
            continue
        requested.append(req)
        out.append(bytes(aus[0]))
        rx.after(ft[0] == 1)
    enc.close()
    syn = L.ref_syntax(b"".join(out))
    assert syn == gold["syntax"] and dropped == gold["log"].count(" failed ")
    hits = [i for i in range(len(syn)) if requested[i] and not syn[i][0]]
    assert hits
    for i in hits:
        assert syn[i][2][0][0] == 2, f"picture {i}: {syn[i]}"


@pytest.mark.gpu
def test_reset_stream_restores_marking_period():
    """a marking period set on a stream does not survive b2h264_enc_reset_stream (what the ISVCEncoder broker does when a slot
    changes owner): the next owner codes with the encoder's own period and produces the golden bitstream"""
    gold = GOLD["cases"]["ltr_p3_cabac_low"]
    n = gold["config"][5]
    pics = clip_pictures(n)
    enc = encoder_for(gold["config"], 1)
    enc.ltr_mark_period(0, 1)
    for i in range(4):                        # a previous owner's pictures, with its own period
        enc.encode([pics[i]])
    enc.reset_stream(0)
    rx = Receiver(gold["script"])
    out = []
    for i in range(n):
        rx.before(enc, 0, i)
        aus, ft = enc.encode([pics[i]])
        if ft[0] > 0:
            out.append(bytes(aus[0]))
            rx.after(ft[0] == 1)
    enc.close()
    assert hashlib.sha1(b"".join(out)).hexdigest() == gold["sha1"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in sorted(GOLD["cases"]) if n.startswith("off_")])
def test_reference_count_without_ltr(name):
    """iNumRefFrame 1..4 / AUTO with LTR off: the reference's bitstream, two pictures per stream on the device"""
    gold = GOLD["cases"][name]
    n = gold["config"][5]
    pics = clip_pictures(n)
    enc = encoder_for(gold["config"], 2)
    assert enc.references()[3] == 2
    rx = [Receiver(gold["script"]), Receiver(gold["script"])]
    out = [[], []]
    for i in range(n):
        for s in range(2):
            rx[s].before(enc, s, i)
        aus, ft = enc.encode([pics[i], pics[i]])
        for s in range(2):
            out[s].append(bytes(aus[s]))
            rx[s].after(ft[s] == 1)
    enc.close()
    for s in range(2):
        assert hashlib.sha1(b"".join(out[s])).hexdigest() == gold["sha1"]
