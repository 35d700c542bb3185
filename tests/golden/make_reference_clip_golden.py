"""Generates tests/golden/reference_clips.json, tests/golden/clips/*.yuv.gz and tests/golden/ref_CiscoVT2people_320x192_qp28.264
from the unmodified reference (oracle/_ref) and its res/ clips, so that the tests that compare with the reference on its own
clips run without it:
  encoder: frame sizes + SHA-1 of the reference encoder's bitstream per (clip, pictures, QP, entropy) case, and the SHA-1 of
           the clip pictures it was given (the small clips' first pictures are committed gzip-compressed under clips/)
  decoder: the reference encoder's stream of its own 320x192 clip and the SHA-1 of what the reference decoder makes of it
  python tests/golden/make_reference_clip_golden.py <reference source directory>"""
import ctypes as C
import gzip
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import h264lib  # noqa: E402
from make_encoder_golden import ref_encode  # noqa: E402

# (clip, width, height, pictures, QP, fps, entropy): the cases of tests/test_encoder_emu.py
OWN = [("CiscoVT2people_320x192_12fps.yuv", 320, 192, 9, qp, 12.0, (0, 66)) for qp in (26, 34)]
OTHER = [("Cisco_Absolute_Power_1280x720_30fps.yuv", 1280, 720, 2, 30, 30.0, (0, 66)),
         ("CiscoVT2people_160x96_6fps.yuv", 160, 96, 5, 24, 30.0, (0, 66)),
         ("Static_152_100.yuv", 152, 100, 8, 28, 30.0, (0, 66))]
CABAC = [(c, w, h, n, qp, fps, (1, prof)) for (c, w, h, n, qp, fps) in
         [("CiscoVT2people_160x96_6fps.yuv", 160, 96, 5, 24, 30.0), ("Static_152_100.yuv", 152, 100, 8, 28, 30.0)] for prof in (0, 77)]
COMMITTED_PREFIXES = {"CiscoVT2people_160x96_6fps.yuv": 5, "Static_152_100.yuv": 8}      # pictures; the 1280x720 clip is too large


def case_key(c, w, h, n, qp, fps, entropy):
    return "%s_n%d_qp%d_fps%g_entropy%d_profile%d" % (c, n, qp, fps, entropy[0], entropy[1])


def main(ref_dir):
    assert h264lib.have_ref(), "build oracle/_ref first (make -f oracle/Makefile.ref)"
    res = os.path.join(ref_dir, "res")
    out = {"encoder": {}, "decoder": {}}
    os.makedirs(os.path.join(HERE, "clips"), exist_ok=True)
    for c, n in COMMITTED_PREFIXES.items():
        w, h = {"CiscoVT2people_160x96_6fps.yuv": (160, 96), "Static_152_100.yuv": (152, 100)}[c]
        data = open(os.path.join(res, c), "rb").read()[:n * w * h * 3 // 2]
        with gzip.GzipFile(os.path.join(HERE, "clips", "%s.first%d.gz" % (c, n)), "wb", mtime=0) as f:
            f.write(data)
    for (c, w, h, n, qp, fps, entropy) in OWN + OTHER + CABAC:
        yuv = np.fromfile(os.path.join(res, c), dtype=np.uint8, count=n * w * h * 3 // 2)
        bs, fb, _ = ref_encode(yuv, w, h, n, qp, fps, entropy=entropy)
        out["encoder"][case_key(c, w, h, n, qp, fps, entropy)] = {"clip_sha1": hashlib.sha1(yuv.tobytes()).hexdigest(),
                                                                 "frame_bytes": list(fb), "sha1": hashlib.sha1(bytes(bs)).hexdigest()}
    # decoder: the reference encoder's stream of its own clip (9 pictures, QP 28, 12 fps), decoded by the reference decoder
    yuv = np.fromfile(os.path.join(res, "CiscoVT2people_320x192_12fps.yuv"), dtype=np.uint8)
    bs = bytes(ref_encode(yuv, 320, 192, 9, 28, 12.0)[0])
    open(os.path.join(HERE, "ref_CiscoVT2people_320x192_qp28.264"), "wb").write(bs)
    R = C.CDLL(h264lib.REFSHIM_SO)
    R.ref_decode.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_double)]
    pics = np.zeros(16 << 20, np.uint8)
    a = np.frombuffer(bs, np.uint8)
    w_, h_, s_ = C.c_int(), C.c_int(), C.c_double()
    nr = R.ref_decode(a.ctypes.data, len(a), pics.ctypes.data, pics.size, C.byref(w_), C.byref(h_), C.byref(s_))
    out["decoder"]["ref_CiscoVT2people_320x192_qp28.264"] = {
        "pictures": nr, "width": w_.value, "height": h_.value,
        "sha1": hashlib.sha1(pics[:nr * w_.value * h_.value * 3 // 2].tobytes()).hexdigest()}
    json.dump(out, open(os.path.join(HERE, "reference_clips.json"), "w"), indent=1, sort_keys=True)


if __name__ == "__main__":
    main(sys.argv[1])
