"""Writes tests/golden/explicit_bipred.json: what the UNMODIFIED reference decoder (oracle/_ref, ISVCDecoder::DecodeFrameNoDelay +
flush behind ref_decode) makes of the committed B-frame vectors once tests/wp_rewrite.py has given their B slices explicit weights
(weighted_bipred_idc 1, a seeded pred_weight_table in every B slice header).  Only the seeds and the hashes are committed; the
rewritten streams are made again from the committed vectors wherever the tests run.

    python tests/golden/make_explicit_bipred_golden.py      (needs oracle/_ref, i.e. a build with the reference's sources)
"""
import ctypes as C
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
import h264lib  # noqa: E402
import wp_rewrite  # noqa: E402

# Main profile, spatial direct, no weights (the Cisco vectors, CAVLC and CABAC); High profile, temporal direct, weighted P slices,
# implicit B weights and three list-0 references (the two VID_1280x544 prefixes)
SOURCES = ["Cisco_Men_whisper_640x320_CAVLC_Bframe_9.264", "Cisco_Men_whisper_640x320_CABAC_Bframe_9.264",
           "Cisco_Adobe_PDF_sample_a_1024x768_CAVLC_Bframe_9.264", "VID_1280x544_cabac_temporal_direct_first14.264",
           "VID_1280x544_cavlc_temporal_direct_first14.264"]
SEEDS = [1, 2, 3]


def ref_decode(bs):
    R = C.CDLL(h264lib.REFSHIM_SO)
    R.ref_decode.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_double)]
    a = np.frombuffer(bs, np.uint8)
    out = np.zeros(64 << 20, np.uint8)
    W, H, s = C.c_int(), C.c_int(), C.c_double()
    n = R.ref_decode(a.ctypes.data, len(a), out.ctypes.data, out.size, C.byref(W), C.byref(H), C.byref(s))
    return n, W.value, H.value, hashlib.sha1(out[:max(n, 0) * W.value * H.value * 3 // 2].tobytes()).hexdigest()


def main():
    jobs = []
    for name in SOURCES:
        src = open(os.path.join(HERE, "conformance_b", name), "rb").read()
        for seed in SEEDS:
            n, w, h, sha = ref_decode(wp_rewrite.rewrite(src, seed))
            assert n > 0, (name, seed, n)
            jobs.append({"source": name, "seed": seed, "pictures": n, "width": w, "height": h, "sha1": sha})
            print(jobs[-1])
    json.dump({"jobs": jobs}, open(os.path.join(HERE, "explicit_bipred.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
