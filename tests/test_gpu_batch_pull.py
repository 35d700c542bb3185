"""GPU: the pulled batches of the encode kernel's short stages (enc_kernels.cu, run_stages, ENC_PULL).

A full batch of list A (skip test) or Bs (skip-candidate intra check) claims up to ENC_PULL x ENC_WPC tasks, and a warp that
finishes its task takes the next one of the block.  A list only holds more than ENC_WPC ready tasks when many streams are in
flight, which the other encoder tests never reach.  This test encodes 96 streams of a clip with a reference golden, asserts
from the kernel's batch statistics that list A ran batches of more than ENC_WPC tasks, and requires every stream's
bitstream to equal the golden byte for byte.

The statistics are switched on by B2H264_ENC_STATS when the library first encodes, so the encode runs in a process of its own."""
import hashlib
import json
import os
import subprocess
import sys

import pytest

import h264lib

pytestmark = pytest.mark.gpu
ROOT = h264lib.ROOT
ENC_WPC = 23                       # worker warps per CTA of k_encode_mbs (enc_kernels.cu)
KEY = "640x360_n5_qp30_fps30"      # tests/golden/encoder.json
STREAMS = 96

_ENCODE = r"""
import ctypes as C, hashlib, json, sys
import numpy as np
import h264lib
from openh264_b200.binding import BatchEncoder, lib
w, h, n, qp, fps, S = json.loads(sys.argv[1])
yuv = h264lib.synth_clip(w, h, n)
fsz = w * h * 3 // 2
L = lib(0)
enc = BatchEncoder(w, h, qp=qp, fps=fps, n_streams=S)
outs = [[] for _ in range(S)]
for f in range(n):
    bs, _ = enc.encode([np.ascontiguousarray(yuv[f * fsz:(f + 1) * fsz])] * S)
    for s in range(S):
        outs[s].append(bytes(bs[s]))
enc.close()
bt = np.zeros((6, 3), np.uint64)
assert L.b2h264_debug_batch_stats(C.c_void_p(bt.ctypes.data), 0) == 0
fs = np.zeros(8 * 128 * 2, np.uint64)
nl, wp = C.c_int(), C.c_int()
L.b2h264_debug_fill_stats.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int]
assert L.b2h264_debug_fill_stats(fs.ctypes.data, C.byref(nl), C.byref(wp), 0) == 0
fs = fs[:nl.value * (wp.value + 1) * 2].reshape(nl.value, wp.value + 1, 2)
print(json.dumps({"sizes": [[len(b) for b in o] for o in outs],
                  "sha1": [hashlib.sha1(b"".join(o)).hexdigest() for o in outs],
                  "batches": bt[:, 0].tolist(), "tasks": bt[:, 1].tolist(),
                  "fill": fs[:, :, 0].tolist()}))
"""


def test_pulled_batches_keep_every_bitstream():
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "encoder.json")))[KEY]
    w, h = map(int, KEY.split("_")[0].split("x"))
    n, qp, fps = int(KEY.split("_n")[1].split("_")[0]), int(KEY.split("_qp")[1].split("_")[0]), float(KEY.split("_fps")[1])
    assert hashlib.sha1(h264lib.synth_clip(w, h, n).tobytes()).hexdigest() == gold["yuv_sha1"]
    env = dict(os.environ, B2H264_ENC_STATS="1",
               PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    r = subprocess.run([sys.executable, "-s", "-c", _ENCODE, json.dumps([w, h, n, qp, fps, STREAMS])],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    # list A (index 0) ran batches of more than ENC_WPC tasks, and those batches hold the tasks the statistics count
    fill_a = res["fill"][0]
    assert sum(fill_a[ENC_WPC + 1:]) > 0, f"no pulled batch on list A: fill histogram {fill_a}"
    assert sum(i * c for i, c in enumerate(fill_a)) == res["tasks"][0]
    assert res["tasks"][0] == STREAMS * (n - 1) * (w // 16) * ((h + 15) // 16)     # every P macroblock runs stage A once
    for s in range(STREAMS):
        assert res["sizes"][s] == gold["frame_bytes"], f"stream {s}"
        assert res["sha1"][s] == gold["sha1"], f"stream {s}"
