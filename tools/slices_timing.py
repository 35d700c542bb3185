"""What several slices per picture cost the batched encoder, on the GPU: S streams of bench.py's synthetic 1080p clip coded with one
slice, with fixed 4 and 8 slices (SM_FIXEDSLCNUM_SLICE), and S streams of the clip down-sampled to 960x540 with one slice and with
one slice per macroblock row (SM_RASTER_SLICE, 34 slices).  Sources are in HBM (b2h264_enc_submit with device pointers), so the
figures leave the host upload out.

Per configuration: resident fps = pictures / (macroblock kernel + deblocking time, from the encoder's CUDA events), and end-to-end
fps = pictures / wall time of submit + collect, one batch at a time (host entropy coding included), both over the timed steps after the warm-up.
Prints the card, its power limit and one JSON line per configuration.  usage: python tools/slices_timing.py [S] [steps] [warmup]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import openh264_b200 as m  # noqa: E402
from openh264_b200.binding import BatchEncoder  # noqa: E402

S = int(sys.argv[1]) if len(sys.argv) > 1 else 256
STEPS = int(sys.argv[2]) if len(sys.argv) > 2 else 8
WARMUP = int(sys.argv[3]) if len(sys.argv) > 3 else 3
FIXED, RASTER = 1, 2
CONFIGS = [(1920, 1080, None), (1920, 1080, (FIXED, 4)), (1920, 1080, (FIXED, 8)), (960, 540, None), (960, 540, (RASTER, 0))]


def half(pic):
    """2:1 down-sampling of a 1920x1080 I420 picture to 960x540 (2x2 means)"""
    y = pic[:bench.W * bench.H].reshape(bench.H, bench.W).astype(np.uint16)
    c = pic[bench.W * bench.H:].reshape(2, bench.H // 2, bench.W // 2).astype(np.uint16)
    ys = (y[0::2, 0::2] + y[1::2, 0::2] + y[0::2, 1::2] + y[1::2, 1::2] + 2) >> 2
    cs = (c[:, 0::2, 0::2] + c[:, 1::2, 0::2] + c[:, 0::2, 1::2] + c[:, 1::2, 1::2] + 2) >> 2
    return np.concatenate([ys.ravel(), cs.ravel()]).astype(np.uint8)


def run(w, h, slices, pics):
    enc = BatchEncoder(w, h, qp=bench.QP, fps=bench.FPS, n_streams=S)
    resolved = enc.set_slices(*slices) if slices else (0, 1, [])
    dev = [m.DeviceArray(p) for p in pics]
    device_us, t_wall, n_bytes = 0.0, 0.0, 0
    for i in range(WARMUP + STEPS):
        ptrs = [dev[(i + s) % len(dev)].ptr for s in range(S)]
        t0 = time.perf_counter()
        enc.submit(ptrs, on_device=True)
        out, _ = enc.collect()
        dt = time.perf_counter() - t0
        if i >= WARMUP:
            t_wall += dt
            us = enc.timing_us()
            device_us += us[0] + us[1]
            n_bytes += sum(len(b) for b in out)
    enc.close()
    n = S * STEPS
    return {"size": f"{w}x{h}", "slice_mode": resolved[0], "slices": resolved[1], "streams": S, "steps": STEPS,
            "resident_fps": round(n / (device_us * 1e-6), 1), "end_to_end_fps": round(n / t_wall, 1),
            "bytes_per_picture": n_bytes // n}


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"gpu": q.stdout.strip()}))
    clip = bench.make_clip(frames=4)
    frames = [np.ascontiguousarray(clip[k * bench.FSZ:(k + 1) * bench.FSZ]) for k in range(4)]
    small = [np.ascontiguousarray(half(f)) for f in frames]
    for w, h, slices in CONFIGS:
        print(json.dumps(run(w, h, slices, frames if w == bench.W else small)), flush=True)


if __name__ == "__main__":
    main()
