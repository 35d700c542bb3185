"""The transcoding ladder timed on the GPU (bench.py's decode workload: S copies of a 1080p Baseline stream of this library's encoder,
one access unit per stream per call, built as tools/transcode_timing.py builds it).

(a) input pictures/s of a 4-rung ladder (1920x1080 QP 26, 1280x720 QP 28: general ratio, 960x540 QP 30: half, 640x360 QP 32: one
    third) in one Transcoder, against four single-output Transcoders, one per rung, run one after another on the same inputs (their
    times add up: each parses and decodes every input again); alternating, two runs each;
(b) the kernel time of one b2h264_k_downsample_ladder launch for the three down-scaled rungs against the nine b2h264_k_downsample
    launches (one per rung and plane) it replaces (torch.profiler, a run of its own), with its algorithmic bytes (per destination
    sample: 4 source bytes + 1 destination byte in every mode, k_vpp.cu) against 3.35 TB/s.
Prints the card, its power limit and clocks, and one JSON line per figure.  usage: python tools/ladder_timing.py [S]"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402
import torch  # noqa: E402
from openh264_b200.binding import DsPlane, check, lib  # noqa: E402
from openh264_b200.transcode import Transcoder, ladder_layout  # noqa: E402
from transcode_timing import N_AU, emit, stream_units  # noqa: E402

S = int(sys.argv[1]) if len(sys.argv) > 1 else 256
LADDER = [dict(width=1920, height=1080, qp=26), dict(width=1280, height=720, qp=28), dict(width=960, height=540, qp=30),
          dict(width=640, height=360, qp=32)]


def run(t, aus):
    """input pictures/s over the timed pushes (two warm-up pushes first) and the output bytes"""
    t.push([aus[0]] * S); t.push([aus[1]] * S)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    outs = [t.push([au] * S) for au in aus[2:]] + [t.flush()]
    dt = time.perf_counter() - t0
    t.close()
    torch.cuda.empty_cache()
    flat = [b for out in outs for o in out for b in (o if isinstance(o, list) else [o])]
    return dt, sum(len(b) for b in flat)


def ladder_rate(aus):
    dt, nb = run(Transcoder(bench.W, bench.H, S, rungs=LADDER), aus)
    return (N_AU - 2) * S / dt, nb


def separate_rate(aus):
    total, nb = 0.0, 0
    for r in LADDER:
        kw = {k: v for k, v in r.items() if k not in ("width", "height")}
        dt, b = run(Transcoder(bench.W, bench.H, S, dst_w=r["width"], dst_h=r["height"], **kw), aus)
        total += dt
        nb += b
    return (N_AU - 2) * S / total, nb


def downsample_kernels():
    """one ladder launch against nine single-plane launches over the same S decoded 1080p pictures"""
    L = lib(0)
    w, h = bench.W, bench.H
    offsets, pitch, planes = ladder_layout(w, h, [(r["width"], r["height"]) for r in LADDER])
    tab = (DsPlane * len(planes))(*[DsPlane(*p) for p in planes])
    buf = torch.randint(0, 256, (S, pitch), dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def ladder():
        check(L.b2h264_k_downsample_ladder(C.addressof(tab), len(planes), buf.data_ptr(), pitch, buf.data_ptr(), pitch, 0, S, st))

    def nine():
        for mode, sx, sy, sw, sh, ss, dw, dh, ds, row0, so, do in planes:
            check(L.b2h264_k_downsample(mode, buf.data_ptr() + do, ds, dw, dh, buf.data_ptr() + so, ss, sw, sh, S, pitch, pitch, st))

    from torch.profiler import ProfilerActivity, profile
    alg = S * sum(5 * p[6] * p[7] for p in planes)
    reps = 10
    for name, fn, per_step in (("ladder (1 launch)", ladder, 1), ("b2h264_k_downsample (9 launches)", nine, 9)):
        fn(); fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
        ks = [e.time_range.elapsed_us() for e in prof.events() if "k_downsample_ladder" in e.name]
        assert len(ks) == reps * per_step, "expected %d down-sampler kernels in the trace, found %d" % (reps * per_step, len(ks))
        us = sum(ks) / reps
        emit(figure="downsample", path=name, launches_per_step=per_step, kernel_us_per_step=us, alg_bytes=alg, tb_s=alg / us / 1e6,
             frac_of_3_35=alg / us / 1e6 / 3.35)


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    emit(card=q.stdout.strip(), streams=S, size="%dx%d" % (bench.W, bench.H), rungs=["%dx%d qp %d" % (r["width"], r["height"], r["qp"])
                                                                                     for r in LADDER])
    aus = stream_units()
    for run_no in (1, 2):
        fps, nb = ladder_rate(aus)
        emit(figure="ladder", path="one Transcoder, 4 rungs", run=run_no, input_pictures_per_s=fps, out_bytes=nb)
        fps, nb = separate_rate(aus)
        emit(figure="ladder", path="4 single-output Transcoders, one after another", run=run_no, input_pictures_per_s=fps, out_bytes=nb)
    downsample_kernels()


if __name__ == "__main__":
    main()
