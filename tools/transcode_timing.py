"""Decoder device output and GPU transcoding, timed on the GPU (bench.py's decode workload: S copies of a 1080p Baseline stream of
this library's encoder, one access unit per stream per call).

(a) decode pictures/s: host output (b2h264_dec_decode into page-locked memory, synchronous) against device output
    (b2h264_dec_decode_device, one synchronize after the timed calls), alternating, two runs each;
(b) k_dec_output's kernel time (torch.profiler, a run of its own) with its algorithmic bytes (read + write of w*h*3/2 per picture)
    against 3.35 TB/s, and the alternative of 3 x S device-to-device cudaMemcpy2DAsync calls per step (CUDA events);
(c) transcode pictures/s (Transcoder) 1080p -> 1080p and 1080p -> 960x540, against the host round trip built from the existing API
    (b2h264_dec_decode2 into page-locked memory, then b2h264_enc_submit with host pictures).
Prints the card, its power limit and one JSON line per figure.  usage: python tools/transcode_timing.py [S]"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import torch  # noqa: E402
from openh264_b200.binding import BatchDecoder, BatchEncoder, check  # noqa: E402
from openh264_b200.transcode import Transcoder  # noqa: E402

S = int(sys.argv[1]) if len(sys.argv) > 1 else 256
N_AU = 8


def emit(**kv):
    print(json.dumps(kv), flush=True)


def stream_units():
    clip = bench.make_clip()
    seq = bench.ping_pong(bench.CLIP_FRAMES)
    enc = BatchEncoder(bench.W, bench.H, qp=bench.QP, fps=bench.FPS, n_streams=1)
    aus = []
    for i in range(N_AU):
        f = bench.stream_frame(seq, 0, i)
        aus.append(bytes(enc.encode([clip[f * bench.FSZ:(f + 1) * bench.FSZ]])[0][0]))
    enc.close()
    return aus


def decode_rate(aus, device_out):
    dec = BatchDecoder(bench.W, bench.H, n_streams=S, pinned_output=not device_out)
    out = torch.empty((S, dec.frame_bytes), dtype=torch.uint8, device="cuda") if device_out else None
    run = (lambda au: dec.decode_device([au] * S, out)) if device_out else (lambda au: dec.decode([au] * S))
    run(aus[0]); run(aus[1])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for au in aus[2:]:
        run(au)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    dec.close()
    return (N_AU - 2) * S / dt


def output_kernel(aus):
    w, h = bench.W, bench.H
    pic = w * h * 3 // 2
    dec = BatchDecoder(w, h, n_streams=S)
    out = torch.empty((S, pic), dtype=torch.uint8, device="cuda")
    dec.decode_device([aus[0]] * S, out); dec.decode_device([aus[1]] * S, out)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for au in aus[2:]:
            dec.decode_device([au] * S, out)
        torch.cuda.synchronize()
    dec.close()
    ks = [e.time_range.elapsed_us() for e in prof.events() if "k_dec_output" in e.name]
    assert ks, "no k_dec_output kernel in the trace"
    us = sum(ks) / len(ks)
    alg = 2 * S * pic
    emit(figure="k_dec_output", launches=len(ks), kernel_us=us, alg_bytes=alg, tb_s=alg / us / 1e6, frac_of_3_35=alg / us / 1e6 / 3.35)
    # the copy engine instead: 3 x S cudaMemcpy2DAsync from padded planes (the decoder's layout) per step
    L = dec.L
    L.cudaMemcpy2DAsync.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int, C.c_void_p]
    sty, stc = w + 64, w // 2 + 32
    ybytes, cbytes = sty * (h + 64), stc * (h // 2 + 32)
    src = torch.empty((S, ybytes + 2 * cbytes), dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def copies():
        for s in range(S):
            base, dst = src[s].data_ptr(), out[s].data_ptr()
            check(L.cudaMemcpy2DAsync(dst, w, base + 32 * sty + 32, sty, w, h, 3, st.cuda_stream))
            for pl in (0, 1):
                check(L.cudaMemcpy2DAsync(dst + w * h + pl * (w // 2) * (h // 2), w // 2, base + ybytes + pl * cbytes + 16 * stc + 16, stc,
                                          w // 2, h // 2, 3, st.cuda_stream))
    copies()
    torch.cuda.synchronize()
    reps = 6
    e0.record()
    for _ in range(reps):
        copies()
    e1.record()
    torch.cuda.synchronize()
    us_c = e0.elapsed_time(e1) * 1e3 / reps
    emit(figure="cudaMemcpy2DAsync_x3S", us_per_step=us_c, alg_bytes=alg, tb_s=alg / us_c / 1e6, frac_of_3_35=alg / us_c / 1e6 / 3.35)


def transcode_rate(aus, dst):
    t = Transcoder(bench.W, bench.H, S, dst_w=dst[0], dst_h=dst[1], qp=bench.QP, fps=bench.FPS)
    t.push([aus[0]] * S); t.push([aus[1]] * S)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    nbytes = 0
    for au in aus[2:]:
        nbytes += sum(len(b) for b in t.push([au] * S))
    nbytes += sum(len(b) for b in t.flush())
    dt = time.perf_counter() - t0
    t.close()
    return (N_AU - 2) * S / dt, nbytes


def host_chain_rate(aus):
    dec = BatchDecoder(bench.W, bench.H, n_streams=S, pinned_output=True)
    enc = BatchEncoder(bench.W, bench.H, qp=bench.QP, fps=bench.FPS, n_streams=S)

    def step(au):
        enc.encode(dec.decode2([au] * S))
    step(aus[0]); step(aus[1])
    t0 = time.perf_counter()
    for au in aus[2:]:
        step(au)
    dt = time.perf_counter() - t0
    dec.close(); enc.close()
    return (N_AU - 2) * S / dt


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    emit(card=q.stdout.strip(), streams=S, size="%dx%d" % (bench.W, bench.H))
    aus = stream_units()
    for run in (1, 2):
        for dev in (False, True):
            emit(figure="decode", output="device" if dev else "host (page-locked)", run=run, pictures_per_s=decode_rate(aus, dev))
    output_kernel(aus)
    for run in (1, 2):
        emit(figure="transcode", path="host round trip (decode2 -> submit from host)", run=run, pictures_per_s=host_chain_rate(aus))
        for dst in ((bench.W, bench.H), (960, 540)):
            fps, nb = transcode_rate(aus, dst)
            emit(figure="transcode", path="Transcoder (device)", dst="%dx%d" % dst, run=run, pictures_per_s=fps, out_bytes=nb)


if __name__ == "__main__":
    main()
