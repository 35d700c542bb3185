"""Batched transcoding on the GPU: Annex-B in, Annex-B out, pictures kept in HBM in between.

The batched decoder writes its pictures into device buffers (b2h264_dec_decode_device), the bilinear down-sampler
(b2h264_k_downsample_ladder) scales them to every output size of the ladder in one launch, and one batched encoder per rung reads
them from there (b2h264_enc_submit with src_on_device = 1).  Decoder and down-sampler share one CUDA stream, each rung's encoder has
its own, which waits for the step's down-sampling: the rungs' encode kernels run side by side, and the host parse of a step overlaps
the encode kernels of the step before."""
import ctypes as C
import inspect
import os
from collections import deque

import numpy as np

from .binding import B2H264Error, BatchDecoder, BatchEncoder, DsPlane, check, load

MAX_RUNGS = 8
_ENCODER_SIGNATURE = inspect.signature(BatchEncoder.__init__)
# BatchEncoder keywords a rung may carry besides width and height
ENCODER_KEYWORDS = [k for k in _ENCODER_SIGNATURE.parameters if k not in ("self", "width", "height", "n_streams", "device")]


def check_scale(src_w, src_h, dst_w, dst_h):
    """refuses an output size the encoder does not take (width % 4, height % 2) and any up-scaling"""
    if dst_w < 16 or dst_h < 16 or dst_w % 4 or dst_h % 2:
        raise ValueError(f"output size {dst_w}x{dst_h}: the encoder needs a width divisible by 4 and an even height, at least 16x16")
    if dst_w > src_w or dst_h > src_h:
        raise ValueError(f"output size {dst_w}x{dst_h} is larger than the input {src_w}x{src_h}: only down-scaling is supported")


class OutputOrder:
    """One stream's output order: the decoder hands pictures back in decoding order; they leave by ascending picture order count
    inside each IDR period, holding at most `depth` pictures back (the bumping process of H.264 C.4.5.3 with the stream's reorder
    depth).  An IDR picture starts a new period: everything held from the period before leaves first."""

    def __init__(self):
        self.held = []
        self.count = 0

    def push(self, item, poc, flags, depth):
        """a decoded picture with the values of BatchDecoder.picture_order(); returns the items now due, in output order"""
        out = self.drain() if flags & 1 else []
        self.held.append((poc, self.count, item))
        self.count += 1
        self.held.sort(key=lambda t: t[:2])
        while len(self.held) > depth:
            out.append(self.held.pop(0)[2])
        return out

    def drain(self):
        out = [t[2] for t in sorted(self.held, key=lambda t: t[:2])]
        self.held = []
        return out


def check_rungs(src_w, src_h, rungs):
    """the rungs as (width, height, encoder keywords); refuses (ValueError) no rungs, more than MAX_RUNGS, a size check_scale
    refuses, a keyword BatchEncoder does not take and two rungs that would give the same bytes (same size, same configuration once
    the encoder's defaults are filled in; the entropy thread count does not change the output)"""
    if not isinstance(rungs, (list, tuple)) or not 1 <= len(rungs) <= MAX_RUNGS:
        raise ValueError(f"a ladder has 1 to {MAX_RUNGS} rungs")
    out, seen = [], []
    for r in rungs:
        kw = dict(r)
        if "width" not in kw or "height" not in kw:
            raise ValueError(f"rung {r}: width and height are required")
        w, h = kw.pop("width"), kw.pop("height")
        check_scale(src_w, src_h, w, h)
        bad = sorted(set(kw) - set(ENCODER_KEYWORDS))
        if bad:
            raise ValueError(f"rung {r}: unknown encoder keywords {bad}")
        b = _ENCODER_SIGNATURE.bind(None, w, h, **kw)
        b.apply_defaults()
        key = [(k, v) for k, v in b.arguments.items() if k not in ("self", "entropy_threads")]
        if key in seen:
            raise ValueError(f"rung {r} repeats an earlier rung")
        seen.append(key)
        out.append((w, h, kw))
    return out


def round_ratio(src, dst, scale):
    """WELS_ROUND(src / dst * scale) in single precision, as the reference (and b2h264_k_downsample) derive the general ratio's steps"""
    return int(0.5 + float(np.float32(src) / np.float32(dst) * np.float32(scale)))


def ladder_layout(src_w, src_h, sizes):
    """The step-buffer layout and the down-sampler's descriptor table of a ladder whose rungs have the output sizes `sizes`.
    A step-buffer row holds one picture of every distinct size, each at a 256-byte aligned offset; the source size (if a rung has
    it, at whatever position) is the decoded picture itself and comes first, at offset 0, where the decoder writes it.  The other
    sizes follow in order of first appearance.  Returns (offset per size, row pitch, descriptors): the descriptors are
    b2h264_ds_plane values as tuples in DsPlane's field order, Y, U, V of each down-scaled size in row order, their source planes
    those of the decoded I420 picture."""
    L = load()
    offsets, planes, pitch, rows = {}, [], 0, 0
    for w, h in sorted(dict.fromkeys(sizes), key=lambda size: size != (src_w, src_h)):      # stable: the source size first
        offsets[(w, h)] = pitch
        if (w, h) != (src_w, src_h):
            so = do = 0
            for pl in range(3):
                c = 1 if pl else 0
                sw, sh, dw, dh = src_w >> c, src_h >> c, w >> c, h >> c
                mode = L.b2h264_downsample_mode(sw, sh, dw, dh, c)
                sx = round_ratio(sw, dw, 1 << (16 if mode == 3 else 15)) if mode >= 3 else 0
                sy = round_ratio(sh, dh, 1 << 15) if mode >= 3 else 0
                planes.append((mode, sx, sy, sw, sh, sw, dw, dh, dw, rows, so, pitch + do))
                rows += dh
                so += sw * sh
                do += dw * dh
        pitch += ((w * h * 3 // 2) + 255) & ~255
    return offsets, pitch, planes


def host_cores():
    """cores this process may really use: the affinity mask, capped by the cgroup CPU quota.  The same rule as bench.py's
    host_cores (not imported: the library does not depend on the benchmark); usable_cores() in csrc/host_pool.h, the encoder's
    default thread count, follows it too but rounds a fractional cgroup quota up.  Keep the three in step."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        q, p = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if q != "max":
            n = min(n, max(1, int(float(q) / float(p))))
    except (OSError, ValueError):
        pass
    try:
        q = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
        p = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
        if q > 0 and p > 0:
            n = min(n, max(1, q // p))
    except (OSError, ValueError):
        pass
    return max(1, n)


def entropy_threads(mbs, cores):
    """host entropy threads per rung: 1 each, and the cores beyond those split in proportion to each rung's macroblocks per
    picture (the largest remainders get what rounding down leaves), so that the total is `cores` (or one per rung where there are
    fewer cores than rungs).  The proportion is a guess that nobody has measured: it assumes a rung's host entropy coding costs in
    proportion to its macroblocks."""
    share = [max(0, cores - len(mbs)) * m / sum(mbs) for m in mbs]
    n = [1 + int(x) for x in share]
    for r in sorted(range(len(mbs)), key=lambda r: int(share[r]) - share[r])[:max(0, cores - sum(n))]:
        n[r] += 1
    return n


class Transcoder:
    """n_streams independent H.264 streams of src_w x src_h decoded once, and re-encoded as a ladder of renditions.

    rungs: a list of 1 to MAX_RUNGS dicts, each with `width` and `height` and any BatchEncoder keywords (qp, entropy_cabac,
    profile_idc, intra_period, complexity_low, loop_filter, fps, num_ref_frames, ltr, ...).  Each rung is down-scaled from the
    decoded picture (never from another rung) and gives the bytes a single-output Transcoder of that rung gives.  Without rungs:
    one rung of dst_w x dst_h (the input size when not given) with encoder_kwargs.

    push(access_units) takes one access unit per stream (or None) and returns per stream the Annex-B bytes that became ready
    (with rungs: per stream a list of one byte string per rung, in rung order); flush() encodes the pictures still held for
    reordering and returns the rest in the same shape.  The bytes of one stream (and rung), concatenated over all calls, are its
    output."""

    def __init__(self, src_w, src_h, n_streams, dst_w=None, dst_h=None, device=0, rungs=None, **encoder_kwargs):
        self.ladder = rungs is not None
        if self.ladder and (dst_w is not None or dst_h is not None or encoder_kwargs):
            raise ValueError("give the rungs, or dst_w / dst_h and the encoder keywords, not both")
        if not self.ladder:
            rungs = [dict(encoder_kwargs, width=src_w if dst_w is None else dst_w, height=src_h if dst_h is None else dst_h)]
        configs = check_rungs(src_w, src_h, rungs)
        self.offsets, self.pitch, planes = ladder_layout(src_w, src_h, [(w, h) for w, h, _ in configs])
        import torch
        self.torch = torch
        self.n = n_streams
        self.dev = torch.device("cuda", device)
        self.stream = torch.cuda.Stream(self.dev)               # decoder and down-sampler
        self.decoded = torch.cuda.Event()                       # the step's down-sampling is done: the rungs' streams wait for it
        self.dec = BatchDecoder(src_w, src_h, n_streams=n_streams, device=device)
        self.src_bytes = src_w * src_h * 3 // 2
        threads = entropy_threads([((w + 15) // 16) * ((h + 15) // 16) for w, h, _ in configs], host_cores())
        self.rungs = []                                         # (encoder, its stream, picture offset in a step-buffer row)
        for (w, h, kw), t in zip(configs, threads):
            st = torch.cuda.Stream(self.dev)
            enc = BatchEncoder(w, h, n_streams=n_streams, device=device, **dict({"entropy_threads": min(t, n_streams)}, **kw))
            enc.set_stream(st.cuda_stream)
            self.rungs.append((enc, st, self.offsets[(w, h)]))
        self.planes = (DsPlane * len(planes))(*[DsPlane(*p) for p in planes]) if planes else None
        self.scratch = None                                     # the decoded pictures when no rung has the input size
        if (src_w, src_h) not in self.offsets:
            self.src_pitch = (self.src_bytes + 255) & ~255
            with torch.cuda.stream(self.stream):
                self.scratch = torch.empty((n_streams, self.src_pitch), dtype=torch.uint8, device=self.dev)
        self.order = [OutputOrder() for _ in range(n_streams)]
        self.ready = [deque() for _ in range(n_streams)]       # released pictures waiting for the encoders
        # step buffers: unused ones / id -> [buffer, pictures x rungs still to collect]; allocated: how many were made
        self.free, self.refs, self.allocated = [], {}, 0
        self.in_flight = None                                   # the pictures of the submission not yet collected

    def _buffer(self):
        if self.free:
            return self.free.pop()
        self.allocated += 1
        return self.torch.empty((self.n, self.pitch), dtype=self.torch.uint8, device=self.dev)

    def _unref(self, buf):
        e = self.refs[id(buf)]
        e[1] -= 1
        if e[1] == 0:
            del self.refs[id(buf)]
            self.free.append(buf)

    def push(self, access_units):
        if len(access_units) != self.n:
            raise ValueError("push takes one access unit (or None) per stream")
        with self.torch.cuda.stream(self.stream):
            buf = self._buffer()
            src = buf if self.scratch is None else self.scratch
            _, status = self.dec.decode_device(access_units, [src[s, :self.src_bytes] for s in range(self.n)])
            self._downsample(buf, status)
            self.decoded.record(self.stream)
            for _, st, _ in self.rungs:
                st.wait_event(self.decoded)
            bad = [(s, v) for s, v in enumerate(status) if v < 0]
            if bad:
                raise B2H264Error("decoder errors (stream, code): %s" % bad)
            got = [s for s in range(self.n) if status[s] == 1]
            if got:
                self.refs[id(buf)] = [buf, len(got) * len(self.rungs)]
            else:
                self.free.append(buf)
            for s in got:
                poc, flags, depth = self.dec.picture_order(s)
                self.ready[s].extend(self.order[s].push((buf, s), poc, flags, depth))
            return self._result(self._encode_ready())

    def flush(self):
        with self.torch.cuda.stream(self.stream):
            for s in range(self.n):
                self.ready[s].extend(self.order[s].drain())
            out = self._encode_ready()
            self._collect(out)
            return self._result(out)

    def _result(self, out):
        return out if self.ladder else [o[0] for o in out]

    def _downsample(self, buf, status):
        """every down-scaled plane of every picture of the step in one launch: the rows from the first to the last stream that got one"""
        got = [s for s in range(self.n) if status[s] == 1]
        if self.planes is None or not got:
            return
        lo, cnt = got[0], got[-1] - got[0] + 1
        src, src_pitch = (buf, self.pitch) if self.scratch is None else (self.scratch, self.src_pitch)
        check(self.dec.L.b2h264_k_downsample_ladder(C.addressof(self.planes), len(self.planes), buf.data_ptr(), self.pitch,
                                                    src.data_ptr(), src_pitch, lo, cnt, self.stream.cuda_stream))

    def _encode_ready(self):
        """one encoder batch per rung and round while pictures wait, one picture per stream each (streams without one sit it out):
        every rung is submitted before any is collected, so that their kernels overlap; the last batches stay in flight until the
        next call, so that their encode overlaps the next step's parse"""
        out = [[b""] * len(self.rungs) for _ in range(self.n)]
        while any(self.ready):
            self._collect(out)
            pics = [self.ready[s].popleft() if self.ready[s] else None for s in range(self.n)]
            for enc, _, off in self.rungs:
                enc.submit([None if p is None else p[0].data_ptr() + p[1] * self.pitch + off for p in pics], on_device=True)
            self.in_flight = [p for p in pics if p is not None]
        return out

    def _collect(self, out):
        if self.in_flight is None:
            return
        for r, (enc, _, _) in enumerate(self.rungs):
            bs, _ = enc.collect()
            for s in range(self.n):
                out[s][r] += bs[s]
            for buf, _ in self.in_flight:                       # this rung's encode kernel has read them
                self._unref(buf)
        self.in_flight = None

    def close(self):
        """releases every encoder, the decoder and the step buffers"""
        for enc, _, _ in self.rungs:
            enc.close()
        self.dec.close()
        self.free, self.refs, self.ready, self.in_flight, self.scratch = [], {}, [deque() for _ in range(self.n)], None, None
