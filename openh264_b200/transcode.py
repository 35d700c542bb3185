"""Batched transcoding on the GPU: Annex-B in, Annex-B out, pictures kept in HBM in between.

The batched decoder writes its pictures into device buffers (b2h264_dec_decode_device), the bilinear down-sampler
(b2h264_k_downsample) scales them when the output size differs, and the batched encoder reads them from there
(b2h264_enc_submit with src_on_device = 1).  Decoder, down-sampler and encoder share one CUDA stream, so no call waits
for another's kernels; the host parse of a step overlaps the encode kernels of the step before."""
from collections import deque

from .binding import B2H264Error, BatchDecoder, BatchEncoder, check


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


class Transcoder:
    """n_streams independent H.264 streams of src_w x src_h decoded, optionally down-scaled to dst_w x dst_h, and re-encoded with
    BatchEncoder's configuration (encoder_kwargs: qp, entropy_cabac, profile_idc, complexity_low, intra_period, loop_filter, fps).

    push(access_units) takes one access unit per stream (or None) and returns per stream the Annex-B bytes that became ready;
    flush() encodes the pictures still held for reordering and returns the rest.  The bytes of one stream, concatenated over all
    calls, are that stream's output."""

    def __init__(self, src_w, src_h, n_streams, dst_w=None, dst_h=None, device=0, **encoder_kwargs):
        dst_w = src_w if dst_w is None else dst_w
        dst_h = src_h if dst_h is None else dst_h
        check_scale(src_w, src_h, dst_w, dst_h)
        import torch
        self.torch = torch
        self.n = n_streams
        self.dev = torch.device("cuda", device)
        self.stream = torch.cuda.Stream(self.dev)
        self.dec = BatchDecoder(src_w, src_h, n_streams=n_streams, device=device)
        self.enc = BatchEncoder(dst_w, dst_h, n_streams=n_streams, device=device, **encoder_kwargs)
        self.enc.set_stream(self.stream.cuda_stream)
        self.src_bytes, self.dst_bytes = src_w * src_h * 3 // 2, dst_w * dst_h * 3 // 2
        self.pitch = (self.dst_bytes + 255) & ~255              # one picture per 256-byte aligned row of a step buffer
        self.planes = None
        if (dst_w, dst_h) != (src_w, src_h):
            L = self.dec.L
            # per plane: mode (the function CDownsampling::Process picks), source / destination offset and size
            self.planes = []
            so = do = 0
            for pl in range(3):
                c = 1 if pl else 0
                sw, sh, dw, dh = src_w >> c, src_h >> c, dst_w >> c, dst_h >> c
                self.planes.append((L.b2h264_downsample_mode(sw, sh, dw, dh, c), so, sw, sh, do, dw, dh))
                so += sw * sh
                do += dw * dh
            self.src_pitch = (self.src_bytes + 255) & ~255
            with torch.cuda.stream(self.stream):
                self.scratch = torch.empty((n_streams, self.src_pitch), dtype=torch.uint8, device=self.dev)
        self.order = [OutputOrder() for _ in range(n_streams)]
        self.ready = [deque() for _ in range(n_streams)]       # released pictures waiting for the encoder
        self.free, self.refs = [], {}                           # step buffers: unused ones / id -> [buffer, pictures still in use]
        self.in_flight = None                                   # the pictures of the submission not yet collected

    def _buffer(self):
        if self.free:
            return self.free.pop()
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
            if self.planes is None:
                _, status = self.dec.decode_device(access_units, [buf[s, :self.dst_bytes] for s in range(self.n)])
            else:
                _, status = self.dec.decode_device(access_units, [self.scratch[s, :self.src_bytes] for s in range(self.n)])
                self._downsample(buf, status)
            bad = [(s, v) for s, v in enumerate(status) if v < 0]
            if bad:
                raise B2H264Error("decoder errors (stream, code): %s" % bad)
            got = [s for s in range(self.n) if status[s] == 1]
            if got:
                self.refs[id(buf)] = [buf, len(got)]
            else:
                self.free.append(buf)
            for s in got:
                poc, flags, depth = self.dec.picture_order(s)
                self.ready[s].extend(self.order[s].push((buf, s), poc, flags, depth))
            return self._encode_ready()

    def flush(self):
        with self.torch.cuda.stream(self.stream):
            for s in range(self.n):
                self.ready[s].extend(self.order[s].drain())
            out = self._encode_ready()
            self._collect(out)
            return out

    def _downsample(self, buf, status):
        """every picture of the step in one launch per plane: the rows from the first to the last stream that got one"""
        got = [s for s in range(self.n) if status[s] == 1]
        if not got:
            return
        lo, cnt = got[0], got[-1] - got[0] + 1
        src0, dst0 = self.scratch[lo].data_ptr(), buf[lo].data_ptr()
        st = self.stream.cuda_stream
        for mode, so, sw, sh, do, dw, dh in self.planes:
            check(self.dec.L.b2h264_k_downsample(mode, dst0 + do, dw, dw, dh, src0 + so, sw, sw, sh, cnt, self.pitch, self.src_pitch, st))

    def _encode_ready(self):
        """one encoder batch per round while pictures wait, one picture per stream each (streams without one sit it out); the
        last batch stays in flight until the next call, so that its encode overlaps the next step's parse"""
        out = [b""] * self.n
        while any(self.ready):
            self._collect(out)
            pics = [self.ready[s].popleft() if self.ready[s] else None for s in range(self.n)]
            self.enc.submit([None if p is None else p[0][p[1]].data_ptr() for p in pics], on_device=True)
            self.in_flight = [p for p in pics if p is not None]
        return out

    def _collect(self, out):
        if self.in_flight is None:
            return
        bs, _ = self.enc.collect()
        for s in range(self.n):
            out[s] += bs[s]
        for buf, _ in self.in_flight:                           # the encode kernel has read them
            self._unref(buf)
        self.in_flight = None

    def close(self):
        self.dec.close()
        self.enc.close()
