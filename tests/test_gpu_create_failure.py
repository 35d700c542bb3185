"""A batched encoder or decoder whose create fails (include/b2h264_codec.h b2h264_enc_create / b2h264_dec_create) returns the error,
hands out no object and releases everything it acquired before the failure: its streams, its buffers and the decoder's parser
threads.  The configurations below ask for a picture store larger than the device's memory, so cudaMalloc refuses the size up
front: nothing is allocated and no kernel runs."""
import ctypes as C
import os

import numpy as np
import pytest

from openh264_b200.binding import DecConfig, EncConfig, lib, vp

pytestmark = pytest.mark.gpu

# 4096x2304 in 6000 streams: two padded pictures of ~14.8 MB per stream make a ~177 GB picture store
W, H, STREAMS = 4096, 2304, 6000
SENTINEL = 0x1234


def _threads():
    return len(os.listdir("/proc/self/task"))


def _dec_create(L):
    h = vp(SENTINEL)
    rc = L.b2h264_dec_create(C.byref(DecConfig(W, H, STREAMS, 0)), C.byref(h))
    return rc, h.value


def _enc_create(L):
    cfg = EncConfig(width=W, height=H, qp=26, fps=30.0, n_streams=STREAMS)
    h = vp(SENTINEL)
    rc = L.b2h264_enc_create(C.byref(cfg), C.byref(h))
    return rc, h.value


def test_decoder_create_failure_releases_everything():
    L = lib(0)
    rc, h = _dec_create(L)                 # the first call may start the runtime's own threads
    assert rc != 0 and h == SENTINEL
    before = _threads()
    for _ in range(50):
        rc, h = _dec_create(L)
        assert rc != 0 and h == SENTINEL
    assert _threads() == before


def test_encoder_create_failure_returns_error():
    L = lib(0)
    for _ in range(3):
        rc, h = _enc_create(L)
        assert rc != 0 and h == SENTINEL


def test_create_after_failure():
    """a failed create leaves no CUDA error behind: the next objects encode, launch and decode as usual"""
    from openh264_b200.binding import BatchDecoder, BatchEncoder
    L = lib(0)
    assert _dec_create(L)[0] != 0 and _enc_create(L)[0] != 0
    enc, dec = BatchEncoder(64, 64), BatchDecoder(64, 64)
    rng = np.random.RandomState(7)
    for _ in range(2):
        aus, _ = enc.encode([rng.randint(0, 256, 64 * 64 * 3 // 2).astype(np.uint8)])
        assert np.array_equal(dec.decode(aus)[0], enc.recon())
    enc.close()
    dec.close()
