"""ctypes binding of libopenh264_b200.so (include/b2h264.h).  No CPU fallback: `load()` raises if the
library has not been built, and every call raises B2H264Error on a non-zero CUDA status."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("B2H264_LIB") or os.path.join(HERE, "libopenh264_b200.so")   # env override: profiling variants only

u8p, i8p = C.POINTER(C.c_uint8), C.POINTER(C.c_int8)
i16p, u16p, i32p = C.POINTER(C.c_int16), C.POINTER(C.c_uint16), C.POINTER(C.c_int32)
vp = C.c_void_p


class B2H264Error(RuntimeError):
    pass


class EdgeJob(C.Structure):
    _fields_ = [("off", C.c_int32), ("sx", C.c_int32), ("sy", C.c_int32), ("alpha", C.c_int16), ("beta", C.c_int16),
                ("tc", C.c_int8 * 4), ("strong", C.c_int32)]


class MeJob(C.Structure):
    _fields_ = [("blk", C.c_int32), ("cur_off", C.c_int32), ("ref_off", C.c_int32),
                ("mvp_x", C.c_int16), ("mvp_y", C.c_int16),
                ("mv_min_x", C.c_int16), ("mv_min_y", C.c_int16), ("mv_max_x", C.c_int16), ("mv_max_y", C.c_int16),
                ("n_mvc", C.c_int32), ("mvc", (C.c_int16 * 2) * 5),
                ("sad_pred", C.c_uint32), ("qp", C.c_int32), ("calc_satd", C.c_int32)]


class MeResult(C.Structure):
    _fields_ = [("mv_x", C.c_int16), ("mv_y", C.c_int16), ("sad_cost", C.c_uint32), ("satd_cost", C.c_uint32),
                ("ref_off", C.c_int32)]


class DsPlane(C.Structure):
    """b2h264_ds_plane: one destination plane of b2h264_k_downsample_ladder"""
    _fields_ = [("mode", C.c_int32), ("sx", C.c_int32), ("sy", C.c_int32), ("src_w", C.c_int32), ("src_h", C.c_int32),
                ("src_stride", C.c_int32), ("dst_w", C.c_int32), ("dst_h", C.c_int32), ("dst_stride", C.c_int32), ("row0", C.c_int32),
                ("src_offset", C.c_uint64), ("dst_offset", C.c_uint64)]


# every symbol include/b2h264.h declares: name -> argtypes (restype int unless noted)
API = {
    "b2h264_init": [C.c_int],
    "b2h264_abi_version": [],
    "b2h264_dev_malloc": [C.POINTER(vp), C.c_size_t],
    "b2h264_dev_free": [vp],
    "b2h264_h2d": [vp, vp, C.c_size_t, vp],
    "b2h264_d2h": [vp, vp, C.c_size_t, vp],
    "b2h264_sync": [vp],
    "b2h264_error_string": [C.c_int],
    "b2h264_launch_count": [],
    "b2h264_k_sad": [vp, C.c_int, vp, vp, C.c_int, vp, C.c_int, C.c_int, vp, vp, vp, vp],
    "b2h264_k_mc_luma": [vp, C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, vp, vp],
    "b2h264_k_mc_chroma": [vp, C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, vp, vp],
    "b2h264_k_halfpel": [C.c_int, vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, vp, vp],
    "b2h264_k_pixel_avg": [vp, C.c_int, vp, vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, vp, vp],
    "b2h264_k_dct_four4x4": [vp, C.c_int, vp, vp, C.c_int, vp, C.c_int, vp, vp],
    "b2h264_k_quant_four4x4": [vp, C.c_int, C.c_int, C.c_int, vp, vp],
    "b2h264_k_quant4x4_dc": [vp, C.c_int, C.c_int, C.c_int, vp],
    "b2h264_k_hadamard_quant2x2": [vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp],
    "b2h264_k_hadamard_t4_dc": [vp, C.c_int, vp, vp],
    "b2h264_k_scan4x4": [vp, C.c_int, vp, vp, vp, vp],
    "b2h264_k_dequant_four4x4": [vp, C.c_int, C.c_int, vp],
    "b2h264_k_dequant_ihadamard4x4": [vp, C.c_int, C.c_int, vp],
    "b2h264_k_dequant_luma_dc": [vp, C.c_int, C.c_int, vp],
    "b2h264_k_dequant_ihadamard2x2": [vp, C.c_int, C.c_int, vp],
    "b2h264_k_idct_four4x4_rec": [vp, C.c_int, vp, vp, C.c_int, vp, vp],
    "b2h264_k_idct_rec_i16x16_dc": [vp, C.c_int, vp, vp, C.c_int, vp, vp],
    "b2h264_k_idct_res_add_pred": [vp, C.c_int, vp, vp, C.c_int, C.c_int, vp],
    "b2h264_k_deblock_luma": [vp, vp, C.c_int, vp],
    "b2h264_k_deblock_chroma": [vp, vp, vp, C.c_int, vp],
    "b2h264_k_expand_plane": [vp, C.c_int, C.c_int, C.c_int, C.c_int, vp],
    "b2h264_k_downsample": [C.c_int, vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_size_t, C.c_size_t, vp],
    "b2h264_downsample_mode": [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int],
    "b2h264_k_downsample_ladder": [vp, C.c_int, vp, C.c_size_t, vp, C.c_size_t, C.c_int, C.c_int, vp],
    "b2h264_k_me_search": [vp, C.c_int, vp, C.c_int, vp, C.c_int, vp, vp],
    "b2h264_k_me_cross_search": [vp, C.c_int, vp, C.c_int, vp, C.c_int, vp, vp],
    "b2h264_k_weighted_pred": [C.c_int, vp, vp, C.c_int, vp, vp, vp, C.c_int, C.c_int, C.c_int, vp],
    "b2h264_k_mc_sad": [vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, vp, vp],
    "b2h264_enc_create": [vp, C.POINTER(vp)],
    "b2h264_enc_destroy": [vp],
    "b2h264_enc_submit": [vp, C.POINTER(vp), C.c_int],
    "b2h264_enc_collect": [vp, C.POINTER(vp), i32p, i32p],
    "b2h264_enc_force_idr": [vp, C.c_int],
    "b2h264_enc_reset_stream": [vp, C.c_int],
    "b2h264_enc_set_mb_bits": [vp, C.c_int],
    "b2h264_enc_get_mb_bits": [vp, C.c_int, i32p, i32p],
    "b2h264_enc_get_recon": [vp, C.c_int, vp],
    "b2h264_enc_set_references": [vp, C.c_int, C.c_int, C.c_int],
    "b2h264_enc_get_references": [vp, i32p],
    "b2h264_enc_set_slices": [vp, C.c_int, C.c_int, C.POINTER(C.c_uint32)],
    "b2h264_enc_get_slices": [vp, i32p, i32p, C.POINTER(C.c_uint32)],
    "b2h264_enc_ltr_recovery_request": [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int],
    "b2h264_enc_ltr_marking_feedback": [vp, C.c_int, C.c_int, C.c_int, C.c_int],
    "b2h264_enc_ltr_mark_period": [vp, C.c_int, C.c_int],
    "b2h264_enc_last_timing": [vp, C.POINTER(C.c_float)],
    "b2h264_enc_last_d2h_bytes": [vp, C.POINTER(C.c_ulonglong)],
    "b2h264_enc_last_coded_mbs": [vp, C.POINTER(C.c_ulonglong)],
    "b2h264_dec_create": [vp, C.POINTER(vp)],
    "b2h264_dec_destroy": [vp],
    "b2h264_dec_decode": [vp, C.POINTER(vp), C.POINTER(C.c_int32), C.POINTER(vp)],
    "b2h264_dec_decode2": [vp, C.POINTER(vp), C.POINTER(C.c_int32), C.POINTER(vp), C.POINTER(C.c_int32)],
    "b2h264_dec_decode3": [vp, C.POINTER(vp), C.POINTER(C.c_int32), C.POINTER(vp), C.POINTER(C.c_int32)],
    "b2h264_dec_decode_device": [vp, C.POINTER(vp), C.POINTER(C.c_int32), C.POINTER(vp), C.POINTER(C.c_int32)],
    "b2h264_dec_set_stream": [vp, vp],
    "b2h264_dec_probe": [vp, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32)],
    "b2h264_dec_reset_stream": [vp, C.c_int32],
    "b2h264_dec_last_picture_order": [vp, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32)],
    "b2h264_host_alloc": [C.c_size_t],
    "b2h264_host_free": [vp],
    "b2h264_enc_set_stream": [vp, vp],
    "b2h264_table_quant_ff": [C.c_int],
    "b2h264_table_quant_mf": [C.c_int],
    "b2h264_table_dequant": [C.c_int],
    "b2h264_table_lambda": [C.c_int],
    "b2h264_table_chroma_qp": [C.c_int],
}
class EncConfig(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("qp", C.c_int32), ("fps", C.c_float),
                ("target_bitrate", C.c_int32), ("n_streams", C.c_int32), ("entropy_threads", C.c_int32),
                ("device", C.c_int32), ("sps_pps_id_strategy", C.c_int32), ("complexity_low", C.c_int32),
                ("entropy_cabac", C.c_int32), ("profile_idc", C.c_int32), ("intra_period", C.c_int32),
                ("loop_filter_idc", C.c_int32), ("loop_filter_alpha_c0_offset", C.c_int32), ("loop_filter_beta_offset", C.c_int32)]


_RESTYPES = {"b2h264_enc_destroy": None, "b2h264_dec_destroy": None, "b2h264_host_alloc": C.c_void_p, "b2h264_host_free": None, "b2h264_error_string": C.c_char_p, "b2h264_launch_count": C.c_ulonglong,
             "b2h264_table_quant_ff": i16p, "b2h264_table_quant_mf": i16p, "b2h264_table_dequant": u16p}

_lib = None
_inited = False


def build(verbose=False):
    """Compile libopenh264_b200.so in-tree for sm_90a (H100) (nvcc cross-compiles without a GPU)."""
    subprocess.check_call(["make", "-C", os.path.join(HERE, "csrc"), "-j", "8"] + ([] if verbose else ["-s"]))


def load():
    """dlopen the product library; raises if it is not built (no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise B2H264Error(f"{SO_PATH} is missing: run openh264_b200.build() / make -C openh264_b200/csrc")
        L = C.CDLL(SO_PATH)
        for name, args in API.items():
            fn = getattr(L, name)           # AttributeError here = header/library mismatch
            fn.argtypes = args
            fn.restype = _RESTYPES.get(name, C.c_int)
        _lib = L
    return _lib


def check(rc):
    if rc != 0:
        raise B2H264Error(f"CUDA error {rc}: {load().b2h264_error_string(rc).decode()}")


def lib(device=0):
    """Loaded library with the device selected and the constant tables uploaded."""
    global _inited
    L = load()
    if not _inited:
        check(L.b2h264_init(device))
        _inited = True
    return L


class DeviceArray:
    """A numpy-shaped buffer in HBM (cudaMalloc through the C-ABI; + slack so word loads stay in bounds)."""

    def __init__(self, arr=None, shape=None, dtype=None):
        L = lib()
        if arr is not None:
            arr = np.ascontiguousarray(arr)
            shape, dtype = arr.shape, arr.dtype
        self.shape, self.dtype = tuple(shape), np.dtype(dtype)
        self.nbytes = int(np.prod(self.shape)) * self.dtype.itemsize
        p = vp()
        check(L.b2h264_dev_malloc(C.byref(p), self.nbytes + 64))
        self.ptr = p.value
        if arr is not None:
            check(L.b2h264_h2d(self.ptr, arr.ctypes.data, self.nbytes, None))
            check(L.b2h264_sync(None))

    def at(self, byte_off):
        return self.ptr + byte_off

    def get(self):
        out = np.empty(self.shape, self.dtype)
        check(load().b2h264_d2h(out.ctypes.data, self.ptr, self.nbytes, None))
        check(load().b2h264_sync(None))
        return out

    def free(self):
        if self.ptr:
            load().b2h264_dev_free(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class BatchEncoder:
    """Host-side mirror of the layer-2 C-ABI (include/b2h264_codec.h): N independent streams, one picture per
    stream per call; returns the Annex-B access units.  No computation happens in Python."""

    def __init__(self, width, height, qp=26, fps=30.0, n_streams=1, target_bitrate=5000000, entropy_threads=0, device=0,
                 sps_pps_id_strategy=1, complexity_low=False, entropy_cabac=False, profile_idc=0, intra_period=0, loop_filter=(0, 0, 0),
                 num_ref_frames=1, ltr=False, ltr_mark_period=30):
        """num_ref_frames (iNumRefFrame: -1 = AUTO_REF_PIC_COUNT, or 1..10), ltr (bEnableLongTermReference) and ltr_mark_period
        (iLtrMarkPeriod): b2h264_enc_set_references"""
        self.L = lib(device)
        self.cfg = EncConfig(width, height, qp, fps, target_bitrate, n_streams, entropy_threads, device, sps_pps_id_strategy,
                             1 if complexity_low else 0, 1 if entropy_cabac else 0, profile_idc, intra_period, *loop_filter)
        self.h = vp()
        check(self.L.b2h264_enc_create(C.byref(self.cfg), C.byref(self.h)))
        self.n = n_streams
        self.frame_bytes = width * height * 3 // 2
        if (num_ref_frames, bool(ltr), ltr_mark_period) != (1, False, 30):
            check(self.L.b2h264_enc_set_references(self.h, num_ref_frames, 1 if ltr else 0, ltr_mark_period))

    def references(self):
        """(iNumRefFrame, max_num_ref_frames, iLTRRefNum, pictures kept per stream) as resolved"""
        v = (C.c_int32 * 4)()
        check(self.L.b2h264_enc_get_references(self.h, v))
        return tuple(v)

    def set_slices(self, mode, num=1, mb_num=()):
        """Slices of every picture of every stream, before the first picture: SSliceArgument's uiSliceMode (0 SM_SINGLE_SLICE,
        1 SM_FIXEDSLCNUM_SLICE, 2 SM_RASTER_SLICE), uiSliceNum and uiSliceMbNum (up to 35 run lengths; none with raster mode: one
        slice per macroblock row).  Returns the partition as the reference resolves it: (mode, slice count, run lengths)."""
        runs = (C.c_uint32 * 35)(*mb_num)
        check(self.L.b2h264_enc_set_slices(self.h, mode, num, runs))
        m, n = C.c_int32(), C.c_int32()
        check(self.L.b2h264_enc_get_slices(self.h, C.byref(m), C.byref(n), runs))
        return m.value, n.value, list(runs[:n.value]) if m.value else []

    def ltr_recovery_request(self, stream, idr_pic_id, cur_frame_num, last_correct_frame_num, feedback_type=1):
        """ENCODER_LTR_RECOVERY_REQUEST for one stream (feedback_type 1 = LTR_RECOVERY_REQUEST); applies to its next picture"""
        check(self.L.b2h264_enc_ltr_recovery_request(self.h, stream, feedback_type, idr_pic_id, cur_frame_num, last_correct_frame_num))

    def ltr_marking_feedback(self, stream, idr_pic_id, ltr_frame_num, success=True):
        """ENCODER_LTR_MARKING_FEEDBACK for one stream (LTR_MARKING_SUCCESS or LTR_MARKING_FAILED); applies to its next picture"""
        check(self.L.b2h264_enc_ltr_marking_feedback(self.h, stream, 4 if success else 5, idr_pic_id, ltr_frame_num))

    def ltr_mark_period(self, stream, period):
        """ENCODER_LTR_MARKING_PERIOD for one stream"""
        check(self.L.b2h264_enc_ltr_mark_period(self.h, stream, period))

    def submit(self, frames, on_device=False):
        """frames: list of n_streams numpy uint8 arrays (host) or raw device pointers (on_device=True)."""
        ptrs = (vp * self.n)(*[(None if f is None else f if on_device else f.ctypes.data) for f in frames])
        # two submissions can be in flight and pinned sources are DMA'd in place: keep both alive until their collect
        self._keep = getattr(self, "_keep", [])[-1:] + [frames]
        check(self.L.b2h264_enc_submit(self.h, ptrs, 1 if on_device else 0))

    def collect(self):
        bs = (vp * self.n)()
        nb = (C.c_int32 * self.n)()
        ft = (C.c_int32 * self.n)()
        check(self.L.b2h264_enc_collect(self.h, bs, nb, ft))
        return [C.string_at(bs[i], nb[i]) if bs[i] else b"" for i in range(self.n)], list(ft)

    def encode(self, frames):
        self.submit(frames)
        return self.collect()

    def set_mb_bits(self, on=True):
        check(self.L.b2h264_enc_set_mb_bits(self.h, 1 if on else 0))

    def mb_bits(self, stream=0):
        """(device count, host writer's count) of CAVLC bits per macroblock of the picture collected last"""
        n = ((self.cfg.width + 15) // 16) * ((self.cfg.height + 15) // 16)
        d, h = np.zeros(n, np.int32), np.zeros(n, np.int32)
        check(self.L.b2h264_enc_get_mb_bits(self.h, stream, d.ctypes.data_as(i32p), h.ctypes.data_as(i32p)))
        return d, h

    def reset_stream(self, stream):
        check(self.L.b2h264_enc_reset_stream(self.h, stream))

    def force_idr(self, stream=-1):
        check(self.L.b2h264_enc_force_idr(self.h, stream))

    def recon(self, stream=0):
        out = np.empty(self.frame_bytes, np.uint8)
        check(self.L.b2h264_enc_get_recon(self.h, stream, out.ctypes.data))
        return out

    def timing_us(self):
        t = (C.c_float * 3)()
        check(self.L.b2h264_enc_last_timing(self.h, t))
        return t[0], t[1], t[2]

    def d2h_bytes(self):
        """bytes the device handed over for the batch collected last (index table + coded records)"""
        v = C.c_ulonglong(0)
        check(self.L.b2h264_enc_last_d2h_bytes(self.h, C.byref(v)))
        return int(v.value)

    def coded_mbs(self):
        """macroblocks of the batch collected last that were coded (not P_SKIP), over all streams"""
        v = C.c_ulonglong(0)
        check(self.L.b2h264_enc_last_coded_mbs(self.h, C.byref(v)))
        return int(v.value)

    def set_stream(self, cuda_stream_handle):
        check(self.L.b2h264_enc_set_stream(self.h, cuda_stream_handle))

    def close(self):
        if self.h:
            self.L.b2h264_enc_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DecConfig(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("n_streams", C.c_int32), ("device", C.c_int32)]


class BatchDecoder:
    """include/b2h264_codec.h b2h264_dec_*: one access unit per stream per call -> one I420 picture per stream."""

    def __init__(self, width, height, n_streams=1, device=0, pinned_output=False):
        """pinned_output: the pictures land in ONE page-locked area owned by the decoder object (b2h264_host_alloc) and the
        arrays decode() returns are views of it, valid until the next call — what a server that consumes each picture at once does."""
        self.L = lib(device)
        self.cfg = DecConfig(width, height, n_streams, device)
        self.h = vp()
        check(self.L.b2h264_dec_create(C.byref(self.cfg), C.byref(self.h)))
        self.n = n_streams
        self.frame_bytes = width * height * 3 // 2
        self._pin = None
        self._stream = None            # the CUDA stream handle the decoder was moved to last (b2h264_dec_set_stream)
        if pinned_output:
            self._pin = self.L.b2h264_host_alloc(self.frame_bytes * n_streams)
            if not self._pin:
                raise MemoryError("b2h264_host_alloc")
            whole = np.ctypeslib.as_array(C.cast(self._pin, C.POINTER(C.c_uint8)), shape=(self.frame_bytes * n_streams,))
            self._outs = [whole[i * self.frame_bytes:(i + 1) * self.frame_bytes] for i in range(n_streams)]

    def _out_buffers(self):
        return self._outs if self._pin else [np.empty(self.frame_bytes, np.uint8) for _ in range(self.n)]

    def decode(self, access_units):
        """access_units: list of n_streams bytes objects; returns a list of numpy uint8 pictures (packed I420)."""
        bufs = [np.frombuffer(bytes(a), np.uint8) for a in access_units]
        outs = self._out_buffers()
        au = (vp * self.n)(*[b.ctypes.data for b in bufs])
        nb = (C.c_int32 * self.n)(*[len(b) for b in bufs])
        yo = (vp * self.n)(*[o.ctypes.data for o in outs])
        check(self.L.b2h264_dec_decode(self.h, au, nb, yo))
        return outs

    def decode2(self, access_units):
        """like decode(); entries may be None (stream sits the call out).  Returns (pictures or None per stream)."""
        bufs = [None if a is None else np.frombuffer(bytes(a), np.uint8) for a in access_units]
        outs = self._out_buffers()
        au = (vp * self.n)(*[None if b is None else b.ctypes.data for b in bufs])
        nb = (C.c_int32 * self.n)(*[0 if b is None else len(b) for b in bufs])
        yo = (vp * self.n)(*[o.ctypes.data for o in outs])
        got = (C.c_int32 * self.n)()
        check(self.L.b2h264_dec_decode2(self.h, au, nb, yo, got))
        return [outs[i] if got[i] else None for i in range(self.n)]

    def decode3(self, access_units):
        """like decode2(), with the outcome of every stream: returns (pictures or None, status) — status 1 picture, 0 none,
        < 0 that stream's error; a failing stream does not stop the others (b2h264_dec_decode3)."""
        bufs = [None if a is None else np.frombuffer(bytes(a), np.uint8) for a in access_units]
        outs = self._out_buffers()
        au = (vp * self.n)(*[None if b is None else b.ctypes.data for b in bufs])
        nb = (C.c_int32 * self.n)(*[0 if b is None else len(b) for b in bufs])
        yo = (vp * self.n)(*[o.ctypes.data for o in outs])
        st = (C.c_int32 * self.n)()
        check(self.L.b2h264_dec_decode3(self.h, au, nb, yo, st))
        return [outs[i] if st[i] == 1 else None for i in range(self.n)], list(st)

    def decode_device(self, access_units, out=None):
        """like decode3(), with the pictures left on the GPU (b2h264_dec_decode_device): returns (out, status).  out: a
        (n_streams, w*h*3//2) uint8 CUDA tensor on the decoder's device, allocated when None; row s receives stream s's picture
        where status[s] == 1 and is left untouched elsewhere.  It may also be a list of n_streams such 1-D tensors (None where the
        unit is None).  The work runs on torch.cuda.current_stream() and is complete when that stream reaches it."""
        import torch
        dev = torch.device("cuda", self.cfg.device)
        if out is None:
            out = torch.empty((self.n, self.frame_bytes), dtype=torch.uint8, device=dev)
        rows = list(out) if isinstance(out, (list, tuple)) else [out[i] for i in range(self.n)] if out.dim() == 2 else None
        if rows is None or len(rows) != self.n:
            raise ValueError("out must hold n_streams pictures")
        for r in rows:
            if r is not None and (r.dtype != torch.uint8 or r.device != dev or r.numel() != self.frame_bytes or (r.numel() > 1 and r.stride(0) != 1)):
                raise ValueError("each picture of out must be %d contiguous uint8 bytes on %s" % (self.frame_bytes, dev))
        st = torch.cuda.current_stream(dev).cuda_stream
        if st != self._stream:
            check(self.L.b2h264_dec_set_stream(self.h, st))
            self._stream = st
        bufs = [None if a is None else np.frombuffer(bytes(a), np.uint8) for a in access_units]
        au = (vp * self.n)(*[None if b is None else b.ctypes.data for b in bufs])
        nb = (C.c_int32 * self.n)(*[0 if b is None else len(b) for b in bufs])
        yo = (vp * self.n)(*[None if r is None else r.data_ptr() for r in rows])
        status = (C.c_int32 * self.n)()
        check(self.L.b2h264_dec_decode_device(self.h, au, nb, yo, status))
        return out, list(status)

    def reset_stream(self, stream):
        check(self.L.b2h264_dec_reset_stream(self.h, stream))

    def picture_order(self, stream=0):
        """(picture order count, flags: bit 0 IDR / bit 1 holds B slices, reorder depth) of the picture `stream` decoded last (b2h264_dec_last_picture_order): pictures
        come back in DECODING order; streams with B slices are output by ascending count inside each IDR period."""
        poc, idr, depth = C.c_int32(), C.c_int32(), C.c_int32()
        check(self.L.b2h264_dec_last_picture_order(self.h, stream, C.byref(poc), C.byref(idr), C.byref(depth)))
        return poc.value, idr.value, depth.value

    def close(self):
        if self.h:
            self.L.b2h264_dec_destroy(self.h)
            self.h = None
        if self._pin:
            self._outs = None
            self.L.b2h264_host_free(self._pin)
            self._pin = None


def probe_access_unit(au):
    """(width, height, has_slice) of an access unit (width / height 0 when it carries no SPS); no device needed"""
    a = np.frombuffer(bytes(au), np.uint8)
    w, h, s = C.c_int32(0), C.c_int32(0), C.c_int32(0)
    check(load().b2h264_dec_probe(a.ctypes.data, len(a), C.byref(w), C.byref(h), C.byref(s)))
    return w.value, h.value, bool(s.value)
