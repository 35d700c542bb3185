"""Test helpers: ctypes bindings for the CPU oracle (oracle/liboracle.so), the compiled reference
behind its plain-C shim (oracle/_ref/librefshim.so, present only where the reference was built) and
the product library (openh264_b200/libopenh264_b200.so).

The oracle and the reference shim export the same signatures under the prefixes ``orc_`` / ``ref_``
so a test can run both on identical buffers.
"""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_SO = os.path.join(ROOT, "oracle", "liboracle.so")
REFSHIM_SO = os.path.join(ROOT, "oracle", "_ref", "librefshim.so")
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
GOLDEN = os.path.join(ROOT, "tests", "golden")
REF_SRC = os.environ.get("OPENH264_REF", "/root/reference")        # the reference's sources, where they exist (as in build())


def reference_vector(rel):
    """path of a bitstream of the reference's res/ directory (`rel` = "res/<name>"): the committed copy under tests/golden
    where there is one, else the reference's own file where its sources exist, else None (the vectors of several MB)"""
    name = os.path.basename(rel)
    for d in ("conformance", "conformance_b", "rejected"):
        p = os.path.join(GOLDEN, d, name)
        if os.path.exists(p):
            return p
    p = os.path.join(REF_SRC, rel)
    return p if os.path.exists(p) else None


def reference_clip(name, w, h, n):
    """the first n pictures of one of the reference's res/*.yuv clips: committed under tests/golden (whole, or the first pictures
    gzip-compressed under tests/golden/clips), else read from the reference's sources where they exist, else None"""
    import gzip
    size = n * w * h * 3 // 2
    whole = os.path.join(GOLDEN, name)
    if os.path.exists(whole):
        data = open(whole, "rb").read()
    else:
        pre = [f for f in os.listdir(os.path.join(GOLDEN, "clips")) if f.startswith(name + ".first")]
        if pre:
            data = gzip.open(os.path.join(GOLDEN, "clips", pre[0])).read()
        elif os.path.exists(os.path.join(REF_SRC, "res", name)):
            data = open(os.path.join(REF_SRC, "res", name), "rb").read(size)
        else:
            return None
    return np.frombuffer(data[:size], np.uint8).copy() if len(data) >= size else None

BLK_DIMS = [(16, 16), (16, 8), (8, 16), (8, 8), (4, 4), (8, 4), (4, 8)]

u8p = C.POINTER(C.c_uint8)
i8p = C.POINTER(C.c_int8)
i16p = C.POINTER(C.c_int16)
u16p = C.POINTER(C.c_uint16)
i32p = C.POINTER(C.c_int32)


class MeJob(C.Structure):
    _fields_ = [("blk", C.c_int32), ("cur_off", C.c_int32), ("ref_off", C.c_int32),
                ("mvp_x", C.c_int16), ("mvp_y", C.c_int16),
                ("mv_min_x", C.c_int16), ("mv_min_y", C.c_int16), ("mv_max_x", C.c_int16), ("mv_max_y", C.c_int16),
                ("n_mvc", C.c_int32), ("mvc", (C.c_int16 * 2) * 5),
                ("sad_pred", C.c_uint32), ("qp", C.c_int32), ("calc_satd", C.c_int32)]


class MeResult(C.Structure):
    _fields_ = [("mv_x", C.c_int16), ("mv_y", C.c_int16), ("sad_cost", C.c_uint32), ("satd_cost", C.c_uint32),
                ("ref_off", C.c_int32)]


class RefineJob(C.Structure):
    _fields_ = [("w", C.c_int32), ("h", C.c_int32), ("cur_off", C.c_int32), ("ref_off", C.c_int32),
                ("mv_x", C.c_int16), ("mv_y", C.c_int16), ("mvp_x", C.c_int16), ("mvp_y", C.c_int16),
                ("qp", C.c_int32), ("satd_in_md", C.c_int32), ("satd", C.c_uint32)]


class RefineResult(C.Structure):
    _fields_ = [("mv_x", C.c_int16), ("mv_y", C.c_int16), ("cost", C.c_uint32)]


class PskipJob(C.Structure):
    _fields_ = [("cur_off", C.c_int32 * 3), ("ref_off", C.c_int32 * 3), ("mb_x", C.c_int32), ("mb_y", C.c_int32),
                ("mb_w", C.c_int32), ("mb_h", C.c_int32), ("qp", C.c_int32), ("md_using_sad", C.c_int32),
                ("ref", C.c_int32 * 4), ("mv", (C.c_int32 * 2) * 4), ("skip", C.c_int32 * 4), ("skip_sad", C.c_int32 * 4),
                ("ref_is_p", C.c_int32), ("col_type", C.c_int32), ("col_skip_sad", C.c_int32)]


class PskipResult(C.Structure):
    _fields_ = [("ok", C.c_int32), ("mv_x", C.c_int32), ("mv_y", C.c_int32), ("sad_pred_skip", C.c_int32),
                ("sad_luma", C.c_int32), ("sad_chroma", C.c_int32), ("cost_luma", C.c_int32), ("cost_skip", C.c_int32),
                ("sad_cost", C.c_int32), ("outcome", C.c_int32), ("score", C.c_int32 * 3)]


# orc_pskip's outcome codes (h264_oracle.h: ORC_PSKIP_*)
PSKIP_OUTCOMES = ["range left", "range right", "range top", "range bottom", "SAD 0", "SAD < predictor", "SAD < co-located",
                  "luma level > 1", "luma score >= 6", "Cb DC", "Cr DC", "Cb level > 1", "Cr level > 1", "Cb score >= 7",
                  "Cr score >= 7", "accepted after the DCT tests"]


# name -> (restype, argtypes) shared by orc_* and ref_*
SIGS = {
    "sad": (C.c_int32, [C.c_int, u8p, C.c_int, u8p, C.c_int]),
    "sad_four": (None, [C.c_int, u8p, C.c_int, u8p, C.c_int, i32p]),
    "satd": (C.c_int32, [C.c_int, u8p, C.c_int, u8p, C.c_int]),
    "mc_luma": (None, [u8p, C.c_int, u8p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "mc_chroma": (None, [u8p, C.c_int, u8p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "pixel_avg": (None, [u8p, C.c_int, u8p, C.c_int, u8p, C.c_int, C.c_int, C.c_int]),
    "dct4x4": (None, [i16p, u8p, C.c_int, u8p, C.c_int]),
    "dct_four4x4": (None, [i16p, u8p, C.c_int, u8p, C.c_int]),
    "quant4x4": (None, [i16p, i16p, i16p]),
    "quant4x4_dc": (None, [i16p, C.c_int16, C.c_int16]),
    "quant_four4x4": (None, [i16p, i16p, i16p]),
    "quant_four4x4_max": (None, [i16p, i16p, i16p, i16p]),
    "hadamard_quant2x2_skip": (C.c_int32, [i16p, C.c_int16, C.c_int16]),
    "hadamard_quant2x2": (C.c_int32, [i16p, C.c_int16, C.c_int16, i16p, i16p]),
    "hadamard_t4_dc": (None, [i16p, i16p]),
    "scan4x4_dcac": (None, [i16p, i16p]),
    "scan4x4_ac": (None, [i16p, i16p]),
    "single_ctr4x4": (C.c_int32, [i16p]),
    "nonzero_count": (C.c_int32, [i16p]),
    "ihadamard4x4_dc": (None, [i16p]),
    "dequant_luma_dc4x4": (None, [i16p, C.c_int]),
    "dequant_ihadamard4x4": (None, [i16p, C.c_uint16]),
    "dequant_ihadamard2x2_dc": (None, [i16p, C.c_uint16]),
    "dequant4x4": (None, [i16p, u16p]),
    "dequant_four4x4": (None, [i16p, u16p]),
    "idct4x4_rec": (None, [u8p, C.c_int, u8p, C.c_int, i16p]),
    "idct_four4x4_rec": (None, [u8p, C.c_int, u8p, C.c_int, i16p]),
    "idct_rec_i16x16_dc": (None, [u8p, C.c_int, u8p, C.c_int, i16p]),
    "idct_res_add_pred": (None, [u8p, C.c_int, i16p]),
    "idct_res_add_pred8x8": (None, [u8p, C.c_int, i16p]),
    "deblock_luma_lt4": (None, [u8p, C.c_int, C.c_int, C.c_int, C.c_int, i8p]),
    "deblock_luma_eq4": (None, [u8p, C.c_int, C.c_int, C.c_int, C.c_int]),
    "deblock_chroma_lt4": (None, [u8p, u8p, C.c_int, C.c_int, C.c_int, C.c_int, i8p]),
    "deblock_chroma_eq4": (None, [u8p, u8p, C.c_int, C.c_int, C.c_int, C.c_int]),
    "expand_plane": (None, [u8p, C.c_int, C.c_int, C.c_int, C.c_int]),
    "me_search": (None, [u8p, C.c_int, u8p, C.c_int, C.POINTER(MeJob), C.POINTER(MeResult)]),
    "me_refine": (None, [u8p, C.c_int, u8p, C.c_int, C.POINTER(RefineJob), C.POINTER(RefineResult), u8p]),
    "pskip": (None, [u8p, C.c_int, C.c_int, u8p, C.c_int, C.c_int, C.POINTER(PskipJob), C.POINTER(PskipResult), u8p]),
    "quant_ff": (i16p, [C.c_int]),
    "quant_mf": (i16p, [C.c_int]),
    "dequant_coeff": (u16p, [C.c_int]),
    "qp_lambda": (C.c_int, [C.c_int]),
    "chroma_qp": (C.c_int, [C.c_int]),
}


class _Lib:
    """`strict` = every signature must be exported.  The oracle is rebuilt from its sources before it is loaded, so it is strict;
    a reference build made before a function was added to the shim lacks it: that function is listed in `missing` (the tests
    of it skip) and every other one stays usable."""

    def __init__(self, path, prefix, strict=True):
        self.lib = C.CDLL(path)
        self.prefix = prefix
        self.missing = set()
        for name, (res, args) in SIGS.items():
            if not strict and not hasattr(self.lib, prefix + name):
                self.missing.add(name)
                continue
            fn = getattr(self.lib, prefix + name)
            fn.restype = res
            fn.argtypes = args
            setattr(self, name, fn)


def build_oracle():
    """(Re)build oracle/liboracle.so from the C restatement (seconds, gcc only)."""
    subprocess.check_call(["make", "-s", "-f", "oracle/Makefile"], cwd=ROOT)


_oracle = None
_ref = None
_emu = None


def emu():
    """tests/emu/libb2h264_emu.so, the host emulation build of the device macroblock code with every stage's test hooks, built
    (make) and loaded once per process.  The library is shared: a test that depends on its settings (emu_set_*) or counters
    sets or resets them itself."""
    global _emu
    if _emu is None:
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "emu")])
        E = C.CDLL(os.path.join(ROOT, "tests", "emu", "libb2h264_emu.so"))
        vp, i = C.c_void_p, C.c_int
        E.emu_encode.restype = C.c_long
        E.emu_encode.argtypes = [vp, i, i, i, i, C.c_float, vp, C.c_long, vp, vp]
        E.emu_stages_run.restype = C.c_uint
        E.emu_decode.restype = C.c_int
        E.emu_decode.argtypes = [vp, C.c_long, vp, C.c_long, C.POINTER(i), C.POINTER(i)]
        E.b2h264_dec_wp_stats.restype = C.c_int
        E.b2h264_dec_wp_stats.argtypes = [C.POINTER(C.c_longlong), i, i]
        E.emu_deblock_picture.restype = C.c_int
        E.emu_deblock_picture.argtypes = [vp] * 3 + [i] * 4 + [vp, vp] + [i] * 4
        E.emu_decode_records.argtypes = [i, i, i, vp, vp, vp, vp, i, vp, vp, vp]
        E.emu_skip_test.argtypes = [i, vp, C.c_longlong, vp, vp]
        E.emu_skip_outcomes.argtypes = [vp, i]
        E.emu_check_chroma_pair.restype = C.c_long
        E.emu_me_partitions.argtypes = [i, vp, C.c_longlong, vp, vp]
        E.emu_intra_tail.argtypes = [i, vp, vp]
        E.emu_i4_ends.argtypes = [vp, i]
        E.emu_inter_residual.argtypes = [i, vp, vp, vp]
        E.emu_res_outcomes.argtypes = [vp, i]
        _emu = E
    return _emu


def oracle():
    global _oracle
    if _oracle is None:
        build_oracle()
        _oracle = _Lib(ORACLE_SO, "orc_")
        _oracle.lib.orc_mvd_cost_init.argtypes = [u16p, C.c_int, C.c_int]
        _oracle.lib.orc_mvd_cost_init.restype = None
    return _oracle


def have_ref():
    return os.path.exists(REFSHIM_SO)


def ref():
    global _ref
    if _ref is None:
        _ref = _Lib(REFSHIM_SO, "ref_", strict=False)
        _ref.lib.ref_mvd_cost_init_all.argtypes = [u16p, C.c_int]
        _ref.lib.ref_halfpel.argtypes = [C.c_int, u8p, C.c_int, u8p, C.c_int, C.c_int, C.c_int]
    return _ref


def ptr(a, ct=None, off=0):
    """ctypes pointer into a numpy array at element offset `off`."""
    if ct is None:
        ct = {np.dtype(np.uint8): C.c_uint8, np.dtype(np.int8): C.c_int8, np.dtype(np.int16): C.c_int16,
              np.dtype(np.uint16): C.c_uint16, np.dtype(np.int32): C.c_int32}[a.dtype]
    return C.cast(a.ctypes.data + off * a.itemsize, C.POINTER(ct))


def sha1(*arrays):
    h = hashlib.sha1()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def synth_frame(w, h, t=0, seed=264):
    """Deterministic natural-ish luma frame: smooth multi-octave pattern + moving rectangles +
    small per-frame noise, global pan (+3,+1)/frame (SURVEY §8(d) generator, numpy form)."""
    yy, xx = np.mgrid[0:h, 0:w].astype(np.int64)
    px, py = xx + 3 * t, yy + 1 * t
    v = (128 + 40 * np.sin(px / 37.0) + 30 * np.cos(py / 23.0) + 20 * np.sin((px + py) / 11.0)
         + 12 * np.sin(px / 5.0) * np.cos(py / 7.0))
    for k in range(8):
        rx = (k * 211 + 5 * t * (k % 3 + 1)) % max(1, w - 64)
        ry = (k * 97 + 3 * t * (k % 2 + 1)) % max(1, h - 48)
        blk = ((xx[ry:ry + 48, rx:rx + 64] * (k + 3) + yy[ry:ry + 48, rx:rx + 64] * (k + 1)) % 64) + 60 + 10 * k
        v[ry:ry + 48, rx:rx + 64] = blk
    rng = np.random.RandomState(seed + t)
    v = v + rng.randint(-3, 4, size=(h, w))
    return np.clip(v, 16, 235).astype(np.uint8)


def synth_clip(w, h, n, seed=264, noise=3):
    """Deterministic INTEGER-ONLY I420 clip (bit-identical on every machine): multi-octave value noise from a
    32-bit LCG, bilinearly upsampled with integer weights, global pan (+3,+1)/frame, 6 moving textured
    rectangles, +-3 per-frame noise; chroma = low-amplitude functions of the half-resolution luma.
    `noise` = amplitude of the per-frame noise (3 = the default clip; 12 = the bench's "hard" workload: far fewer
    skipped macroblocks, several times the bits).  Returns a uint8 array of n*w*h*3/2 bytes."""
    def lcg_field(gh, gw, s):
        idx = (np.arange(gh * gw, dtype=np.uint64).reshape(gh, gw) + np.uint64(s) * np.uint64(7919)) & np.uint64(0xffffffff)
        x = (idx * np.uint64(1664525) + np.uint64(1013904223)) & np.uint64(0xffffffff)
        x = (x * np.uint64(1664525) + np.uint64(1013904223)) & np.uint64(0xffffffff)
        x = (x ^ (x >> np.uint64(15))) * np.uint64(2246822519) & np.uint64(0xffffffff)
        return ((x >> np.uint64(13)) & np.uint64(255)).astype(np.int64)

    def upsample(f, cell, H, W):       # integer bilinear, weights in 1/cell units
        yy = np.arange(H, dtype=np.int64); xx = np.arange(W, dtype=np.int64)
        y0, fy = yy // cell, yy % cell
        x0, fx = xx // cell, xx % cell
        a = f[y0][:, x0]; b = f[y0][:, x0 + 1]; c = f[y0 + 1][:, x0]; d = f[y0 + 1][:, x0 + 1]
        fy = fy[:, None]; fx = fx[None, :]
        return (a * (cell - fy) * (cell - fx) + b * (cell - fy) * fx + c * fy * (cell - fx) + d * fy * fx) // (cell * cell)

    PW, PH = w + 3 * n + 64, h + n + 64            # panned canvas
    base = np.zeros((PH, PW), np.int64)
    for k, (cell, amp) in enumerate([(64, 6), (16, 3), (4, 1)]):
        f = lcg_field(PH // cell + 3, PW // cell + 3, seed + k)
        base += upsample(f, cell, PH, PW) * amp
    base = 40 + base * 150 // (255 * 10)
    frames = []
    for t in range(n):
        y = base[t:t + h, 3 * t:3 * t + w].copy()
        yy, xx = np.mgrid[0:h, 0:w].astype(np.int64)
        for k in range(6):
            rw, rh = 48 + 8 * k, 32 + 8 * (k % 3)
            rx = (k * 211 + (2 * (k % 3) + 1) * t * 2) % max(1, w - rw)
            ry = (k * 97 + ((k % 2) + 1) * t) % max(1, h - rh)
            y[ry:ry + rh, rx:rx + rw] = ((xx[ry:ry + rh, rx:rx + rw] * (k + 3) + yy[ry:ry + rh, rx:rx + rw] * (k + 1)) % 64) + 60 + 12 * k
        nz = lcg_field(h, w, seed + 1000 + t) % (2 * noise + 1) - noise
        y = np.clip(y + nz, 16, 235).astype(np.uint8)
        sub = y[::2, ::2].astype(np.int64)
        u = np.clip(128 + (sub - 128) // 4, 16, 240).astype(np.uint8)
        v = np.clip(128 - (sub - 128) // 6, 16, 240).astype(np.uint8)
        frames.append(np.concatenate([y.ravel(), u[:h // 2, :w // 2].ravel(), v[:h // 2, :w // 2].ravel()]))
    return np.concatenate(frames)


def split_access_units(bs):
    """Annex-B stream -> list of access units (bytes).  An access unit ends with a slice NAL (type 1 / 5) that is followed by a
    non-slice NAL or by a slice with first_mb_in_slice == 0 (its ue(v) is the single bit 1 right after the NAL header)."""
    bs = bytes(bs)
    starts, i, n = [], 0, len(bs)
    while i + 3 <= n:
        if bs[i] == 0 and bs[i + 1] == 0 and bs[i + 2] == 1:
            starts.append((i - 1 if i > 0 and bs[i - 1] == 0 else i, i + 3))      # (unit start incl. zero_byte, header position)
            i += 3
        else:
            i += 1
    aus, begin = [], starts[0][0] if starts else 0
    for k, (_, hdr) in enumerate(starts):
        t = bs[hdr] & 31
        if t not in (1, 5):
            continue
        last = True
        if k + 1 < len(starts):
            nh = starts[k + 1][1]
            if (bs[nh] & 31) in (1, 5) and nh + 1 < n and not (bs[nh + 1] & 0x80):
                last = False
        if last:
            end = starts[k + 1][0] if k + 1 < len(starts) else n
            aus.append(bs[begin:end])
            begin = end
    return aus
