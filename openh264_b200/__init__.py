"""openh264_b200 — H100-native H.264 macroblock pipeline (drop-in for the hot path of cisco/openh264).

The product is the C-ABI shared library ``libopenh264_b200.so`` (hand-written sm_90a CUDA + C++ host
code, sources under ``openh264_b200/csrc``, headers under ``include/``).  This Python package is only a
thin ctypes mirror used by the tests and the benchmark; it never computes anything itself and it
fails loudly when the CUDA library is missing (there is no CPU fallback).
"""
from .binding import B2H264Error, DeviceArray, build, lib, load  # noqa: F401
