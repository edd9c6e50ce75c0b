"""Loader of tests/video_convert_oracle.c, the CPU oracle of smr_video_nv12_to_rgba.  Test infrastructure.

The C file is compiled on first use into a temporary directory (the tree may be read-only) with -ffp-contract=off, so that
every f32 operation rounds on its own, and OpenMP over target rows.  RGBA -> NV12 is K11: `oracle.rgba_to_nv12_scaled`.
"""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "video_convert_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="video_convert_oracle_")
        atexit.register(shutil.rmtree, d, ignore_errors=True)
        so = os.path.join(d, "libvideo_convert_oracle.so")
        subprocess.check_call(["gcc", "-O2", "-std=gnu99", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared", "-o", so, _SRC, "-lm"])
        _lib = C.CDLL(so)
        _lib.orc_video_nv12_to_rgba.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int] + [C.c_int] * 4 + [C.c_void_p]
        _lib.orc_video_nv12_to_rgba.restype = None
    return _lib


def nv12_to_rgba(y, uv, out_w=None, out_h=None):
    """y is the (h, w) luma crop, uv the (h / 2, w / 2, 2) chroma crop (views into a larger surface are fine: rows are read
    at their stride).  Returns the (out_h, out_w, 4) RGBA8 target (default: the source size)."""
    h, w = y.shape
    assert uv.shape == (h // 2, w // 2, 2) and y.dtype == np.uint8 and uv.dtype == np.uint8
    assert y.strides[1] == 1 and uv.strides[1:] == (2, 1)
    out_w, out_h = (w, h) if out_w is None else (int(out_w), int(out_h))
    out = np.empty((out_h, out_w, 4), np.uint8)
    lib().orc_video_nv12_to_rgba(y.ctypes.data, y.strides[0], uv.ctypes.data, uv.strides[0], w, h, out_w, out_h, out.ctypes.data)
    return out
