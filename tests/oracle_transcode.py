"""Loader of tests/transcode_oracle.c, the CPU oracle of smr_transcode_resize.  Test infrastructure.

The C file is compiled on first use into a temporary directory (the tree may be read-only) with -ffp-contract=off, so that
every f32 operation rounds on its own, and OpenMP over output rows.
"""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "transcode_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="transcode_oracle_")
        atexit.register(shutil.rmtree, d, ignore_errors=True)
        so = os.path.join(d, "libtranscode_oracle.so")
        subprocess.check_call(["gcc", "-O2", "-std=gnu99", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared", "-o", so, _SRC, "-lm"])
        _lib = C.CDLL(so)
        _lib.orc_transcode_resize.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int] + [C.c_int] * 5 + [C.c_void_p, C.c_void_p]
        _lib.orc_transcode_resize.restype = None
    return _lib


def transcode_resize(y, uv, out_w, out_h, scaling):
    """One rendition: y is the (h, w) luma crop, uv the (h / 2, w / 2, 2) chroma crop (views into a larger surface are
    fine: rows are read at their stride).  Returns the rendition's (out_h, out_w) Y and (out_h / 2, out_w / 2, 2) UV."""
    h, w = y.shape
    assert uv.shape == (h // 2, w // 2, 2) and y.dtype == np.uint8 and uv.dtype == np.uint8
    assert y.strides[1] == 1 and uv.strides[1:] == (2, 1)
    oy = np.empty((out_h, out_w), np.uint8)
    ouv = np.empty((out_h // 2, out_w // 2, 2), np.uint8)
    lib().orc_transcode_resize(y.ctypes.data, y.strides[0], uv.ctypes.data, uv.strides[0], w, h, int(out_w), int(out_h),
                               int(scaling), oy.ctypes.data, ouv.ctypes.data)
    return oy, ouv
