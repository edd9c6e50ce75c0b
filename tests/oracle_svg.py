"""Loader of tests/svg_oracle.c, the CPU oracle of SVG image node textures (orc_render_svg, orc_check_same_size_taps).
Test infrastructure.

Compiled on first use into a temporary directory (the tree may be read-only) with the flags tests/oracle_image.py uses
for the image oracle it includes: -ffp-contract=off, so that only the fmaf() calls are fused.
"""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "svg_oracle.c")
_lib = None


def _load():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="svg_oracle_")
        atexit.register(shutil.rmtree, d, ignore_errors=True)
        so = os.path.join(d, "libsvg_oracle.so")
        subprocess.check_call(["gcc", "-O2", "-std=gnu99", "-ffp-contract=off", "-mfma", "-fPIC", "-shared", "-o", so, _SRC, "-lm"])
        L = C.CDLL(so)
        L.orc_render_svg.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        L.orc_render_svg.restype = None
        L.orc_check_same_size_taps.argtypes = [C.c_int]
        L.orc_check_same_size_taps.restype = C.c_long
        _lib = L
    return _lib


def render_svg(raster, mode=0):
    """SvgAsset::render: the caller's premultiplied (h, w, 4) raster at the node's size -> the (h, w, 4) node texture"""
    raster = np.ascontiguousarray(raster, np.uint8)
    h, w = raster.shape[:2]
    mid, out = np.empty((h, w, 4), np.uint8), np.empty((h, w, 4), np.uint8)
    _load().orc_render_svg(raster.ctypes.data, w, h, int(mode), mid.ctypes.data, out.ctypes.data)
    return out


def same_size_taps_off_texel(max_dim):
    return _load().orc_check_same_size_taps(int(max_dim))
