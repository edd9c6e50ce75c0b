"""Loader of tests/image_oracle.c, the CPU oracle of image node textures.  Test infrastructure.

The C file is compiled on first use into a temporary directory (the tree may be read-only), with the flags the committed
oracle is built with where they matter to the numbers: -ffp-contract=off, so that only the fmaf() calls are fused.
"""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "image_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="image_oracle_")
        atexit.register(shutil.rmtree, d, ignore_errors=True)
        so = os.path.join(d, "libimage_oracle.so")
        subprocess.check_call(["gcc", "-O2", "-std=gnu99", "-ffp-contract=off", "-mfma", "-fPIC", "-shared", "-o", so, _SRC, "-lm"])
        _lib = C.CDLL(so)
        _lib.orc_render_image.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
        _lib.orc_render_image.restype = None
    return _lib


def render_image(rgba, ow, oh, mode=0):
    """ImageNode::render: a straight-alpha (h, w, 4) frame -> the premultiplied (oh, ow, 4) node texture"""
    rgba = np.ascontiguousarray(rgba, np.uint8)
    sh, sw = rgba.shape[:2]
    out = np.empty((oh, ow, 4), np.uint8)
    lib().orc_render_image(rgba.ctypes.data, sw, sh, int(ow), int(oh), int(mode), out.ctypes.data)
    return out
