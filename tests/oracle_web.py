"""Loader of tests/web_oracle.c, the CPU oracle of web view node textures.  Test infrastructure.

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

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "web_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="web_oracle_")
        atexit.register(shutil.rmtree, d, ignore_errors=True)
        so = os.path.join(d, "libweb_oracle.so")
        subprocess.check_call(["gcc", "-O2", "-std=gnu99", "-ffp-contract=off", "-mfma", "-fPIC", "-shared", "-o", so, _SRC, "-lm"])
        _lib = C.CDLL(so)
        _lib.orc_render_web.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        _lib.orc_render_web.restype = None
    return _lib


def render_web(prev, bgra, children, rects, embedding, mode=0):
    """WebRenderer::render: `prev` the (H, W, 4) node texture before the tick, `bgra` the page or None (no frame: `prev`
    stays), `children` each child's (h, w, 4) premultiplied RGBA8 node texture or None (the empty view), `rects` a list of
    (x, y, width, height).  Returns the node texture after the tick."""
    out = np.ascontiguousarray(prev, np.uint8).copy()
    H, W = out.shape[:2]
    kids = [None if c is None else np.ascontiguousarray(c, np.uint8) for c in children]
    ptrs = (C.c_void_p * max(1, len(kids)))(*[None if c is None else c.ctypes.data for c in kids])
    cw = (C.c_int * max(1, len(kids)))(*[1 if c is None else c.shape[1] for c in kids])
    ch = (C.c_int * max(1, len(kids)))(*[1 if c is None else c.shape[0] for c in kids])
    r = np.ascontiguousarray(np.asarray(rects, np.float64).reshape(-1, 4))
    page = None if bgra is None else np.ascontiguousarray(bgra, np.uint8)
    assert page is None or page.shape == (H, W, 4)
    lib().orc_render_web(W, H, int(mode), int(embedding), None if page is None else page.ctypes.data, ptrs, cw, ch, len(kids),
                         r.ctypes.data if len(r) else None, len(r), out.ctypes.data)
    return out
