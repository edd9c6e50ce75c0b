"""Loader of the WGSL shader oracle: a hand-written C++ restatement of one WGSL module's vs_main and fs_main, compiled for
the CPU against tests/wgsl_oracle_shim.h (its own rasteriser).  Test infrastructure.

Compiled on first use into a temporary directory with g++ -ffp-contract=off, so that the arithmetic rounds as the GPU's
does under --fmad=false.  Restatements that call transcendentals are compared within a tolerance, not bit for bit."""
import ctypes as C
import os

import numpy as np

from tests import oracle_shader

_SHIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "wgsl_oracle_shim.h")


def lib(restatement):
    L = oracle_shader.lib(f'#define WO_PRE\n#include "{_SHIM}"\n#undef WO_PRE\n{restatement}\n#include "{_SHIM}"\n')
    if not hasattr(L, "_wgsl_ready"):
        L.orc_render_wgsl.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_int, C.c_void_p]
        L.orc_render_wgsl.restype = None
        L._wgsl_ready = True
    return L


def render(restatement, W, H, children, pts=0.0, params=b"", mode=0):
    """the (H, W, 4) node texture a WGSL shader node draws: `children` each child's RGBA8 node texture or None"""
    out = np.zeros((H, W, 4), np.uint8)
    kids = [None if c is None else np.ascontiguousarray(c, np.uint8) for c in children]
    ptrs = (C.c_void_p * max(1, len(kids)))(*[None if c is None else c.ctypes.data for c in kids])
    cw = (C.c_int * max(1, len(kids)))(*[1 if c is None else c.shape[1] for c in kids])
    ch = (C.c_int * max(1, len(kids)))(*[1 if c is None else c.shape[0] for c in kids])
    pb = C.create_string_buffer(bytes(params), max(1, len(params)))
    lib(restatement).orc_render_wgsl(W, H, int(mode), float(oracle_shader.time_of(pts)), pb if params else None, ptrs, cw, ch,
                                     len(kids), out.ctypes.data)
    return out
