"""Loader of the shader oracle: a test shader's CUDA C++ source compiled for the CPU against tests/shader_oracle_shim.h.
Test infrastructure.

Each source is compiled on first use into a temporary directory (the tree may be read-only) with g++ -ffp-contract=off,
so that only its fmaf() calls are fused, as on the GPU (--fmad=false).  The shaders pinned this way use only operations
IEEE 754 rounds exactly (+ - * /, sqrtf, fminf / fmaxf, floorf, fmaf); a shader calling transcendentals (sinf, expf, powf)
is not reproducible bit for bit between the GPU's and the C library's implementations and is not pinned here.
"""
import atexit
import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile

import numpy as np

_SHIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "shader_oracle_shim.h")
_dir = None
_libs = {}


def lib(source):
    global _dir
    key = hashlib.sha1(source.encode()).hexdigest()[:16]
    if key not in _libs:
        if _dir is None:
            _dir = tempfile.mkdtemp(prefix="shader_oracle_")
            atexit.register(shutil.rmtree, _dir, ignore_errors=True)
        cpp, so = os.path.join(_dir, key + ".cpp"), os.path.join(_dir, key + ".so")
        with open(cpp, "w") as f:
            f.write(f'#include "{_SHIM}"\n#line 1 "shader"\n{source}\n')
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-mfma", "-fPIC", "-shared", "-o", so, cpp, "-lm"])
        L = C.CDLL(so)
        L.orc_render_shader.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_int, C.c_void_p]
        L.orc_render_shader.restype = None
        _libs[key] = L
    return _libs[key]


def time_of(pts):
    """BaseShaderParameters::time: Duration::as_secs_f32 of pts (seconds), whole seconds plus nanoseconds / 1e9 in f32"""
    ns = int(round(pts * 1e9))
    return np.float32(np.float32(ns // 1_000_000_000) + np.float32(ns % 1_000_000_000) / np.float32(1e9))


def render_shader(source, W, H, children, pts=0.0, params=b"", mode=0):
    """ShaderNode::render: `children` each child's (h, w, 4) premultiplied RGBA8 node texture or None (the empty view),
    `params` the parameter bytes.  Returns the (H, W, 4) node texture."""
    out = np.zeros((H, W, 4), np.uint8)
    kids = [None if c is None else np.ascontiguousarray(c, np.uint8) for c in children]
    ptrs = (C.c_void_p * max(1, len(kids)))(*[None if c is None else c.ctypes.data for c in kids])
    cw = (C.c_int * max(1, len(kids)))(*[1 if c is None else c.shape[1] for c in kids])
    ch = (C.c_int * max(1, len(kids)))(*[1 if c is None else c.shape[0] for c in kids])
    pb = C.create_string_buffer(bytes(params), max(1, len(params)))
    lib(source).orc_render_shader(W, H, int(mode), float(time_of(pts)), pb if params else None, ptrs, cw, ch, len(kids),
                                  out.ctypes.data)
    return out
