"""The CPU oracles written in C and C++ under tests/, their one build and their wrappers.  Test infrastructure.

Each library is compiled on first use into one temporary directory per session (the tree may be read-only) and cached by
the hash of its sources, with the flags the committed oracle is built with where they matter to the numbers:
-ffp-contract=off, so that only the fmaf() calls are fused, as on the GPU (--fmad=false).  The image, SVG, web, transcode
and video-convert oracles are one library; each shader source and each WGSL restatement is one more.

The shaders pinned through `render_shader` use only operations IEEE 754 rounds exactly (+ - * /, sqrtf, fminf / fmaxf,
floorf, fmaf); a shader calling transcendentals (sinf, expf, powf) is not reproducible bit for bit between the GPU's and
the C library's implementations and is not pinned here.  WGSL restatements that call transcendentals are compared within a
tolerance, not bit for bit.  RGBA -> NV12 is K11: `oracle.rgba_to_nv12_scaled`.
"""
import atexit
import ctypes as C
import functools
import hashlib
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_FLAGS = ["-O2", "-ffp-contract=off", "-mfma", "-fopenmp", "-fPIC", "-shared"]
_tmp = None
_libs = {}


def _dir():
    """the session's directory for sources and libraries"""
    global _tmp
    if _tmp is None:
        _tmp = tempfile.mkdtemp(prefix="c_oracles_")
        atexit.register(shutil.rmtree, _tmp, ignore_errors=True)
    return _tmp


def build(sources, cxx=False):
    """the library of `sources` (paths), compiled as C or, with `cxx`, as C++; built once per session and content"""
    h = hashlib.sha1(b"c++" if cxx else b"c")
    for s in sources:
        with open(s, "rb") as f:
            h.update(f.read())
    key = h.hexdigest()[:16]
    if key not in _libs:
        so = os.path.join(_dir(), key + ".so")
        cc = ["g++", "-std=c++17"] if cxx else ["gcc", "-std=gnu99"]
        subprocess.check_call(cc + _FLAGS + ["-o", so, *sources, "-lm"])
        _libs[key] = C.CDLL(so)
    return _libs[key]


def _fn(L, name, argtypes, restype=None):
    f = getattr(L, name)
    f.argtypes, f.restype = argtypes, restype


_DRAW = [C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]


@functools.cache
def _oracles():
    L = build([os.path.join(_HERE, f) for f in ("image_oracle.c", "svg_oracle.c", "web_oracle.c", "transcode_oracle.c",
                                                "video_convert_oracle.c")])
    _fn(L, "orc_render_image", [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p])
    _fn(L, "orc_render_svg", [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p])
    _fn(L, "orc_check_same_size_taps", [C.c_int], C.c_long)
    _fn(L, "orc_render_web", [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                              C.c_void_p, C.c_int, C.c_void_p])
    _fn(L, "orc_transcode_resize", [C.c_void_p, C.c_int, C.c_void_p, C.c_int] + [C.c_int] * 5 + [C.c_void_p, C.c_void_p])
    _fn(L, "orc_video_nv12_to_rgba", [C.c_void_p, C.c_int, C.c_void_p, C.c_int] + [C.c_int] * 4 + [C.c_void_p])
    return L


def _unit(text):
    """a C++ source file holding `text`, in the session's directory"""
    path = os.path.join(_dir(), hashlib.sha1(text.encode()).hexdigest()[:16] + ".cpp")
    with open(path, "w") as f:
        f.write(text)
    return path


@functools.cache
def shader_lib(source):
    """the library of a test shader's CUDA C++ source compiled against tests/shader_oracle_shim.h"""
    shim = os.path.join(_HERE, "shader_oracle_shim.h")
    L = build([_unit(f'#include "{shim}"\n#line 1 "shader"\n{source}\n')], cxx=True)
    _fn(L, "orc_render_shader", _DRAW)
    return L


@functools.cache
def wgsl_lib(restatement):
    """the library of a hand-written C++ restatement of one WGSL module's vs_main and fs_main, compiled against
    tests/wgsl_oracle_shim.h (its own rasteriser)"""
    shim = os.path.join(_HERE, "wgsl_oracle_shim.h")
    L = shader_lib(f'#define WO_PRE\n#include "{shim}"\n#undef WO_PRE\n{restatement}\n#include "{shim}"\n')
    _fn(L, "orc_render_wgsl", _DRAW)
    return L


def _children(children):
    """the children's pointers, widths and heights as the C draws take them (None: the empty view, 1 x 1), and the
    contiguous arrays the pointers point into"""
    kids = [None if c is None else np.ascontiguousarray(c, np.uint8) for c in children]
    n = max(1, len(kids))
    ptrs = (C.c_void_p * n)(*[None if c is None else c.ctypes.data for c in kids])
    cw = (C.c_int * n)(*[1 if c is None else c.shape[1] for c in kids])
    ch = (C.c_int * n)(*[1 if c is None else c.shape[0] for c in kids])
    return kids, ptrs, cw, ch


def time_of(pts):
    """BaseShaderParameters::time: Duration::as_secs_f32 of pts (seconds), whole seconds plus nanoseconds / 1e9 in f32"""
    ns = int(round(pts * 1e9))
    return np.float32(np.float32(ns // 1_000_000_000) + np.float32(ns % 1_000_000_000) / np.float32(1e9))


def _draw(fn, W, H, children, pts, params, mode):
    """a shader or WGSL draw into a cleared (H, W, 4) node texture"""
    out = np.zeros((H, W, 4), np.uint8)
    kids, ptrs, cw, ch = _children(children)
    pb = C.create_string_buffer(bytes(params), max(1, len(params)))
    fn(W, H, int(mode), float(time_of(pts)), pb if params else None, ptrs, cw, ch, len(kids), out.ctypes.data)
    return out


def render_image(rgba, ow, oh, mode=0):
    """ImageNode::render: a straight-alpha (h, w, 4) frame -> the premultiplied (oh, ow, 4) node texture"""
    rgba = np.ascontiguousarray(rgba, np.uint8)
    sh, sw = rgba.shape[:2]
    out = np.empty((oh, ow, 4), np.uint8)
    _oracles().orc_render_image(rgba.ctypes.data, sw, sh, int(ow), int(oh), int(mode), out.ctypes.data)
    return out


def render_svg(raster, mode=0):
    """SvgAsset::render: the caller's premultiplied (h, w, 4) raster at the node's size -> the (h, w, 4) node texture"""
    raster = np.ascontiguousarray(raster, np.uint8)
    h, w = raster.shape[:2]
    mid, out = np.empty((h, w, 4), np.uint8), np.empty((h, w, 4), np.uint8)
    _oracles().orc_render_svg(raster.ctypes.data, w, h, int(mode), mid.ctypes.data, out.ctypes.data)
    return out


def same_size_taps_off_texel(max_dim):
    return _oracles().orc_check_same_size_taps(int(max_dim))


def render_web(prev, bgra, children, rects, embedding, mode=0):
    """WebRenderer::render: `prev` the (H, W, 4) node texture before the tick, `bgra` the page or None (no frame: `prev`
    stays), `children` each child's (h, w, 4) premultiplied RGBA8 node texture or None (the empty view), `rects` a list of
    (x, y, width, height).  Returns the node texture after the tick."""
    out = np.ascontiguousarray(prev, np.uint8).copy()
    H, W = out.shape[:2]
    kids, ptrs, cw, ch = _children(children)
    r = np.ascontiguousarray(np.asarray(rects, np.float64).reshape(-1, 4))
    page = None if bgra is None else np.ascontiguousarray(bgra, np.uint8)
    assert page is None or page.shape == (H, W, 4)
    _oracles().orc_render_web(W, H, int(mode), int(embedding), None if page is None else page.ctypes.data, ptrs, cw, ch,
                              len(kids), r.ctypes.data if len(r) else None, len(r), out.ctypes.data)
    return out


def transcode_resize(y, uv, out_w, out_h, scaling):
    """One rendition: y is the (h, w) luma crop, uv the (h / 2, w / 2, 2) chroma crop (views into a larger surface are
    fine: rows are read at their stride).  Returns the rendition's (out_h, out_w) Y and (out_h / 2, out_w / 2, 2) UV."""
    h, w = y.shape
    assert uv.shape == (h // 2, w // 2, 2) and y.dtype == np.uint8 and uv.dtype == np.uint8
    assert y.strides[1] == 1 and uv.strides[1:] == (2, 1)
    oy = np.empty((out_h, out_w), np.uint8)
    ouv = np.empty((out_h // 2, out_w // 2, 2), np.uint8)
    _oracles().orc_transcode_resize(y.ctypes.data, y.strides[0], uv.ctypes.data, uv.strides[0], w, h, int(out_w),
                                    int(out_h), int(scaling), oy.ctypes.data, ouv.ctypes.data)
    return oy, ouv


def nv12_to_rgba(y, uv, out_w=None, out_h=None):
    """y is the (h, w) luma crop, uv the (h / 2, w / 2, 2) chroma crop (views into a larger surface are fine: rows are read
    at their stride).  Returns the (out_h, out_w, 4) RGBA8 target (default: the source size)."""
    h, w = y.shape
    assert uv.shape == (h // 2, w // 2, 2) and y.dtype == np.uint8 and uv.dtype == np.uint8
    assert y.strides[1] == 1 and uv.strides[1:] == (2, 1)
    out_w, out_h = (w, h) if out_w is None else (int(out_w), int(out_h))
    out = np.empty((out_h, out_w, 4), np.uint8)
    _oracles().orc_video_nv12_to_rgba(y.ctypes.data, y.strides[0], uv.ctypes.data, uv.strides[0], w, h, out_w, out_h,
                                      out.ctypes.data)
    return out


def render_shader(source, W, H, children, pts=0.0, params=b"", mode=0):
    """ShaderNode::render: `children` each child's (h, w, 4) premultiplied RGBA8 node texture or None (the empty view),
    `params` the parameter bytes.  Returns the (H, W, 4) node texture."""
    return _draw(shader_lib(source).orc_render_shader, W, H, children, pts, params, mode)


def render_wgsl(restatement, W, H, children, pts=0.0, params=b"", mode=0):
    """the (H, W, 4) node texture a WGSL shader node draws: `children` each child's RGBA8 node texture or None"""
    return _draw(wgsl_lib(restatement).orc_render_wgsl, W, H, children, pts, params, mode)

