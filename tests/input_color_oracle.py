"""The oracle of an input's colour setting (smr_set_input_color, DESIGN.md NC-13): `input_color_oracle.c`, built with
`tests/c_oracles.build`.  Test infrastructure.  matrix 0 BT.709, 1 BT.601; full_range applies to every YUV format."""
import ctypes as C
import functools
import os

import numpy as np

from tests.c_oracles import build

_HERE = os.path.dirname(os.path.abspath(__file__))


@functools.cache
def _lib():
    L = build([os.path.join(_HERE, "input_color_oracle.c")])
    p, i = C.c_void_p, C.c_int
    L.ico_yuv_planar_to_rgba.argtypes = [p, p, p, i, i, i, i, i, i, p]
    L.ico_nv12_to_rgba.argtypes = [p, p, i, i, i, i, p]
    L.ico_interleaved422_to_rgba.argtypes = [p, i, i, i, i, i, p]
    for f in (L.ico_yuv_planar_to_rgba, L.ico_nv12_to_rgba, L.ico_interleaved422_to_rgba):
        f.restype = None
    return L


def _u8(a):
    return np.ascontiguousarray(a, dtype=np.uint8)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def yuv_planar_to_rgba(y, u, v, w, h, cw, ch, full_range, matrix):
    """planar 4:2:0 / 4:2:2 / 4:4:4 (chroma planes cw x ch) -> (h, w, 4) RGBA8"""
    y, u, v = _u8(y), _u8(u), _u8(v)
    out = np.empty((h, w, 4), np.uint8)
    _lib().ico_yuv_planar_to_rgba(_p(y), _p(u), _p(v), w, h, cw, ch, int(full_range), int(matrix), _p(out))
    return out


def nv12_to_rgba(y, uv, w, h, full_range, matrix):
    y, uv = _u8(y), _u8(uv)
    out = np.empty((h, w, 4), np.uint8)
    _lib().ico_nv12_to_rgba(_p(y), _p(uv), w, h, int(full_range), int(matrix), _p(out))
    return out


def interleaved422_to_rgba(data, w, h, yuyv, full_range, matrix):
    """UYVY (yuyv False) / YUYV, h rows of (w / 2) texels of 4 bytes"""
    data = _u8(data)
    assert data.size >= (w // 2) * 4 * h
    out = np.empty((h, w, 4), np.uint8)
    _lib().ico_interleaved422_to_rgba(_p(data), w, h, int(bool(yuyv)), int(full_range), int(matrix), _p(out))
    return out
