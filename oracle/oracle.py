"""ctypes loader for the CPU oracle (TEST INFRASTRUCTURE ONLY -- never imported by smelter_b200/).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may
import this module.  See oracle/smelter_oracle.h for what the oracle is pinned by.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")

MODE_GPU_OPTIMIZED = 0
MODE_CPU_OPTIMIZED = 1
LAYOUT_TEXTURE, LAYOUT_COLOR, LAYOUT_BOX_SHADOW = 0, 1, 2
MAX_MASKS = 20


class Mask(C.Structure):
    _fields_ = [("radius", C.c_float * 4), ("top", C.c_float), ("left", C.c_float),
                ("width", C.c_float), ("height", C.c_float)]


class Layout(C.Structure):
    _fields_ = [
        ("type", C.c_int32),
        ("top", C.c_float), ("left", C.c_float), ("width", C.c_float), ("height", C.c_float),
        ("rotation_degrees", C.c_float),
        ("border_radius", C.c_float * 4),
        ("color", C.c_uint8 * 4), ("border_color", C.c_uint8 * 4),
        ("border_width", C.c_float), ("blur_radius", C.c_float),
        ("child_index", C.c_int32),
        ("crop_top", C.c_float), ("crop_left", C.c_float),
        ("crop_width", C.c_float), ("crop_height", C.c_float),
        ("masks_len", C.c_int32),
        ("masks", Mask * MAX_MASKS),
    ]


class Texture(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("data", C.c_void_p)]


def build(force=False):
    if force or not os.path.exists(_LIB_PATH) or (
            os.path.getmtime(_LIB_PATH) < os.path.getmtime(os.path.join(_HERE, "smelter_oracle.c"))):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_srgb_decode_u8.restype = C.c_float
        _lib.orc_render_text.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_uint8), C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                         C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
        _lib.orc_render_text.restype = None
        _lib.orc_srgb_decode_u8.argtypes = [C.c_uint8]
        _lib.orc_srgb_encode_u8.restype = C.c_uint8
        _lib.orc_srgb_encode_u8.argtypes = [C.c_float]
        _lib.orc_unorm8.restype = C.c_uint8
        _lib.orc_unorm8.argtypes = [C.c_float]
        _lib.orc_f32_to_f16.restype = C.c_uint16
        _lib.orc_f32_to_f16.argtypes = [C.c_float]
        _lib.orc_f16_to_f32.restype = C.c_float
        _lib.orc_f16_to_f32.argtypes = [C.c_uint16]
        _lib.orc_predecimate_levels.argtypes = [C.c_float, C.c_int]
        _lib.orc_plan_passes.argtypes = [C.c_float] * 4 + [C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        _lib.orc_resample_taps.argtypes = [C.c_float]
        _lib.orc_resample_weights.argtypes = [C.c_float, C.c_float, C.c_int, C.c_void_p, C.c_void_p]
        _lib.orc_resample.argtypes = [C.POINTER(Texture)] + [C.c_float] * 4 + [C.c_int, C.c_int, C.c_void_p]
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _u8(a):
    a = np.ascontiguousarray(a, dtype=np.uint8)
    return a


def yuv420_to_rgba(y, u, v, w, h, full_range=False):
    y, u, v = _u8(y), _u8(u), _u8(v)
    out = np.empty((h, w, 4), np.uint8)
    lib().orc_yuv420_to_rgba(_p(y), _p(u), _p(v), w, h, int(full_range), _p(out))
    return out


def yuv_planar_to_rgba(y, u, v, w, h, cw, ch, full_range=False):
    """planar 4:2:0 / 4:2:2 / 4:4:4 by chroma plane size (texture/planar_yuv.rs:64-83)"""
    y, u, v = _u8(y), _u8(u), _u8(v)
    out = np.empty((h, w, 4), np.uint8)
    lib().orc_yuv_planar_to_rgba(_p(y), _p(u), _p(v), w, h, cw, ch, int(full_range), _p(out))
    return out


def interleaved422_to_rgba(data, w, h, yuyv):
    """K3: UYVY (yuyv=False) / YUYV (yuyv=True), h rows of 2*(w//2)*2 bytes"""
    data = _u8(data)
    assert data.size >= (w // 2) * 4 * h
    out = np.empty((h, w, 4), np.uint8)
    lib().orc_interleaved422_to_rgba(_p(data), w, h, int(bool(yuyv)), _p(out))
    return out


def nv12_to_rgba(y, uv, w, h):
    y, uv = _u8(y), _u8(uv)
    out = np.empty((h, w, 4), np.uint8)
    lib().orc_nv12_to_rgba(_p(y), _p(uv), w, h, _p(out))
    return out


def bgra_to_rgba(d, w, h):
    d = _u8(d)
    out = np.empty((h, w, 4), np.uint8)
    lib().orc_bgra_to_rgba(_p(d), w, h, _p(out))
    return out


def argb_to_rgba(d, w, h):
    d = _u8(d)
    out = np.empty((h, w, 4), np.uint8)
    lib().orc_argb_to_rgba(_p(d), w, h, _p(out))
    return out


def rgba_to_yuv420(rgba):
    rgba = _u8(rgba)
    h, w = rgba.shape[:2]
    y = np.empty((h, w), np.uint8)
    u = np.empty((h // 2, w // 2), np.uint8)
    v = np.empty((h // 2, w // 2), np.uint8)
    lib().orc_rgba_to_yuv420(_p(rgba), w, h, _p(y), _p(u), _p(v))
    return y, u, v


def rgba_to_nv12(rgba):
    rgba = _u8(rgba)
    h, w = rgba.shape[:2]
    y = np.empty((h, w), np.uint8)
    uv = np.empty((h // 2, w // 2, 2), np.uint8)
    lib().orc_rgba_to_nv12(_p(rgba), w, h, _p(y), _p(uv))
    return y, uv


def rgba_to_yuv420_scaled(rgba, w, h):
    rgba = _u8(rgba)
    sh, sw = rgba.shape[:2]
    y = np.empty((h, w), np.uint8)
    u = np.empty((h // 2, w // 2), np.uint8)
    v = np.empty((h // 2, w // 2), np.uint8)
    lib().orc_rgba_to_yuv420_scaled(_p(rgba), sw, sh, w, h, _p(y), _p(u), _p(v))
    return y, u, v


def rgba_to_yuv_planar_scaled(rgba, w, h, cw, ch):
    rgba = _u8(rgba)
    sh, sw = rgba.shape[:2]
    y = np.empty((h, w), np.uint8)
    u = np.empty((ch, cw), np.uint8)
    v = np.empty((ch, cw), np.uint8)
    lib().orc_rgba_to_yuv_planar_scaled(_p(rgba), sw, sh, w, h, cw, ch, _p(y), _p(u), _p(v))
    return y, u, v


def add_premultiplied_alpha(rgba, mode=0):
    """PremultiplyAlphaPipeline: straight-alpha RGBA8 -> premultiplied RGBA8 (add_premultiplied_alpha.wgsl)"""
    rgba = _u8(rgba)
    h, w = rgba.shape[:2]
    out = np.empty((h, w, 4), np.uint8)
    lib().orc_add_premultiplied_alpha(_p(rgba), w, h, int(mode), _p(out))
    return out


GLYPH_DTYPE = [("x", "<i4"), ("y", "<i4"), ("width", "<u2"), ("height", "<u2"), ("atlas_x", "<u2"), ("atlas_y", "<u2"),
               ("color", "u1", (4,)), ("content", "<i4")]   # orc_glyph


def render_text(width, height, background, glyphs, mask_atlas=None, color_atlas=None, color_mode=0, mode=0):
    """TextRendererNode::render: clear + glyph quads (orc_render_text).  background: 4 bytes; glyphs: GLYPH_DTYPE records."""
    if width == 0 or height == 0:
        return np.zeros((1, 1, 4), np.uint8)
    g = np.ascontiguousarray(glyphs, dtype=np.dtype(GLYPH_DTYPE))
    bg = (C.c_uint8 * 4)(*[int(v) for v in background])
    m = _u8(mask_atlas) if mask_atlas is not None else None
    c = _u8(color_atlas) if color_atlas is not None else None
    out = np.empty((height, width, 4), np.uint8)
    lib().orc_render_text(int(width), int(height), bg, g.ctypes.data_as(C.c_void_p) if len(g) else None, len(g),
                          _p(m) if m is not None else None, m.shape[1] if m is not None else 0, m.shape[0] if m is not None else 0,
                          _p(c) if c is not None else None, c.shape[1] if c is not None else 0, c.shape[0] if c is not None else 0,
                          int(color_mode), int(mode), _p(out))
    return out


def rescale_rgba(rgba, ow, oh, mode=0):
    """FramePreProcessor rescale: bilinear (NC-6) sample of the node texture, stored through the target format"""
    rgba = _u8(rgba)
    sh, sw = rgba.shape[:2]
    out = np.empty((oh, ow, 4), np.uint8)
    lib().orc_rescale_rgba(_p(rgba), sw, sh, ow, oh, int(mode), _p(out))
    return out


def rgba_to_nv12_scaled(rgba, w, h):
    rgba = _u8(rgba)
    sh, sw = rgba.shape[:2]
    y = np.empty((h, w), np.uint8)
    uv = np.empty((h // 2, w // 2, 2), np.uint8)
    lib().orc_rgba_to_nv12_scaled(_p(rgba), sw, sh, w, h, _p(y), _p(uv))
    return y, uv


def rgb_to_yuv_bytes(r, g, b):
    out = (C.c_uint8 * 3)()
    lib().orc_rgb_to_yuv_bytes(r, g, b, out)
    return tuple(out)


def harness_yuv420_to_rgba(y, u, v, w, h):
    """integration-tests/src/render_tests/harness/utils.rs:31-65"""
    y, u, v = _u8(y), _u8(u), _u8(v)
    cw, ch = w - (w % 2), h - (h % 2)
    out = np.empty((ch, cw, 4), np.uint8)
    lib().orc_harness_yuv420_to_rgba(_p(y), _p(u), _p(v), w, h, _p(out))
    return out


def plan_passes(crop_left, crop_top, crop_w, crop_h, dst_w, dst_h):
    """-> list of (axis, perp_offset); [] when direct."""
    ax = (C.c_int * 2)()
    pp = (C.c_int * 2)()
    n = lib().orc_plan_passes(crop_left, crop_top, crop_w, crop_h, dst_w, dst_h, ax, pp)
    return [(ax[i], pp[i]) for i in range(n)]


def predecimate_levels(crop_len, dst_len):
    return lib().orc_predecimate_levels(crop_len, dst_len)


def resample_weights(scale, offset, out_coord):
    taps = lib().orc_resample_taps(scale)
    w = np.zeros(taps, np.float32)
    ws = C.c_float()
    first = lib().orc_resample_weights(scale, offset, out_coord, _p(w), C.byref(ws))
    return first, w, ws.value


def resample(src_rgba, crop_left, crop_top, crop_w, crop_h, dst_w, dst_h):
    src = _u8(src_rgba)
    t = Texture(src.shape[1], src.shape[0], src.ctypes.data)
    out = np.zeros((dst_h, dst_w, 4), np.uint8)
    n = lib().orc_resample(C.byref(t), crop_left, crop_top, crop_w, crop_h, dst_w, dst_h, _p(out))
    return out if n else None


def make_layout(type, top, left, width, height, rotation_degrees=0.0, border_radius=(0, 0, 0, 0),
                color=(0, 0, 0, 0), border_color=(0, 0, 0, 0), border_width=0.0, blur_radius=0.0,
                child_index=0, crop=(0, 0, 0, 0), masks=()):
    """crop = (top, left, width, height); masks = [(radius4, top, left, width, height), ...]"""
    L = Layout()
    L.type = type
    L.top, L.left, L.width, L.height = top, left, width, height
    L.rotation_degrees = rotation_degrees
    L.border_radius = (C.c_float * 4)(*border_radius)
    L.color = (C.c_uint8 * 4)(*color)
    L.border_color = (C.c_uint8 * 4)(*border_color)
    L.border_width, L.blur_radius = border_width, blur_radius
    L.child_index = child_index
    L.crop_top, L.crop_left, L.crop_width, L.crop_height = crop
    L.masks_len = len(masks)
    for i, m in enumerate(masks[:MAX_MASKS]):
        L.masks[i].radius = (C.c_float * 4)(*m[0])
        L.masks[i].top, L.masks[i].left, L.masks[i].width, L.masks[i].height = m[1:5]
    return L


def _textures(arrs):
    keep = [None if a is None else _u8(a) for a in arrs]
    tex = (Texture * max(1, len(keep)))()
    for i, a in enumerate(keep):
        if a is None:
            tex[i] = Texture(0, 0, None)
        else:
            tex[i] = Texture(a.shape[1], a.shape[0], a.ctypes.data)
    return tex, keep


def apply_layouts(out_w, out_h, layouts, textures, mode=MODE_GPU_OPTIMIZED, max_layouts=100):
    arr = (Layout * max(1, len(layouts)))(*layouts)
    tex, keep = _textures(textures)
    out = np.empty((out_h, out_w, 4), np.uint8)
    lib().orc_apply_layouts(out_w, out_h, arr, tex, len(layouts), max_layouts, mode, _p(out))
    return out


def bare_map(out_w, out_h, layout, mode=MODE_GPU_OPTIMIZED):
    """(out_h, out_w) bool: where `layout` covers the pixel and its fragment is the bare colour or sample (every alpha
    factor exactly 1, no border colour mixed in)."""
    out = np.empty((out_h, out_w), np.uint8)
    lib().orc_bare_map(out_w, out_h, C.byref(layout), mode, _p(out))
    return out.astype(bool)


def render_layout_node(out_w, out_h, layouts, nodes, mode=MODE_GPU_OPTIMIZED, max_layouts=100):
    """LayoutNode::render: nodes[i] = premultiplied RGBA8 node texture (h, w, 4) or None."""
    arr = (Layout * max(1, len(layouts)))(*layouts)
    tex, keep = _textures(nodes)
    out = np.empty((out_h, out_w, 4), np.uint8)
    lib().orc_render_layout_node(out_w, out_h, arr, len(layouts), tex, len(nodes), max_layouts, mode, _p(out))
    return out


def num_threads():
    return lib().orc_num_threads()


def set_num_threads(n):
    lib().orc_set_num_threads(int(n))
