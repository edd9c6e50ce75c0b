"""smr_transcode_resize on the CPU: its refusals on a host-only handle, the host tables its kernel reads
(smr_debug_transcode_taps) against an independent restatement of gpu-video's transcoder shader, and known answers of the
CPU oracle (tests/transcode_oracle.c)."""
import ctypes as C
import math

import numpy as np
import pytest

from smelter_b200 import _ffi as F
from tests.c_oracles import transcode_resize

f32 = np.float32
ALGOS = (F.SCALE_NEAREST, F.SCALE_BILINEAR, F.SCALE_LANCZOS3)

# (source, renditions) of the GPU tests; every axis pair they need is checked here
LADDERS = [((3840, 2160), [(1920, 1080), (1280, 720), (854, 480), (640, 360)]),
           ((1920, 1080), [(1280, 720), (640, 360), (426, 240), (1920, 1080)]),
           ((640, 360), [(1920, 1080)]),
           ((2, 2), [(16, 16)]),
           ((1918, 1078), [(1000, 562)]),
           ((16384, 2), [(16384, 2), (1000, 2), (2, 16)])]


def axis_pairs():
    pairs = {(2, 16384), (16384, 2)}
    for (sw, sh), outs in LADDERS:
        for ow, oh in outs:
            pairs |= {(sw, ow), (sh, oh), (sw // 2, ow // 2), (sh // 2, oh // 2)}
    return sorted(pairs)


# ---------------------------------------------------------------------------------------------------------------------
# an independent restatement of shader.wgsl's per-axis arithmetic: np.float32 at every step, sin in fp64 (math.sin)
# ---------------------------------------------------------------------------------------------------------------------
PI = f32(math.pi)


def sinc(x):
    x = f32(x)
    if abs(x) < f32(1e-6):
        return f32(1.0)
    px = f32(PI * x)
    return f32(f32(math.sin(float(px))) / px)


def lanczos3_weight(x):
    x = f32(x)
    if abs(x) >= f32(3.0):
        return f32(0.0)
    return f32(sinc(x) * sinc(f32(x / f32(3.0))))


def axis_taps(n_in, n_out):
    k = np.arange(n_out, dtype=f32)
    coords = (k + f32(0.5)) / f32(n_out)
    scaled = f32(n_in) * coords
    nearest = scaled.astype(np.uint32).astype(np.int32)
    fc = scaled - f32(0.5)
    fl = np.floor(fc)
    lo = np.maximum(fl, f32(0)).astype(np.uint32).astype(np.int32)
    hi = np.minimum(lo + 1, n_in - 1).astype(np.int32)
    frac = fc - fl
    w = np.array([[lanczos3_weight(f32(a - f32(b + f32(d)))) for d in range(-2, 4)] for a, b in zip(fc, fl)], f32)
    return nearest, np.stack([lo, hi], 1), frac, fl.astype(np.int32), w


def debug_taps(n_in, n_out):
    nearest, bil, frac = np.empty(n_out, np.int32), np.empty((n_out, 2), np.int32), np.empty(n_out, f32)
    center, w = np.empty(n_out, np.int32), np.empty((n_out, 6), f32)
    st = F.lib().smr_debug_transcode_taps(n_in, n_out, nearest.ctypes.data, bil.ctypes.data, frac.ctypes.data,
                                          center.ctypes.data, w.ctypes.data)
    assert st == F.SMR_OK
    return nearest, bil, frac, center, w


@pytest.mark.parametrize("n_in,n_out", axis_pairs())
def test_debug_taps_match_the_restatement_bit_for_bit(n_in, n_out):
    got, exp = debug_taps(n_in, n_out), axis_taps(n_in, n_out)
    for name, g, e in zip(("nearest", "bilinear", "frac", "center", "lanczos"), got, exp):
        assert g.dtype == e.dtype and np.array_equal(g.view(np.int32), e.view(np.int32)), (name, n_in, n_out)
    nearest, bil, _, _, _ = got
    assert nearest.min() >= 0 and nearest.max() < n_in and bil.min() >= 0 and bil.max() < n_in


def test_debug_taps_refusals():
    buf = np.zeros(16 * 6, np.float32)
    p = buf.ctypes.data
    L = F.lib()
    for n_in, n_out in ((0, 4), (4, 0), (16385, 4), (4, 16385)):
        assert L.smr_debug_transcode_taps(n_in, n_out, p, p, p, p, p) == 1
    assert L.smr_debug_transcode_taps(4, 4, None, p, p, p, p) == 1


# ---------------------------------------------------------------------------------------------------------------------
# refusals, on a host-only handle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def host_handle():
    L = F.lib()
    h = C.c_void_p()
    assert L.smr_create(C.byref(F.Options(-1, 0, 100, 3_000_000_000, 30, 1)), C.byref(h)) == F.SMR_OK
    yield L, h
    L.smr_destroy(h)


def nv12_src(w=64, h=32, fmt=F.FRAME_NV12, mem=F.MEM_HOST, ptr=0x1000, pitch=0):
    f = F.InputFrame()
    f.input_id, f.format, f.width, f.height, f.mem_kind = b"src", fmt, w, h, mem
    for p in range(3):
        f.planes[p] = ptr
        f.pitch[p] = pitch
    return f


def renditions(*specs):
    arr = (F.Rendition * max(1, len(specs)))()
    for i, (w, h, algo) in enumerate(specs):
        arr[i].width, arr[i].height, arr[i].scaling, arr[i].mem_kind = w, h, algo, F.MEM_HOST
        arr[i].planes[0], arr[i].planes[1] = 0x2000, 0x3000
    return arr


def call(handle, src, outs, n=None):
    L, h = handle
    return L.smr_transcode_resize(h, C.byref(src), outs, len(outs) if n is None else n)


def test_valid_call_reaches_the_device_check(host_handle):
    assert call(host_handle, nv12_src(), renditions((32, 16, 2), (16, 8, 1))) == 2      # SMR_ERR_CUDA: no device


@pytest.mark.parametrize("n", [0, 9])
def test_wrong_output_number(host_handle, n):
    outs = renditions(*[(32, 16, 0)] * 9)
    assert call(host_handle, nv12_src(), outs, n) == 1


@pytest.mark.parametrize("w,h", [(0, 16), (16, 0), (15, 16), (16, 15), (16386, 16), (16, 16386), (1, 1)])
def test_rendition_size_refused(host_handle, w, h):
    assert call(host_handle, nv12_src(), renditions((32, 16, 0), (w, h, 1))) == 1


@pytest.mark.parametrize("algo", [-1, 3, 100])
def test_unknown_scaling_refused(host_handle, algo):
    assert call(host_handle, nv12_src(), renditions((32, 16, algo))) == 1


@pytest.mark.parametrize("plane", [0, 1])
def test_null_rendition_plane_refused(host_handle, plane):
    outs = renditions((32, 16, 0))
    outs[0].planes[plane] = None
    assert call(host_handle, nv12_src(), outs) == 1


@pytest.mark.parametrize("plane", [0, 1])
def test_short_rendition_pitch_refused(host_handle, plane):
    outs = renditions((32, 16, 0))
    outs[0].pitch[plane] = 31
    assert call(host_handle, nv12_src(), outs) == 1
    outs[0].pitch[plane] = 32
    assert call(host_handle, nv12_src(), outs) == 2


def test_unknown_mem_kind_refused(host_handle):
    outs = renditions((32, 16, 0))
    outs[0].mem_kind = 2
    assert call(host_handle, nv12_src(), outs) == 1


@pytest.mark.parametrize("w,h", [(63, 32), (64, 31), (0, 32), (1, 1), (16386, 32)])
def test_source_size_refused(host_handle, w, h):
    assert call(host_handle, nv12_src(w, h), renditions((32, 16, 0))) == 1


def test_source_planes_and_pitch_refused(host_handle):
    src = nv12_src()
    src.planes[1] = None
    assert call(host_handle, src, renditions((32, 16, 0))) == 1
    assert call(host_handle, nv12_src(pitch=63), renditions((32, 16, 0))) == 1


@pytest.mark.parametrize("ptr,pitch", [(0x1001, 64), (0x1000, 65)])
def test_device_source_alignment_refused(host_handle, ptr, pitch):
    assert call(host_handle, nv12_src(mem=F.MEM_DEVICE, ptr=ptr, pitch=pitch), renditions((32, 16, 0))) == 1
    assert call(host_handle, nv12_src(mem=F.MEM_DEVICE, ptr=0x1000, pitch=64), renditions((32, 16, 0))) == 2


@pytest.mark.parametrize("fmt", [F.FRAME_PLANAR_YUV420, F.FRAME_PLANAR_YUVJ420, F.FRAME_BGRA, F.FRAME_ARGB, F.FRAME_RGBA8,
                                 F.FRAME_PLANAR_YUV422, F.FRAME_PLANAR_YUV444, F.FRAME_UYVY422, F.FRAME_YUYV422])
def test_other_formats_unsupported(host_handle, fmt):
    assert call(host_handle, nv12_src(fmt=fmt), renditions((32, 16, 0))) == 5


# ---------------------------------------------------------------------------------------------------------------------
# oracle known answers
# ---------------------------------------------------------------------------------------------------------------------
def random_nv12(w, h, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (h, w), np.uint8), rng.integers(0, 256, (h // 2, w // 2, 2), np.uint8)


@pytest.mark.parametrize("algo", ALGOS)
def test_oracle_identity_at_one_to_one(algo):
    y, uv = random_nv12(96, 54, 1)
    oy, ouv = transcode_resize(y, uv, 96, 54, algo)
    assert np.array_equal(oy, y) and np.array_equal(ouv, uv)


def test_oracle_nearest_two_to_one_picks_odd_columns_and_rows():
    y, uv = random_nv12(128, 72, 2)
    oy, ouv = transcode_resize(y, uv, 64, 36, F.SCALE_NEAREST)
    assert np.array_equal(oy, y[1::2, 1::2]) and np.array_equal(ouv, uv[1::2, 1::2])


def test_oracle_nearest_copies_source_bytes():
    y, uv = random_nv12(100, 60, 3)
    oy, ouv = transcode_resize(y, uv, 302, 118, F.SCALE_NEAREST)
    nx, ny = axis_taps(100, 302)[0], axis_taps(60, 118)[0]
    cx, cy = axis_taps(50, 151)[0], axis_taps(30, 59)[0]
    assert np.array_equal(oy, y[np.ix_(ny, nx)]) and np.array_equal(ouv, uv[np.ix_(cy, cx)])


def test_oracle_bilinear_left_edge_at_two_times():
    """At a 2x upscale output column 0 samples fc = -0.25: the shader's weight comes from the unclamped fc, so the column
    is 0.25 p0 + 0.75 p1, not p0 (no clamp-to-edge)."""
    w, h = 16, 8
    y = np.full((h, w), 77, np.uint8)
    y[:, 0], y[:, 1] = 0, 200
    uv = np.full((h // 2, w // 2, 2), 77, np.uint8)
    uv[:, 0], uv[:, 1] = (100, 8), (20, 40)
    oy, ouv = transcode_resize(y, uv, 2 * w, 2 * h, F.SCALE_BILINEAR)
    assert (oy[:, 0] == 150).all()
    assert (ouv[:, 0] == (40, 32)).all()


def f64_resample(plane, out_w, out_h, algo):
    """the same formulas in float64 on one (h, w, c) plane"""
    h, w, _ = plane.shape
    t = plane.astype(np.float64) / 255.0

    def axis(n_in, n_out):
        fcoord = (np.arange(n_out) + 0.5) / n_out
        return fcoord * n_in, fcoord * n_in - 0.5

    (sx, fcx), (sy, fcy) = axis(w, out_w), axis(h, out_h)
    if algo == F.SCALE_NEAREST:
        v = t[np.ix_(sy.astype(int), sx.astype(int))]
    elif algo == F.SCALE_BILINEAR:
        x0 = np.maximum(np.floor(fcx), 0).astype(int)
        y0 = np.maximum(np.floor(fcy), 0).astype(int)
        x1, y1 = np.minimum(x0 + 1, w - 1), np.minimum(y0 + 1, h - 1)
        ax, ay = (fcx - np.floor(fcx))[None, :, None], (fcy - np.floor(fcy))[:, None, None]
        top = t[np.ix_(y0, x0)] * (1 - ax) + t[np.ix_(y0, x1)] * ax
        bot = t[np.ix_(y1, x0)] * (1 - ax) + t[np.ix_(y1, x1)] * ax
        v = top * (1 - ay) + bot * ay
    else:
        def weights(fc, n_in):
            c = np.floor(fc)
            d = np.arange(-2, 4)
            x = fc[:, None] - (c[:, None] + d)
            wt = np.where(np.abs(x) < 3, np.sinc(x) * np.sinc(x / 3), 0.0)
            return np.clip(c[:, None].astype(int) + d, 0, n_in - 1), wt

        ix, wx = weights(fcx, w)
        iy, wy = weights(fcy, h)
        num = np.zeros((out_h, out_w, plane.shape[2]))
        den = np.zeros((out_h, out_w, 1))
        for a in range(6):
            for b in range(6):
                wgt = (wy[:, a][:, None] * wx[:, b][None, :])[..., None]
                num += t[np.ix_(iy[:, a], ix[:, b])] * wgt
                den += wgt
        v = num / den
    return np.rint(np.clip(v, 0, 1) * 255)


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("src,dst", [((96, 54), (40, 24)), ((64, 36), (150, 86)), ((90, 50), (62, 34)), ((2, 2), (16, 16))])
def test_oracle_within_one_of_float64(algo, src, dst):
    y, uv = random_nv12(*src, seed=sum(src) + algo)
    oy, ouv = transcode_resize(y, uv, *dst, algo)
    ey = f64_resample(y[..., None], *dst, algo)[..., 0]
    euv = f64_resample(uv, dst[0] // 2, dst[1] // 2, algo)
    assert np.abs(oy.astype(int) - ey).max() <= 1 and np.abs(ouv.astype(int) - euv).max() <= 1
