"""gpu-video's frame converters on the CPU: every refusal of smr_video_nv12_to_rgba / smr_video_rgba_to_nv12 on a host-only
handle, and the NV12 -> RGBA oracle (tests/video_convert_oracle.c, DESIGN.md NC-11) over the whole joint byte space
against a float64 restatement of nv12_to_rgba.wgsl, with known answers and a check that it is not smelter-render's K2.

The content generators, the exact NC-6u chroma sums and the tie rule are those of tests/test_color_conversion_space.py: a
byte may differ from rint(float64) by exactly 1 only where the float64 value lies within 10^-3 LSB of a rounding tie."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as orc
from smelter_b200 import _ffi as F
from tests.c_oracles import nv12_to_rgba
from tests.test_color_conversion_space import (CHUNK, N, SIDE, coverage, report, tie_rule, upsample2_sum16,
                                               yuv420_block_triples, yuv420_chroma_sums)

f32 = np.float32
BT709_LIMITED = (F.COLOR_SPACE_BT709, F.COLOR_RANGE_LIMITED)
SPACES = (F.COLOR_SPACE_UNSPECIFIED, F.COLOR_SPACE_BT709, F.COLOR_SPACE_BT601_NTSC, F.COLOR_SPACE_BT601_PAL)
RANGES = (F.COLOR_RANGE_FULL, F.COLOR_RANGE_LIMITED)
OTHER_CONVERTERS = [(cs, cr) for cs in SPACES for cr in RANGES if (cs, cr) != BT709_LIMITED]


# ---------------------------------------------------------------------------------------------------------------------
# refusals, on a host-only handle (SMR_ERR_CUDA = 2 means every check passed and a device was needed)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def host_handle():
    L = F.lib()
    h = C.c_void_p()
    assert L.smr_create(C.byref(F.Options(-1, 0, 100, 3_000_000_000, 30, 1)), C.byref(h)) == F.SMR_OK
    yield L, h
    L.smr_destroy(h)


def src_frame(w=64, h=32, fmt=F.FRAME_NV12, mem=F.MEM_HOST, ptr=0x1000, pitch=0):
    f = F.InputFrame()
    f.input_id, f.format, f.width, f.height, f.mem_kind = b"src", fmt, w, h, mem
    for p in range(3):
        f.planes[p] = ptr
        f.pitch[p] = pitch
    return f


def to_rgba(handle, src=None, converter=BT709_LIMITED, frame=(F.COLOR_SPACE_UNSPECIFIED, F.COLOR_RANGE_LIMITED), ow=32,
            oh=16, rgba=0x2000, pitch=0, mem=F.MEM_HOST):
    L, h = handle
    src = src_frame() if src is None else src
    return L.smr_video_nv12_to_rgba(h, F.VideoColor(*converter), C.byref(src), F.VideoColor(*frame), ow, oh, rgba, pitch, mem)


def to_nv12(handle, src=None, converter=BT709_LIMITED, ow=32, oh=16, planes=(0x2000, 0x3000), pitch=(0, 0), mem=F.MEM_HOST):
    L, h = handle
    src = src_frame(fmt=F.FRAME_RGBA8) if src is None else src
    return L.smr_video_rgba_to_nv12(h, F.VideoColor(*converter), C.byref(src), ow, oh, (C.c_void_p * 2)(*planes),
                                    (C.c_uint32 * 2)(*pitch), mem)


@pytest.mark.parametrize("frame", [(F.COLOR_SPACE_UNSPECIFIED, F.COLOR_RANGE_LIMITED), BT709_LIMITED],
                         ids=["unspecified", "bt709"])
def test_valid_calls_reach_the_device_check(host_handle, frame):
    assert to_rgba(host_handle, frame=frame) == 2
    assert to_rgba(host_handle, frame=frame, ow=0, oh=0) == 2          # 0 x 0: the source size
    assert to_rgba(host_handle, frame=frame, ow=1, oh=1) == 2
    assert to_nv12(host_handle) == 2
    assert to_nv12(host_handle, pitch=(32, 40)) == 2
    L, h = host_handle   # a NULL pitch array: both planes tightly packed
    assert L.smr_video_rgba_to_nv12(h, F.VideoColor(*BT709_LIMITED), C.byref(src_frame(fmt=F.FRAME_RGBA8)), 32, 16,
                                    (C.c_void_p * 2)(0x2000, 0x3000), None, F.MEM_HOST) == 2


@pytest.mark.parametrize("converter", OTHER_CONVERTERS, ids=[f"{cs}_{cr}" for cs, cr in OTHER_CONVERTERS])
def test_only_limited_bt709_converters(host_handle, converter):
    assert len(OTHER_CONVERTERS) == 7
    assert to_rgba(host_handle, converter=converter, frame=converter) == 5
    assert to_nv12(host_handle, converter=converter) == 5


@pytest.mark.parametrize("frame", [(F.COLOR_SPACE_UNSPECIFIED, F.COLOR_RANGE_FULL), (F.COLOR_SPACE_BT709, F.COLOR_RANGE_FULL),
                                   (F.COLOR_SPACE_BT601_NTSC, F.COLOR_RANGE_LIMITED), (F.COLOR_SPACE_BT601_PAL, F.COLOR_RANGE_LIMITED),
                                   (F.COLOR_SPACE_BT601_NTSC, F.COLOR_RANGE_FULL), (F.COLOR_SPACE_BT601_PAL, F.COLOR_RANGE_FULL)])
def test_incompatible_frame(host_handle, frame):
    assert to_rgba(host_handle, frame=frame) == 1


@pytest.mark.parametrize("color", [(4, 1), (-1, 1), (1, 2), (1, -1), (100, 0)])
def test_unknown_enum_values(host_handle, color):
    assert to_rgba(host_handle, converter=color, frame=color) == 1
    assert to_rgba(host_handle, frame=color) == 1
    assert to_nv12(host_handle, converter=color) == 1


@pytest.mark.parametrize("w,h", [(63, 32), (64, 31)])
def test_odd_nv12_sides(host_handle, w, h):
    assert to_rgba(host_handle, src=src_frame(w, h)) == 1
    assert to_nv12(host_handle, ow=w, oh=h) == 1


@pytest.mark.parametrize("w,h", [(0, 16), (16, 0), (16385, 16), (16, 16385), (16386, 16)])
def test_target_size_refused(host_handle, w, h):
    assert to_rgba(host_handle, ow=w, oh=h) == 1
    assert to_nv12(host_handle, ow=w, oh=h) == 1
    assert to_nv12(host_handle, ow=0, oh=0) == 1


def test_largest_targets_accepted(host_handle):
    assert to_rgba(host_handle, ow=16384, oh=16384) == 2
    assert to_nv12(host_handle, ow=16384, oh=16384) == 2


def test_null_targets_and_frames(host_handle):
    L, h = host_handle
    assert to_rgba(host_handle, rgba=None) == 1
    assert to_nv12(host_handle, planes=(None, 0x3000)) == 1
    assert to_nv12(host_handle, planes=(0x2000, None)) == 1
    assert L.smr_video_nv12_to_rgba(h, F.VideoColor(*BT709_LIMITED), None, F.VideoColor(0, 1), 32, 16, 0x2000, 0, 0) == 1
    assert L.smr_video_rgba_to_nv12(h, F.VideoColor(*BT709_LIMITED), None, 32, 16, (C.c_void_p * 2)(1, 2), None, 0) == 1
    assert L.smr_video_rgba_to_nv12(h, F.VideoColor(*BT709_LIMITED), C.byref(src_frame(fmt=F.FRAME_RGBA8)), 32, 16, None,
                                    None, 0) == 1


def test_short_pitch_refused(host_handle):
    assert to_rgba(host_handle, ow=32, pitch=127) == 1
    assert to_rgba(host_handle, ow=32, pitch=128) == 2
    assert to_rgba(host_handle, ow=0, oh=0, pitch=255) == 1       # the source size: 64 x 4 bytes
    assert to_rgba(host_handle, ow=0, oh=0, pitch=256) == 2
    for p in range(2):
        pitch = [0, 0]
        pitch[p] = 31
        assert to_nv12(host_handle, ow=32, pitch=tuple(pitch)) == 1


def test_unknown_mem_kind_refused(host_handle):
    assert to_rgba(host_handle, mem=2) == 1
    assert to_nv12(host_handle, mem=2) == 1
    assert to_rgba(host_handle, mem=-1) == 1


@pytest.mark.parametrize("ptr,pitch", [(0x2002, 0), (0x2001, 0), (0x2000, 130), (0x2000, 129)])
def test_unaligned_device_rgba_target_refused(host_handle, ptr, pitch):
    assert to_rgba(host_handle, rgba=ptr, pitch=pitch, mem=F.MEM_DEVICE) == 1
    assert to_rgba(host_handle, rgba=ptr, pitch=pitch, mem=F.MEM_HOST) == 2   # host targets are staged: no rule
    assert to_rgba(host_handle, rgba=0x2000, pitch=132, mem=F.MEM_DEVICE) == 2


def test_nv12_planes_may_start_at_any_byte(host_handle):
    assert to_nv12(host_handle, planes=(0x2001, 0x3003), pitch=(33, 35), mem=F.MEM_DEVICE) == 2


@pytest.mark.parametrize("fmt", [F.FRAME_PLANAR_YUV420, F.FRAME_PLANAR_YUVJ420, F.FRAME_BGRA, F.FRAME_ARGB, F.FRAME_RGBA8,
                                 F.FRAME_PLANAR_YUV422, F.FRAME_PLANAR_YUV444, F.FRAME_UYVY422, F.FRAME_YUYV422])
def test_nv12_to_rgba_takes_only_nv12(host_handle, fmt):
    assert to_rgba(host_handle, src=src_frame(fmt=fmt)) == 5


@pytest.mark.parametrize("fmt", [F.FRAME_PLANAR_YUV420, F.FRAME_PLANAR_YUVJ420, F.FRAME_NV12, F.FRAME_BGRA, F.FRAME_ARGB,
                                 F.FRAME_PLANAR_YUV422, F.FRAME_PLANAR_YUV444, F.FRAME_UYVY422, F.FRAME_YUYV422])
def test_rgba_to_nv12_takes_only_rgba8(host_handle, fmt):
    assert to_nv12(host_handle, src=src_frame(fmt=fmt)) == 5


@pytest.mark.parametrize("w,h", [(0, 32), (1, 1), (16386, 32)])
def test_source_size_refused(host_handle, w, h):
    assert to_rgba(host_handle, src=src_frame(w, h)) == 1
    assert to_nv12(host_handle, src=src_frame(w, h, fmt=F.FRAME_RGBA8)) == 1


def test_source_planes_pitch_and_alignment_refused(host_handle):
    s = src_frame()
    s.planes[1] = None
    assert to_rgba(host_handle, src=s) == 1
    assert to_rgba(host_handle, src=src_frame(pitch=63)) == 1
    assert to_nv12(host_handle, src=src_frame(fmt=F.FRAME_RGBA8, pitch=255)) == 1
    assert to_rgba(host_handle, src=src_frame(mem=F.MEM_DEVICE, ptr=0x1001, pitch=64)) == 1
    assert to_rgba(host_handle, src=src_frame(mem=F.MEM_DEVICE, ptr=0x1000, pitch=65)) == 1
    assert to_rgba(host_handle, src=src_frame(mem=F.MEM_DEVICE, ptr=0x1000, pitch=66)) == 2
    assert to_nv12(host_handle, src=src_frame(fmt=F.FRAME_RGBA8, mem=F.MEM_DEVICE, ptr=0x1002, pitch=256)) == 1
    assert to_nv12(host_handle, src=src_frame(fmt=F.FRAME_RGBA8, mem=F.MEM_DEVICE, ptr=0x1000, pitch=258)) == 1
    assert to_nv12(host_handle, src=src_frame(fmt=F.FRAME_RGBA8, mem=F.MEM_DEVICE, ptr=0x1000, pitch=260)) == 2


# ---------------------------------------------------------------------------------------------------------------------
# restatements of nv12_to_rgba.wgsl fs_main: float64 (exact) and float32 (NC-11, every operation rounded)
# ---------------------------------------------------------------------------------------------------------------------
def gpu_video_rgb64(y, cb, cr):
    """fs_main at sampled values y, cb, cr in [0, 1] -> exact (r, g, b) in byte units (clamped, times 255): no clamp before
    the matrix, scale 255/219 and 255/224, `s * M` with M's columns (1, 0, 1.5748), (1, -0.1873, -0.4681), (1, 1.8556, 0)"""
    s0 = (np.asarray(y, np.float64) - 16.0 / 255.0) * (255.0 / 219.0)
    s1 = (np.asarray(cb, np.float64) - 0.5) * (255.0 / 224.0)
    s2 = (np.asarray(cr, np.float64) - 0.5) * (255.0 / 224.0)
    rgb = (s0 + 1.5748 * s2, s0 - 0.1873 * s1 - 0.4681 * s2, s0 + 1.8556 * s1)
    return tuple(np.clip(c, 0.0, 1.0) * 255.0 for c in rgb)


def nc11_f32(y, cb, cr):
    """NC-11 steps 3-5 in numpy float32 (each operation rounds once) -> uint8 (r, g, b)"""
    y, cb, cr = (np.asarray(a, f32) for a in (y, cb, cr))
    s = [(y - f32(16 / 255)) * f32(255 / 219), (cb - f32(0.5)) * f32(255 / 224), (cr - f32(0.5)) * f32(255 / 224)]
    cols = ((1.0, 0.0, 1.5748), (1.0, -0.1873, -0.4681), (1.0, 1.8556, 0.0))
    out = []
    for m in cols:
        v = (s[0] * f32(m[0]) + s[1] * f32(m[1])) + s[2] * f32(m[2])
        out.append(np.rint(np.clip(v, f32(0), f32(1)) * f32(255)).astype(np.uint8))
    return tuple(out)


def sampled_chroma(sum16):
    """NC-6u value of an interpolated chroma sample, 16 x byte value sum16: f32(sum16 / (16 * 255))"""
    return (np.asarray(sum16, np.float64) / (16.0 * 255.0)).astype(f32)


def nv12_of(planes):
    y, u, v = planes
    return y, np.ascontiguousarray(np.stack([u, v], axis=-1))


def check_frame_against_float64(planes):
    """oracle at the source size on one 4096 x 4096 frame vs rint(float64) under the tie rule -> bytes off rint per channel"""
    y, uv = nv12_of(planes)
    got = nv12_to_rgba(y, uv)
    assert (got[..., 3] == 255).all()
    n = {}
    for r0 in range(0, SIDE, CHUNK):
        rows = np.arange(r0, r0 + CHUNK)
        su, sv = upsample2_sum16(planes[1], rows), upsample2_sum16(planes[2], rows)
        ex = gpu_video_rgb64(y[rows] / 255.0, su / (16.0 * 255.0), sv / (16.0 * 255.0))
        for c, e in enumerate(ex):
            n["rgb"[c]] = n.get("rgb"[c], 0) + tie_rule(got[rows, :, c], e, f"NC-11 {'rgb'[c]}")
    return n


def test_oracle_every_exact_chroma_triple():
    """every (Y, Cb, Cr) with an uninterpolated chroma sample: the four block frames of the colour-space test"""
    seen = np.zeros(N, bool)
    n = {}
    for part in range(4):
        planes, cov = yuv420_block_triples(part)
        seen |= cov
        for k, v in check_frame_against_float64(planes).items():
            n[k] = n.get(k, 0) + v
    assert coverage(seen) == N
    report("NV12 -> RGBA (gpu-video) block frames, bytes off rint(float64)", n)


def test_oracle_every_interpolated_chroma_with_every_luma():
    """every same-size interpolated chroma value n / 16 (n = 0 .. 4080) with every Y, on both channels"""
    planes, cov = yuv420_chroma_sums()
    assert cov["u"] == cov["v"] == cov["uv"] == 256 * 4081, cov
    report("NV12 -> RGBA (gpu-video) chroma sums, bytes off rint(float64)", check_frame_against_float64(planes))


# ---------------------------------------------------------------------------------------------------------------------
# known answers
# ---------------------------------------------------------------------------------------------------------------------
def random_nv12(w, h, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (h, w), np.uint8), rng.integers(0, 256, (h // 2, w // 2, 2), np.uint8)


@pytest.mark.parametrize("w,h", [(2, 2), (6, 4), (96, 54), (130, 18)])
def test_source_size_is_luma_texel_and_quarter_chroma_taps(w, h):
    """at W_t = W, H_t = H luma is texel (x, y) and chroma the .25 / .75 pair: the oracle equals NC-11's f32 steps applied
    to f32(Y / 255) and the exact interpolant, bit for bit"""
    y, uv = random_nv12(w, h, w * h)
    got = nv12_to_rgba(y, uv)
    rows = np.arange(h)
    su, sv = upsample2_sum16(uv[..., 0], rows), upsample2_sum16(uv[..., 1], rows)
    want = nc11_f32((y / np.float64(255)).astype(f32), sampled_chroma(su), sampled_chroma(sv))
    for c in range(3):
        assert np.array_equal(got[..., c], want[c]), c
    assert (got[..., 3] == 255).all()


@pytest.mark.parametrize("w,h", [(2, 2), (4, 4), (8, 6), (1920, 1080), (6, 10)])
def test_one_by_one_target_samples_the_centre(w, h):
    """a 1 x 1 target samples (.5, .5): luma halfway between the two middle texels of each axis, chroma likewise when the
    chroma side is even and the middle texel itself when it is odd"""
    y, uv = random_nv12(w, h, 5 + w)
    got = nv12_to_rgba(y, uv, 1, 1)

    def centre(p):
        n_y, n_x = p.shape
        ys = [n_y // 2 - 1, n_y // 2] if n_y % 2 == 0 else [n_y // 2] * 2
        xs = [n_x // 2 - 1, n_x // 2] if n_x % 2 == 0 else [n_x // 2] * 2
        n = sum(int(p[a, b]) * 128 * 128 for a in ys for b in xs)
        return f32(n / (255.0 * 65536.0))

    want = nc11_f32(centre(y), centre(uv[..., 0]), centre(uv[..., 1]))
    assert tuple(int(got[0, 0, c]) for c in range(3)) == tuple(int(v) for v in want)
    assert got[0, 0, 3] == 255


def test_constant_frames_any_size():
    """a constant frame converts to one colour at every size, up or down; alpha is 255"""
    for yv, cb, cr in ((16, 128, 128), (235, 128, 128), (0, 0, 255), (255, 255, 0), (81, 90, 240)):
        y = np.full((36, 64), yv, np.uint8)
        uv = np.empty((18, 32, 2), np.uint8)
        uv[..., 0], uv[..., 1] = cb, cr
        want = nc11_f32(f32(yv / 255.0), f32(cb / 255.0), f32(cr / 255.0))
        for ow, oh in ((64, 36), (1, 1), (7, 3), (200, 90)):
            got = nv12_to_rgba(y, uv, ow, oh)
            assert (got[..., 3] == 255).all()
            for c in range(3):
                assert (got[..., c] == want[c]).all(), (yv, cb, cr, ow, oh, c)
    # the chroma offset is 0.5, not 128 / 255, so limited-range black with neutral chroma byte 128 keeps a trace of
    # colour: r = b = rint(255 * 1.5748 * (128 / 255 - 0.5) * 255 / 224) = 1
    y = np.full((2, 2), 16, np.uint8)
    assert tuple(nv12_to_rgba(y, np.full((1, 1, 2), 128, np.uint8))[0, 0]) == (1, 0, 1, 255)
    y[:] = 235
    assert tuple(nv12_to_rgba(y, np.full((1, 1, 2), 128, np.uint8))[0, 0]) == (255, 255, 255, 255)


def test_scaled_oracle_within_one_of_float64():
    """at other sizes the samples are NC-6u's four taps; the oracle stays within 1 of a float64 evaluation of the same taps"""
    y, uv = random_nv12(96, 54, 3)
    for ow, oh in ((40, 24), (150, 86), (1, 1), (97, 55)):
        got = nv12_to_rgba(y, uv, ow, oh)

        def taps(n_out, n_in):
            c = ((np.arange(n_out) + 0.5) / n_out) * n_in - 0.5
            fl = np.floor(c)
            w1 = np.rint((c - fl) * 256) / 256
            return np.clip(fl, 0, n_in - 1).astype(int), np.clip(fl + 1, 0, n_in - 1).astype(int), w1

        def sample(p):
            x0, x1, wx = taps(ow, p.shape[1])
            y0, y1, wy = taps(oh, p.shape[0])
            p = p.astype(np.float64) / 255.0
            top = p[np.ix_(y0, x0)] * (1 - wx) + p[np.ix_(y0, x1)] * wx
            bot = p[np.ix_(y1, x0)] * (1 - wx) + p[np.ix_(y1, x1)] * wx
            return top * (1 - wy)[:, None] + bot * wy[:, None]

        ex = gpu_video_rgb64(sample(y), sample(uv[..., 0]), sample(uv[..., 1]))
        for c in range(3):
            assert np.abs(got[..., c].astype(int) - np.rint(ex[c])).max() <= 1, (ow, oh, c)


# ---------------------------------------------------------------------------------------------------------------------
# not smelter-render's K2
# ---------------------------------------------------------------------------------------------------------------------
def test_differs_from_smelter_render_k2():
    """gpu-video's shader does not clamp Y, Cb, Cr before the matrix and scales by 255/219, 255/224 instead of dividing by
    0.8588.. / 0.8784..: on the exact-chroma block frames it gives other bytes than orc_nv12_to_rgba (K2) for a set of
    triples that includes out-of-range and in-range values"""
    differ = np.zeros(N, bool)
    in_range = 0
    for part in range(4):
        planes, _ = yuv420_block_triples(part)
        y, uv = nv12_of(planes)
        a, b = nv12_to_rgba(y, uv), orc.nv12_to_rgba(y, uv, SIDE, SIDE)
        inner = np.zeros((SIDE, SIDE), bool)   # the block frames' inner pixels see their block's chroma exactly
        for r in (1, 2):
            for c in (1, 2):
                inner[r::4, c::4] = True
        d = np.any(a[..., :3] != b[..., :3], axis=-1) & inner
        u = np.repeat(np.repeat(planes[1], 2, 0), 2, 1)
        v = np.repeat(np.repeat(planes[2], 2, 0), 2, 1)
        yy, uu, vv = y[d].astype(np.int64), u[d].astype(np.int64), v[d].astype(np.int64)
        differ[yy | (uu << 8) | (vv << 16)] = True
        in_range += int(np.count_nonzero((yy >= 16) & (yy <= 235) & (uu >= 16) & (uu <= 240) & (vv >= 16) & (vv <= 240)))
        if part == 0:
            first = [(int(p), int(q), int(s), tuple(int(t) for t in a[d][i, :3]), tuple(int(t) for t in b[d][i, :3]))
                     for i, (p, q, s) in enumerate(zip(yy[:5], uu[:5], vv[:5]))]
    n = coverage(differ)
    print(f"\ngpu-video NV12->RGBA differs from K2 on {n} (Y, Cb, Cr) triples ({in_range} in-range pixels); "
          f"first (Y, Cb, Cr, gpu-video, K2): {first}")
    assert n > 0 and in_range > 0
