"""smr_set_input_color on the CPU: the status rules on a host-only handle, a float64 restatement of DESIGN.md NC-13, known
answers on SMPTE colour bars, and the colour oracle (`tests/input_color_oracle.c`) over the whole joint (Y, U, V) byte
space.  At BT.709 and a format's own range that oracle writes the committed oracle's bytes.

NC-13 is K1/K2/K3 (`k1_rgb` in `tests/test_color_conversion_space.py`) with the chroma coefficients of BT.601
(Kr = 0.299, Kb = 0.114) rounded to four decimals, and a range that is set per input instead of per format.  The content
generators, the tie rule and TIE_DELTA are those of that file: every byte the colour oracle writes equals rint of the
float64 value, or differs by exactly 1 where that value lies within TIE_DELTA of a rounding tie.
"""
import ctypes as C

import numpy as np
import pytest

import smelter_b200 as s
from smelter_b200 import _ffi as F
from oracle import oracle as orc
from tests import input_color_oracle as ico
from tests.test_color_conversion_space import (CHUNK, N, SIDE, TIE_DELTA, all_triples, coverage, interleaved_all_triples,
                                               interleaved_planes, k1_rgb, report, tie_distance, tie_rule,
                                               upsample2_sum16, yuv420_block_triples, yuv420_chroma_sums,
                                               yuv444_all_triples)

BT709, BT601 = 0, 1          # the colour oracle's matrix argument (Tex::matrix)
MATRICES = {"bt709": BT709, "bt601": BT601}
# the chroma coefficients (rv, gu, gv, bu) of r = y + rv (v - .5), g = y + gu (u - .5) + gv (v - .5), b = y + bu (u - .5)
COEF = {BT709: (1.5748, -0.1873, -0.4681, 1.8556),                       # K1-K3, as the reference's shaders write them
        BT601: (1.402, -0.3441, -0.7141, 1.772)}                         # NC-13


# ------------------------------------------------------------------------------------------------
# float64 restatement of NC-13
# ------------------------------------------------------------------------------------------------
def nc13_rgb(y, u, v, full_range, matrix):
    """sampled y, u, v in [0, 1] -> exact r, g, b in byte units (clamped, times 255): limited range expands by 219 / 255 and
    224 / 255 and clamps, full range does not; then the matrix's rows"""
    y, u, v = (np.asarray(a, np.float64) for a in (y, u, v))
    if not full_range:
        y = np.clip((y - (16.0 / 255.0)) / 0.85882352941, 0.0, 1.0)
        u = np.clip((u - (16.0 / 255.0)) / 0.87843137254, 0.0, 1.0)
        v = np.clip((v - (16.0 / 255.0)) / 0.87843137254, 0.0, 1.0)
    rv, gu, gv, bu = COEF[matrix]
    r = y + rv * (v - 0.5)
    g = y + gu * (u - 0.5) + gv * (v - 0.5)
    b = y + bu * (u - 0.5)
    return tuple(np.clip(c, 0.0, 1.0) * 255.0 for c in (r, g, b))


def test_coefficients_come_from_kr_and_kb():
    """NC-13's constants are 2 (1 - Kr), -2 Kb (1 - Kb) / Kg, -2 Kr (1 - Kr) / Kg and 2 (1 - Kb) at four decimals, and the
    BT.709 ones the same expressions at Kr = 0.2126, Kb = 0.0722"""
    for m, (kr, kb) in ((BT601, (0.299, 0.114)), (BT709, (0.2126, 0.0722))):
        kg = 1.0 - kr - kb
        want = (2 * (1 - kr), -2 * kb * (1 - kb) / kg, -2 * kr * (1 - kr) / kg, 2 * (1 - kb))
        assert np.allclose(COEF[m], want, atol=5e-5), (m, want)


@pytest.mark.parametrize("full_range", [0, 1], ids=["limited", "full"])
def test_bt709_rows_are_k1(full_range):
    """the restatement at BT.709 is the existing K1-K3 restatement, value for value, over every (Y, U, V)"""
    Y, U, V = (c / 255.0 for c in all_triples())
    for a, b in zip(nc13_rgb(Y, U, V, full_range, BT709), k1_rgb(Y, U, V, full_range)):
        assert np.array_equal(a, b)


# SMPTE colour bars, BT.601 8-bit limited range (Y, Cb, Cr): white, yellow, cyan, green, magenta, red, blue, black
BARS_75 = [(180, 128, 128), (162, 44, 142), (131, 156, 44), (112, 72, 58), (84, 184, 198), (65, 100, 212), (35, 212, 114),
           (16, 128, 128)]
BARS_100 = [(235, 128, 128), (210, 16, 146), (170, 166, 16), (145, 54, 34), (106, 202, 222), (81, 90, 240), (41, 240, 110),
            (16, 128, 128)]
BAR_RGB = [(1, 1, 1), (1, 1, 0), (0, 1, 1), (0, 1, 0), (1, 0, 1), (1, 0, 0), (0, 0, 1), (0, 0, 0)]
# the bytes NC-13 gives them (the bars' 8-bit values are themselves rounded, so a channel may sit 1 off the nominal level)
BARS_75_RGB = [(191, 191, 191), (192, 192, 1), (0, 191, 190), (0, 191, 0), (191, 0, 192), (191, 0, 1), (0, 1, 192), (0, 0, 0)]
BARS_100_RGB = [(255, 255, 255), (255, 255, 0), (1, 255, 255), (0, 255, 1), (255, 0, 254), (254, 0, 0), (0, 0, 255), (0, 0, 0)]


def bar_frame(bars):
    """a 4:4:4 frame of one pixel per bar, 8 x 2"""
    t = np.array(bars, np.uint8)
    return [np.ascontiguousarray(np.tile(t[:, c], (2, 1))) for c in range(3)]


@pytest.mark.parametrize("level,bars,want", [(191, BARS_75, BARS_75_RGB), (255, BARS_100, BARS_100_RGB)], ids=["75", "100"])
def test_colour_bars(level, bars, want):
    """BT.601 limited-range bars come out at their nominal RGB within 1, through the restatement and the oracle alike; read
    as BT.709 (the rule without the setting), the green bar loses more than a tenth of its level"""
    y, u, v = bar_frame(bars)
    got = ico.yuv_planar_to_rgba(y, u, v, 8, 2, 8, 2, False, BT601)
    ex = np.stack(nc13_rgb(y / 255.0, u / 255.0, v / 255.0, False, BT601), axis=-1)
    assert np.array_equal(got[0, :, :3], np.array(want, np.uint8)), got[0, :, :3]
    assert np.array_equal(np.rint(ex[0]).astype(np.uint8), np.array(want, np.uint8))
    assert np.abs(got[0, :, :3].astype(int) - level * np.array(BAR_RGB)).max() <= 1
    old = orc.yuv_planar_to_rgba(y, u, v, 8, 2, 8, 2)
    assert level - int(old[0, 3, 1]) > level // 10, old[0, 3]


def test_issue_examples():
    """the two bars quoted when the setting was asked for: BT.601 100 % green and red"""
    for (yy, uu, vv), want, old in (((145, 54, 34), (0, 255, 1), (0, 216, 0)), ((81, 90, 240), (254, 0, 0), (255, 24, 0))):
        y, u, v = (np.full((2, 2), c, np.uint8) for c in (yy, uu, vv))
        assert tuple(ico.yuv_planar_to_rgba(y, u, v, 2, 2, 2, 2, False, BT601)[0, 0, :3]) == want
        assert tuple(orc.yuv_planar_to_rgba(y, u, v, 2, 2, 2, 2)[0, 0, :3]) == old


# ------------------------------------------------------------------------------------------------
# the colour oracle over the joint byte space
# ------------------------------------------------------------------------------------------------
_NEAR = {}


def near_ties(full_range, matrix):
    """the (Y, U, V) triples whose float64 NC-13 r, g or b lies within TIE_DELTA of a tie"""
    key = (full_range, matrix)
    if key not in _NEAR:
        Y, U, V = all_triples()
        near = np.zeros(N, bool)
        for c in nc13_rgb(Y / 255.0, U / 255.0, V / 255.0, full_range, matrix):
            near |= tie_distance(c) < TIE_DELTA
        _NEAR[key] = near
    return _NEAR[key]


def test_bt601_has_near_ties():
    """the tie rule is exercised at BT.601 too: both ranges have triples within TIE_DELTA of a tie"""
    sizes = {f"{'full' if fr else 'limited'}": coverage(near_ties(fr, BT601)) for fr in (0, 1)}
    report("NC-13 BT.601 near-tie set sizes", sizes)
    assert all(v > 1000 for v in sizes.values()), sizes


def legacy_entry(kind, full_range):
    """the existing converter that computes the same bytes, where one exists (BT.709 at the format's own range)"""
    if kind == "planar":
        return lambda y, u, v, w, h, cw, ch: orc.yuv_planar_to_rgba(y, u, v, w, h, cw, ch, full_range=bool(full_range))
    if kind == "nv12" and not full_range:
        return lambda y, uv, w, h: orc.nv12_to_rgba(y, uv, w, h)
    if kind in ("uyvy", "yuyv") and not full_range:
        return lambda t, w, h: orc.interleaved422_to_rgba(t, w, h, kind == "yuyv")
    return None


@pytest.mark.parametrize("matrix", list(MATRICES), ids=list(MATRICES))
@pytest.mark.parametrize("full_range", [0, 1], ids=["limited", "full"])
def test_planar_444_every_triple(full_range, matrix):
    """the colour oracle's planar converter at 4:4:4 on every (Y, U, V); at BT.709 its bytes are orc_yuv_planar_to_rgba's"""
    m = MATRICES[matrix]
    (y, u, v), n = yuv444_all_triples()
    assert n == N
    got = ico.yuv_planar_to_rgba(y, u, v, SIDE, SIDE, SIDE, SIDE, full_range, m)
    counts = {}
    for r0 in range(0, SIDE, CHUNK):
        sl = slice(r0, r0 + CHUNK)
        for c, e in enumerate(nc13_rgb(y[sl] / 255.0, u[sl] / 255.0, v[sl] / 255.0, full_range, m)):
            counts["rgb"[c]] = counts.get("rgb"[c], 0) + tie_rule(got[sl, :, c], e, f"4:4:4 {matrix} {'rgb'[c]}")
    assert np.all(got[..., 3] == 255)
    if m == BT709:
        assert np.array_equal(got, legacy_entry("planar", full_range)(y, u, v, SIDE, SIDE, SIDE, SIDE))
    report(f"NC-13 4:4:4 {matrix} {'full' if full_range else 'limited'}, bytes off rint(float64)", counts)


def _check_420_frame(planes, full_range, m, what):
    """the colour oracle at 4:2:0 and NV12 on one frame against the restatement with the exactly
    interpolated chroma -> bytes off rint"""
    y, u, v = planes
    got = {"planar": ico.yuv_planar_to_rgba(y, u, v, SIDE, SIDE, SIDE // 2, SIDE // 2, full_range, m),
           "nv12": ico.nv12_to_rgba(y, np.stack([u, v], axis=-1), SIDE, SIDE, full_range, m)}
    assert np.array_equal(got["planar"], got["nv12"])
    n = 0
    for r0 in range(0, SIDE, CHUNK):
        rows = np.arange(r0, r0 + CHUNK)
        ex = nc13_rgb(y[rows] / 255.0, upsample2_sum16(u, rows) / (16.0 * 255.0), upsample2_sum16(v, rows) / (16.0 * 255.0),
                      full_range, m)
        for c, e in enumerate(ex):
            n += tie_rule(got["planar"][rows, :, c], e, f"{what} {'rgb'[c]}")
    return n


@pytest.mark.parametrize("full_range", [0, 1], ids=["limited", "full"])
def test_420_bt601_every_triple(full_range):
    """the 4:2:0 and NV12 entry points at BT.601 on the four block frames (every (Y, U, V) with the chroma delivered
    exactly) and on the chroma-sum frame (every interpolated chroma value with every Y)"""
    seen = np.zeros(N, bool)
    n = 0
    for part in range(4):
        planes, cov = yuv420_block_triples(part)
        seen |= cov
        n += _check_420_frame(planes, full_range, BT601, f"4:2:0 blocks {part}")
    assert coverage(seen) == N
    planes, cov = yuv420_chroma_sums()
    assert cov["u"] == cov["v"] == 256 * 4081
    n += _check_420_frame(planes, full_range, BT601, "4:2:0 chroma sums")
    report(f"NC-13 4:2:0 / NV12 BT.601 {'full' if full_range else 'limited'}, bytes off rint(float64)", {"rgb": n})


def test_420_bt709_entry_points_are_the_legacy_ones():
    """at BT.709 and the format's own range the colour oracle's 4:2:0 / NV12 converters write the committed oracle's bytes"""
    (y, u, v), _ = yuv420_chroma_sums()
    uv = np.stack([u, v], axis=-1)
    assert np.array_equal(ico.nv12_to_rgba(y, uv, SIDE, SIDE, 0, BT709), orc.nv12_to_rgba(y, uv, SIDE, SIDE))
    for fr in (0, 1):
        assert np.array_equal(ico.yuv_planar_to_rgba(y, u, v, SIDE, SIDE, SIDE // 2, SIDE // 2, fr, BT709),
                              orc.yuv420_to_rgba(y, u, v, SIDE, SIDE, full_range=bool(fr)))


@pytest.mark.parametrize("matrix", list(MATRICES), ids=list(MATRICES))
@pytest.mark.parametrize("full_range", [0, 1], ids=["limited", "full"])
@pytest.mark.parametrize("yuyv", [0, 1], ids=["uyvy", "yuyv"])
def test_interleaved_every_triple(yuyv, full_range, matrix):
    """the colour oracle's UYVY / YUYV converter on every (Y, U, V), both ranges; at BT.709 limited it is
    orc_interleaved422_to_rgba"""
    m = MATRICES[matrix]
    t, n = interleaved_all_triples(yuyv)
    assert n == N
    got = ico.interleaved422_to_rgba(t, SIDE, SIDE, yuyv, full_range, m)
    y, u, v = interleaved_planes(t, yuyv)
    counts = 0
    for r0 in range(0, SIDE, CHUNK):
        sl = slice(r0, r0 + CHUNK)
        for c, e in enumerate(nc13_rgb(y[sl] / 255.0, u[sl] / 255.0, v[sl] / 255.0, full_range, m)):
            counts += tie_rule(got[sl, :, c], e, f"{'yuyv' if yuyv else 'uyvy'} {matrix} {'rgb'[c]}")
    legacy = legacy_entry("yuyv" if yuyv else "uyvy", full_range)
    if m == BT709 and legacy is not None:
        assert np.array_equal(got, legacy(t, SIDE, SIDE))
    report(f"NC-13 {'yuyv' if yuyv else 'uyvy'} {matrix} {'full' if full_range else 'limited'}", {"rgb": counts})


# ------------------------------------------------------------------------------------------------
# status rules, on a host-only handle
# ------------------------------------------------------------------------------------------------
INVALID = 1   # SMR_ERR_INVALID_ARGUMENT


@pytest.fixture
def host_handle():
    L = F.lib()
    h = C.c_void_p()
    assert L.smr_create(C.byref(F.Options(-1, 0, 100, 3_000_000_000, 30, 1)), C.byref(h)) == F.SMR_OK
    assert L.smr_register_input(h, b"in") == F.SMR_OK
    yield L, h
    L.smr_destroy(h)


def set_color(handle, input_id=b"in", matrix=F.MATRIX_BT601, rng=F.RANGE_LIMITED):
    L, h = handle
    return L.smr_set_input_color(h, input_id, C.byref(F.InputColor(matrix, rng)))


@pytest.mark.parametrize("matrix", [F.MATRIX_DEFAULT, F.MATRIX_BT709, F.MATRIX_BT601])
@pytest.mark.parametrize("rng", [F.RANGE_DEFAULT, F.RANGE_LIMITED, F.RANGE_FULL])
def test_accepted(host_handle, matrix, rng):
    assert set_color(host_handle, matrix=matrix, rng=rng) == F.SMR_OK


def test_refusals(host_handle):
    L, h = host_handle
    assert L.smr_set_input_color(h, None, C.byref(F.InputColor(1, 1))) == INVALID
    assert L.smr_set_input_color(h, b"in", None) == INVALID
    assert L.smr_set_input_color(None, b"in", C.byref(F.InputColor(1, 1))) == INVALID
    assert set_color(host_handle, input_id=b"other") == INVALID
    for m in (-1, 3, 1 << 30):
        assert set_color(host_handle, matrix=m) == INVALID
    for r in (-1, 3, -(1 << 31)):
        assert set_color(host_handle, rng=r) == INVALID


def test_setting_belongs_to_a_registered_input(host_handle):
    L, h = host_handle
    assert set_color(host_handle) == F.SMR_OK
    assert L.smr_unregister_input(h, b"in") == F.SMR_OK
    assert set_color(host_handle) == INVALID
    assert L.smr_register_input(h, b"in") == F.SMR_OK
    assert set_color(host_handle, matrix=F.MATRIX_DEFAULT, rng=F.RANGE_FULL) == F.SMR_OK


def test_python_interface():
    r = s.Renderer(s.RendererOptions(cuda_device=-1))
    r.register_input("in")
    r.set_input_color("in", s.YuvMatrix.BT601, s.YuvRange.Full)
    r.set_input_color("in", s.YuvMatrix.BT709)
    r.set_input_color("in")
    with pytest.raises(s.RendererError):
        r.set_input_color("in", 3)
    with pytest.raises(s.RendererError):
        r.set_input_color("in", s.YuvMatrix.BT601, 7)
    with pytest.raises(s.RendererError):
        r.set_input_color("nope", s.YuvMatrix.BT601)
    r.close()
    assert (s.YuvMatrix.Default, s.YuvMatrix.BT709, s.YuvMatrix.BT601) == (0, 1, 2)
    assert (s.YuvRange.Default, s.YuvRange.Limited, s.YuvRange.Full) == (0, 1, 2)


def test_inspection_records_end_in_the_matrix():
    """smr_fused_job_info and smr_composite_layer_info gained one trailing int32 each: the ctypes mirrors follow the header"""
    assert F.FusedJobInfo._fields_[-1] == ("matrix", C.c_int32)
    assert F.CompositeLayerInfo._fields_[-1] == ("tex_matrix", C.c_int32)
    assert F.FusedJobInfo.matrix.offset == C.sizeof(F.FusedJobInfo) - 4
    assert F.CompositeLayerInfo.tex_matrix.offset == C.sizeof(F.CompositeLayerInfo) - 4
