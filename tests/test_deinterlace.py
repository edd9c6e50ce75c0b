"""Deinterlacing on the CPU: the status rules of smr_set_input_deinterlace on a host-only handle, and a numpy restatement of
DESIGN.md NC-12 (the field and motion-adaptive rules, per plane, and the per-input history) with the properties that pin
it.  tests/test_gpu_deinterlace.py holds k_deinterlace and the renderer to this restatement byte for byte."""
import ctypes as C
import os

import numpy as np
import pytest

import smelter_b200 as s
from smelter_b200 import _ffi as F
from smelter_b200.renderer import plane_shapes

OFF, FIELD, MOTION = F.DEINTERLACE_OFF, F.DEINTERLACE_FIELD, F.DEINTERLACE_MOTION_ADAPTIVE
TOP, BOTTOM = F.FIELD_TOP_FIRST, F.FIELD_BOTTOM_FIRST
FORMATS = [F.FRAME_PLANAR_YUV420, F.FRAME_PLANAR_YUVJ420, F.FRAME_NV12, F.FRAME_BGRA, F.FRAME_ARGB, F.FRAME_RGBA8,
           F.FRAME_PLANAR_YUV422, F.FRAME_PLANAR_YUV444, F.FRAME_UYVY422, F.FRAME_YUYV422]


# ---------------------------------------------------------------------------------------------------------------------
# NC-12, restated
# ---------------------------------------------------------------------------------------------------------------------
def deinterlace_plane(cur, mode, field_order, threshold=10, prev=None):
    """one plane, (rows, row bytes) uint8: the kept field as it is, the other rebuilt.  prev: the previous frame's plane
    (MOTION_ADAPTIVE; None: the rebuilt rows follow FIELD)"""
    cur = np.asarray(cur, np.uint8)
    if mode == OFF:
        return cur.copy()
    rows = cur.shape[0]
    out = cur.copy()
    if rows == 1:
        return out
    ys = np.arange(1 if field_order == TOP else 0, rows, 2)
    ia = np.where(ys - 1 >= 0, ys - 1, ys + 1)
    ib = np.where(ys + 1 < rows, ys + 1, ys - 1)
    a, b = cur[ia].astype(np.int32), cur[ib].astype(np.int32)
    field = (a + b + 1) >> 1
    if mode == MOTION and prev is not None:
        p = np.asarray(prev, np.int32)
        c = cur[ys].astype(np.int32)
        m = np.maximum(np.maximum(np.abs(c - p[ys]), np.abs(a - p[ia])), np.abs(b - p[ib]))
        field = np.where(m <= threshold, c, field)
    out[ys] = field.astype(np.uint8)
    return out


class InputModel:
    """One input's NC-12 state: its setting and the last two frames of distinct pts (the history)"""

    def __init__(self):
        self.mode, self.order, self.threshold = OFF, TOP, 10
        self.clear()

    def clear(self):
        self.last = None     # ((format, width, height, pts), planes)
        self.before = None

    def set(self, mode, order=TOP, threshold=10):
        if (mode, order) != (self.mode, self.order):
            self.clear()
        self.mode, self.order, self.threshold = mode, order, threshold

    def frame(self, fmt, width, height, pts, planes):
        """the planes a tick with this live frame reads"""
        prev = None
        if self.mode == MOTION:
            if self.last is not None and self.last[0][:3] != (fmt, width, height):
                self.clear()
            if self.last is not None and self.last[0][3] == pts:   # the same frame again: the history stays
                prev = self.before
            else:
                prev = self.last
                self.before, self.last = self.last, ((fmt, width, height, pts), [np.array(p, np.uint8) for p in planes])
            prev = None if prev is None else prev[1]
        return [deinterlace_plane(p, self.mode, self.order, self.threshold, None if prev is None else prev[i])
                for i, p in enumerate(planes)]


def random_planes(fmt, w, h, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, shape, np.uint8) for shape in plane_shapes(fmt, w, h)]


# ---------------------------------------------------------------------------------------------------------------------
# properties of the restatement
# ---------------------------------------------------------------------------------------------------------------------
def test_known_answer():
    cur = np.array([[10, 200], [0, 0], [20, 100], [255, 255], [31, 0]], np.uint8)
    top = deinterlace_plane(cur, FIELD, TOP)
    assert top.tolist() == [[10, 200], [15, 150], [20, 100], [26, 50], [31, 0]]   # (10 + 20 + 1) >> 1, ...
    bottom = deinterlace_plane(cur, FIELD, BOTTOM)
    assert bottom.tolist() == [[0, 0], [0, 0], [128, 128], [255, 255], [255, 255]]   # row 0 takes row 1, row 4 row 3
    prev = cur.copy()
    prev[1, 0] = 5                  # |c - p| = 5 at (1, 0); elsewhere no motion
    got = deinterlace_plane(cur, MOTION, TOP, threshold=4, prev=prev)
    assert got[1].tolist() == [15, 0] and got[3].tolist() == [255, 255]
    assert deinterlace_plane(cur, MOTION, TOP, threshold=5, prev=prev)[1].tolist() == [0, 0]


@pytest.mark.parametrize("order", [TOP, BOTTOM])
@pytest.mark.parametrize("rows", [2, 3, 36, 37])
def test_field_of_constant_columns_is_the_input(order, rows):
    col = np.random.default_rng(rows).integers(0, 256, 53, np.uint8)
    cur = np.tile(col, (rows, 1))
    assert np.array_equal(deinterlace_plane(cur, FIELD, order), cur)


@pytest.mark.parametrize("order", [TOP, BOTTOM])
@pytest.mark.parametrize("rows", [2, 3, 36, 37])
def test_motion_adaptive_at_255_is_the_input(order, rows):
    rng = np.random.default_rng(rows + 7)
    cur, prev = rng.integers(0, 256, (rows, 40), np.uint8), rng.integers(0, 256, (rows, 40), np.uint8)
    assert np.array_equal(deinterlace_plane(cur, MOTION, order, 255, prev), cur)


@pytest.mark.parametrize("order", [TOP, BOTTOM])
@pytest.mark.parametrize("rows", [2, 3, 36, 37])
def test_motion_adaptive_at_0_with_every_byte_moved_is_field(order, rows):
    rng = np.random.default_rng(rows + 11)
    cur = rng.integers(0, 256, (rows, 40), np.uint8)
    prev = cur ^ rng.integers(1, 256, cur.shape, np.uint8)   # differs from cur in every byte
    assert np.array_equal(deinterlace_plane(cur, MOTION, order, 0, prev), deinterlace_plane(cur, FIELD, order))


def test_motion_adaptive_without_a_previous_frame_is_field():
    cur = np.random.default_rng(3).integers(0, 256, (9, 12), np.uint8)
    for order in (TOP, BOTTOM):
        assert np.array_equal(deinterlace_plane(cur, MOTION, order, 10, None), deinterlace_plane(cur, FIELD, order))


@pytest.mark.parametrize("rows", [2, 3, 36, 37])
def test_edge_rows_replicate(rows):
    cur = np.random.default_rng(rows + 5).integers(0, 256, (rows, 24), np.uint8)
    bottom = deinterlace_plane(cur, FIELD, BOTTOM)
    assert np.array_equal(bottom[0], cur[1])               # row 0 is rebuilt from row 1 alone
    top = deinterlace_plane(cur, FIELD, TOP)
    if rows % 2 == 0:
        assert np.array_equal(top[rows - 1], cur[rows - 2])   # the last row is odd: rebuilt from the row above alone
    else:
        assert np.array_equal(bottom[rows - 1], cur[rows - 2])
    assert np.array_equal(top[0::2], cur[0::2]) and np.array_equal(bottom[1::2], cur[1::2])   # the kept field


def test_one_row_is_copied():
    cur = np.arange(17, dtype=np.uint8).reshape(1, 17)
    for mode in (FIELD, MOTION):
        for order in (TOP, BOTTOM):
            assert np.array_equal(deinterlace_plane(cur, mode, order, 0, cur ^ 1), cur)


def test_history_model():
    m = InputModel()
    m.set(MOTION, TOP, 0)
    f0, f1, f2 = (random_planes(F.FRAME_NV12, 8, 6, k) for k in range(3))
    field = lambda planes: [deinterlace_plane(p, FIELD, TOP) for p in planes]   # noqa: E731
    motion = lambda planes, prev: [deinterlace_plane(p, MOTION, TOP, 0, q) for p, q in zip(planes, prev)]   # noqa: E731
    eq = lambda a, b: all(np.array_equal(x, y) for x, y in zip(a, b))   # noqa: E731
    assert eq(m.frame(F.FRAME_NV12, 8, 6, 0, f0), field(f0))              # first frame
    assert eq(m.frame(F.FRAME_NV12, 8, 6, 0, f0), field(f0))              # repeated pts: no previous frame yet
    assert eq(m.frame(F.FRAME_NV12, 8, 6, 1, f1), motion(f1, f0))
    assert eq(m.frame(F.FRAME_NV12, 8, 6, 1, f1), motion(f1, f0))         # repeated pts: the same bytes
    assert eq(m.frame(F.FRAME_NV12, 8, 6, 2, f2), motion(f2, f1))
    g = random_planes(F.FRAME_NV12, 8, 8, 9)
    assert eq(m.frame(F.FRAME_NV12, 8, 8, 3, g), field(g))                # a resize clears the history
    m.set(MOTION, BOTTOM, 0)
    assert m.last is None                                                 # so does a change of field order
    m.set(MOTION, BOTTOM, 7)
    m.frame(F.FRAME_NV12, 8, 8, 4, g)
    m.set(MOTION, BOTTOM, 9)
    assert m.last is not None                                             # a threshold alone keeps it


# ---------------------------------------------------------------------------------------------------------------------
# status rules, on a host-only handle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def host_handle():
    L = F.lib()
    h = C.c_void_p()
    assert L.smr_create(C.byref(F.Options(-1, 0, 100, 3_000_000_000, 30, 1)), C.byref(h)) == F.SMR_OK
    assert L.smr_register_input(h, b"in") == F.SMR_OK
    yield L, h
    L.smr_destroy(h)


def set_cfg(handle, input_id=b"in", mode=FIELD, order=TOP, threshold=10):
    L, h = handle
    return L.smr_set_input_deinterlace(h, input_id, C.byref(F.Deinterlace(mode, order, threshold)))


INVALID = 1   # SMR_ERR_INVALID_ARGUMENT


@pytest.mark.parametrize("mode", [OFF, FIELD, MOTION])
@pytest.mark.parametrize("order", [TOP, BOTTOM])
@pytest.mark.parametrize("threshold", [0, 10, 255])
def test_accepted(host_handle, mode, order, threshold):
    assert set_cfg(host_handle, mode=mode, order=order, threshold=threshold) == F.SMR_OK


def test_refusals(host_handle):
    L, h = host_handle
    assert L.smr_set_input_deinterlace(h, None, C.byref(F.Deinterlace(FIELD, TOP, 10))) == INVALID
    assert L.smr_set_input_deinterlace(h, b"in", None) == INVALID
    assert L.smr_set_input_deinterlace(None, b"in", C.byref(F.Deinterlace(FIELD, TOP, 10))) == INVALID
    assert set_cfg(host_handle, input_id=b"other") == INVALID
    for mode in (-1, 3, 1 << 30):
        assert set_cfg(host_handle, mode=mode) == INVALID
    for order in (-1, 2):
        assert set_cfg(host_handle, order=order) == INVALID
    for t in (256, 1 << 31, 0xFFFFFFFF):
        assert set_cfg(host_handle, threshold=t) == INVALID


def test_setting_belongs_to_a_registered_input(host_handle):
    L, h = host_handle
    assert set_cfg(host_handle) == F.SMR_OK
    assert L.smr_unregister_input(h, b"in") == F.SMR_OK
    assert set_cfg(host_handle) == INVALID
    assert L.smr_register_input(h, b"in") == F.SMR_OK
    assert set_cfg(host_handle, mode=MOTION) == F.SMR_OK


def test_debug_input_planes_refusals(host_handle):
    L, h = host_handle
    buf = (C.c_void_p * 3)(0x1000, 0x2000, 0x3000)
    pitch = (C.c_uint32 * 3)()
    assert L.smr_debug_input_planes(h, None, C.byref(buf), C.byref(pitch), F.MEM_HOST) == INVALID
    assert L.smr_debug_input_planes(h, b"in", None, C.byref(pitch), F.MEM_HOST) == INVALID
    assert L.smr_debug_input_planes(h, b"in", C.byref(buf), C.byref(pitch), 7) == INVALID
    assert L.smr_debug_input_planes(h, b"other", C.byref(buf), C.byref(pitch), F.MEM_HOST) == INVALID
    assert L.smr_debug_input_planes(h, b"in", C.byref(buf), C.byref(pitch), F.MEM_HOST) == INVALID   # no frame yet


def test_python_interface():
    r = s.Renderer(s.RendererOptions(cuda_device=-1))
    r.register_input("in")
    r.set_input_deinterlace("in", s.DeinterlaceMode.MotionAdaptive, s.FieldOrder.BottomFirst, 20)
    r.set_input_deinterlace("in", s.DeinterlaceMode.Off)
    with pytest.raises(s.RendererError):
        r.set_input_deinterlace("in", s.DeinterlaceMode.Field, motion_threshold=256)
    with pytest.raises(s.RendererError):
        r.set_input_deinterlace("nope", s.DeinterlaceMode.Field)
    with pytest.raises(s.RendererError):
        r.debug_input_planes("in")
    r.close()


def test_kernel_class_is_appended():
    header = open(os.path.join(os.path.dirname(os.path.dirname(__file__)), "include", "smelter_b200.h")).read()
    assert "SMR_KERNEL_DEINTERLACE = 14" in header and "SMR_KERNEL_CLASSES = 15" in header
    assert F.KERNEL_CLASSES[14] == "deinterlace" and len(F.KERNEL_CLASSES) == 15


def test_plane_shapes_follow_the_frame_formats():
    want = {F.FRAME_PLANAR_YUV420: [(37, 70), (18, 35), (18, 35)], F.FRAME_PLANAR_YUVJ420: [(37, 70), (18, 35), (18, 35)],
            F.FRAME_NV12: [(37, 70), (18, 70)], F.FRAME_BGRA: [(37, 280)], F.FRAME_ARGB: [(37, 280)], F.FRAME_RGBA8: [(37, 280)],
            F.FRAME_PLANAR_YUV422: [(37, 70), (37, 35), (37, 35)], F.FRAME_PLANAR_YUV444: [(37, 70)] * 3,
            F.FRAME_UYVY422: [(37, 140)], F.FRAME_YUYV422: [(37, 140)]}
    assert sorted(want) == sorted(FORMATS)
    for fmt in FORMATS:
        assert plane_shapes(fmt, 70, 37) == want[fmt], fmt
