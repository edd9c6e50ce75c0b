"""Deinterlacing on an H100: k_deinterlace and the renderer's per-input history against the numpy restatement of NC-12
(tests/test_deinterlace.py), byte for byte.

(a) smr_debug_input_planes after one and after two ticks, for every frame format, both modes, both field orders, odd and
    even heights, host and device frames, packed and pitched planes;
(b) sequences: first frame, repeated pts, new pts, a stale tick, a resize, unregister / re-register, and ticks in flight
    through smr_render_begin / smr_render_end with the device planes rewritten after each tick retires;
(c) end to end: scenes on a deinterlacing handle give the bytes a second handle gives when fed the restatement's planes
    as progressive frames (the fused Lanczos 4:1 path with direct tiles, a 1:1 child, the generic path for 4:2:2);
(d) OFF gives the bytes and the launch count of a handle where the call was never made."""
import ctypes as C

import numpy as np
import pytest
import torch

import smelter_b200 as s
from smelter_b200 import _ffi as F
from smelter_b200.renderer import _FRAME_KIND, plane_shapes
from tests.test_deinterlace import BOTTOM, FIELD, FORMATS, MOTION, OFF, TOP, InputModel, random_planes

pytestmark = pytest.mark.gpu

KIND = {v: k for k, v in _FRAME_KIND.items()}
T = 12


@pytest.fixture(scope="module")
def r():
    rr = s.Renderer()
    yield rr
    rr.close()


def moved(planes, seed):
    """the next frame: half the bytes move a little (below and above T), the rest anywhere"""
    rng = np.random.default_rng(seed)
    out = []
    for p in planes:
        small = (p.astype(np.int32) + rng.integers(-2 * T, 2 * T + 1, p.shape)).clip(0, 255).astype(np.uint8)
        out.append(np.where(rng.random(p.shape) < 0.5, small, rng.integers(0, 256, p.shape, np.uint8)))
    return out


class Frames:
    """smr_input_frame records over planes placed in host or device memory: layout "packed" (pitch 0), or "pitched"
    (rows of row bytes + 6 rounded up to 4, the device planes starting 4 bytes past a 16-byte boundary)"""

    def __init__(self, n):
        self.arr = (F.InputFrame * max(1, n))()
        self.keep = []

    def set(self, i, input_id, fmt, w, h, pts_ns, planes, mem="host", layout="packed"):
        f = self.arr[i]
        bid = input_id.encode()
        self.keep.append(bid)
        f.input_id, f.format, f.width, f.height, f.pts_ns = bid, fmt, w, h, pts_ns
        f.mem_kind = F.MEM_DEVICE if mem == "device" else F.MEM_HOST
        for p, plane in enumerate(planes):
            rows, rb = plane.shape
            pitch = rb if layout == "packed" else (rb + 6 + 3) // 4 * 4
            off = 4 if (layout == "pitched" and mem == "device") else 0
            host = np.full(rows * pitch + off, 0xAB, np.uint8)
            host[off:off + rows * pitch].reshape(rows, pitch)[:, :rb] = plane
            if mem == "device":
                buf = torch.from_numpy(host).to("cuda:0")
                ptr = buf.data_ptr() + off
            else:
                buf, ptr = host, host.ctypes.data
            self.keep.append(buf)
            f.planes[p] = ptr
            f.pitch[p] = 0 if layout == "packed" else pitch
        torch.cuda.synchronize()


def tick(r, pts_ns, frames, n):
    r.render_raw(pts_ns, frames.arr, n, None, 0)


def assert_planes(got, want, what):
    assert len(got) == len(want), what
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape, (what, i, g.shape, w.shape)
        bad = g != w
        assert not bad.any(), (what, "plane", i, int(bad.sum()), tuple(np.argwhere(bad)[0]))


# ---------------------------------------------------------------------------------------------------------------------
# (a) the planes, per format, mode, field order, height and memory
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem,layout", [("host", "packed"), ("host", "pitched"), ("device", "packed"), ("device", "pitched")])
@pytest.mark.parametrize("h", [36, 37])
@pytest.mark.parametrize("order", [TOP, BOTTOM])
@pytest.mark.parametrize("mode", [FIELD, MOTION])
@pytest.mark.parametrize("fmt", FORMATS)
def test_planes(r, fmt, mode, order, h, mem, layout):
    w = 70   # chroma rows of 35 bytes, RGBA rows of 280: partial 16-byte columns everywhere
    r.register_input("in")
    try:
        r.set_input_deinterlace("in", mode, order, T)
        model = InputModel()
        model.set(mode, order, T)
        f0 = random_planes(fmt, w, h, fmt * 100 + h)
        for k, planes in enumerate((f0, moved(f0, h + order))):
            fr = Frames(1)
            fr.set(0, "in", fmt, w, h, 1000 + k, planes, mem, layout)
            tick(r, 1000 + k, fr, 1)
            assert_planes(r.debug_input_planes("in"), model.frame(fmt, w, h, 1000 + k, planes), (KIND[fmt], mode, order, h, k))
    finally:
        r.unregister_input("in")


@pytest.mark.parametrize("fmt", [F.FRAME_PLANAR_YUV420, F.FRAME_NV12, F.FRAME_UYVY422, F.FRAME_BGRA])
@pytest.mark.parametrize("size", [(1920, 1080), (1918, 1081)])
def test_planes_full_size(r, fmt, size):
    w, h = size
    r.register_input("in")
    try:
        r.set_input_deinterlace("in", MOTION, BOTTOM, T)
        model = InputModel()
        model.set(MOTION, BOTTOM, T)
        f0 = random_planes(fmt, w, h, fmt + w)
        for k, planes in enumerate((f0, moved(f0, 5), moved(f0, 6))):
            fr = Frames(1)
            fr.set(0, "in", fmt, w, h, k, planes, "device" if k % 2 else "host")
            tick(r, k, fr, 1)
            assert_planes(r.debug_input_planes("in"), model.frame(fmt, w, h, k, planes), (KIND[fmt], size, k))
    finally:
        r.unregister_input("in")


def test_several_inputs_in_one_launch(r):
    """three deinterlaced inputs of different formats and settings and one left alone: one k_deinterlace launch"""
    ids = ["a", "b", "c", "d"]
    setup = {"a": (F.FRAME_NV12, FIELD, TOP), "b": (F.FRAME_UYVY422, MOTION, BOTTOM), "c": (F.FRAME_PLANAR_YUV444, MOTION, TOP),
             "d": (F.FRAME_RGBA8, OFF, TOP)}
    models = {}
    for i in ids:
        r.register_input(i)
        fmt, mode, order = setup[i]
        r.set_input_deinterlace(i, mode, order, T)
        models[i] = InputModel()
        models[i].set(mode, order, T)
    try:
        r.set_profiling(True)
        frames = {i: random_planes(setup[i][0], 96, 54, ord(i)) for i in ids}
        for k in range(2):
            fr = Frames(len(ids))
            for n, i in enumerate(ids):
                fr.set(n, i, setup[i][0], 96, 54, k, frames[i])
            tick(r, k, fr, len(ids))
            for i in ids:
                assert_planes(r.debug_input_planes(i), models[i].frame(setup[i][0], 96, 54, k, frames[i]), (i, k))
            frames = {i: moved(frames[i], k) for i in ids}
        assert r.kernel_times()["deinterlace"][1] == 2
        assert r.stats()["last_render_kernel_launches"] == 1
    finally:
        r.set_profiling(False)
        for i in ids:
            r.unregister_input(i)


# ---------------------------------------------------------------------------------------------------------------------
# (b) sequences
# ---------------------------------------------------------------------------------------------------------------------
def test_sequence(r):
    fmt, w = F.FRAME_NV12, 64
    a = random_planes(fmt, w, 36, 0)
    b, c = moved(a, 1), moved(a, 2)
    d = random_planes(fmt, w, 40, 3)
    e = moved(d, 4)
    sec = 1_000_000_000
    r.register_input("in")
    r.set_input_deinterlace("in", MOTION, TOP, T)
    model = InputModel()
    model.set(MOTION, TOP, T)

    def step(pts, planes, h, frame_pts=None, live=True, what=""):
        fr = Frames(1)
        fr.set(0, "in", fmt, w, h, pts if frame_pts is None else frame_pts, planes, "device")
        tick(r, pts, fr, 1)
        if live:
            assert_planes(r.debug_input_planes("in"), model.frame(fmt, w, h, pts, planes), what)

    try:
        step(0, a, 36, what="first frame")
        step(0, a, 36, what="repeated pts, no history yet")
        step(sec, b, 36, what="new pts")
        step(sec, b, 36, what="repeated pts")
        step(10 * sec, b, 36, frame_pts=sec, live=False)   # stale: older than the 3 s fallback timeout, no live frame
        step(11 * sec, c, 36, what="new pts after a stale tick: the history is b")
        step(12 * sec, d, 40, what="resize: no history")
        step(13 * sec, e, 40, what="after the resize")
        r.set_input_deinterlace("in", MOTION, TOP, T + 1)   # the threshold alone keeps the history
        model.set(MOTION, TOP, T + 1)
        step(14 * sec, d, 40, what="threshold changed")
        r.set_input_deinterlace("in", MOTION, BOTTOM, T)    # the field order clears it
        model.set(MOTION, BOTTOM, T)
        step(15 * sec, e, 40, what="field order changed")
        r.unregister_input("in")
        r.register_input("in")
        model = InputModel()                                 # the setting and the history are gone: OFF
        step(16 * sec, a, 36, what="re-registered, off")
        r.set_input_deinterlace("in", MOTION, TOP, T)
        model.set(MOTION, TOP, T)
        step(17 * sec, b, 36, what="enabled again: no history")
        step(18 * sec, c, 36, what="and then with b")
    finally:
        r.unregister_input("in")


def yuv420_out(r, w, h):
    sizes = (C.c_size_t * 3)()
    assert r._lib.smr_output_plane_sizes(w, h, F.OUT_PLANAR_YUV420, C.byref(sizes)) == F.SMR_OK
    return [np.zeros(sizes[p], np.uint8) for p in range(3)]


def test_ticks_in_flight():
    """three ticks in flight on a ring of three device plane sets; each set is rewritten with the next frame once the tick
    that read it has retired.  Every tick's output equals a second handle's fed the restatement's planes."""
    fmt, w, h = F.FRAME_NV12, 128, 72
    pts_seq = [0, 1, 1, 2, 3, 3, 3, 4, 5, 6]
    content = {}
    for p in pts_seq:
        content.setdefault(p, moved(random_planes(fmt, w, h, 50), p) if p else random_planes(fmt, w, h, 50))
    ra, rb = s.Renderer(), s.Renderer()
    try:
        for rr in (ra, rb):
            rr.register_input("in")
            rr.update_scene("out", s.Resolution(w, h), s.OutputFrameFormat.PlanarYuv420Bytes, s.InputStreamComponent(input_id="in"))
        ra.set_input_deinterlace("in", MOTION, BOTTOM, T)
        ring = [torch.zeros(h * w * 3 // 2, dtype=torch.uint8, device="cuda:0") for _ in range(3)]
        outs, keep = [], []
        for k, pts in enumerate(pts_seq):
            if k >= 3:
                ra.wait()   # retires tick k - 3, the last reader of ring[k % 3]
            y, uv = content[pts]
            ring[k % 3].copy_(torch.from_numpy(np.concatenate([y.ravel(), uv.ravel()])))
            torch.cuda.synchronize()
            f = (F.InputFrame * 1)()
            f[0].input_id, f[0].format, f[0].width, f[0].height, f[0].pts_ns, f[0].mem_kind = b"in", fmt, w, h, pts, F.MEM_DEVICE
            f[0].planes[0], f[0].planes[1] = ring[k % 3].data_ptr(), ring[k % 3].data_ptr() + w * h
            o = (F.OutputFrame * 1)()
            o[0].output_id, o[0].mem_kind = b"out", F.MEM_HOST
            planes = yuv420_out(ra, w, h)
            for p in range(3):
                o[0].planes[p] = planes[p].ctypes.data
            keep.append((f, o))
            outs.append(planes)
            ra.render_raw(pts, f, 1, o, 1, wait=False)
        for _ in range(3):
            ra.wait()
        model = InputModel()
        model.set(MOTION, BOTTOM, T)
        for k, pts in enumerate(pts_seq):
            want_planes = model.frame(fmt, w, h, pts, content[pts])
            fs = s.FrameSet(frames={"in": s.Frame(s.FrameData(KIND[fmt], tuple(want_planes)), s.Resolution(w, h), pts / 1e9)},
                            pts=pts / 1e9)
            want = rb.render(fs).frames["out"].data.planes
            for p in range(3):
                assert np.array_equal(outs[k][p], np.ascontiguousarray(want[p]).ravel()), ("tick", k, "plane", p)
    finally:
        ra.close()
        rb.close()


# ---------------------------------------------------------------------------------------------------------------------
# (c) end to end, and (d) OFF
# ---------------------------------------------------------------------------------------------------------------------
def scene_inputs(name):
    """(output size, output format, scene root, {input id: (format, width, height)})"""
    if name == "fused_4to1_direct":   # cfg3's shape at 1080p: 16 x 1080p in 4 x 4 tiles of 480 x 270
        ins = {f"in{i}": (F.FRAME_PLANAR_YUV420 if i % 2 else F.FRAME_NV12, 1920, 1080) for i in range(16)}
        root = s.TilesComponent(children=[s.InputStreamComponent(input_id=i) for i in ins])
        return (1920, 1080), s.OutputFrameFormat.PlanarYuv420Bytes, root, ins
    if name == "one_to_one":          # an input shown at its size: the composite reads it 1:1
        ins = {"in0": (F.FRAME_NV12, 1280, 720)}
        return (1280, 720), s.OutputFrameFormat.Nv12WgpuTexture, s.InputStreamComponent(input_id="in0"), ins
    # planar and interleaved 4:2:2 at 2:1: the generic passes (planar) and the LDG fused kernel (UYVY)
    ins = {"in0": (F.FRAME_PLANAR_YUV422, 1280, 720), "in1": (F.FRAME_UYVY422, 1280, 720)}
    root = s.TilesComponent(children=[s.InputStreamComponent(input_id=i) for i in ins])
    return (1280, 720), s.OutputFrameFormat.PlanarYuv420Bytes, root, ins


def render_scene(rr, name, planes_of, pts):
    size, _, _, ins = scene_inputs(name)
    frames = {i: s.Frame(s.FrameData(KIND[fmt], tuple(planes_of[i])), s.Resolution(w, h), pts) for i, (fmt, w, h) in ins.items()}
    return [np.array(p) for p in rr.render(s.FrameSet(frames=frames, pts=pts)).frames["out"].data.planes]


def make_handle(name):
    size, fmt, root, ins = scene_inputs(name)
    rr = s.Renderer()
    for i in ins:
        rr.register_input(i)
    rr.update_scene("out", s.Resolution(*size), fmt, root)
    return rr


@pytest.mark.parametrize("mode", [FIELD, MOTION])
@pytest.mark.parametrize("name", ["fused_4to1_direct", "one_to_one", "generic_422"])
def test_end_to_end(name, mode):
    _, _, _, ins = scene_inputs(name)
    ra, rb = make_handle(name), make_handle(name)
    try:
        models = {}
        for n, i in enumerate(ins):
            order = TOP if n % 2 == 0 else BOTTOM
            ra.set_input_deinterlace(i, mode, order, T)
            models[i] = InputModel()
            models[i].set(mode, order, T)
        content = {i: random_planes(fmt, w, h, n) for n, (i, (fmt, w, h)) in enumerate(ins.items())}
        for k in range(2):
            got = render_scene(ra, name, content, k * 0.04)
            launches = ra.stats()["last_render_kernel_launches"]
            direct = ra.stats()["last_render_direct_tiles"]
            fused = [(j["kernel"], j["ratio"]) for j in ra.debug_fused_jobs()]
            want_planes = {i: models[i].frame(*ins[i], k, content[i]) for i in ins}
            want = render_scene(rb, name, want_planes, k * 0.04)
            for p, (g, wnt) in enumerate(zip(got, want)):
                assert np.array_equal(g, wnt), (name, mode, k, "plane", p, int((g != wnt).sum()))
            assert launches == rb.stats()["last_render_kernel_launches"] + 1   # k_deinterlace, and nothing else changed
            assert direct == rb.stats()["last_render_direct_tiles"]
            if name == "fused_4to1_direct":
                assert direct > 0 and fused and all(ratio == 4 for _, ratio in fused), (direct, fused)
            content = {i: moved(content[i], k + 10) for i in ins}
    finally:
        ra.close()
        rb.close()


@pytest.mark.parametrize("name", ["fused_4to1_direct", "generic_422"])
def test_off_is_unchanged(name):
    _, _, _, ins = scene_inputs(name)
    ra, rb = make_handle(name), make_handle(name)
    try:
        for i in ins:   # set, then switched off again
            ra.set_input_deinterlace(i, MOTION, BOTTOM, T)
            ra.set_input_deinterlace(i, OFF)
        content = {i: random_planes(fmt, w, h, n + 40) for n, (i, (fmt, w, h)) in enumerate(ins.items())}
        for k in range(2):
            got, want = render_scene(ra, name, content, k * 0.04), render_scene(rb, name, content, k * 0.04)
            for p, (g, wnt) in enumerate(zip(got, want)):
                assert np.array_equal(g, wnt), (name, k, "plane", p)
            assert ra.stats()["last_render_kernel_launches"] == rb.stats()["last_render_kernel_launches"]
            for i in ins:
                assert_planes(ra.debug_input_planes(i), content[i], (name, i))
            content = {i: moved(content[i], k) for i in ins}
    finally:
        ra.close()
        rb.close()
