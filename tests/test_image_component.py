"""Image components (smr_register_image, smr_component.image_id): registered bitmap and animated assets as scene nodes.

The reference's pictures are not in the tree (a JPEG behind a URL, GIFs in a submodule), so the six non-SVG scenes of
integration-tests/src/render_tests/image.rs are typed here over seeded stand-in pixels: an opaque 1200 x 630 bitmap for the
JPEG, and two animated assets with uneven delays for the GIFs.

CPU (host-only handle): the registry, the argument and scene errors, layouts and image node state against the independent
engine (tests/layout_ref_image.py), and the image oracle (tests/image_oracle.c) against the committed premultiply oracle.
GPU: every output byte against the oracle (the image oracle for the node textures, then the oracle's layout node).
"""
import ctypes as C

import numpy as np
import pytest

import smelter_b200 as s
from oracle import oracle as orc
from smelter_b200 import _ffi as F
from tests import harness
from tests import layout_ref_image as LR
from tests import c_oracles
from tests.parity import assert_identical, black, chroma_size, from_ref_layout, layouts_equal, node_texture, yuv_frame
from tests.test_layout_independent import diff, product_layouts, ref_layouts

V, R, IN, IMG = s.ViewComponent, s.RescalerComponent, s.InputStreamComponent, s.ImageComponent
YUV, NV12, RGBA = s.OutputFrameFormat.PlanarYuv420Bytes, s.OutputFrameFormat.Nv12WgpuTexture, s.OutputFrameFormat.RgbaWgpuTexture
MODES = [s.RenderingMode.GpuOptimized, s.RenderingMode.CpuOptimized]
FORMATS = [YUV, NV12, RGBA]
MS = 1_000_000


def pixels(w, h, n=1, seed=0, opaque=False):
    """n seeded straight-alpha frames: a smooth ramp plus noise, alpha over its whole range"""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        f = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        f[..., 0] = (np.arange(w)[None, :] * 255 // max(1, w - 1) + 40 * k) % 256
        f[::3, ::2, 3] = 255
        f[1::3, 1::2, 3] = 0
        if opaque:
            f[..., 3] = 255
        out.append(f)
    return out


JPEG = ("image_jpeg", pixels(1200, 630, 1, 1, opaque=True), None)
GIF1 = ("image_gif1", pixels(96, 64, 5, 2), [100 * MS, 150 * MS, 0, 200 * MS, 100 * MS])
GIF2 = ("image_gif2", pixels(80, 120, 3, 3), [300 * MS, 300 * MS, 400 * MS])


class Pair:
    """a renderer and the independent engine driven together; the pixels of every asset by its independent Asset object"""

    def __init__(self, out=(640, 360), fmt=YUV, mode=s.RenderingMode.GpuOptimized, device=None, inputs=()):
        opts = s.RendererOptions(rendering_mode=mode) if device is None else s.RendererOptions(rendering_mode=mode, cuda_device=device)
        self.r, self.ref = s.Renderer(opts), LR.StatefulScene(*out)
        self.out, self.fmt, self.mode, self.scene, self.px = out, fmt, mode, None, {}
        self.inputs = {i: (640, 360) for i in inputs}
        for i in inputs:
            self.r.register_input(i)

    def register(self, image_id, frames, delays=None):
        self.r.register_image(image_id, frames, delays)
        h, w = frames[0].shape[:2]
        self.ref.register_image(image_id, w, h, delays if delays is not None else [0] * len(frames))
        self.px[self.ref.images[image_id]] = frames

    def unregister(self, image_id):
        self.r.unregister_image(image_id)
        self.ref.unregister_image(image_id)

    def update(self, scene, out=None):
        if out is not None:
            self.out = out
            self.ref.out_w, self.ref.out_h = out
        self.r.update_scene("output_1", s.Resolution(*self.out), self.fmt, scene)
        self.ref.update_scene(scene)
        self.scene = scene

    def check_state(self, pts):
        """layouts field for field, and every image node's resolution, start pts and frame; returns the ref layouts"""
        self.r.debug_set_inputs(pts, {k: s.Resolution(*v) for k, v in self.inputs.items()})
        got, root = product_layouts(self.r, pts)
        exp, exp_root = self.ref.layouts(pts, self.inputs)
        assert root == exp_root, f"pts {pts}: root {root} expected {exp_root}"
        d = diff(got, ref_layouts(exp))
        assert d is None, f"pts {pts}: {d}"
        nodes = [(res, start, a.frame_at(LR.LR.to_ns(pts), start)) for _, a, start, res in self.ref.image_nodes()]
        assert self.r.debug_image_nodes("output_1", pts) == nodes
        return nodes

    # ---- GPU ----
    def frames(self, pts):
        return {k: yuv_frame(harness.test_input(i + 1, w, h), w, h, pts) for i, (k, (w, h)) in enumerate(sorted(self.inputs.items()))}

    def expected(self, pts, frames):
        m = orc.MODE_GPU_OPTIMIZED if self.mode == s.RenderingMode.GpuOptimized else orc.MODE_CPU_OPTIMIZED
        ns = LR.LR.to_ns(pts)
        res = {k: (f.resolution.width, f.resolution.height) for k, f in frames.items()}
        layouts, (rw, rh) = self.ref.layouts(pts, res)
        tex = {id(c): c_oracles.render_image(self.px[a][a.frame_at(ns, start)], w, h, m)
               for c, a, start, (w, h) in self.ref.image_nodes()}
        if isinstance(self.scene, IMG):
            return to_format(tex[id(self.scene)], self.out, self.fmt)
        got, root = self.r.debug_layouts("output_1", pts)
        assert root == (rw, rh)
        d = layouts_equal(got, layouts)
        assert d is None, d
        if rw == 0 or rh == 0:
            return black(s.Resolution(*self.out), self.fmt)
        nodes = [tex[id(c)] if isinstance(c, IMG) else node_texture(frames[c.input_id]) for c in leaves(self.scene)]
        rgba = orc.render_layout_node(rw, rh, [from_ref_layout(l) for l in layouts], nodes, mode=m, max_layouts=100)
        return to_format(rgba, self.out, self.fmt)

    def render_check(self, pts, what=""):
        frames = self.frames(pts)
        got = self.r.render(s.FrameSet(frames=frames, pts=pts)).frames["output_1"]
        assert_identical(tuple(np.asarray(p) for p in got.data.planes), self.expected(pts, frames), f"{what} pts {pts}")
        return self.r.stats()["last_render_kernel_launches"]


def leaves(comp):
    if isinstance(comp, (IN, IMG)):
        return [comp]
    if isinstance(comp, R):
        return leaves(comp.child)
    return [x for c in comp.children for x in leaves(c)]


def to_format(rgba, out, fmt):
    W, H = out
    if fmt == RGBA:
        assert rgba.shape[:2] == (H, W)
        return (rgba,)
    if fmt == NV12:
        return orc.rgba_to_nv12_scaled(rgba, W, H)
    return orc.rgba_to_yuv_planar_scaled(rgba, W, H, *chroma_size(fmt, W, H))


# ---- the reference's scenes: steps ("register", asset) | ("update", scene, root image size or None) | ("snapshot", pts) ----
def _jpeg(scene, then=None):
    steps = [("register", JPEG), ("update", scene)]
    if then is not None:
        steps.append(("update", then))
    return steps + [("snapshot", 0.0)]


def _gif(image_id):
    return IMG(id="gif", image_id=image_id)


SCENES = {
    "jpeg_as_root": lambda: _jpeg(IMG(image_id="image_jpeg")),
    "jpeg_in_view": lambda: _jpeg(V(children=[IMG(image_id="image_jpeg")])),
    "jpeg_in_view_overflow_fit": lambda: _jpeg(V(children=[IMG(image_id="image_jpeg")], overflow=s.Overflow.Fit)),
    "remove_jpeg_as_root": lambda: _jpeg(IMG(image_id="image_jpeg"), V()),
    "remove_jpeg_in_view": lambda: _jpeg(V(children=[IMG(image_id="image_jpeg")]), V()),
    "gif_progress_between_updates": lambda: [
        ("register", GIF1), ("register", GIF2),
        ("update", _gif("image_gif1")), ("snapshot", 0.5),
        ("update", _gif("image_gif1")), ("snapshot", 1.0),       # the update does not reset the progress
        ("update", _gif("image_gif2")), ("snapshot", 1.001)],    # the image changed: the progress restarts
}


def root_size(p, scene):
    """an RGBA output of an Image root has the node's size (render_loop.rs:81-103)"""
    if isinstance(scene, IMG) and p.fmt == RGBA:
        a = p.ref.images[scene.image_id]
        return LR.resolution(a, scene.width, scene.height)
    return (640, 360)


def play(p, steps, on_snapshot):
    n = 0
    for step in steps:
        if step[0] == "register":
            p.register(*step[1])
        elif step[0] == "update":
            p.update(step[1], out=root_size(p, step[1]))
        else:
            on_snapshot(step[1])
            n += 1
    return n


# ---- CPU ------------------------------------------------------------------------------------------------------------
def host(**kw):
    return Pair(device=-1, **kw)


@pytest.mark.parametrize("name", sorted(SCENES))
def test_reference_scenes_layouts_and_state(name):
    p = host(inputs=("input_1",))
    assert play(p, SCENES[name](), p.check_state) > 0


def test_gif_progress_story():
    p = host()
    play(p, SCENES["gif_progress_between_updates"](), p.check_state)
    # kept across the identical update (start 0), restarted at the last render's pts by the other asset
    assert [n[1] for n in p.check_state(1.001)] == [1000 * MS]
    small = lambda **kw: IMG(image_id="image_gif2", width=40.0, height=60.0, **kw)
    p.update(small(id="gif"))                                              # a changed component restarts too
    assert p.check_state(1.5)[0][:2] == ((40, 60), 1001 * MS)
    p.update(small(id="gif"))
    assert [n[1] for n in p.check_state(1.75)] == [1001 * MS]
    p.unregister("image_gif2")                                            # re-registration makes a new asset: restart
    p.register(*GIF2)
    p.update(small(id="gif"))
    assert [n[1] for n in p.check_state(2.0)] == [1750 * MS]
    p.update(small())                                                     # no component id: nothing to inherit from
    assert [n[1] for n in p.check_state(2.25)] == [2000 * MS]


def _raw_register(r, image_id, w, h, frames, n=None, pitch=0, delays=None, null_frame=False):
    arr = (F.ImageFrame * max(1, len(frames)))()
    for i, f in enumerate(frames):
        arr[i] = F.ImageFrame(None if null_frame else f.ctypes.data, pitch, delays[i] if delays else 0)
    spec = F.ImageSpec(w, h, arr, len(frames) if n is None else n)
    return F.lib().smr_register_image(r._h, image_id, C.byref(spec))


def test_registry_rules():
    r = s.Renderer(s.RendererOptions(cuda_device=-1))
    one = pixels(8, 4, 1)
    shown = lambda i: F.lib().smr_update_scene(r._h, b"o", 64, 64, YUV, C.byref(_image_c(i)))
    bad = [dict(w=0, h=4), dict(w=8, h=0), dict(w=16385, h=4), dict(w=8, h=16385), dict(w=8, h=4, pitch=31), dict(w=8, h=4, n=0),
           dict(w=8, h=4, null_frame=True)]
    for kw in bad:
        assert _raw_register(r, b"x", frames=one, **kw) == 1, kw
        assert shown(b"x") == 4                                            # a failed call registers nothing
    assert _raw_register(r, None, 8, 4, one) == 1
    assert F.lib().smr_register_image(r._h, b"x", None) == 1
    assert _raw_register(r, b"x", 8, 4, pixels(8, 4, 1001)) == 1          # TooManyFrames
    assert _raw_register(r, b"x", 8, 4, pixels(8, 4, 2), delays=[2 ** 63, 2 ** 63]) == 1
    assert shown(b"x") == 4
    assert _raw_register(r, b"x", 8, 4, [np.zeros((4, 10, 4), np.uint8)], pitch=40) == 0     # a pitch above the row is fine
    assert _raw_register(r, b"x", 8, 4, one) == 1                         # KeyTaken
    for n, image_id in ((1, b"n1"), (2, b"n2"), (1000, b"n1000")):
        assert _raw_register(r, image_id, 8, 4, pixels(8, 4, n)) == 0
        assert shown(image_id) == 0
    assert F.lib().smr_unregister_image(r._h, b"nope") == 1
    assert F.lib().smr_unregister_image(r._h, None) == 1
    assert F.lib().smr_unregister_image(r._h, b"x") == 0 and F.lib().smr_unregister_image(r._h, b"x") == 1
    assert shown(b"x") == 4
    ref = LR.StatefulScene(64, 64)                                        # the independent registry says the same
    ref.register_image("x", 8, 4, [0])
    for call in (lambda: ref.register_image("x", 8, 4, [0]), lambda: ref.unregister_image("nope"),
                 lambda: ref.register_image("y", 8, 4, []), lambda: ref.register_image("y", 8, 4, [0] * 1001)):
        with pytest.raises(LR.RegistryError):
            call()
    ref.register_image("y", 8, 4, [0] * 1000)


def _image_c(image_id, kind=F.COMPONENT_IMAGE):
    c = F.Component()
    F.lib().smr_component_default(kind, C.byref(c))
    c.image_id = image_id
    return c


def _status(r, scene):
    with pytest.raises(s.RendererError) as e:
        r.update_scene("output_1", s.Resolution(640, 360), YUV, scene)
    return e.value.status


def test_scene_errors():
    p = host()
    p.register(*JPEG)
    c = _image_c(None)
    assert not c.image_id and not c.image_width.has_value and not c.image_height.has_value       # NULL / None / None
    assert F.lib().smr_update_scene(p.r._h, b"output_1", 640, 360, YUV, C.byref(c)) == 5        # what an older caller sends
    assert _status(p.r, IMG(image_id="missing")) == 4
    assert _status(p.r, IMG(image_id="")) == 4                                                   # the reference's Default
    assert _status(p.r, V(children=[V(children=[IMG(image_id="missing")])])) == 4
    assert _status(p.r, V(children=[IMG(id="a", image_id="image_jpeg"), IMG(id="a", image_id="image_jpeg")])) == 4
    assert _status(p.r, V(id="a", children=[IMG(id="a", image_id="image_jpeg")])) == 4
    with pytest.raises(LR.SceneError):
        p.ref.update_scene(V(children=[IMG(id="a", image_id="image_jpeg"), IMG(id="a", image_id="image_jpeg")]))
    with pytest.raises(LR.SceneError):
        p.ref.update_scene(IMG(image_id=""))


ASSETS = {"landscape": (640, 360), "square": (100, 100), "portrait": (360, 640), "wide": (300, 100)}
SIDES = [(None, None), (200.0, 90.4), (150.5, None), (None, 60.5), (0.4, None), (None, 0.2), (20000.0, 10.0), (3.0, 17000.0),
         (float("nan"), 10.0), (-5.0, None), (1e30, None)]


@pytest.mark.parametrize("asset", sorted(ASSETS))
def test_resolution_rule(asset):
    """every width / height combination; the integer aspect ratio makes a portrait asset divide by zero"""
    w, h = ASSETS[asset]
    p = host()
    p.register("a", pixels(w, h, 1))
    p.update(V())
    accepted = refused = 0
    for sides in SIDES:
        scene = V(children=[IMG(image_id="a", width=sides[0], height=sides[1])])
        res = LR.resolution(p.ref.images["a"], *sides)
        if all(1 <= v <= 16384 for v in res):
            p.update(scene)
            assert [n[0] for n in p.check_state(0.0)] == [res]
            accepted += 1
        else:
            before = p.r.debug_layouts("output_1", 0.0)[1], p.r.debug_image_nodes("output_1", 0.0)
            assert _status(p.r, scene) == 4, (sides, res)
            with pytest.raises(LR.SceneError):
                p.ref.update_scene(scene)
            assert (p.r.debug_layouts("output_1", 0.0)[1], p.r.debug_image_nodes("output_1", 0.0)) == before   # as it was
            refused += 1
    assert accepted >= 2 and refused >= 5
    # 150.5 rounds to 151 wide; the height is the unrounded width over the integer ratio 640 / 360 = 1, 1, 0 and 3
    one_side = {"landscape": (151, 151), "square": (151, 151), "portrait": (151, LR.USIZE_MAX), "wide": (151, 50)}
    assert LR.resolution(p.ref.images["a"], 150.5, None) == one_side[asset]
    if asset == "portrait":
        assert LR.resolution(p.ref.images["a"], None, 60.5) == (0, 61)


@pytest.mark.parametrize("delays", [[100 * MS, 150 * MS, 0, 200 * MS, 100 * MS], [0, 0, 0], [40 * MS, 40 * MS], [1, 1, 1, 1]])
def test_frame_choice_over_a_period(delays):
    """1 ms steps over more than one period, from a start pts that is not zero: ties (the midpoint of two frames, frames
    with equal pts) go to the first frame, and a zero-delay animation has a 1 ns period"""
    p = host()
    p.register("g", pixels(8, 8, len(delays)), delays)
    p.update(V())
    p.check_state(0.25)                                                   # the last render: where the image starts
    p.update(V(children=[IMG(image_id="g")]))
    period_ms = max(1, sum(delays) // MS)
    seen = set()
    for k in range(0, period_ms * 2 + 3):
        nodes = p.check_state(0.25 + k / 1000.0)
        assert nodes[0][1] == 250 * MS
        seen.add(nodes[0][2])
    a = p.ref.images["g"]
    assert a.duration == (sum(delays) or 1)
    if sum(delays) >= MS:
        assert len(seen) > 1
    if delays[:3] == [100 * MS, 150 * MS, 0]:
        assert a.frame_pts == [0, 100 * MS, 250 * MS, 250 * MS, 450 * MS]
        assert a.frame_at(300 * MS, 250 * MS) == 0 and a.frame_at(301 * MS, 250 * MS) == 1      # the midpoint: the first
        assert a.frame_at(500 * MS, 250 * MS) == 2 and 3 not in seen                             # equal pts: the first
    # a pts before the start: the subtraction saturates
    assert p.r.debug_image_nodes("output_1", 0.1)[0][2] == 0


@pytest.mark.parametrize("mode", [orc.MODE_GPU_OPTIMIZED, orc.MODE_CPU_OPTIMIZED])
def test_image_oracle_at_equal_size_is_the_premultiply_oracle(mode):
    full = np.zeros((256, 256, 4), np.uint8)           # every colour byte against every alpha byte
    full[..., 0] = np.arange(256)[None, :]
    full[..., 1] = np.arange(256)[None, ::-1]
    full[..., 2] = (np.arange(256)[None, :] * 7) % 256
    full[..., 3] = np.arange(256)[:, None]
    for src in (full, pixels(37, 23, 1, 5)[0], pixels(1, 1, 1, 6)[0]):
        h, w = src.shape[:2]
        assert np.array_equal(c_oracles.render_image(src, w, h, mode), orc.add_premultiplied_alpha(src, mode))


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", sorted(SCENES))
def test_reference_scenes_match_oracle(name, mode, fmt):
    p = Pair(fmt=fmt, mode=mode, inputs=("input_1",))
    assert play(p, SCENES[name](), lambda pts: p.render_check(pts, name)) > 0


def _full_range(w, h):
    f = pixels(w, h, 1, 9)[0]
    f[0, :, 3] = np.arange(w) % 256
    f[:, 0, :3] = (np.arange(h) % 256)[:, None]
    return f


K_IMAGE_CASES = [((256, 256), (256, 256)), ((64, 48), (64, 48)), ((64, 48), (200, 131)), ((300, 200), (75, 50)),
                 ((120, 90), (37, 161)), ((1, 1), (33, 9)), ((17, 31), (31, 17)), ((33, 7), (1, 1)), ((5, 3), (640, 360))]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("src,dst", K_IMAGE_CASES)
def test_k_image_alone(src, dst, mode):
    """an Image root with an RGBA output is the node texture itself"""
    p = Pair(out=dst, fmt=RGBA, mode=mode)
    p.register("a", [_full_range(*src)])
    p.update(IMG(image_id="a", width=float(dst[0]), height=float(dst[1])))
    p.render_check(0.0, f"{src} -> {dst}")
    if src == dst:
        got = p.r.render(s.FrameSet(pts=0.04)).frames["output_1"]
        assert np.array_equal(np.asarray(got.data.planes[0]).reshape(dst[1], dst[0], 4), p.r.premultiply_rgba8(_full_range(*src)))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_animation_over_a_period(mode):
    p = Pair(mode=mode, inputs=("input_1",))
    p.register(*GIF1)
    p.update(V(background_color=s.RGBAColor(20, 30, 40, 255), children=[
        R(child=IN(input_id="input_1")),
        V(position=s.Position.Absolute(width=192.0, height=128.0, left=30.0, top=40.0), children=[IMG(image_id="image_gif1", width=192.0, height=128.0)])]))
    p.r.set_profiling(True)
    a = p.ref.images["image_gif1"]
    held, draws, launches = None, 0, {}
    for k in range(0, 24):
        pts = k * 0.05
        frame = a.frame_at(LR.LR.to_ns(pts), 0)
        n = p.render_check(pts, "animation")
        launches.setdefault(frame != held, set()).add(n)
        draws += frame != held
        held = frame
    assert draws >= 8 and p.r.kernel_times()["image"][1] == draws            # no image launch on ticks that keep the frame
    assert len(launches[True]) == 1 and len(launches[False]) == 1 and launches[True].pop() == launches[False].pop() + 1


@pytest.mark.gpu
def test_nodes_share_a_launch_and_an_asset_and_outlive_the_registry():
    p = Pair(inputs=("input_1",))
    p.register(*GIF1)
    p.register(*JPEG)
    cell = lambda x, y, w, h, child, **kw: V(position=s.Position.Absolute(width=float(w), height=float(h), left=float(x), top=float(y)),
                                              children=[child], **kw)
    p.update(V(children=[
        R(child=IN(input_id="input_1")),
        cell(10, 10, 96, 64, IMG(image_id="image_gif1")),                                        # 1:1
        cell(150, 20, 240, 160, IMG(image_id="image_gif1", width=240.0, height=160.0)),           # the same asset, scaled by k_image
        cell(400, 30, 200, 105, R(child=IMG(image_id="image_jpeg"))),                             # a resampled child
        cell(60, 200, 300, 140, IMG(image_id="image_jpeg", width=300.0, height=157.0),            # under a rounded mask
             border_radius=s.BorderRadius(30.0, 10.0, 40.0, 5.0), overflow=s.Overflow.Hidden)]))
    p.r.set_profiling(True)
    p.render_check(0.0, "four nodes")
    assert p.r.kernel_times()["image"][1] == 1                                # every node of the tick in one launch
    p.unregister("image_gif1")                                                # the scene keeps drawing the asset
    p.unregister("image_jpeg")
    for pts in (0.1, 0.3, 0.45):
        p.render_check(pts, "unregistered")
    assert _status(p.r, IMG(image_id="image_gif1")) == 4


class _Tick:
    """one smr_render_begin with host output planes that stay alive until its smr_render_end"""

    def __init__(self, r, pts, frames, out, fmt):
        self.keep = []
        self.in_arr = r._input_frames(s.FrameSet(frames=frames, pts=pts), self.keep)
        sizes = (C.c_size_t * 3)()
        F.lib().smr_output_plane_sizes(out[0], out[1], fmt, C.byref(sizes))
        self.planes = [np.zeros(sizes[p], np.uint8) if sizes[p] else None for p in range(3)]
        self.out_arr = (F.OutputFrame * 1)()
        self.out_arr[0].output_id = b"output_1"
        self.out_arr[0].mem_kind = F.MEM_HOST
        for p in range(3):
            if self.planes[p] is not None:
                self.out_arr[0].planes[p] = self.planes[p].ctypes.data
        r.render_raw(int(round(pts * 1e9)), self.in_arr, len(frames), self.out_arr, 1, wait=False)


@pytest.mark.gpu
def test_four_ticks_in_flight_over_an_animated_node():
    p = Pair(inputs=("input_1",))
    p.register(*GIF2)
    p.update(V(children=[R(child=IN(input_id="input_1")),
                         V(position=s.Position.Absolute(width=160.0, height=240.0, left=50.0, top=60.0),
                           children=[IMG(image_id="image_gif2", width=160.0, height=240.0)])]))
    pts_list = [0.0, 0.2, 0.5, 0.9, 1.0, 1.4, 1.45, 1.8]
    done = []
    for base in (0, 4):
        ticks = [(_Tick(p.r, pts, p.frames(pts), p.out, p.fmt), pts) for pts in pts_list[base:base + 4]]
        for _ in ticks:
            p.r.wait()
        done += ticks
    for t, pts in done:
        assert_identical([pl for pl in t.planes if pl is not None], p.expected(pts, p.frames(pts)), f"tick at {pts}")
