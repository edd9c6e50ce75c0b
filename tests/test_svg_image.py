"""SVG image assets (smr_register_svg_image): the caller rasterises at each node's resolution during smr_update_scene, and
k_image converts the raster into the node texture (svg_image.rs: two passes in GpuOptimized, the bytes as they are in
CpuOptimized).

There is no resvg here: the rasteriser is a stand-in (tests/svg_standin.py) drawing two shapes of the reference's
integration-tests/assets/image.svg, whose intrinsic size is 666 x 524.  svg_as_root and svg_in_view are the two SVG
scenes of integration-tests/src/render_tests/image.rs.

CPU (host-only handle): the registry and argument errors, layouts and image node state against the independent engine
(the SVG registered there as a one-frame asset of its intrinsic size), when and with what the rasteriser is called, and
the oracle's arithmetic.  GPU: every output byte against the oracle (tests/svg_oracle.c: orc_render_svg for the node
texture, then the layout, shader and web oracles).
"""
import ctypes as C

import numpy as np
import pytest

import smelter_b200 as s
from smelter_b200 import _ffi as F
from tests import layout_ref_image as LI
from tests import c_oracles
from tests import svg_standin
from tests import test_shader_component as TS
from tests import test_web_view_component as TW
from tests import test_web_view_layout_children as TWL
from tests.test_image_component import _Tick, pixels
from tests.test_layout_independent import product_layouts

V, R, IN, IMG, SH = s.ViewComponent, s.RescalerComponent, s.InputStreamComponent, s.ImageComponent, s.ShaderComponent
YUV, RGBA = TW.YUV, TW.RGBA
web, cell, sized = TW.web, TW.cell, TWL.sized
SVG = "image_svg"
MS = 1_000_000


class Asset:
    """what the resolution rule reads of an asset (LI.resolution); kept after an unregister for the scenes still showing it"""

    def __init__(self, w, h):
        self.width, self.height = w, h


class Pair(TWL.Pair):
    """the renderer and the independent engine with SVG assets: each SVG asset is a rasteriser of (w, h), and a log of the
    (image id, w, h) it was called with"""

    def __init__(self, **kw):
        super().__init__(**kw)
        self.svg, self.calls = {}, []

    def register_svg(self, image_id=SVG, size=svg_standin.SIZE, fn=svg_standin.rasterize):
        def rasterize(w, h):
            self.calls.append((image_id, w, h))
            return fn(w, h)
        self.r.register_svg_image(image_id, size[0], size[1], rasterize)
        self.ref.register_image(image_id, size[0], size[1], [0])
        self.svg[image_id] = (Asset(*size), fn)

    def unregister(self, image_id):
        self.r.unregister_image(image_id)
        self.ref.unregister_image(image_id)

    def check_state(self, pts):
        """root layouts, every layout node's, and every image node's resolution, start pts and frame"""
        self.check_layouts(pts)
        self.check_node_layouts(pts)
        nodes = [(res, start, 0) for _, _, start, res in self.ref.image_nodes()]
        assert self.r.debug_image_nodes("output_1", pts) == nodes
        return nodes

    def leaf_texture(self, c, frames, live, pts=0.0):
        if isinstance(c, IMG) and c.image_id in self.svg:
            asset, fn = self.svg[c.image_id]
            w, h = LI.resolution(asset, c.width, c.height)
            return c_oracles.render_svg(fn(w, h), self.m)
        return super().leaf_texture(c, frames, live, pts)

    def expected(self, pts, frames, stale=()):
        if isinstance(self.scene, IMG):
            self.ref.layouts(pts, {})
            return TW.to_format(self.leaf_texture(self.scene, frames, set(frames), pts), self.out, self.fmt)
        return super().expected(pts, frames, stale)

    def launches(self):
        return self.r.stats()["last_render_kernel_launches"]


def host(**kw):
    return Pair(device=-1, **kw)


def _status(r, scene):
    with pytest.raises(s.RendererError) as e:
        r.update_scene("output_1", s.Resolution(640, 360), YUV, scene)
    return e.value.status


def _state(p):
    return product_layouts(p.r, 0.0), p.r.debug_image_nodes("output_1", 0.0)


# the reference's two SVG scenes, and sized variants of the view one: (scene, the node's resolution or None if refused)
PORTRAIT = (524, 666)      # the landscape asset on its side: the integer aspect ratio 524 / 666 is 0
SCENES = {
    "svg_as_root": (lambda: IMG(image_id=SVG), (666, 524)),
    "svg_in_view": (lambda: V(children=[IMG(image_id=SVG)]), (666, 524)),
    "width_only": (lambda: V(children=[IMG(image_id=SVG, width=300.4)]), (300, 300)),    # 666 / 524 = 1: a square
    "height_only": (lambda: V(children=[IMG(image_id=SVG, height=120.5)]), (121, 121)),
    "both_sides": (lambda: V(children=[IMG(image_id=SVG, width=333.0, height=400.6)]), (333, 401)),
    "root_both_sides": (lambda: IMG(image_id=SVG, width=99.5, height=77.2), (100, 77)),
}


def root_size(p, scene):
    """an RGBA output of an Image root has the node's size (render_loop.rs:81-103)"""
    if isinstance(scene, IMG) and p.fmt == RGBA:
        asset, _ = p.svg[scene.image_id]
        return LI.resolution(asset, scene.width, scene.height)
    return (640, 360)


# ---- CPU ------------------------------------------------------------------------------------------------------------
def _raw(r, image_id, w, h, fn):
    return F.lib().smr_register_svg_image(r._h, image_id, C.byref(F.SvgSpec(w, h, fn, None)))


def test_registry_and_argument_errors():
    p = host()
    r = p.r
    ok = F.SVG_RASTERIZE_FN(lambda user, w, h, rgba, pitch: 0)
    shown = lambda i: F.lib().smr_update_scene(r._h, b"output_1", 64, 64, YUV, C.byref(_image_c(i)))
    for w, h, fn in ((0, 10, ok), (10, 0, ok), (16385, 10, ok), (10, 16385, ok), (10, 10, F.SVG_RASTERIZE_FN())):
        assert _raw(r, b"x", w, h, fn) == 1, (w, h)
        assert shown(b"x") == 4                                    # a failed call registers nothing
    assert _raw(r, None, 10, 10, ok) == 1
    assert F.lib().smr_register_svg_image(r._h, b"x", None) == 1
    assert _raw(r, b"x", 16384, 16384, ok) == 0
    assert _raw(r, b"x", 10, 10, ok) == 1                          # KeyTaken, SVG over SVG
    r.register_image("bitmap", pixels(8, 4, 1)[0])
    assert _raw(r, b"bitmap", 10, 10, ok) == 1                     # ... SVG over bitmap
    with pytest.raises(s.RendererError) as e:                      # ... bitmap over SVG
        r.register_image("x", pixels(8, 4, 1)[0])
    assert e.value.status == 1
    assert F.lib().smr_unregister_image(r._h, b"x") == 0 and F.lib().smr_unregister_image(r._h, b"x") == 1
    assert shown(b"x") == 4
    assert _raw(r, b"x", 10, 10, ok) == 0 and shown(b"x") == 0     # the id is free again


def _image_c(image_id):
    c = F.Component()
    F.lib().smr_component_default(F.COMPONENT_IMAGE, C.byref(c))
    c.image_id = image_id
    return c


def test_reregistration_makes_a_new_asset():
    """a component with an id keeps its start pts across updates while the asset is the same object; re-registering the
    id makes a new asset, and the node restarts at the last render's pts"""
    p = host()
    p.register_svg()
    scene = lambda: V(children=[IMG(id="s", image_id=SVG, width=100.0)])
    p.update(V())
    p.check_state(0.25)
    p.update(scene())
    assert p.check_state(0.5)[0][:2] == ((100, 100), 250 * MS)
    p.update(scene())
    assert p.check_state(0.75)[0][:2] == ((100, 100), 250 * MS)
    p.unregister(SVG)
    p.register_svg()
    p.update(scene())
    assert p.check_state(1.0)[0][:2] == ((100, 100), 750 * MS)


@pytest.mark.parametrize("name", sorted(SCENES))
def test_scenes_layouts_and_state(name):
    p = host(inputs=("input_1",))
    p.register_svg()
    scene, res = SCENES[name]
    p.update(scene())
    assert p.check_state(0.0) == [(res, 0, 0)]
    assert p.calls == [(SVG, *res)]
    p.check_state(0.5)
    assert len(p.calls) == 1                                       # rendering does not rasterise


@pytest.mark.parametrize("sides", [(200.0, None), (None, 90.0)])
def test_portrait_asset_with_one_side_is_refused(sides):
    """the integer aspect ratio of a portrait asset is 0: one side given divides by it (width only) or multiplies by it
    (height only), and either way a side leaves the texture range"""
    p = host()
    p.register_svg("portrait", size=PORTRAIT)
    p.update(V(children=[IMG(image_id="portrait", width=50.0, height=60.0)]))
    before, calls = _state(p), list(p.calls)
    scene = V(children=[IMG(image_id="portrait", width=sides[0], height=sides[1])])
    assert _status(p.r, scene) == 4
    with pytest.raises(LI.SceneError):
        p.ref.update_scene(scene)
    assert _state(p) == before and p.calls == calls
    assert LI.resolution(Asset(*PORTRAIT), *sides) in ((200, LI.USIZE_MAX), (0, 90))


def test_rasteriser_arguments():
    """once per SVG node per update, at the node's resolution, pitch 4 * width, into a zeroed buffer"""
    p = host()
    log = []

    def raw(user, w, h, rgba, pitch):
        buf = np.ctypeslib.as_array(rgba, shape=(h * pitch,))
        log.append((w, h, pitch, not buf.any()))
        buf[:] = 0x7f
        return 0
    fn = F.SVG_RASTERIZE_FN(raw)
    assert _raw(p.r, SVG.encode(), 666, 524, fn) == 0
    p.ref.register_image(SVG, 666, 524, [0])
    scene = V(children=[IMG(image_id=SVG), IMG(image_id=SVG, width=31.0, height=7.0), V(children=[IMG(image_id=SVG, height=3.0)])])
    p.update(scene)
    assert log == [(666, 524, 666 * 4, True), (31, 7, 31 * 4, True), (3, 3, 12, True)]
    p.update(scene)                                                # every update rasterises again
    assert len(log) == 6 and log[3:] == log[:3]
    p.check_state(0.0)


def test_refused_scenes_never_rasterise():
    p = host(inputs=("input_1",))
    p.register_svg()
    TWL._register(p)
    p.update(V(children=[IN(input_id="input_1"), IMG(image_id=SVG, width=64.0)]))
    before = _state(p)
    svg = lambda **kw: IMG(image_id=SVG, **kw)
    refused = [V(children=[svg(id="a"), svg(id="a")]),                                   # duplicate ids
               V(children=[svg(), IMG(image_id="missing")]),                              # ImageNotFound
               V(children=[svg(), svg(width=0.2)]),                                       # a node of 0 x 0
               V(children=[svg(), svg(width=17000.0, height=10.0)]),                      # above 16384
               V(children=[svg(), SH(shader_id="missing", width=8, height=8)]),           # ShaderNotFound
               SH(shader_id="gradient", width=8, height=8, children=[V(children=[svg()])]),   # a sizeless layout root
               V(children=[svg(), web("missing")]),                                       # WebRendererNotFound
               web(children=[svg()])]                                                     # WebViewChildWithoutId
    n = len(p.calls)
    for scene in refused:
        assert _status(p.r, scene) == 4, scene
        assert _state(p) == before and len(p.calls) == n, scene


@pytest.mark.parametrize("failure", ["status", "exception", "shape", "dtype"])
def test_rasteriser_failure_refuses_the_update(failure):
    p = host(inputs=("input_1",))
    bad = {"status": None, "exception": lambda w, h: 1 // 0, "shape": lambda w, h: np.zeros((h + 1, w, 4), np.uint8),
           "dtype": lambda w, h: np.zeros((h, w, 4), np.float32)}[failure]
    p.register_svg()
    p.register_svg("bad", fn=bad or svg_standin.rasterize)
    if failure == "status":     # the C rasteriser's own non-zero status
        p.r.unregister_image("bad")
        refuse = F.SVG_RASTERIZE_FN(lambda user, w, h, rgba, pitch: 3)   # alive while registered
        assert _raw(p.r, b"bad", 666, 524, refuse) == 0
    p.update(V(children=[IN(input_id="input_1"), IMG(id="s", image_id=SVG, width=128.0)]))
    p.check_state(0.5)
    before = _state(p)
    with pytest.raises(s.RendererError) as e:
        p.r.update_scene("output_1", s.Resolution(640, 360), YUV, V(children=[IMG(image_id=SVG), IMG(image_id="bad", height=48.0)]))
    assert e.value.status == 4 and '"bad"' in str(e.value) and "48 x 48" in str(e.value)
    assert _state(p) == before
    p.check_state(0.5)


def test_nodes_under_shaders_webs_and_layout_nodes_are_rasterised():
    p = host(inputs=("input_1",))
    p.register_svg()
    TWL._register(p)
    p.update(V(children=[
        SH(shader_id="grade", shader_param=TS.grade(), width=320, height=180, children=[IMG(image_id=SVG, width=64.0)]),
        web(children=[IMG(id="w", image_id=SVG, height=50.0), V(id="v", position=sized(320, 180), children=[
            IMG(image_id=SVG, width=20.0, height=30.0)])]),
        SH(shader_id="bands", width=200, height=100, children=[V(position=sized(200, 100), children=[IMG(image_id=SVG, width=10.0)])])]))
    assert sorted(c[1:] for c in p.calls) == sorted([(64, 64), (50, 50), (20, 30), (10, 10)])
    assert len(p.r.debug_image_nodes("output_1", 0.0)) == 4
    p.check_layouts(0.0)
    p.check_node_layouts(0.0)


def test_unregister_keeps_the_scene_and_stops_the_rasteriser():
    p = host(inputs=("input_1",))
    p.register_svg()
    p.update(V(children=[IN(input_id="input_1"), IMG(image_id=SVG, width=64.0)]))
    before, n = _state(p), len(p.calls)
    p.unregister(SVG)
    assert _state(p) == before
    assert _status(p.r, V(children=[IMG(image_id=SVG)])) == 4       # ImageNotFound
    assert len(p.calls) == n and SVG not in p.r._svg_rasterizers


def test_oracle_conversion():
    """the oracle's two passes: an opaque raster comes back as it is (division by 1, then sRGB decode and encode), a
    transparent pixel stays 0, and the sampled taps of a texture of the target's size are its own texels at every size
    the renderer accepts, which is what lets k_image take pass 1's bytes as pass 2's texel"""
    opaque = svg_standin.rasterize(40, 30)
    opaque[..., 3] = 255
    assert np.array_equal(c_oracles.render_svg(opaque, 0), opaque)
    raster = svg_standin.rasterize(67, 52)
    assert np.array_equal(c_oracles.render_svg(raster, 1), raster)
    got = c_oracles.render_svg(raster, 0)
    assert np.array_equal(got[..., 3], raster[..., 3]) and not got[raster[..., 3] == 0].any()
    assert c_oracles.same_size_taps_off_texel(16384) == 0


def test_standin_draws_partial_coverage_at_scale():
    a, b = svg_standin.rasterize(666, 524), svg_standin.rasterize(333, 262)
    for x in (a, b):
        assert (x[..., :3] <= x[..., 3:]).all()                                # premultiplied
        assert len(np.unique(x.reshape(-1, 4), axis=0)) > 8                     # the sun's edge blends into the sky
    assert ((a[..., 3] > 0) & (a[..., 3] < 255)).any()                        # the sky's edge is translucent at 1:1
    assert np.array_equal(a, svg_standin.rasterize(666, 524))


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _full_range():
    """every (colour byte, alpha byte) pair: colour > alpha, alpha 0 with colour, and the premultiplied ones"""
    f = np.zeros((256, 256, 4), np.uint8)
    f[..., 0] = np.arange(256)[None, :]
    f[..., 1] = np.arange(256)[None, ::-1]
    f[..., 2] = (np.arange(256)[None, :] * 7) % 256
    f[..., 3] = np.arange(256)[:, None]
    return f


@pytest.mark.gpu
@pytest.mark.parametrize("mode", TW.MODES)
def test_exhaustive_conversion(mode):
    full = _full_range()
    p = Pair(out=(256, 256), fmt=RGBA, mode=mode)
    p.register_svg("full", size=(256, 256), fn=lambda w, h: full)
    p.update(IMG(image_id="full"))
    got = np.asarray(p.r.render(s.FrameSet(pts=0.0)).frames["output_1"].data.planes[0]).reshape(256, 256, 4)
    exp = c_oracles.render_svg(full, p.m)
    assert np.array_equal(got, exp), np.argwhere(np.any(got != exp, axis=-1))[:8]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", TW.FORMATS)
@pytest.mark.parametrize("mode", TW.MODES)
@pytest.mark.parametrize("name", sorted(SCENES))
def test_scenes_match_oracle(name, mode, fmt):
    p = Pair(fmt=fmt, mode=mode, inputs=("input_1",))
    p.register_svg()
    scene = SCENES[name][0]()
    p.update(scene, out=root_size(p, scene))
    p.render_check(0.0, name)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", TW.MODES)
def test_resize_rerasterises_and_later_ticks_launch_nothing_for_it(mode):
    p = Pair(mode=mode, inputs=("input_1",))
    p.register_svg()
    scene = lambda w: V(background_color=s.RGBAColor(20, 30, 40, 255), children=[
        R(child=IN(input_id="input_1")), cell(40, 30, 300, 240, IMG(id="s", image_id=SVG, width=w))])
    p.update(scene(200.0))
    p.render_check(0.0, "first")
    first = p.launches()
    p.render_check(0.04, "second")
    assert p.launches() == first - 1                       # the node texture already holds the raster
    p.update(scene(271.0))
    assert p.calls[-1] == (SVG, 271, 271)
    p.render_check(0.08, "resized")
    assert p.launches() == first
    p.render_check(0.12, "resized, again")
    assert p.launches() == first - 1


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", TW.FORMATS)
@pytest.mark.parametrize("mode", TW.MODES)
def test_under_shader_web_and_layout_node(mode, fmt):
    p = Pair(fmt=fmt, mode=mode, inputs=("input_1",))
    p.register_svg()
    for k in TS.SOURCES:
        p.register_shader(k)
    p.register_web("page", 640, 360, TW.OVER)
    p.update(V(background_color=s.RGBAColor(10, 20, 30, 255), children=[
        cell(0, 0, 320, 180, SH(shader_id="grade", shader_param=TS.grade(), width=320, height=180,
                                children=[IMG(image_id=SVG, width=320.0, height=180.0)])),
        cell(320, 0, 320, 180, R(child=web(children=[IMG(id="w", image_id=SVG, height=150.0),
                                                    V(id="v", position=sized(300, 200), background_color=s.RGBAColor(0, 0, 90, 255),
                                                      children=[IMG(image_id=SVG, width=150.0, height=97.0)])]))),
        cell(0, 180, 640, 180, R(child=IN(input_id="input_1")))]))
    p.set_frame("page", TW.page(640, 360, 3))
    p.set_rects("page", [(20.5, 10, 150, 150), (300, 100.25, 300, 200)])
    p.render_check(0.0, "nested")
    p.render_check(0.04, "nested, again")


@pytest.mark.gpu
def test_ticks_in_flight_across_an_update():
    """three ticks submitted under one SVG node, the scene replaced by a node of another size, one more tick: each output
    is that of the scene it was submitted under"""
    p = Pair(inputs=("input_1",))
    p.register_svg()
    scene = lambda w: V(children=[R(child=IN(input_id="input_1")), cell(60, 40, 300, 240, IMG(image_id=SVG, width=w))])
    p.update(scene(180.0))
    ticks = []
    for pts in (0.0, 0.04, 0.08):
        ticks.append((_Tick(p.r, pts, p.frames(pts), p.out, p.fmt), p.expected(pts, p.frames(pts)), pts))
    p.update(scene(250.0))
    ticks.append((_Tick(p.r, 0.12, p.frames(0.12), p.out, p.fmt), p.expected(0.12, p.frames(0.12)), 0.12))
    for _ in ticks:
        p.r.wait()
    for t, exp, pts in ticks:
        TW.assert_identical([pl for pl in t.planes if pl is not None], exp, f"tick at {pts}")
