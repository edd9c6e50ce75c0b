"""Text components in the scene tree (smr_component.text): a caller-shaped glyph run is a leaf of the layout tree with a
static size, drawn once per scene update into its node texture and composited like any premultiplied RGBA8 child.

The reference's glyph pixels cannot be pinned here (glyphon is not in the tree), so every Text component is a stand-in
laid-out payload: the resolution is TextDimensions::Fixed when the scene gives one and (13 x len(text), line height)
otherwise (standing in for cosmic-text's measurement); the glyphs are seeded quads over one seeded mask / colour atlas.

CPU: the product's layouts (host-only handle) against the independent engine (tests/layout_ref_text.py), and the argument
checks of smr_update_scene.  GPU: output planes byte-identical to the oracle (orc.render_text for the node texture, then
the oracle's layout node), the once-per-update rendering, ticks in flight across a scene update, and Text roots.
"""
import ctypes as C

import numpy as np
import pytest

import smelter_b200 as s
from oracle import oracle as orc
from smelter_b200 import _ffi as F
from tests import harness
from tests import layout_ref_text as LR
from tests import ref_scene_rt as rt
from tests.golden import ref_scenes
from tests.parity import assert_identical, black, chroma_size, from_ref_layout, layouts_equal, node_texture, yuv_frame
from tests.test_layout_independent import diff, product_layouts, ref_layouts
from tests.test_text import MASK, COLOR, color_atlas, random_glyphs, soft_mask_atlas

MASK_ATLAS = soft_mask_atlas(256, 96, 31)      # shared by every label: one upload per scene
COLOR_ATLAS = color_atlas(128, 96, 32)
V, R, T, IN = s.ViewComponent, s.RescalerComponent, s.TilesComponent, s.InputStreamComponent


def label(w, h, seed, id=None, bg=(40, 40, 40, 200), n=None, contents=(MASK, COLOR), color_mode=0):
    g = random_glyphs(n if n is not None else max(4, w // 10), w, h, 128, 96, seed, contents=contents)
    return s.TextComponent(id=id, width=w, height=h, background_color=s.RGBAColor(*bg), glyphs=g, mask_atlas=MASK_ATLAS,
                           color_atlas=COLOR_ATLAS, color_mode=color_mode)


def stand_in_text(text="", font_size=None, line_height=None, color=None, background_color=None, dimensions=None,
                  id=None, **kw):
    """rt.TextComponent -> a stand-in laid-out payload"""
    if dimensions is not None and dimensions[0] == "fixed":
        w, h = int(dimensions[1]["width"]), int(dimensions[1]["height"])
    else:
        w, h = 13 * len(text), int(line_height or font_size or 0)
    seed = sum(map(ord, text)) + 7 * w + h
    c = label(w, h, seed, id=id, contents=(MASK,))
    if color is not None:
        c.glyphs["color"][:] = (color.r, color.g, color.b, color.a)
    if background_color is not None:
        c.background_color = background_color
    return c


@pytest.fixture
def text_catalogue(monkeypatch):
    """the re-typed scene catalogue with Text components replaced by stand-in payloads"""
    monkeypatch.setattr(rt, "TextComponent", stand_in_text)
    monkeypatch.setattr(rt.Component, "Text", staticmethod(lambda c: c))
    monkeypatch.setattr(rt.TextDimensions, "Fixed", staticmethod(lambda **kw: ("fixed", kw)))
    monkeypatch.setattr(rt.TextDimensions, "Fitted", staticmethod(lambda **kw: ("fitted", kw)))
    monkeypatch.setattr(rt.TextDimensions, "FittedColumn", staticmethod(lambda **kw: ("fitted_column", kw)))
    rec = rt.record(ref_scenes.MODULES["tiles"]["video_call_with_labels"])
    assert rec is not None
    return rec


# ---- scenes: (inputs {id: (w, h)}, output (w, h), steps [("update", scene) | ("snapshot", pts)]) --------------------
def _inputs(n, w=640, h=360):
    return {f"input_{i}": (w, h) for i in range(1, n + 1)}


def _one(scene, inputs=None, out=(640, 360)):
    return inputs if inputs is not None else _inputs(1), out, [("update", scene), ("snapshot", 0.0)]


def _transition():
    def scene(width, t):
        return V(background_color=s.RGBAColor(20, 20, 60, 255), children=[
            V(id="bar", position=s.Position.Static(width=width), transition=t, direction=s.ViewChildrenDirection.Column,
              children=[label(150, 30, 3), IN(input_id="input_1")]),
            label(90, 25, 4)])
    steps = [("update", scene(100.0, None)), ("update", scene(400.0, s.Transition(duration=10.0)))]
    steps += [("snapshot", p) for p in (0.0, 2.5, 5.0, 7.5, 10.0)]
    return _inputs(1), (640, 360), steps


SCENES = {
    "row_fit": lambda: _one(V(overflow=s.Overflow.Fit, children=[label(300, 40, 1), IN(input_id="input_1"), label(420, 60, 2)])),
    "row_hidden": lambda: _one(V(overflow=s.Overflow.Hidden, children=[label(300, 40, 1), IN(input_id="input_1"), label(420, 60, 2)])),
    "column_fit": lambda: _one(V(direction=s.ViewChildrenDirection.Column, overflow=s.Overflow.Fit,
                                 children=[label(200, 150, 5), IN(input_id="input_1"), label(100, 200, 6)])),
    "column_hidden": lambda: _one(V(direction=s.ViewChildrenDirection.Column, background_color=s.RGBAColor(9, 80, 9, 255),
                                    children=[label(200, 150, 5), label(700, 120, 6), IN(input_id="input_1")])),
    "rescaler_fit": lambda: _one(V(children=[R(mode=s.RescaleMode.Fit, child=label(220, 48, 7)), IN(input_id="input_1")])),
    "rescaler_fill": lambda: _one(V(children=[R(mode=s.RescaleMode.Fill, child=label(220, 48, 8)),
                                              R(child=IN(input_id="input_1"))])),
    "absolute_rotated": lambda: _one(V(background_color=s.RGBAColor(50, 50, 50, 255), children=[
        R(child=IN(input_id="input_1")),
        V(position=s.Position.Absolute(width=220.0, height=48.0, left=30.0, bottom=20.0), children=[label(220, 48, 9)]),
        V(position=s.Position.Absolute(width=160.0, height=40.0, right=40.5, top=60.0, rotation_degrees=30.0),
          children=[label(160, 40, 10)])])),
    "tiles": lambda: _one(T(margin=8.0, background_color=s.RGBAColor(30, 30, 30, 255),
                            children=[IN(input_id="input_1"), label(200, 60, 11), IN(input_id="input_2"), label(64, 64, 12)]),
                          inputs=_inputs(2)),
    "transition": _transition,
    "zero_size": lambda: _one(V(children=[label(0, 0, 13), R(child=label(0, 0, 14)), IN(input_id="input_1"),
                                          V(position=s.Position.Absolute(width=50.0, height=50.0, left=10.0, top=10.0),
                                            children=[label(0, 0, 15)])])),
}
TEXT_ROOT = label(200, 80, 16)


def leaves(comp):
    """the node children of a layout tree in DFS order (scene/layout.rs:95-103): InputStream and Text components"""
    if isinstance(comp, (s.InputStreamComponent, s.TextComponent)):
        return [comp]
    if isinstance(comp, s.RescalerComponent):
        return leaves(comp.child)
    return [x for c in comp.children for x in leaves(c)]


# ---- CPU ------------------------------------------------------------------------------------------------------------
def host_handle(inputs):
    r = s.Renderer(s.RendererOptions(cuda_device=-1))
    for i in inputs:
        r.register_input(i)
    return r


def check_layouts(inputs, out, steps):
    r = host_handle(inputs)
    ref = LR.StatefulScene(*out)
    snaps = 0
    for kind, arg in steps:
        if kind == "update":
            r.update_scene("output_1", s.Resolution(*out), s.OutputFrameFormat.PlanarYuv420Bytes, arg)
            ref.update_scene(arg)
            continue
        r.debug_set_inputs(arg, {k: s.Resolution(*v) for k, v in inputs.items()})
        got, root = product_layouts(r, arg)
        exp, exp_root = ref.layouts(arg, inputs)
        assert root == exp_root, f"pts {arg}: root {root} expected {exp_root}"
        d = diff(got, ref_layouts(exp))
        assert d is None, f"pts {arg}: {d}"
        snaps += 1
    return snaps


@pytest.mark.parametrize("name", sorted(SCENES))
def test_text_layouts_match_independent_engine(name):
    assert check_layouts(*SCENES[name]()) > 0


def test_video_call_with_labels_layouts(text_catalogue):
    rec = text_catalogue
    inputs = {i.name: (i.resolution.width, i.resolution.height) for i in rec.inputs}
    steps = [(k, a) for k, a in rec.steps if k in ("update", "snapshot")]
    assert check_layouts(inputs, (rec.resolution.width, rec.resolution.height), steps) == 1
    scene = [a for k, a in rec.steps if k == "update"][-1]
    assert sum(isinstance(c, s.TextComponent) for c in leaves(scene)) == 3


def test_text_children_are_node_children_with_static_size():
    """a Text is a node child (child_index counts it) whose size is known before any frame arrives"""
    r = host_handle(_inputs(1))
    scene = V(children=[label(300, 40, 1), IN(input_id="input_1"), label(120, 60, 2)])
    r.update_scene("output_1", s.Resolution(640, 360), s.OutputFrameFormat.PlanarYuv420Bytes, scene)
    got, _ = product_layouts(r, 0.0)          # no frame yet: the input is 0 x 0, the labels are not
    kids = [l for l in got if l["kind"] == "child"]
    assert [(l["index"], l["width"], l["height"]) for l in kids] == [(0, 300.0, 40.0), (2, 120.0, 60.0)]
    assert kids[1]["left"] == 300.0


def test_text_root_has_no_layouts():
    r = host_handle({})
    r.update_scene("output_1", s.Resolution(200, 80), s.OutputFrameFormat.PlanarYuv420Bytes, TEXT_ROOT)
    assert r.debug_layouts("output_1", 0.0) == ([], (0, 0))


def _status(r, scene):
    with pytest.raises(s.RendererError) as e:
        r.update_scene("output_1", s.Resolution(640, 360), s.OutputFrameFormat.PlanarYuv420Bytes, scene)
    return e.value.status


def test_text_payload_validation():
    r = host_handle(_inputs(1))
    ok = label(100, 20, 1)
    r.update_scene("output_1", s.Resolution(640, 360), s.OutputFrameFormat.PlanarYuv420Bytes, V(children=[ok]))
    bad = label(100, 20, 1)
    bad.glyphs["content"][2] = 7
    assert _status(r, V(children=[bad])) == 1
    no_color = label(100, 20, 1, contents=(COLOR,))
    no_color.color_atlas = None
    assert _status(r, V(children=[no_color])) == 1
    no_mask = label(100, 20, 1, contents=(MASK,))
    no_mask.mask_atlas = None
    assert _status(r, V(children=[no_mask])) == 1
    assert _status(r, V(children=[label(16385, 20, 1)])) == 1
    assert _status(r, label(20, 16385, 1, n=0)) == 1
    assert _status(r, V(id="a", children=[label(10, 10, 1, id="a")])) == 4          # duplicate id: SceneError
    # a Text without its payload (only a C caller can send one)
    c = F.Component()
    F.lib().smr_component_default(F.COMPONENT_TEXT, C.byref(c))
    assert not c.text
    assert F.lib().smr_update_scene(r._h, b"output_1", 640, 360, s.OutputFrameFormat.PlanarYuv420Bytes, C.byref(c)) == 1
    # 0 x 0 without glyphs or atlases is legal, colour glyphs need no mask atlas
    r.update_scene("output_1", s.Resolution(640, 360), s.OutputFrameFormat.PlanarYuv420Bytes,
                   V(children=[s.TextComponent(width=0, height=0), label(30, 30, 2, contents=(COLOR,))]))


@pytest.mark.parametrize("kind", [F.COMPONENT_SHADER, F.COMPONENT_WEB_VIEW, F.COMPONENT_IMAGE])
def test_other_components_stay_unsupported(kind):
    class Other:
        component_type = kind
    assert _status(host_handle({}), V(children=[Other()])) == 5


# ---- GPU ------------------------------------------------------------------------------------------------------------
def text_texture(c, mode):
    bg = c.background_color
    return orc.render_text(c.width, c.height, (bg.r, bg.g, bg.b, bg.a), c.glyphs, c.mask_atlas, c.color_atlas,
                           c.color_mode, mode)


def to_format(rgba, out, fmt):
    W, H = out
    if fmt == s.OutputFrameFormat.RgbaWgpuTexture:
        assert rgba.shape[:2] == (H, W)
        return (rgba,)
    if fmt == s.OutputFrameFormat.Nv12WgpuTexture:
        return orc.rgba_to_nv12_scaled(rgba, W, H)
    return orc.rgba_to_yuv_planar_scaled(rgba, W, H, *chroma_size(fmt, W, H))


def expected(scene, frames, out, fmt, mode, ref, pts, product=None):
    """the oracle's planes: node textures of the inputs (K1 / K2) and of the Text leaves (orc.render_text), composited
    with the independent engine's layouts (which the product's must equal)"""
    m = orc.MODE_GPU_OPTIMIZED if mode == s.RenderingMode.GpuOptimized else orc.MODE_CPU_OPTIMIZED
    if isinstance(scene, s.TextComponent):
        return to_format(text_texture(scene, m), out, fmt)
    res = {k: (f.resolution.width, f.resolution.height) for k, f in frames.items()}
    layouts, (rw, rh) = ref.layouts(pts, res)
    if product is not None:
        got, root = product.debug_layouts("output_1", pts)
        assert root == (rw, rh)
        d = layouts_equal(got, layouts)
        assert d is None, d
    if rw == 0 or rh == 0:
        return black(s.Resolution(*out), fmt)
    nodes = [text_texture(c, m) if isinstance(c, s.TextComponent) else node_texture(frames[c.input_id]) for c in leaves(scene)]
    rgba = orc.render_layout_node(rw, rh, [from_ref_layout(l) for l in layouts], nodes, mode=m, max_layouts=100)
    return to_format(rgba, out, fmt)


def frames_for(inputs, pts=0.0):
    return {k: yuv_frame(harness.test_input(i % 16 + 1, w, h), w, h, pts) for i, (k, (w, h)) in enumerate(sorted(inputs.items()))}


def run_steps(inputs, out, steps, fmt, mode):
    r = s.Renderer(s.RendererOptions(rendering_mode=mode))
    for i in inputs:
        r.register_input(i)
    ref = LR.StatefulScene(*out)
    scene = None
    n = 0
    for kind, arg in steps:
        if kind == "update":
            scene = arg
            r.update_scene("output_1", s.Resolution(*out), fmt, scene)
            ref.update_scene(scene)
            continue
        frames = frames_for(inputs, arg)
        got = r.render(s.FrameSet(frames=frames, pts=arg)).frames["output_1"]
        exp = expected(scene, frames, out, fmt, mode, ref, arg, product=r)
        assert_identical(tuple(np.asarray(p) for p in got.data.planes), exp, f"pts {arg}")
        n += 1
    return r, n


MODES = [s.RenderingMode.GpuOptimized, s.RenderingMode.CpuOptimized]
FORMATS = [s.OutputFrameFormat.PlanarYuv420Bytes, s.OutputFrameFormat.Nv12WgpuTexture, s.OutputFrameFormat.RgbaWgpuTexture]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", sorted(SCENES))
def test_text_scenes_match_oracle(name, mode, fmt):
    assert run_steps(*SCENES[name](), fmt, mode)[1] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("mode", MODES)
def test_video_call_with_labels_matches_oracle(text_catalogue, mode, fmt):
    rec = text_catalogue
    inputs = {i.name: (i.resolution.width, i.resolution.height) for i in rec.inputs}
    steps = [(k, a) for k, a in rec.steps if k in ("update", "snapshot")]
    assert run_steps(inputs, (rec.resolution.width, rec.resolution.height), steps, fmt, mode)[1] == 1


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", [s.OutputFrameFormat.PlanarYuv420Bytes, s.OutputFrameFormat.Nv12WgpuTexture])
@pytest.mark.parametrize("mode", MODES)
def test_label_over_a_4to1_child_beside_direct_tiles(mode, fmt):
    """cfg3's shape: 1920 x 1080 inputs shown 4:1 in a grid, whose 1:1 interiors the fused resample writes directly; a
    label overlaps one child, so the tiles under it go through the composite"""
    inputs = _inputs(4, 1920, 1080)
    cells = [V(position=s.Position.Absolute(width=480.0, height=270.0, left=480.0 * (i % 2), top=270.0 * (i // 2)),
               children=[R(child=IN(input_id=f"input_{i + 1}"))]) for i in range(4)]
    over = V(position=s.Position.Absolute(width=220.0, height=48.0, left=100.0, top=240.0), children=[label(220, 48, 40)])
    r, _ = run_steps(inputs, (960, 540), [("update", V(children=cells + [over])), ("snapshot", 0.0)], fmt, mode)
    if mode == s.RenderingMode.GpuOptimized:
        assert r.stats()["last_render_direct_tiles"] > 0


def _render(r, frames, pts=0.0):
    r.render(s.FrameSet(frames=frames, pts=pts))
    return r.stats()["last_render_kernel_launches"]


@pytest.mark.gpu
def test_text_is_drawn_once_per_scene_update():
    r = s.Renderer()
    scene = lambda seed: V(background_color=s.RGBAColor(10, 10, 10, 255), children=[label(200, 40, seed), label(120, 40, seed + 1)])
    fmt = s.OutputFrameFormat.PlanarYuv420Bytes
    r.update_scene("output_1", s.Resolution(640, 360), fmt, scene(1))
    r.set_profiling(True)
    first, second = _render(r, {}), _render(r, {})
    assert first == second + 1
    assert r.kernel_times()["convert"][1] == 1          # the text launch, both nodes; none in the second tick
    r.update_scene("output_1", s.Resolution(640, 360), fmt, scene(5))
    assert _render(r, {}) == second + 1 and _render(r, {}) == second
    # two outputs updated before the same tick: one launch draws the text nodes of both
    r.update_scene("output_2", s.Resolution(320, 180), fmt, scene(9))
    r.update_scene("output_1", s.Resolution(640, 360), fmt, scene(12))
    r.set_profiling(True)
    both, after = _render(r, {}), _render(r, {})
    assert both == after + 1 and r.kernel_times()["convert"][1] == 1


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
        r.render_raw(int(pts * 1e9), self.in_arr, len(frames), self.out_arr, 1, wait=False)


@pytest.mark.gpu
def test_ticks_in_flight_keep_the_scene_they_were_submitted_with():
    inputs, out, fmt = _inputs(1), (640, 360), s.OutputFrameFormat.PlanarYuv420Bytes
    scenes = [V(children=[R(child=IN(input_id="input_1")),
                          V(position=s.Position.Absolute(width=300.0, height=60.0, left=20.0, top=30.0),
                            children=[label(300, 60, seed, bg=(200, 20, 20, 180))]), label(90 + seed, 30, seed + 1)])
              for seed in (21, 57)]
    r = s.Renderer()
    r.register_input("input_1")
    refs = []
    ticks = []
    for k, scene in enumerate(scenes):
        r.update_scene("output_1", s.Resolution(*out), fmt, scene)
        ref = LR.StatefulScene(*out)
        ref.update_scene(scene)
        for j in range(3 if k == 0 else 2):
            pts = 0.04 * len(ticks)
            ticks.append((_Tick(r, pts, frames_for(inputs, pts), out, fmt), scene, ref, pts))
    for _ in ticks:
        r.wait()
    for t, scene, ref, pts in ticks:
        exp = expected(scene, frames_for(inputs, pts), out, fmt, s.RenderingMode.GpuOptimized, ref, pts)
        assert_identical([p for p in t.planes if p is not None], exp, f"tick at {pts}")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_text_root(mode):
    r = s.Renderer(s.RendererOptions(rendering_mode=mode))
    for fmt, out in ((s.OutputFrameFormat.PlanarYuv420Bytes, (640, 360)), (s.OutputFrameFormat.PlanarYuv420Bytes, (200, 80)),
                     (s.OutputFrameFormat.Nv12WgpuTexture, (320, 180)), (s.OutputFrameFormat.RgbaWgpuTexture, (200, 80))):
        r.update_scene("output_1", s.Resolution(*out), fmt, TEXT_ROOT)
        got = r.render(s.FrameSet(pts=0.0)).frames["output_1"]
        assert_identical(tuple(np.asarray(p) for p in got.data.planes), expected(TEXT_ROOT, {}, out, fmt, mode, None, 0.0),
                         f"text root {out} format {fmt}")
    r.update_scene("output_1", s.Resolution(640, 360), s.OutputFrameFormat.RgbaWgpuTexture, TEXT_ROOT)
    with pytest.raises(s.RenderSceneError) as e:
        r.render(s.FrameSet(pts=0.0))
    assert e.value.status == 5
