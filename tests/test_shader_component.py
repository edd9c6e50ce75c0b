"""Shader components (smr_register_shader, smr_unregister_shader, smr_component.shader_id / shader_param / size).

A shader here is CUDA C++ compiled by NVRTC at registration.  The test shaders use only operations IEEE 754 rounds exactly
(+ - * /, sqrtf, fminf / fmaxf, floorf, fmaf), so the same sources compiled for the CPU against
tests/shader_oracle_shim.h pin every byte; shaders that call transcendentals are not pinned bit for bit.  There are no
reference snapshots of CUDA shaders: parity with the reference rests on the shared contract (NC-6 sampling, one
PREMULTIPLIED_ALPHA_BLENDING pass with an 8-bit store per plane, BaseShaderParameters).

CPU (host-only handle): layouts against the independent engine (tests/layout_ref_shader.py), the registry, the compile
errors and the scene refusals.  GPU: every output byte against the oracle, both rendering modes and three output formats.
"""
import ctypes as C
import json
import os
import struct

import numpy as np
import pytest

import bench
import smelter_b200 as s
from smelter_b200 import _ffi as F
from tests import layout_ref_shader as LS
from tests import oracle_shader
from tests import test_web_view_component as TW
from tests.test_gpu_bench_scenes import bench_frames
from tests.test_image_component import pixels
from tests.parity import run_case
from tests.test_layout_independent import diff, product_layouts, ref_layouts
from tests.test_text_component import label

V, R, T, IN, IMG, WEB, SH = (s.ViewComponent, s.RescalerComponent, s.TilesComponent, s.InputStreamComponent, s.ImageComponent,
                             s.WebViewComponent, s.ShaderComponent)
P, PT = s.ShaderParam, s.ShaderParamType
YUV, NV12, RGBA = TW.YUV, TW.NV12, TW.RGBA

# a colour grade of child 0: gain per channel, then lift scaled by alpha (stays premultiplied), clamped to alpha
GRADE = r'''
struct Grade { float gain[3]; float lift; };
__device__ float4 smr_fragment(smr_fragment_in in, const smr_base_params &base, const void *params, const smr_textures &tex) {
    const Grade &g = *(const Grade *)params;
    float4 c = tex.sample(0, in.tex_coords);
    float r = fminf(fmaf(c.x, g.gain[0], g.lift * c.w), c.w);
    float gg = fminf(fmaf(c.y, g.gain[1], g.lift * c.w), c.w);
    float b = fminf(fmaf(c.z, g.gain[2], g.lift * c.w), c.w);
    return make_float4(r, gg, b, c.w);
}
'''
GRADE_TYPE = PT("struct", fields=[("gain", PT("list", item=PT("f32"), length=3)), ("lift", PT("f32"))])


def grade(gain=(1.25, 0.75, 1.0), lift=0.0625):
    return P.struct([("gain", P.list([P.f32(g) for g in gain])), ("lift", P.f32(lift))])


# a wipe between children 0 and 1: plane 0 draws child 0, plane 1 child 1 left of an edge that moves with time
WIPE = r'''
struct Wipe { float speed; float softness; unsigned flip; };
__device__ float4 smr_fragment(smr_fragment_in in, const smr_base_params &base, const void *params, const smr_textures &tex) {
    const Wipe &w = *(const Wipe *)params;
    float4 c = tex.sample((unsigned)base.plane_id, in.tex_coords);
    if (base.plane_id == 0) return c;
    float x = w.flip ? 1.0f - in.tex_coords.x : in.tex_coords.x;
    float edge = base.time * w.speed - floorf(base.time * w.speed);
    float k = fminf(fmaxf((edge - x) / w.softness, 0.0f), 1.0f);
    return make_float4(c.x * k, c.y * k, c.z * k, c.w * k);
}
'''
WIPE_TYPE = PT("struct", fields=[("speed", PT("f32")), ("softness", PT("f32")), ("flip", PT("u32"))])


def wipe(speed=0.5, softness=0.125, flip=0):
    return P.struct([("speed", P.f32(speed)), ("softness", P.f32(softness)), ("flip", P.u32(flip))])


# no children: a radial gradient from position, output_resolution and plane_id (-1)
GRADIENT = r'''
__device__ float4 smr_fragment(smr_fragment_in in, const smr_base_params &base, const void *params, const smr_textures &tex) {
    float dx = in.position.x - 0.5f * (float)base.output_resolution[0];
    float dy = in.position.y - 0.5f * (float)base.output_resolution[1];
    float d = sqrtf(dx * dx + dy * dy) / (float)base.output_resolution[1];
    float a = base.plane_id == -1 && base.texture_count == 0 ? fminf(fmaxf(1.0f - d, 0.0f), 1.0f) : 0.0f;
    return make_float4(a * in.tex_coords.x, a * 0.5f, a * in.tex_coords.y, a);
}
'''

# every child at once, each in its own vertical band: plane p draws child p into band p
BANDS = r'''
__device__ float4 smr_fragment(smr_fragment_in in, const smr_base_params &base, const void *params, const smr_textures &tex) {
    float n = (float)base.texture_count;
    float band = floorf(in.tex_coords.x * n);
    if (band != (float)base.plane_id) return make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    float2 uv = make_float2(in.tex_coords.x * n - band, in.tex_coords.y);
    return tex.sample((unsigned)base.plane_id, uv);
}
'''

SOURCES = {"grade": (GRADE, GRADE_TYPE), "wipe": (WIPE, WIPE_TYPE), "gradient": (GRADIENT, None), "bands": (BANDS, None)}


def param_bytes(p):
    """ShaderParam::to_bytes: the scalars, little-endian, tightly concatenated"""
    if p is None:
        return b""
    if p.kind in ("f32", "u32", "i32"):
        return struct.pack({"f32": "<f", "u32": "<I", "i32": "<i"}[p.kind], p.value)
    return b"".join(param_bytes(v if p.kind == "list" else v[1]) for v in p.value)


class Pair(TW.Pair):
    """the web test's renderer / independent engine pair, with shader nodes"""

    def __init__(self, **kw):
        super().__init__(**kw)
        self.ref = LS.StatefulScene(*self.out)
        self.sources = {}

    def register_shader(self, shader_id, name=None):
        src, ty = SOURCES[name or shader_id]
        self.r.register_shader(shader_id, src, ty)
        self.ref.register_shader(shader_id, ty)
        self.sources[shader_id] = src

    def update(self, scene, out=None):
        super().update(scene, out)
        # the layout nodes below the root, by component (render graph order, as smr_debug_node_layouts numbers them)
        self.nested = {id(n.comp): k for k, n in enumerate(LS.render_nodes(self.ref.render_tree))}

    def node_index(self, k):
        """smr_debug_node_layouts' index of layout node k below the root"""
        return k + (0 if self.ref.render_tree.kind in LS.LEAVES else 1)

    def check_node_layouts(self, pts):
        self.r.debug_set_inputs(pts, {k: s.Resolution(*v) for k, v in self.inputs.items()})
        for k in range(len(self.nested)):
            got, root = self.r.debug_node_layouts("output_1", self.node_index(k), pts)
            exp, exp_root = self.ref.node_layouts(k, pts, self.inputs)
            assert root == exp_root, f"node {k} pts {pts}: root {root} expected {exp_root}"
            d = diff(product_layouts(_Node(self.r, self.node_index(k)), pts)[0], ref_layouts(exp))
            assert d is None, f"node {k} pts {pts}: {d}"

    def leaf_texture(self, c, frames, live, pts=0.0):
        if id(c) in self.nested:   # a layout node below the root: its layouts composited into its own texture
            res = {k: (f.resolution.width, f.resolution.height) for k, f in frames.items() if k in live}
            k = self.nested[id(c)]
            got, root = self.r.debug_node_layouts("output_1", self.node_index(k), pts)
            layouts, (rw, rh) = self.ref.node_layouts(k, pts, res)
            assert root == (rw, rh) and TW.layouts_equal(got, layouts) is None, f"layout node {k} at {pts}"
            kids = [self.leaf_texture(x, frames, live, pts) for x in leaves(c)]
            if rw == 0 or rh == 0:
                return None
            kids = [x if x is not None else np.zeros((1, 1, 4), np.uint8) for x in kids]
            return TW.orc.render_layout_node(rw, rh, [TW.from_ref_layout(l) for l in layouts], kids, mode=self.m, max_layouts=100)
        if not isinstance(c, SH):
            return super().leaf_texture(c, frames, live)
        kids = [self.leaf_texture(k, frames, live, pts) for k in c.children]
        return oracle_shader.render_shader(self.sources[c.shader_id], int(c.width), int(c.height), kids, pts,
                                           param_bytes(c.shader_param), self.m)

    def expected(self, pts, frames, stale=()):
        live = {k for k in frames if k not in stale}
        if isinstance(self.scene, SH):
            return TW.to_format(self.leaf_texture(self.scene, frames, live, pts), self.out, self.fmt)
        layouts, (rw, rh) = self.ref.layouts(pts, {k: (f.resolution.width, f.resolution.height) for k, f in frames.items() if k in live})
        got, root = self.r.debug_layouts("output_1", pts)
        assert root == (rw, rh)
        d = TW.layouts_equal(got, layouts)
        assert d is None, d
        nodes = [self.leaf_texture(c, frames, live, pts) for c in leaves(self.scene)]
        nodes = [n if n is not None else np.zeros((1, 1, 4), np.uint8) for n in nodes]
        rgba = TW.orc.render_layout_node(rw, rh, [TW.from_ref_layout(l) for l in layouts], nodes, mode=self.m, max_layouts=100)
        return TW.to_format(rgba, self.out, self.fmt)


class _Node:
    """a renderer whose debug_layouts are those of one layout node (smr_debug_node_layouts)"""

    def __init__(self, r, node):
        self.r, self.node = r, node

    def debug_layouts(self, output_id, pts):
        return self.r.debug_node_layouts(output_id, self.node, pts)


def leaves(comp):
    if isinstance(comp, (IN, IMG, s.TextComponent, WEB, SH)):
        return [comp]
    if isinstance(comp, R):
        return leaves(comp.child)
    return [x for c in comp.children for x in leaves(c)]


def host(**kw):
    return Pair(device=-1, **kw)


# ---- CPU ------------------------------------------------------------------------------------------------------------
LAYOUT_SCENES = {
    "root": lambda: SH(shader_id="grade", shader_param=grade(), width=320, height=180, children=[IN(input_id="input_1")]),
    "in_view": lambda: V(children=[IN(input_id="input_1"), SH(shader_id="gradient", width=200.7, height=100.2)]),
    "absolute_in_view": lambda: V(children=[TW.cell(40, 30, 320, 180, SH(shader_id="gradient", width=640, height=360))]),
    "in_tiles": lambda: T(children=[IN(input_id="input_1"), SH(shader_id="gradient", width=64, height=64), IN(input_id="input_2")]),
    "in_rescaler": lambda: V(children=[R(mode=s.RescaleMode.Fill, child=SH(shader_id="wipe", shader_param=wipe(), width=800,
                                                                           height=450, children=[IN(input_id="input_1"), IN(input_id="input_2")]))]),
}


@pytest.mark.parametrize("name", sorted(LAYOUT_SCENES))
def test_layouts_match_independent_engine(name):
    p = host(inputs=("input_1", "input_2"))
    for k in SOURCES:
        p.register_shader(k)
    p.update(LAYOUT_SCENES[name]())
    for pts in (0.0, 0.5):
        p.check_layouts(pts)


def test_layouts_across_a_transition_and_a_tiles_reorder():
    p = host(inputs=("input_1", "input_2"))
    p.register_shader("gradient")
    g = lambda i: SH(id=f"g{i}", shader_id="gradient", width=160, height=90)
    tr = s.Transition(duration=1.0)
    p.update(V(id="v", children=[T(id="t", children=[g(1), IN(id="a", input_id="input_1"), g(2)])]))
    p.check_layouts(0.0)
    p.update(V(id="v", direction=s.ViewChildrenDirection.Column, transition=tr,
               children=[T(id="t", transition=tr, children=[g(2), g(1), IN(id="a", input_id="input_1")])]))
    for pts in (0.0, 0.25, 0.5, 0.99, 1.5):
        p.check_layouts(pts)


def _tiles_of(ids, **kw):
    return T(id="t", width=600.0, height=300.0, children=[IN(id=i, input_id="input_1" if i < "c" else "input_2") for i in ids], **kw)


def test_nested_layout_nodes_match_independent_engine():
    """View, Tiles and Rescaler children of shaders, at two depths: each a layout node of its own, whose layouts equal the
    independent engine's across a transition and a Tiles reorder, and whose state survives scene updates"""
    p = host(inputs=("input_1", "input_2"))
    for k in SOURCES:
        p.register_shader(k)
    tr = s.Transition(duration=1.0)

    def scene(direction, ids, transition=None):
        inner = V(id="inner", position=s.Position.Static(width=320.0, height=180.0), direction=direction, transition=transition,
                  children=[IN(id="x", input_id="input_1"), R(child=IN(input_id="input_2"))])
        return V(children=[
            SH(id="w", shader_id="wipe", shader_param=wipe(), width=640, height=360, children=[
                inner, SH(shader_id="bands", width=600, height=300, children=[_tiles_of(ids, transition=transition)])]),
            SH(shader_id="grade", shader_param=grade(), width=300, height=200, children=[
                R(id="r", position=s.Position.Static(width=300.0, height=200.0), child=IN(input_id="input_2"))])])
    p.update(scene(s.ViewChildrenDirection.Row, ["a", "b", "c"]))
    assert len(p.nested) == 3
    for pts in (0.0, 0.5):
        p.check_layouts(pts)
        p.check_node_layouts(pts)
    p.update(scene(s.ViewChildrenDirection.Column, ["c", "a", "b"], tr))
    for pts in (0.5, 0.75, 1.0, 1.4, 1.6):
        p.check_layouts(pts)
        p.check_node_layouts(pts)
    p.update(scene(s.ViewChildrenDirection.Column, ["b", "c"], tr))   # a tile leaves while the last transition is done
    for pts in (1.6, 2.0, 2.7):
        p.check_node_layouts(pts)
    with pytest.raises(s.RendererError):
        p.r.debug_node_layouts("output_1", 5, 0.0)


def test_registry_and_compile_errors():
    r = s.Renderer(s.RendererOptions(cuda_device=-1))
    r.register_shader("g", GRADE, GRADE_TYPE)
    with pytest.raises(s.RendererError) as e:                       # KeyTaken
        r.register_shader("g", GRADIENT)
    assert e.value.status == 1
    with pytest.raises(s.RendererError) as e:                       # CreateShaderError, with NVRTC's log
        r.register_shader("bad", GRADIENT.replace("sqrtf(dx * dx + dy * dy)", "sqrtf(undefined_distance)"))
    assert e.value.status == 1 and "undefined_distance" in str(e.value) and "shader(" in str(e.value)
    for bad_type in (PT("list", item=PT("f32"), length=0), PT("list", length=2), PT("struct"), PT("struct", fields=[("", PT("f32"))])):
        spec_keep = []
        t = s.renderer._param_type_to_c(bad_type, spec_keep)
        if bad_type.kind == "struct" and bad_type.fields:
            t.items[0].name = None
        spec = F.ShaderSpec(GRADIENT.encode(), C.pointer(t))
        assert F.lib().smr_register_shader(r._h, b"t", C.byref(spec)) == 1, bad_type
    assert F.lib().smr_register_shader(r._h, b"t", None) == 1
    assert F.lib().smr_register_shader(r._h, b"t", C.byref(F.ShaderSpec(None, None))) == 1
    with pytest.raises(s.RendererError):
        r.unregister_shader("nope")
    r.unregister_shader("g")
    with pytest.raises(s.RendererError):
        r.unregister_shader("g")


def _status(r, scene, output_id="output_1"):
    with pytest.raises(s.RendererError) as e:
        r.update_scene(output_id, s.Resolution(640, 360), YUV, scene)
    return e.value.status


def test_scene_refusals_leave_the_scene_as_it_was():
    p = host(inputs=("input_1",))
    for k in ("grade", "gradient"):
        p.register_shader(k)
    p.register_web("page", 320, 180)
    good = V(children=[IN(input_id="input_1"), SH(id="s", shader_id="grade", shader_param=grade(), width=320, height=180,
                                                     children=[IN(input_id="input_1")])])
    p.update(good)
    before = product_layouts(p.r, 0.0)
    c = F.Component()
    F.lib().smr_component_default(F.COMPONENT_SHADER, C.byref(c))
    assert not c.shader_id
    assert F.lib().smr_update_scene(p.r._h, b"output_1", 640, 360, YUV, C.byref(c)) == 5       # what an older caller sends
    g = lambda param, **kw: SH(shader_id="grade", shader_param=param, width=kw.get("w", 320), height=kw.get("h", 180))
    refused = {
        4: [SH(shader_id="missing", width=64, height=64),                                        # ShaderNotFound
            V(children=[g(P.f32(1.0))]),                                                         # wrong kind
            g(P.struct([("gain", P.list([P.f32(1)] * 4)), ("lift", P.f32(0))])),                 # list too long
            g(P.struct([("gain", P.list([P.f32(1)] * 3))])),                                     # a field missing
            g(P.struct([("lift", P.f32(0)), ("gain", P.list([P.f32(1)] * 3))])),                 # field names out of order
            g(P.struct([("gain", P.list([P.u32(1)] * 3)), ("lift", P.f32(0))])),                 # wrong element kind
            SH(shader_id="gradient", shader_param=P.f32(1.0), width=64, height=64),              # NoBindingInShader
            g(grade(), w=0), g(grade(), h=0.5), g(grade(), w=16385), g(grade(), w=-3.0),         # node size
            V(children=[SH(id="a", shader_id="gradient", width=8, height=8, children=[IN(id="a", input_id="input_1")])]),
            SH(shader_id="gradient", width=8, height=8, children=[IMG(id="i", image_id="missing")]),
            SH(shader_id="gradient", width=8, height=8, children=[V()]),                          # UnknownDimensionsForLayoutNodeRoot
            SH(shader_id="gradient", width=8, height=8, children=[V(position=s.Position.Static(width=64.0))]),
            V(children=[SH(shader_id="gradient", width=8, height=8, children=[R(child=IN(input_id="input_1"))])]),
            SH(shader_id="gradient", width=8, height=8, children=[T(width=64.0)])],
        5: [SH(shader_id="gradient", width=8, height=8, children=[IN(input_id="input_1")] * 17),   # more than 16 textures
            TW.web(children=[SH(id="x", shader_id="gradient", width=8, height=8)])],             # a Shader inside a WebView
    }
    for status, scenes in refused.items():
        for scene in scenes:
            assert _status(p.r, scene) == status, scene
            if status == 4:
                with pytest.raises(LS.SceneError):
                    p.ref.update_scene(scene)
            assert product_layouts(p.r, 0.0) == before
    p.check_layouts(0.0)
    # a short list is accepted (validation.rs: ListTooLong only above the length); sixteen children are accepted
    p.update(g(P.struct([("gain", P.list([P.f32(1)] * 2)), ("lift", P.f32(0))])))
    p.update(SH(shader_id="gradient", width=8, height=8, children=[IN(input_id="input_1")] * 16))
    # unregistering a shader a scene shows keeps that scene; a new scene cannot name it
    p.r.unregister_shader("gradient")
    assert _status(p.r, SH(shader_id="gradient", width=8, height=8)) == 4


def test_param_bytes_are_tight_little_endian():
    p = P.struct([("a", P.f32(1.5)), ("b", P.list([P.u32(7), P.i32(-2)])), ("c", P.struct([("d", P.f32(-0.0))]))])
    assert param_bytes(p) == struct.pack("<fIif", 1.5, 7, -2, -0.0)


def test_oracle_identity_shader_is_the_child():
    """a shader that returns its child's sample at the texel centres is the child, in both modes"""
    ident = "__device__ float4 smr_fragment(smr_fragment_in in, const smr_base_params &b, const void *p, const smr_textures &t) " \
            "{ return t.sample(0, in.tex_coords); }"
    px = TW.page(37, 23, 4, translucent=False)
    for m in (0, 1):
        assert np.array_equal(oracle_shader.render_shader(ident, 37, 23, [px], mode=m), px)
    assert not oracle_shader.render_shader(ident, 5, 4, [None]).any()


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _gpu_pair(fmt, mode, out=(640, 360), inputs=("input_1", "nv12_2")):
    p = Pair(out=out, fmt=fmt, mode=mode, inputs=inputs)
    for k in SOURCES:
        p.register_shader(k)
    return p


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", TW.FORMATS)
@pytest.mark.parametrize("mode", TW.MODES)
def test_colour_grade_wipe_and_gradient_match_oracle(mode, fmt):
    """a single-input grade as the root, a two-input wipe driven by time and a struct parameter, a shader without children"""
    p = _gpu_pair(fmt, mode, out=(640, 360))
    p.update(SH(shader_id="grade", shader_param=grade(), width=640, height=360, children=[IN(input_id="input_1")]))
    p.render_check(0.0, "grade root")
    p.update(V(background_color=s.RGBAColor(10, 20, 30, 255), children=[
        SH(shader_id="wipe", shader_param=wipe(), width=640, height=360, children=[IN(input_id="input_1"), IN(input_id="nv12_2")])]))
    p.r.set_profiling(True)
    for pts in (0.0, 0.5, 1.25, 1.9):
        p.render_check(pts, "wipe")
    assert p.r.kernel_times()["shader"][1] == 4                 # one launch per tick: one shader at one depth
    p.update(V(children=[IN(input_id="input_1"), SH(shader_id="gradient", width=300.9, height=170.2)]))
    p.render_check(0.5, "gradient")


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", TW.FORMATS)
@pytest.mark.parametrize("mode", TW.MODES)
def test_children_of_every_kind_and_nested_shaders_match_oracle(mode, fmt):
    """a shader over inputs, an Image, a Text and a WebView, Lanczos-scaled and under a rounded mask; a shader over a View
    holding inputs, an Image and a Text with a rounded mask and a Lanczos-scaled child; a shader under a shader under a
    View; a stale input"""
    p = _gpu_pair(fmt, mode, inputs=("input_1", "nv12_2", "input_3"))
    p.register_image("img", pixels(90, 60, 1, 5)[0])
    p.register_web("page", 320, 180, TW.OVER)
    p.set_frame("page", TW.page(320, 180, 2))
    p.set_rects("page", [(20.5, 10, 160, 90)])
    kids = [IN(input_id="input_1"), IN(input_id="nv12_2"), IMG(image_id="img"), label(120, 24, 3),
            TW.web(children=[IN(id="a", input_id="input_3")]), IN(input_id="input_3")]
    inner = SH(shader_id="grade", shader_param=grade((0.5, 1.5, 1.0), 0.125), width=200, height=120,
               children=[IN(input_id="nv12_2")])
    view = V(position=s.Position.Static(width=400.0, height=240.0), background_color=s.RGBAColor(40, 0, 60, 200), children=[
        R(child=IN(input_id="input_1")),                                                     # 640 x 360 -> Lanczos
        TW.cell(20, 130, 120, 90, IMG(image_id="img"), border_radius=s.BorderRadius(20.0, 5.0, 30.0, 10.0),
                overflow=s.Overflow.Hidden),
        TW.cell(200, 10, 120, 24, label(120, 24, 4)),
        TW.cell(180, 120, 200, 112, IN(input_id="input_3"))])
    p.update(V(background_color=s.RGBAColor(10, 20, 30, 255), children=[
        R(child=SH(shader_id="bands", width=960, height=540, children=kids)),                # 960 x 540 -> Lanczos
        TW.cell(330, 170, 300, 170, SH(shader_id="grade", shader_param=grade(), width=300, height=170,
                                       children=[SH(shader_id="wipe", shader_param=wipe(0.25), width=300, height=170,
                                                    children=[inner, IN(input_id="input_1")])]),
                border_radius=s.BorderRadius(30.0, 10.0, 40.0, 5.0), overflow=s.Overflow.Hidden),
        TW.cell(20, 20, 200, 120, SH(shader_id="grade", shader_param=grade((1.0, 1.0, 0.5), 0.0), width=400, height=240,
                                     children=[view]))]))
    p.r.set_profiling(True)
    p.render_check(6.0, "children", stale=("input_3",))
    # one launch per distinct (shader, depth): (grade, 1) `inner`; (bands, 2) over a web node; (wipe, 2) over `inner`;
    # (grade, 2) over the View's layout node (depth 1); (grade, 3) over the wipe
    assert p.r.kernel_times()["shader"][1] == 5
    p.render_check(6.04, "children, input_3 live")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", TW.MODES)
def test_tiles_reorder_inside_a_shader_over_a_transition(mode):
    """a Tiles child of a shader, its tiles reordered and one removed under a transition: the layout node's state carries
    over the scene updates"""
    p = _gpu_pair(YUV, mode, inputs=("input_1", "nv12_2"))
    tr = s.Transition(duration=1.0)
    sc = lambda ids, t=None: V(children=[SH(shader_id="grade", shader_param=grade(), width=640, height=360,
                                            children=[_tiles_of(ids, transition=t)])])
    p.update(sc(["a", "b", "c"]))
    p.render_check(0.0)
    p.update(sc(["c", "a", "b"], tr))
    for pts in (0.0, 0.5, 1.5):
        p.render_check(pts, "reorder")
    p.update(sc(["b", "c"], tr))
    for pts in (1.5, 2.0, 2.6):
        p.render_check(pts, "removed")


@pytest.mark.gpu
def test_shaders_in_tiles_and_unregistered_shader_keeps_drawing():
    p = _gpu_pair(YUV, s.RenderingMode.GpuOptimized)
    g = lambda i, src: SH(id=f"g{i}", shader_id="grade", shader_param=grade(), width=320, height=180, children=[IN(input_id=src)])
    tr = s.Transition(duration=1.0)
    p.update(T(id="t", children=[g(1, "input_1"), g(2, "nv12_2")]))
    p.render_check(0.0)
    p.update(T(id="t", transition=tr, children=[g(2, "nv12_2"), g(1, "input_1")]))
    for pts in (0.0, 0.5, 1.5):
        p.render_check(pts, "reorder")
    p.r.unregister_shader("grade")
    p.render_check(1.6, "unregistered")
    p.update(V(children=[IN(input_id="input_1")]))               # the last user lets go: the module is unloaded later
    p.render_check(1.7, "shader gone")


@pytest.mark.gpu
def test_four_ticks_in_flight():
    """four ticks submitted behind a busy render stream, each with its own pts (the wipe's edge moves with time) and
    frames: every tick shows its own, the layout node textures of the frame arena included"""
    torch = pytest.importorskip("torch")
    p = _gpu_pair(YUV, s.RenderingMode.GpuOptimized)
    p.update(SH(shader_id="wipe", shader_param=wipe(0.5), width=640, height=360, children=[
        V(position=s.Position.Static(width=640.0, height=360.0), children=[R(child=IN(input_id="nv12_2"))]),
        IN(input_id="input_1")]))
    p.r.render(s.FrameSet(frames=p.frames(0.0), pts=0.0))
    stream = torch.cuda.ExternalStream(p.r.cuda_stream(), device=torch.device("cuda:0"))
    frames = {k: p.frames(1.0 + 0.3 * k) for k in range(4)}
    with torch.cuda.stream(stream):
        torch.cuda._sleep(1_000_000_000)   # about half a second: the ticks below wait behind it on the render stream
    ticks = []
    for k in range(4):
        pts = 1.0 + 0.3 * k
        ticks.append((TW._Tick(p.r, pts, frames[k], p.out, p.fmt, torch), pts, frames[k]))
    assert not stream.query(), "the render stream drained before the ticks were checked"
    for _ in ticks:
        p.r.wait()
    for t, pts, fr in ticks:
        TW.assert_identical([pl for pl in t.planes if pl is not None], p.expected(pts, fr), f"tick at {pts}")


_LAUNCHES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bench_scene_launches.json")


@pytest.mark.gpu
def test_bench_scenes_plan_the_same_launches():
    """every scene of tests/test_gpu_bench_scenes.py launches as many kernels per tick as before shader nodes existed
    (tests/golden/bench_scene_launches.json, counted on an H100 with the library of the commit before them), with a shader
    registered"""
    with open(_LAUNCHES) as f:
        before = json.load(f)
    got = {}
    for name, seed in (("cfg3", 7000), ("cfg3b", 7100), ("cfg2", 7200), ("grid25", 7600), ("cfg5", 7500)):
        wl = bench.workload(name)
        fr = bench_frames(wl, seed)
        _, _, r = run_case(wl["scene"], fr, resolution=s.Resolution(wl["W"], wl["H"]), out_format=NV12, mode=wl["mode"])
        got[name] = r.stats()["last_render_kernel_launches"]
    wl = bench.workload("cfg4")
    fr = bench_frames(wl, 7300)
    r = s.Renderer(s.RendererOptions(rendering_mode=wl["mode"]))
    r.register_shader("grade", GRADE, GRADE_TYPE)
    for iid in fr:
        r.register_input(iid)
    for k in range(wl["n_out"]):
        r.update_scene(f"output_{k + 1}", s.Resolution(wl["W"], wl["H"]), NV12, bench.cfg4_scene(k, wl["n"]))
    r.render(s.FrameSet(frames=fr, pts=0.0))
    got["cfg4"] = r.stats()["last_render_kernel_launches"]
    assert got == before
