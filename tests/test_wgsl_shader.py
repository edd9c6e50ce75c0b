"""WGSL shaders (smr_register_wgsl_shader): the reference's shader dialect translated to CUDA and drawn with its vertex
stage.

The WGSL files under tests/golden/wgsl/ are the reference's own (its render tests load them with include_str!), kept
verbatim.  CPU (host-only handle): every corpus file registers (NVRTC compiles the translation for sm_90a), the derived
parameter type, the refusals, and scene-update validation against WGSL vector, matrix and array types.  GPU: the
reference's yuv_test_gradient known answer; the reference's shader render tests re-typed as scenes, every output byte
against an independent oracle (tests/wgsl_oracle_shim.h: its own rasteriser, and a hand-written C++ restatement of each
module's two stages); the translator's integer and conversion rules against numpy; the rasteriser's edges.
"""
import os
import struct

import numpy as np
import pytest

import smelter_b200 as s
from smelter_b200 import _ffi as F
from tests import oracle_wgsl
from tests import test_shader_component as TS
from tests import test_web_view_component as TW
from tests.test_oracle_kat import GRADIENT_RGBA_EXPECTED, GRADIENT_YUV_EXPECTED
from oracle import oracle as orc

V, IN, SH, P, PT = s.ViewComponent, s.InputStreamComponent, s.ShaderComponent, s.ShaderParam, s.ShaderParamType
YUV, NV12, RGBA = TW.YUV, TW.NV12, TW.RGBA
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wgsl")
CORPUS = sorted(f[:-5] for f in os.listdir(GOLDEN) if f.endswith(".wgsl"))


def wgsl(name):
    with open(os.path.join(GOLDEN, name + ".wgsl")) as f:
        return f.read()


HEADER = wgsl("gradient").split("@fragment")[0]   # the shader header with an identity vs_main


def with_fs(body, extra=""):
    return HEADER + extra + "\n@fragment\nfn fs_main(input: VertexOutput) -> @location(0) vec4<f32> {\n" + body + "\n}\n"


def host():
    return s.Renderer(s.RendererOptions(cuda_device=-1))


def status(r, src, shader_id="x"):
    with pytest.raises(s.RendererError) as e:
        r.register_wgsl_shader(shader_id, src)
    return e.value.status, str(e.value)


# ---- CPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CORPUS)
def test_corpus_registers(name):
    r = host()
    r.register_wgsl_shader(name, wgsl(name))
    assert status(r, wgsl(name), name)[0] == 1    # KeyTaken
    r.unregister_shader(name)


def test_circle_layout_parameter_type():
    """the uniform array<CircleLayout, 4> becomes the parameter type: validation accepts the reference's parameter and
    the same rules as a hand-written tree refuse the rest"""
    p = TS.host(inputs=("input_1",))
    p.r.register_wgsl_shader("circle", wgsl("circle_layout"))
    p.ref.register_shader("circle", PT("list", item=PT("struct", fields=[
        ("left_px", PT("u32")), ("top_px", PT("u32")), ("width_px", PT("u32")), ("height_px", PT("u32")),
        ("background_color", PT("list", item=PT("f32"), length=4))]), length=4))
    ok = SH(shader_id="circle", shader_param=circle_param(), width=640, height=360, children=[IN(input_id="input_1")] * 4)
    p.update(ok)
    bad = [P.list([circle_item(0, 0, 1, 1, (1, 0, 0, 1))] * 5),                          # ListTooLong
           P.list([P.struct([("left_px", P.u32(0))])]),                                   # fields missing
           P.f32(1.0)]
    for param in bad:
        assert TS._status(p.r, SH(shader_id="circle", shader_param=param, width=64, height=64)) == 4


def circle_item(l, t, w, h, c):
    return P.struct([("left_px", P.u32(l)), ("top_px", P.u32(t)), ("width_px", P.u32(w)), ("height_px", P.u32(h)),
                     ("background_color", P.list([P.f32(x) for x in c]))])


def circle_param(W=640, H=360):
    hw, hh = W // 2, H // 2
    cols = [(1, 0, 0, 1), (0, 1, 0, 1), (0, 0, 1, 1), (1, 1, 1, 1)]
    return P.list([circle_item(x, y, hw, hh, c) for (x, y), c in zip([(0, 0), (hw, 0), (0, hh), (hw, hh)], cols)])


REFUSED_INVALID = {
    "parse": with_fs("return vec4(1.0, 0.0, 0.0 1.0);"),
    "type": with_fs("let a: u32 = 1.5; return vec4(1.0);"),
    "unknown identifier": with_fs("return vec4(nope);"),
    "missing textures": with_fs("return vec4(1.0);").replace("@group(0) @binding(0) var textures: binding_array<texture_2d<f32>, 16>;", ""),
    "missing sampler": with_fs("return vec4(1.0);").replace("@group(2) @binding(0) var sampler_: sampler;", ""),
    "textures of 8": with_fs("return vec4(1.0);").replace("texture_2d<f32>, 16>", "texture_2d<f32>, 8>"),
    "sampler wrong type": with_fs("return vec4(1.0);").replace("var sampler_: sampler;", "var sampler_: texture_2d<f32>;"),
    "base params field": with_fs("return vec4(1.0);").replace("texture_count: u32,", "texture_count: i32,"),
    "push constant": with_fs("return vec4(1.0);").replace("var<immediate>", "var<push_constant>"),
    "non-uniform user binding": with_fs("return vec4(1.0);", "@group(1) @binding(0) var<storage, read> p: array<f32, 4>;"),
    "vs_main two arguments": with_fs("return vec4(1.0);").replace("fn vs_main(input: VertexInput)", "fn vs_main(input: VertexInput, b: VertexInput)"),
    "no vs_main": with_fs("return vec4(1.0);").replace("fn vs_main", "fn vs_other"),
    "uniform stride": with_fs("return vec4(1.0);", "@group(1) @binding(0) var<uniform> p: array<f32, 4>;"),
}
REFUSED_UNSUPPORTED = {
    "dpdx": with_fs("return vec4(dpdx(input.tex_coords.x));"),
    "fwidth": with_fs("return vec4(fwidth(input.tex_coords.x));"),
    "storage": with_fs("return vec4(1.0);", "@group(3) @binding(0) var<storage, read> p: array<f32>;"),
    "atomic": with_fs("return vec4(1.0);", "struct A { a: atomic<u32> }"),
    "override": with_fs("return vec4(1.0);", "override k: f32 = 1.0;"),
    "pointers": with_fs("var a = 1.0; let p = &a; return vec4(1.0);"),
    "texture_3d": with_fs("return vec4(1.0);", "@group(3) @binding(0) var t3: texture_3d<f32>;"),
    "textureLoad": with_fs("return textureLoad(textures[0], vec2<i32>(0, 0), 0);"),
}


@pytest.mark.parametrize("name", sorted(REFUSED_INVALID))
def test_invalid_wgsl_is_refused_with_a_position(name):
    st, msg = status(host(), REFUSED_INVALID[name])
    assert st == 1, msg
    assert "WGSL " in msg and ":" in msg


@pytest.mark.parametrize("name", sorted(REFUSED_UNSUPPORTED))
def test_unsupported_constructs_are_named(name):
    st, msg = status(host(), REFUSED_UNSUPPORTED[name])
    assert st == 5, msg
    assert "unsupported" in msg


def test_semantics_and_edge_shaders_register():
    r = host()
    r.register_wgsl_shader("sem", sem_shader())
    r.register_wgsl_shader("edge", EDGE_SRC)


VEC_MAT = with_fs("return u.c * u.m[0].x;", """struct U { c: vec4<f32>, m: mat2x3<f32>, a: array<vec4<u32>, 2>, }
@group(1) @binding(0) var<uniform> u: U;""")


def test_vector_matrix_and_array_parameters_validate_as_validation_rs():
    p = TS.host(inputs=("input_1",))
    p.r.register_wgsl_shader("vm", VEC_MAT)
    f = lambda n: P.list([P.f32(0.5)] * n)
    good = P.struct([("c", f(4)), ("m", P.list([f(2)] * 3)), ("a", P.list([P.list([P.u32(1)] * 4)]))])
    p.r.update_scene("output_1", s.Resolution(640, 360), YUV, V(children=[SH(shader_id="vm", shader_param=good, width=64, height=64)]))
    before = TS.product_layouts(p.r, 0.0)
    bad = [P.struct([("c", f(3)), ("m", P.list([f(2)] * 3)), ("a", P.list([]))]),                 # vector of 3
           P.struct([("c", f(4)), ("m", P.list([f(2)] * 2)), ("a", P.list([]))]),                 # 2 rows
           P.struct([("c", f(4)), ("m", P.list([f(3)] * 3)), ("a", P.list([]))]),                 # rows of 3
           P.struct([("c", f(4)), ("m", P.list([f(2)] * 3)), ("a", P.list([P.list([P.u32(1)] * 4)] * 3))]),   # too long
           P.struct([("c", P.f32(1)), ("m", P.list([f(2)] * 3)), ("a", P.list([]))]),             # a scalar for a vector
           P.struct([("c", f(4)), ("m", P.list([f(2)] * 3)), ("a", P.list([P.list([P.f32(1)] * 4)]))])]   # f32 for u32
    for param in bad:
        assert TS._status(p.r, SH(shader_id="vm", shader_param=param, width=64, height=64)) == 4, param
        assert TS.product_layouts(p.r, 0.0) == before


# ---- oracle restatements (C++, compiled for the CPU against tests/wgsl_oracle_shim.h) --------------------------------
IDENTITY_VS = r'''
#define WO_NVARY 2
static const int wo_interp[2] = {0, 0};
static void wo_vs(const wo_base &, const void *, const float *p, const float *tc, float *pos, float *vary) {
    pos[0] = p[0]; pos[1] = p[1]; pos[2] = p[2]; pos[3] = 1.0f; vary[0] = tc[0]; vary[1] = tc[1];
}
'''
SAMPLE = "static float4 S(const smr_textures &t, int i, float u, float v) { return t.sample((unsigned)i, make_float2(u, v)); }\n"
FS = "static bool wo_fs(const wo_base &b, const void *params, const smr_textures &t, const float *fp, const float *tc, float4 &out) {\n"
RESTATED = {
    "gradient": IDENTITY_VS + FS + "out = make_float4(tc[0], 0.0f, 0.0f, 1.0f); return true; }",
    "color_output_with_texture_count": IDENTITY_VS + FS + r'''
    out = b.count == 0 ? make_float4(1, 0, 0, 1) : b.count == 1 ? make_float4(0, 1, 0, 1) : make_float4(0, 0, 1, 1);
    return true; }''',
    "layout_planes": r'''
#define WO_NVARY 2
static const int wo_interp[2] = {0, 0};
static void wo_vs(const wo_base &b, const void *, const float *p, const float *tc, float *pos, float *vary) {
    float sx = p[0] / 2.0f, sy = p[1] / 2.0f;
    int id = b.plane_id;
    if (id == -1) { pos[0] = p[0]; pos[1] = p[1]; }
    else if (id == 0) { pos[0] = sx - 0.5f; pos[1] = sy + 0.5f; }
    else if (id == 1) { pos[0] = sx + 0.5f; pos[1] = sy + 0.5f; }
    else if (id == 2) { pos[0] = sx - 0.5f; pos[1] = sy - 0.5f; }
    else if (id == 3) { pos[0] = sx + 0.5f; pos[1] = sy - 0.5f; }
    else { pos[0] = sx; pos[1] = sy; }
    pos[2] = p[2]; pos[3] = 1.0f; vary[0] = tc[0]; vary[1] = tc[1];
}
''' + SAMPLE + FS + r'''
    if (b.plane_id == -1) { out = make_float4(1, 0, 0, 1); return true; }
    out = S(t, b.plane_id, tc[0], tc[1]); return true; }''',
    "red_border": IDENTITY_VS + SAMPLE + FS + r'''
    float4 smp = S(t, 0, tc[0], tc[1]);
    if (fp[0] > 50.0f && fp[0] < (float)b.res[0] - 50.0f && fp[1] > 50.0f && fp[1] < (float)b.res[1] - 50.0f) { out = smp; return true; }
    out = make_float4(1, 0, 0, 1); return true; }''',
    "circle_layout": r'''
#define WO_NVARY 2
static const int wo_interp[2] = {0, 0};
struct CL { unsigned l, t, w, h; float c[4]; };
static CL cl(const wo_base &b, const void *params) {
    unsigned i = (unsigned)b.plane_id < 4u ? (unsigned)b.plane_id : 3u;
    CL r; memcpy(&r, (const char *)params + 32 * i, sizeof r); return r;
}
static void wo_vs(const wo_base &b, const void *params, const float *p, const float *tc, float *pos, float *vary) {
    CL c = cl(b, params);
    float xs = (float)c.w / (float)b.res[0], ys = (float)c.h / (float)b.res[1];
    float cx = (((float)c.l + (float)c.w / 2.0f) / (float)b.res[0]) * 2.0f - 1.0f;
    float cy = 1.0f - (((float)c.t + (float)c.h / 2.0f) / (float)b.res[1]) * 2.0f;
    pos[0] = p[0] * xs + cx; pos[1] = p[1] * ys + cy; pos[2] = p[2]; pos[3] = 1.0f; vary[0] = tc[0]; vary[1] = tc[1];
}
''' + SAMPLE + FS + r'''
    CL c = cl(b, params);
    float ux = tc[0] - 0.5f, uy = tc[1] - 0.5f, len = sqrtf(ux * ux + uy * uy);
    float in = len < 0.5f ? 1.0f : 0.0f;
    float4 smp = S(t, b.plane_id, tc[0], tc[1]);
    out = make_float4(smp.x * in + c.c[0] * (1.0f - in), smp.y * in + c.c[1] * (1.0f - in), smp.z * in + c.c[2] * (1.0f - in),
                      smp.w * in + c.c[3] * (1.0f - in));
    return true; }''',
    "fade_to_ball": IDENTITY_VS + SAMPLE + r'''
static float ss(float lo, float hi, float x) { float t = fminf(fmaxf((x - lo) / (hi - lo), 0.0f), 1.0f); return t * t * (3.0f - 2.0f * t); }
''' + FS + r'''
    float4 smp = S(t, 0, tc[0], tc[1]);
    float r = b.time / 5.0f, eps = 0.15f;
    float ux = tc[0] - 0.5f, uy = tc[1] - 0.5f, len = sqrtf(ux * ux + uy * uy);
    float k = ss(r + eps, r - eps, len);
    out = make_float4(smp.x * k, smp.y * k, smp.z * k, smp.w * k); return true; }''',
    "silly": IDENTITY_VS + SAMPLE + r'''
static float ss(float lo, float hi, float x) { float t = fminf(fmaxf((x - lo) / (hi - lo), 0.0f), 1.0f); return t * t * (3.0f - 2.0f * t); }
''' + FS + r'''
    if (b.count != 1u) { out = make_float4(0, 0, 0, 0); return true; }
    float pi = 3.14159f, er = fabsf(sinf(b.time) / 2.0f), ea = 2.0f * pi * fabsf(sinf(b.time) / 2.0f);
    float ux = tc[0] - 0.5f, uy = tc[1] - 0.5f, len = sqrtf(ux * ux + uy * uy);
    float a = atan2f(uy, ux) + ea * ss(er, 0.0f, len);
    out = S(t, 0, len * cosf(a) + 0.5f, len * sinf(a) + 0.5f); return true; }''',
}
RESTATED["component_shader"] = RESTATED["silly"]
TOLERANT = {"silly", "component_shader"}   # sin / cos / atan2: the GPU's and the C library's differ in the last bits


class Pair(TS.Pair):
    """the shader test's pair, with WGSL shaders drawn by their restatements"""

    def __init__(self, **kw):
        super().__init__(**kw)
        self.wgsl = {}

    def register_wgsl(self, shader_id, name, src=None, restated=None, param_type=None):
        self.r.register_wgsl_shader(shader_id, src or wgsl(name))
        self.ref.register_shader(shader_id, param_type)
        self.wgsl[shader_id] = (restated or RESTATED[name], name)

    def leaf_texture(self, c, frames, live, pts=0.0):
        if isinstance(c, SH) and c.shader_id in self.wgsl:
            kids = [self.leaf_texture(k, frames, live, pts) for k in c.children]
            pb = TS.param_bytes(c.shader_param)
            return oracle_wgsl.render(self.wgsl[c.shader_id][0], int(c.width), int(c.height), kids, pts, pb.ljust(256, b"\0"), self.m)
        return super().leaf_texture(c, frames, live, pts)


def inputs(n):
    return [IN(input_id=f"input_{i + 1}") for i in range(n)]


CIRCLE_TYPE = PT("list", item=PT("struct", fields=[("left_px", PT("u32")), ("top_px", PT("u32")), ("width_px", PT("u32")),
                                                   ("height_px", PT("u32")), ("background_color", PT("list", item=PT("f32"), length=4))]), length=4)
# the reference's shader render tests (shader.rs), re-typed: (shader, scene, snapshot pts)
RENDER_TESTS = {
    "base_params_plane_id_no_inputs": ("layout_planes", lambda: SH(shader_id="layout_planes", width=640, height=360), [0.0]),
    "base_params_plane_id_5_inputs": ("layout_planes", lambda: SH(shader_id="layout_planes", width=640, height=360, children=inputs(5)), [0.0]),
    "base_params_time": ("fade_to_ball", lambda: SH(shader_id="fade_to_ball", width=640, height=360, children=inputs(1)), [0.0, 1.0, 2.0]),
    "base_params_output_resolution": ("red_border", lambda: SH(shader_id="red_border", width=640, height=360, children=inputs(1)), [0.0]),
    "base_params_texture_count_no_inputs": ("color_output_with_texture_count", lambda: SH(shader_id="color_output_with_texture_count", width=640, height=360), [0.0]),
    "base_params_texture_count_1_input": ("color_output_with_texture_count", lambda: SH(shader_id="color_output_with_texture_count", width=640, height=360, children=inputs(1)), [0.0]),
    "base_params_texture_count_2_inputs": ("color_output_with_texture_count", lambda: SH(shader_id="color_output_with_texture_count", width=640, height=360, children=inputs(2)), [0.0]),
    "user_params_circle_layout": ("circle_layout", lambda: SH(shader_id="circle_layout", shader_param=circle_param(), width=640, height=360, children=inputs(4)), [0.0]),
}


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_yuv_test_gradient_reference_known_answer():
    """yuv_tests.rs: the reference's gradient.wgsl on an 8 x 2 node; RGBA output equal to its bytes, the YUV output through
    the harness's conversion equal to its YUV-case bytes"""
    for fmt in (RGBA, YUV):
        r = s.Renderer(s.RendererOptions())
        r.register_wgsl_shader("example_shader", wgsl("gradient"))
        r.update_scene("output_1", s.Resolution(8, 2), fmt, SH(shader_id="example_shader", width=8.0, height=2.0))
        got = [np.asarray(p) for p in r.render(s.FrameSet(frames={}, pts=0.0)).frames["output_1"].data.planes]
        if fmt == RGBA:
            assert got[0].reshape(-1).tolist() == GRADIENT_RGBA_EXPECTED
        else:
            back = orc.harness_yuv420_to_rgba(got[0], got[1], got[2], 8, 2)
            assert back.reshape(-1).tolist() == GRADIENT_YUV_EXPECTED


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", TW.FORMATS)
@pytest.mark.parametrize("mode", TW.MODES)
@pytest.mark.parametrize("name", sorted(RENDER_TESTS))
def test_reference_shader_render_tests_match_oracle(name, mode, fmt):
    shader, scene, snapshots = RENDER_TESTS[name]
    p = Pair(out=(640, 360), fmt=fmt, mode=mode, inputs=tuple(f"input_{i + 1}" for i in range(5)))
    p.register_wgsl(shader, shader, param_type=CIRCLE_TYPE if shader == "circle_layout" else None)
    p.update(scene())
    p.r.set_profiling(True)
    for pts in snapshots:
        p.render_check(pts, name)
    assert p.r.kernel_times()["shader"][1] == len(snapshots)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", TW.MODES)
@pytest.mark.parametrize("name", sorted(TOLERANT))
def test_transcendental_shaders_within_tolerance(name, mode):
    p = Pair(out=(640, 360), fmt=RGBA, mode=mode, inputs=("input_1",))
    p.register_wgsl(name, name)
    p.update(SH(shader_id=name, width=640, height=360, children=inputs(1)))
    for pts in (0.0, 0.7, 2.3):
        frames = p.frames(pts)
        got = np.asarray(p.r.render(s.FrameSet(frames=frames, pts=pts)).frames["output_1"].data.planes[0]).astype(int)
        exp = p.expected(pts, frames)[0].astype(int)
        d = np.abs(got - exp)
        # a last-bit difference in an angle moves a sample by at most a fraction of a texel: within 3 levels everywhere,
        # and identical almost everywhere
        assert d.max() <= 3 and (d > 0).mean() < 0.01, (name, pts, d.max(), (d > 0).mean())


# the translator's rules, evaluated on the GPU: each fragment writes one 16-bit half of one 32-bit result into r and g
SEM_N = 64
SEM = r'''
struct U { a: array<vec4<i32>, 16>, b: array<vec4<i32>, 16>, f: array<vec4<f32>, 16>, }
@group(1) @binding(0) var<uniform> u: U;
fn pick(v: vec4<i32>, k: u32) -> i32 {
    switch k { case 0u: { return v.x; } case 1u: { return v.y; } case 2u: { return v.z; } default: { return v.w; } }
}
fn pickf(v: vec4<f32>, k: u32) -> f32 { var r = v.w; if k == 0u { r = v.x; } else if k == 1u { r = v.y; } else if k == 2u { r = v.z; } return r; }
fn op(which: u32, i: u32) -> u32 {
    let a = pick(u.a[i / 4u], i % 4u);
    let b = pick(u.b[i / 4u], i % 4u);
    let f = pickf(u.f[i / 4u], i % 4u);
    switch which {
        case 0u: { return bitcast<u32>(a + b); }
        case 1u: { return bitcast<u32>(a - b * 3); }
        case 2u: { return bitcast<u32>(a * b); }
        case 3u: { return bitcast<u32>(a / b); }
        case 4u: { return bitcast<u32>(a % b); }
        case 5u: { return u32(a) / u32(b); }
        case 6u: { return u32(a) % u32(b); }
        case 7u: { return bitcast<u32>(a << u32(b)); }
        case 8u: { return bitcast<u32>(a >> u32(b)); }
        case 9u: { return u32(a) >> u32(b); }
        case 10u: { return bitcast<u32>(i32(f)); }
        case 11u: { return u32(f); }
        case 12u: { return bitcast<u32>(-a); }
        case 13u: { return bitcast<u32>(select(a, b, a < b)); }
        case 14u: {
            var s = 0u;
            for (var k = 0u; k < (u32(b) & 15u); k++) { if k == 3u { continue; } s += u32(a) ^ k; }
            var j = 0;
            loop { j += 1; if j > 4 { break; } continuing { s = s * 3u + u32(j); } }
            while s > 1000000u { s = s >> 1u; }
            return s;
        }
        case 15u: { return bitcast<u32>(f * 3.0 - 1.5 + f32(a) * 0.25); }
        case 16u: { return bitcast<u32>(abs(a) + max(a, b) - min(a, b)); }
        case 17u: { let v = vec3(1, 2, 3) * a + vec3<i32>(b); return bitcast<u32>(v.z - v.x + (v.yx).y); }
        default: { return bitcast<u32>(f32(a < b) + f32(true) * 2.0 + 0.5); }
    }
}
'''
SEM_OPS = 19


def sem_shader():
    return with_fs(r'''
    let x = u32(input.position.x);
    let y = u32(input.position.y);
    let v = op(y, x / 2u);
    let h = select(v & 0xFFFFu, v >> 16u, (x & 1u) == 1u);
    return vec4(f32(h & 255u) / 255.0, f32(h >> 8u) / 255.0, 0.0, 1.0);''', SEM)


def sem_expected(a, b, f):
    out = []
    w = lambda x: int(x) & 0xFFFFFFFF
    s32 = lambda x: ((int(x) + 2**31) % 2**32) - 2**31
    for op in range(SEM_OPS):
        row = []
        for i in range(32):
            A, B, Fv = int(a[i]), int(b[i]), np.float32(f[i])
            ua, ub = A & 0xFFFFFFFF, B & 0xFFFFFFFF
            if op == 0: r = w(A + B)
            elif op == 1: r = w(A - B * 3)
            elif op == 2: r = w(A * B)
            elif op in (3, 4):
                if B == 0 or (A == -2**31 and B == -1):
                    r = w(A) if op == 3 else 0
                else:
                    q = abs(A) // abs(B) * (1 if (A < 0) == (B < 0) else -1)
                    r = w(q) if op == 3 else w(A - B * q)
            elif op == 5: r = ua if ub == 0 else ua // ub
            elif op == 6: r = 0 if ub == 0 else ua % ub
            elif op == 7: r = w(ua << (ub & 31))
            elif op == 8: r = w(A >> (ub & 31))
            elif op == 9: r = ua >> (ub & 31)
            elif op == 10: r = w(0 if np.isnan(Fv) else 2**31 - 1 if Fv >= 2**31 else -2**31 if Fv < -2**31 else int(np.trunc(Fv)))
            elif op == 11: r = 0 if np.isnan(Fv) else 2**32 - 1 if Fv >= 2**32 else 0 if Fv <= -1 else int(np.trunc(Fv))
            elif op == 12: r = w(-A)
            elif op == 13: r = w(B if A < B else A)
            elif op == 14:
                s = 0
                for k in range(ub & 15):
                    if k == 3:
                        continue
                    s = (s + (ua ^ k)) & 0xFFFFFFFF
                j = 0
                while True:
                    j += 1
                    if j > 4:
                        break
                    s = (s * 3 + j) & 0xFFFFFFFF
                while s > 1000000:
                    s >>= 1
                r = s
            elif op == 15:
                x = np.float32(np.float32(np.float32(Fv * np.float32(3)) - np.float32(1.5)) + np.float32(np.float32(s32(A)) * np.float32(0.25)))
                r = int(np.array([x], np.float32).view(np.uint32)[0])
            elif op == 16:
                absA = A if A != -2**31 else A
                r = w(s32(w(abs(A) if A != -2**31 else A) + max(A, B)) - min(A, B))
            elif op == 17:
                v = [w(1 * A + B), w(2 * A + B), w(3 * A + B)]
                r = w(s32(v[2]) - s32(v[0]) + s32(v[0]))
            else:
                x = np.float32(np.float32(float(A < B)) + np.float32(2.0)) + np.float32(0.5)
                r = int(np.array([x], np.float32).view(np.uint32)[0])
            row.append(r)
        out.append(row)
    return out


@pytest.mark.gpu
def test_translator_semantics_bit_exact():
    """wrap, division by 0, INT_MIN / -1, shift masking, saturating conversions, select, loops, switch and abstract
    literals, evaluated by translated WGSL on the GPU against a numpy restatement of WGSL's rules"""
    rng = np.random.default_rng(11)
    a = rng.integers(-2**31, 2**31, 32).astype(np.int64)
    b = rng.integers(-40, 40, 32).astype(np.int64)
    a[:6] = [-2**31, -2**31, 2**31 - 1, 7, -7, 0]
    b[:6] = [-1, 0, 1, 0, 33, -1]
    f = rng.uniform(-3e9, 5e9, 32).astype(np.float32)
    f[:6] = [np.nan, 3e9, -3e9, 4.5e9, -0.75, 2147483520.0]
    # every array given in full: the bytes are tight and the shader reads each array at its uniform offset
    full = lambda arr: np.concatenate([arr, np.zeros(64 - len(arr), arr.dtype)])
    plist = lambda arr, mk: P.list([P.list([mk(full(arr)[4 * k + j]) for j in range(4)]) for k in range(16)])
    param = P.struct([("a", plist(a, lambda v: P.i32(int(v)))), ("b", plist(b, lambda v: P.i32(int(v)))),
                      ("f", plist(f, lambda v: P.f32(float(v))))])
    r = s.Renderer(s.RendererOptions(rendering_mode=s.RenderingMode.CpuOptimized))
    r.register_wgsl_shader("sem", sem_shader())
    r.update_scene("output_1", s.Resolution(64, SEM_OPS), RGBA, SH(shader_id="sem", shader_param=param, width=64, height=SEM_OPS))
    px = np.asarray(r.render(s.FrameSet(frames={}, pts=0.0)).frames["output_1"].data.planes[0]).astype(np.uint32)
    half = px[:, :, 0] | (px[:, :, 1] << 8)
    got = half[:, 0::2] | (half[:, 1::2] << 16)
    exp = np.array(sem_expected(a, b, f), np.uint64).astype(np.uint32)
    nan = lambda x: np.isnan(x.view(np.float32))
    same = (got == exp) | (nan(got) & nan(exp))   # op 15 of a NaN: any NaN
    bad = np.argwhere(~same)
    assert bad.size == 0, [(int(o), int(i), int(a[i]), int(b[i]), float(f[i]), hex(got[o, i]), hex(exp[o, i])) for o, i in bad[:10]]


# the rasteriser's edges: a plane placed by the uniform, a colour per vertex (flat / linear / perspective) and a discard
EDGE = r'''
struct E { v: array<vec4<f32>, 4>, c: vec4<f32>, d: vec4<f32>, }
@group(1) @binding(0) var<uniform> e: E;
struct VOut {
    @builtin(position) position: vec4<f32>,
    @location(0) @interpolate(flat) flat_c: f32,
    @location(1) @interpolate(linear) lin_c: f32,
    @location(2) persp_c: f32,
}
@vertex
fn vs_main(input: VertexInput) -> VOut {
    var o: VOut;
    var i = 3;
    if (input.tex_coords.x == 1.0) { i = select(0, 1, input.tex_coords.y == 0.0); } else { i = select(3, 2, input.tex_coords.y == 0.0); }
    o.position = e.v[i];
    o.flat_c = f32(i) / 3.0;
    o.lin_c = input.tex_coords.x;
    o.persp_c = input.tex_coords.y;
    return o;
}
@fragment
fn fs_main(input: VOut) -> @location(0) vec4<f32> {
    if (input.lin_c < e.d.x) { discard; }
    return vec4(input.flat_c, input.lin_c, input.persp_c, 1.0) * e.c.w + vec4(e.c.xyz, 0.0) * input.position.z;
}
'''
EDGE_SRC = """enable wgpu_binding_array;
struct VertexInput { @location(0) position: vec3<f32>, @location(1) tex_coords: vec2<f32>, }
struct BaseShaderParameters { plane_id: i32, time: f32, output_resolution: vec2<u32>, texture_count: u32, }
@group(0) @binding(0) var textures: binding_array<texture_2d<f32>, 16>;
@group(2) @binding(0) var sampler_: sampler;
var<immediate> base_params: BaseShaderParameters;
""" + EDGE
V4 = PT("list", item=PT("f32"), length=4)
EDGE_TYPE = PT("struct", fields=[("v", PT("list", item=V4, length=4)), ("c", V4), ("d", V4)])
EDGE_RESTATED = r'''
#define WO_NVARY 3
static const int wo_interp[3] = {2, 1, 0};
static const float *EP(const void *p) { return (const float *)p; }
static void wo_vs(const wo_base &, const void *params, const float *p, const float *tc, float *pos, float *vary) {
    int i = tc[0] == 1.0f ? (tc[1] == 0.0f ? 1 : 0) : (tc[1] == 0.0f ? 2 : 3);
    for (int k = 0; k < 4; k++) pos[k] = EP(params)[4 * i + k];
    vary[0] = (float)i / 3.0f; vary[1] = tc[0]; vary[2] = tc[1];
}
static bool wo_fs(const wo_base &, const void *params, const smr_textures &, const float *fp, const float *v, float4 &out) {
    const float *c = EP(params) + 16, *d = EP(params) + 20;
    if (v[1] < d[0]) return false;
    out = make_float4(v[0] * c[3] + c[0] * fp[2], v[1] * c[3] + c[1] * fp[2], v[2] * c[3] + c[2] * fp[2], 1.0f * c[3] + 0.0f * fp[2]);
    return true;
}
'''


def edge_param(verts, c=(0.0, 0.0, 0.0, 1.0), discard_below=-1.0):
    v4 = lambda x: P.list([P.f32(float(t)) for t in x])
    return P.struct([("v", P.list([v4(v) for v in verts])), ("c", v4(c)), ("d", v4((discard_below, 0, 0, 0)))])


PLANE = [(1, -1, 0, 1), (1, 1, 0, 1), (-1, 1, 0, 1), (-1, -1, 0, 1)]
EDGE_CASES = {
    "full plane": edge_param(PLANE),
    "mirrored plane is culled": edge_param([(-x, y, z, w) for x, y, z, w in PLANE]),
    "partly off the target": edge_param([(1.7, -0.3, 0, 1), (1.7, 1.9, 0, 1), (-0.4, 1.9, 0, 1), (-0.4, -0.3, 0, 1)]),
    "fractional edges, translucent": edge_param([(0.613, -0.377, 0, 1), (0.7, 0.811, 0, 1), (-0.523, 0.59, 0, 1), (-0.61, -0.6, 0, 1)],
                                                c=(0.0, 0.0, 0.0, 0.5)),
    "depth outside [0, 1]": edge_param([(1, -1, -0.5, 1), (1, 1, 0.5, 1), (-1, 1, 1.5, 1), (-1, -1, 0.5, 1)], c=(0.3, 0.2, 0.1, 0.25)),
    "perspective": edge_param([(2, -2, 0.5, 2), (0.5, 0.5, 0.25, 0.5), (-1, 1, 0.5, 1), (-1.5, -1.5, 0.5, 1.5)]),
    "discard": edge_param(PLANE, discard_below=0.37),
    "w <= 0 draws no plane": edge_param([(1, -1, 0, 1), (1, 1, 0, 1), (-1, 1, 0, -1), (-1, -1, 0, 1)]),
}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", TW.MODES)
@pytest.mark.parametrize("case", sorted(EDGE_CASES))
def test_rasteriser_edges_match_oracle(case, mode):
    p = Pair(out=(97, 61), fmt=RGBA, mode=mode, inputs=())
    p.register_wgsl("edge", None, src=EDGE_SRC, restated=EDGE_RESTATED, param_type=EDGE_TYPE)
    p.update(SH(shader_id="edge", shader_param=EDGE_CASES[case], width=97, height=61))
    p.render_check(0.0, case)
    got = np.asarray(p.r.render(s.FrameSet(frames={}, pts=0.0)).frames["output_1"].data.planes[0])
    if case in ("mirrored plane is culled", "w <= 0 draws no plane"):
        assert not got.any()
    elif case == "fractional edges, translucent":   # the diagonal is blended once: no pixel darker than one layer's alpha
        assert set(np.unique(got[..., 3]).tolist()) <= {0, 128}
    elif case not in ("full plane", "perspective"):
        assert got[..., 3].any() and not got[..., 3].all()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", TW.FORMATS)
@pytest.mark.parametrize("mode", TW.MODES)
def test_mixed_wgsl_and_cuda_shaders_match_oracle(mode, fmt):
    """WGSL and CUDA shader nodes in one scene, nested both ways, over layouts and inputs; one launch per (depth, shader)"""
    p = Pair(out=(640, 360), fmt=fmt, mode=mode, inputs=("input_1", "input_2", "input_3"))
    for k in TS.SOURCES:
        p.register_shader(k)
    p.register_wgsl("layout_planes", "layout_planes")
    p.register_wgsl("circle_layout", "circle_layout", param_type=CIRCLE_TYPE)
    inner = lambda: SH(shader_id="grade", shader_param=TS.grade(), width=320, height=180, children=[IN(input_id="input_2")])
    view = lambda: V(position=s.Position.Static(width=320.0, height=180.0), background_color=s.RGBAColor(40, 0, 60, 200),
                     children=[IN(input_id="input_1"), IN(input_id="input_3")])
    p.update(V(background_color=s.RGBAColor(10, 20, 30, 255), children=[
        SH(shader_id="layout_planes", width=640, height=360, children=[
            inner(), view(), SH(shader_id="circle_layout", shader_param=circle_param(320, 180), width=320, height=180,
                                children=[IN(input_id="input_1"), inner(), view(), IN(input_id="input_2")]),
            IN(input_id="input_3")])]))
    p.r.set_profiling(True)
    p.render_check(0.5, "mixed")
    # (grade, 1); (circle_layout, 2) over inner and the View node; (layout_planes, 3)
    assert p.r.kernel_times()["shader"][1] == 3
