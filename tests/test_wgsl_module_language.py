"""WGSL module language in registered shaders (smr_register_wgsl_shader): var<private>, texture and sampler values, alias,
const_assert, hexadecimal float literals, @size / @align, an fs_main struct result and diagnostic filters.

CPU (host-only handle): every construct registers, every misuse answers SMR_ERR_INVALID_ARGUMENT at its line and column,
hexadecimal literals and const-evaluation through const_assert, and the parameter type derived through aliases and
@size / @align.  GPU, byte for byte, both modes, three NV12 children: each construct renders what the same shader written
without it renders; private state starts afresh in every vs_main and fs_main invocation; fields moved by @align / @size
read the words a numpy restatement of WGSL's uniform layout places there; and a shader with texture parameters and
private state matches a hand-written restatement on tests/wgsl_oracle_shim.h.
"""
import numpy as np
import pytest

import smelter_b200 as s
from tests import test_shader_component as TS
from tests import test_web_view_component as TW
from tests.test_wgsl_builtins import _line_col, tex_shader
from tests.test_wgsl_shader import FS, HEADER, IDENTITY_VS, SAMPLE, Pair, host, status

IN, SH, P = s.InputStreamComponent, s.ShaderComponent, s.ShaderParam
RGBA = TW.RGBA


def fs(body, extra="", result="@location(0) vec4<f32>"):
    return HEADER + extra + f"\n@fragment\nfn fs_main(input: VertexOutput) -> {result} {{\n{body}\n}}\n"


# ---- CPU ------------------------------------------------------------------------------------------------------------
TAP = "fn tap(t: texture_2d<f32>, s: sampler, uv: vec2<f32>) -> vec4<f32> { return textureSample(t, s, uv); }\n"
REGISTERS = {
    "var<private> forms": fs("a += 1; b = b * 2.0; c.x = 1.0; return vec4(f32(a), b, c.x, c.y);",
                            "var<private> a: i32;\nvar<private> b: f32 = 0.5;\nvar<private> c = vec2(1.0, 2.0);\n"),
    "var<private> of a struct and an array": fs("s.v[1] = 2.0; return vec4(s.v[1], f32(s.n), k[2], 1.0);",
                                                "struct St { v: vec4<f32>, n: u32 }\nconst K = 3.0;\nvar<private> s: St;\n"
                                                "var<private> k = array<f32, 3>(1.0, 2.0, K);\n"),
    "texture parameters": fs("return tap(textures[0], sampler_, input.tex_coords);", TAP),
    "texture lets": fs("let t = textures[1];\n    let s = sampler_;\n    return tap(t, s, input.tex_coords) + textureGather(1, t, s, input.tex_coords)"
                       " + vec4(f32(textureDimensions(t).x + textureNumLevels(t))) + textureSampleLevel(t, s, input.tex_coords, 0.0);", TAP),
    "alias": fs("let v: V = V(1.0, 2.0, 3.0, 4.0);\n    let a = A(F(1), 2.0);\n    return v * a[1];",
                "alias F = f32;\nalias V = vec4<F>;\nalias A = array<F, 2>;\n"),
    "alias in the header": fs("return vec4(1.0);").replace("var textures: binding_array<texture_2d<f32>, 16>", "var textures: Tex")
                                                  .replace("var<immediate> base_params: BaseShaderParameters", "var<immediate> base_params: B")
                           + "alias Tex = binding_array<texture_2d<f32>, 16>;\nalias B = BaseShaderParameters;\n",
    "const_assert": fs("const_assert 2 > 1;\n    return vec4(1.0);", "const_assert 0x1.8p1 == 3.0;\nconst k = 4u;\nconst_assert k * 2u == 8u;\n"),
    "hexadecimal floats": fs("return vec4(0x1.8p1, 0x.8p0, 0X1P-2f, 0x1.8) * 0x1p-3 + vec4(f32(0x1f));"),
    "@size and @align": fs("return u.b;", "struct U { a: f32, @align(32) b: vec4<f32>, @size(20) c: f32, d: vec2<f32> }\n"
                                         "@group(1) @binding(0) var<uniform> u: U;\n"),
    "fs_main struct result": fs("var o: FragmentOutput;\n    o.color = vec4(1.0);\n    return o;",
                                "struct FragmentOutput { @location(0) color: vec4<f32> }\n", "FragmentOutput"),
    "diagnostic": "diagnostic(off, derivative_uniformity);\ndiagnostic(warning, my.rule,);\n" +
                  fs("@diagnostic(off, derivative_uniformity) { }\n    return vec4(1.0);").replace("@fragment", "@diagnostic(info, derivative_uniformity)\n@fragment"),
}


@pytest.mark.parametrize("name", sorted(REGISTERS))
def test_construct_registers(name):
    host().register_wgsl_shader("x", REGISTERS[name])


UNI = "@group(1) @binding(0) var<uniform> u: U;\n"
MISUSES = {   # (source, the text at the position the refusal names)
    "private initializer not const": (fs("return vec4(p);", "struct U { a: f32 }\n" + UNI + "var<private> p = u.a;\n"), ".a;"),
    "private initializer calls a function": (fs("return vec4(p);", "fn one() -> f32 { return 1.0; }\nvar<private> p = one();\n"), "one();"),
    "private texture": (fs("return vec4(1.0);", "var<private> t: texture_2d<f32>;\n"), "var<private> t"),
    "private sampler": (fs("return vec4(1.0);", "var<private> q: sampler;\n"), "var<private> q"),
    "private with a binding": (fs("return vec4(1.0);", "@group(3) @binding(0) var<private> z: f32;\n"), "var<private> z"),
    "var of a texture": (fs("var t = textures[0];\n    return vec4(1.0);"), "var t = "),
    "typed var of a sampler": (fs("var q: sampler;\n    return vec4(1.0);"), "var q"),
    "returning a texture": (fs("return vec4(1.0);", "fn pick() -> texture_2d<f32> { return textures[0]; }\n"), "texture_2d<f32> { return"),
    "returning a sampler": (fs("return vec4(1.0);", "fn smp() -> sampler { return sampler_; }\n"), "sampler { return"),
    "struct member texture": (fs("return vec4(1.0);", "struct H { t: texture_2d<f32> }\n"), "t: texture_2d<f32> }"),
    "fs_main texture parameter": (fs("return vec4(1.0);").replace("fn fs_main(input: VertexOutput)", "fn fs_main(input: VertexOutput, tt: texture_2d<f32>)"), "tt:"),
    "alias cycle": (fs("return vec4(1.0);", "alias A1 = B1;\nalias B1 = A1;\n"), "alias B1"),
    "alias cycle through an array": (fs("return vec4(1.0);", "alias C1 = array<C1, 2>;\n"), "alias C1"),
    "alias redeclared": (fs("return vec4(1.0);", "alias V = vec4<f32>;\nalias V = vec2<f32>;\n"), "alias V = vec2"),
    "alias named as a struct": (fs("return vec4(1.0);", "alias VertexOutput = vec4<f32>;\n"), "alias VertexOutput"),
    "alias unknown target": (fs("return vec4(1.0);", "alias X = nope;\n"), "nope"),
    "const_assert false": (fs("return vec4(1.0);", "const_assert 0x1.8p1 == 3.5;\n"), "const_assert"),
    "const_assert false in a function": (fs("const k = 2;\n    const_assert k == 3;\n    return vec4(1.0);"), "const_assert"),
    "const_assert of a let": (fs("let y = 1;\n    const_assert y == 1;\n    return vec4(1.0);"), "y == 1"),
    "const_assert of a uniform": (fs("return vec4(1.0);", "struct U { a: f32 }\n" + UNI + "const_assert u.a == 0.0;\n"), "u.a == 0.0"),
    "const_assert not bool": (fs("return vec4(1.0);", "const_assert 1;\n"), "1;"),
    "hex float not exact in f32": (fs("return vec4(0x1.000001p0f);"), "0x1.000001p0f"),
    "hex float not exact in f64": (fs("return vec4(0x1.00000000000001p0);"), "0x1.00000000000001p0"),
    "hex float out of range": (fs("return vec4(0x1p128f);"), "0x1p128f"),
    "@align not a power of two": (fs("return u.b;", "struct U { a: f32, @align(24) b: vec4<f32> }\n" + UNI), "align(24)"),
    "@align of zero": (fs("return u.b;", "struct U { a: f32, @align(0) b: vec4<f32> }\n" + UNI), "align(0)"),
    "@size below SizeOf": (fs("return u.b;", "struct U { @size(8) a: vec4<f32>, b: vec4<f32> }\n" + UNI), "size(8)"),
    "@align below the type's alignment": (fs("return u.b;", "struct U { a: f32, @align(4) b: vec4<f32> }\n" + UNI), "align(4)"),
    "@align below the type's alignment, value type": (fs("return vec4(1.0);", "struct Q { a: f32, @align(8) b: vec3<f32> }\n"), "align(8)"),
    "diagnostics in conflict": ("diagnostic(off, derivative_uniformity);\ndiagnostic(error, derivative_uniformity);\n" + fs("return vec4(1.0);"),
                                "diagnostic(error"),
    "attributes in conflict": (fs("return vec4(1.0);").replace("@fragment", "@diagnostic(off, x) @diagnostic(info, x) @fragment"), "diagnostic(info"),
    "unknown severity": ("diagnostic(loud, derivative_uniformity);\n" + fs("return vec4(1.0);"), "loud"),
    "diagnostic directive after a declaration": (fs("return vec4(1.0);") + "diagnostic(off, derivative_uniformity);\n", "diagnostic(off"),
    "@diagnostic on a struct member": (fs("return vec4(1.0);", "struct D { @diagnostic(off, x) a: f32 }\n"), "diagnostic(off, x) a"),
    "@diagnostic on a global": (fs("return vec4(1.0);", "@diagnostic(off, x) var<private> dg: f32;\n"), "diagnostic(off, x) var"),
    "@diagnostic on a let": (fs("@diagnostic(off, x) let y = 1.0;\n    return vec4(y);"), "diagnostic(off, x) let"),
}


@pytest.mark.parametrize("name", sorted(MISUSES))
def test_misuse_is_invalid_with_a_position(name):
    src, at = MISUSES[name]
    st, msg = status(host(), src)
    assert st == 1, msg
    assert "WGSL " + _line_col(src, at) + ":" in msg, (msg, _line_col(src, at))


STILL_UNSUPPORTED = {
    "requires": "requires readonly_and_readwrite_storage_textures;\n" + fs("return vec4(1.0);"),
    "h suffix on a hex float": fs("return vec4(f32(0x1p1h));"),
    "two-member result": fs("var o: O2;\n    return o;", "struct O2 { @location(0) c: vec4<f32>, @location(1) d: vec4<f32> }\n", "O2"),
    "result at location 1": fs("var o: O1;\n    return o;", "struct O1 { @location(1) c: vec4<f32> }\n", "O1"),
    "binding array let": fs("let a = textures;\n    return vec4(1.0);"),
    "workgroup": fs("return vec4(1.0);", "var<workgroup> w: f32;\n"),
}


@pytest.mark.parametrize("name", sorted(STILL_UNSUPPORTED))
def test_still_unsupported(name):
    st, msg = status(host(), STILL_UNSUPPORTED[name])
    assert st == 5, msg


# const-evaluation and hexadecimal literals, both sides of each assert: (holds, does not hold)
CONST_ASSERTS = [
    ("0x1.8p1 == 3.0", "0x1.8p1 == 3.5"),
    ("0x.8p0 == 0.5", "0x.8p0 == 0.25"),
    ("0X1P-2f == 0.25f", "0X1P-2f == 0.5f"),
    ("0x1.8 == 1.5", "0x1.8 == 1.8"),
    ("0x1f == 31", "0x1f == 1.0"),
    ("0x1.fffffep127f > 3.4e38f", "0x1.fffffep127f < 3.4e38f"),
    ("0x1p-149f > 0.0f", "0x1p-149f == 0.0f"),
    ("0x1.8p-1 + 0x.4p0 == 1.0", "0x1.8p-1 + 0x.4p0 == 1.25"),
    ("0.1 + 0.2 != 0.3", "0.1 + 0.2 == 0.3"),                       # abstract floats compare in f64
    ("0.1f + 0.2f == 0.3f", "0.1f + 0.2f != 0.3f"),                  # f32 arithmetic rounds each step
    ("-7 / 2 == -3 && -7 % 2 == -1", "-7 / 2 == -4"),
    ("(1u << 31u) == 0x80000000u", "(1u << 31u) == 0u"),
    ("i32(2.9) == 2 && u32(-1.5f) == 0u && i32(3e9f) == 2147483647", "i32(2.9) == 3"),
    ("all(vec3(1, 2, 3) == vec3<i32>(1, 2, 3))", "all(vec3(1, 2, 3) != vec3<i32>(1, 2, 4))"),
    ("vec4(1.0, 2.0, 3.0, 4.0).zy.x == 3.0", "vec4(1.0, 2.0, 3.0, 4.0).w == 3.0"),
    ("select(1, 2, true) == 2 && max(3u, 5u) == 5u && abs(-2.5) == 2.5", "select(1, 2, false) == 2"),
    ("KF * 2.0 == 3.0f && KI + 1 == 8 && KV.y == 2.0", "KF == 1.0"),
]
CONSTS = "const KF: f32 = 0x1.8p0;\nconst KI = 7;\nconst KV = vec2<f32>(1.0, 2.0);\n"


@pytest.mark.parametrize("i", range(len(CONST_ASSERTS)))
def test_const_assert_evaluates(i):
    holds, fails = CONST_ASSERTS[i]
    r = host()
    r.register_wgsl_shader("ok", fs("const_assert " + holds + ";\n    return vec4(1.0);", CONSTS + f"const_assert {holds};\n"))
    src = fs("return vec4(1.0);", CONSTS + f"const_assert {fails};\n")
    st, msg = status(r, src, "bad")
    assert st == 1 and "const_assert failed" in msg and _line_col(src, "const_assert " + fails) in msg, msg


def test_const_assert_over_an_unevaluated_builtin_is_unsupported():
    st, msg = status(host(), fs("return vec4(1.0);", "const k = sqrt(4.0);\nconst_assert k == 2.0;\n"))
    assert st == 5, msg


def test_parameter_type_through_aliases_and_layout_attributes():
    """the aliased shader, whose struct members move under @align / @size, accepts and refuses the same parameters as
    the spelled-out one: the derived parameter types are the same"""
    spelled = fs("return u.b;", "struct S3 { x: f32 }\nstruct U { a: f32, b: vec4<f32>, c: f32, d: vec2<u32>, n: S3 }\n" + UNI)
    aliased = fs("return u.b;", "alias F = f32;\nstruct S3 { @size(16) x: F }\nalias N = S3;\n"
                                "struct U { a: F, @align(32) b: vec4<F>, @size(20) c: F, d: vec2<u32>, @align(16) n: N }\nalias UU = U;\n"
                                "@group(1) @binding(0) var<uniform> u: UU;\n")
    f, u = P.f32, P.u32
    fields = [("a", f(1)), ("b", P.list([f(2)] * 4)), ("c", f(3)), ("d", P.list([u(4)] * 2)), ("n", P.struct([("x", f(5))]))]
    with_field = lambda k, v: P.struct([(i, v if i == k else x) for i, x in fields])
    bad = [with_field("b", P.list([f(2)] * 3)),                 # a vector of 3
           with_field("d", P.list([f(4)] * 2)),                 # f32 for u32
           with_field("n", P.struct([("y", f(5))])),            # another member name
           with_field("a", P.u32(1)),                           # u32 for f32
           P.struct(fields[:4]),                                # a field missing
           f(1.0)]
    p = TS.host(inputs=("input_1",))
    p.r.register_wgsl_shader("spelled", spelled)
    p.r.register_wgsl_shader("aliased", aliased)
    for sid in ("spelled", "aliased"):
        p.r.update_scene("output_1", s.Resolution(640, 360), TW.YUV, SH(shader_id=sid, shader_param=P.struct(fields), width=64, height=64))
        for param in bad:
            assert TS._status(p.r, SH(shader_id=sid, shader_param=param, width=64, height=64)) == 4, (sid, param)


# ---- the uniform layout, restated -----------------------------------------------------------------------------------
# WGSL (memory layout): AlignOf / SizeOf of f32 4 / 4, vec2 8 / 8, vec4 16 / 16; array<E, N>: AlignOf(E), stride
# roundUp(AlignOf(E), SizeOf(E)); struct: members at roundUp(AlignOfMember, end of the previous one), AlignOfMember @align
# or AlignOf(T), SizeOfMember @size or SizeOf(T); AlignOf the members' largest, SizeOf roundUp(AlignOf, end).
def _up(k, n):
    return (n + k - 1) // k * k


def wgsl_layout(t):
    """(align, size, [(leaf path, byte offset)]) of a type: 'f32', ('vec', n), ('array', elem, n), ('struct', members)
    with members (name, type, align or None, size or None)"""
    if t == "f32":
        return 4, 4, [("", 0)]
    if t[0] == "vec":
        return (8 if t[1] == 2 else 16), 4 * t[1], [(f".{'xyzw'[i]}", 4 * i) for i in range(t[1])]
    if t[0] == "array":
        a, sz, leaves = wgsl_layout(t[1])
        stride = _up(a, sz)
        return a, stride * t[2], [(f"[{i}]{p}", i * stride + o) for i in range(t[2]) for p, o in leaves]
    off, al, out = 0, 1, []
    for name, mt, ma, ms in t[1]:
        a, sz, leaves = wgsl_layout(mt)
        a, sz = ma or a, ms or sz
        off = _up(a, off)
        out += [(f".{name}{p}", off + o) for p, o in leaves]
        off += sz
        al = max(al, a)
    return al, _up(al, off), out


LAYOUT_T = ("struct", [("a", "f32", None, None), ("b", ("vec", 4), 32, None), ("c", "f32", None, 20), ("d", ("vec", 2), None, None),
                       ("e", ("array", ("struct", [("x", "f32", 16, 36)]), 2), None, None), ("f", "f32", 16, None),
                       ("g", ("array", ("vec", 4), 8), None, None)])
LAYOUT_WGSL = """struct S2 { @align(16) @size(36) x: f32 }
struct U { a: f32, @align(32) b: vec4<f32>, @size(20) c: f32, d: vec2<f32>, e: array<S2, 2>, @align(16) f: f32, g: array<vec4<f32>, 8> }
@group(1) @binding(0) var<uniform> u: U;
"""
LEAVES = [".a", ".b.x", ".b.y", ".b.w", ".c", ".d.x", ".d.y", ".e[0].x", ".e[1].x", ".f", ".g[0].x", ".g[3].w", ".g[7].y"]


def test_layout_restatement_offsets():
    al, size, leaves = wgsl_layout(LAYOUT_T)
    off = dict(leaves)
    assert (al, size) == (32, 320)
    assert [off[k] for k in (".a", ".b.x", ".c", ".d.x", ".e[0].x", ".e[1].x", ".f", ".g[0].x")] == [0, 32, 48, 72, 80, 128, 176, 192]


def layout_shaders():
    """the shader reading LEAVES through U, and the same reads at the restatement's offsets into raw vec4 words"""
    _, size, leaves = wgsl_layout(LAYOUT_T)
    off = dict(leaves)
    n = len(LEAVES)
    body = "    let k = u32(input.position.x) % {n}u;\n    let v = array<f32, {n}>({vals});\n" \
           "    return vec4(v[k], v[(k + 5u) % {n}u], v[(k + 9u) % {n}u], 1.0);"
    a = fs(body.format(n=n, vals=", ".join("u" + p for p in LEAVES)), LAYOUT_WGSL)
    raw = ", ".join(f"raw[{off[p] // 16}][{off[p] % 16 // 4}]" for p in LEAVES)
    b = fs(body.format(n=n, vals=raw), f"@group(1) @binding(0) var<uniform> raw: array<vec4<f32>, {size // 16}>;\n")
    return a, b, size


def layout_params(size):
    """the same tight bytes (ShaderParam::to_bytes) for both: U's 43 scalars, and those zero-padded as raw words"""
    vals = [(j + 1) / 64.0 for j in range(43)]
    it = iter(vals)
    f = lambda: P.f32(next(it))
    pu = P.struct([("a", f()), ("b", P.list([f() for _ in range(4)])), ("c", f()), ("d", P.list([f(), f()])),
                   ("e", P.list([P.struct([("x", f())]) for _ in range(2)])), ("f", f()),
                   ("g", P.list([P.list([f() for _ in range(4)]) for _ in range(8)]))])
    words = vals + [0.0] * (size // 4 - len(vals))
    praw = P.list([P.list([P.f32(words[4 * i + c]) for c in range(4)]) for i in range(size // 16)])
    assert TS.param_bytes(pu) + bytes(size - 4 * len(vals)) == TS.param_bytes(praw)
    return pu, praw


def test_layout_shaders_register():
    a, b, size = layout_shaders()
    r = host()
    r.register_wgsl_shader("a", a)
    r.register_wgsl_shader("b", b)
    layout_params(size)


# ---- GPU: equivalence ---------------------------------------------------------------------------------------------
INPUTS = ("nv12_1", "nv12_2", "nv12_3")
W, H = 320, 180


def _tap(T, uv):
    return (f"(textureSample({T}, sampler_, {uv}) * 0.5 + textureGather(2, {T}, sampler_, ({uv}).yx) * 0.25"
            f" + textureSampleLevel({T}, sampler_, ({uv}) * 0.5, 1.0) * 0.125"
            f" + vec4(f32(textureDimensions({T}).x) / 4096.0, f32(textureDimensions({T}).y) / 4096.0, 0.0, 0.0))")


ORDER_PRE = """var<private> state: u32;
var<private> acc: f32;
var<private> arr: array<f32, 3>;
fn rand() -> f32 {
    state = state * 747796405u + 2891336453u;
    return f32(state >> 8u) / 16777216.0;
}
fn ri() -> u32 { return u32(rand() * 3.0); }
fn bump() -> f32 {
    acc = acc * 4.0 + 0.25;
    return acc;
}
"""
ORDER_SEED = """    state = u32(input.position.x) * 1973u + u32(input.position.y) * 9277u + u32(base_params.plane_id) * 26699u;
    acc = 0.5;
"""
ORDER_OUT = """
    let o = vec4(fract(v.x * 3.0 + v.y), fract(m * 5.0 + q[0].y * 2.0 + q[1].x), fract(acc + arr[0] + arr[1] * 2.0 + arr[2] * 4.0), 0.5);
    return o * 0.5 + c * 0.25 + g * 0.125;"""
EQUIVALENT = {   # (with the construct, written without it)
    "var<private>": (
        tex_shader("""    let i = u32(base_params.plane_id);
    add(textureSample(textures[i], sampler_, input.tex_coords));
    add(textureSample(textures[(i + 1u) % 3u], sampler_, input.tex_coords.yx));
    return acc * 0.125 + vec4(0.0, 0.0, f32(n) * 0.03125, 0.0);
}
var<private> acc: vec4<f32>;
var<private> n = 2;
fn add(c: vec4<f32>) {
    acc += c * f32(n);
    n += 1;"""),
        tex_shader("""    let i = u32(base_params.plane_id);
    var acc: vec4<f32>;
    var n = 2;
    acc += textureSample(textures[i], sampler_, input.tex_coords) * f32(n);
    n += 1;
    acc += textureSample(textures[(i + 1u) % 3u], sampler_, input.tex_coords.yx) * f32(n);
    n += 1;
    return acc * 0.125 + vec4(0.0, 0.0, f32(n) * 0.03125, 0.0);""")),
    "texture values": (
        tex_shader("""    let i = u32(base_params.plane_id);
    let t = textures[i + 1u];
    let s = sampler_;
    return twice(t, s, input.tex_coords) * 0.5 + tap(textures[i], sampler_, input.tex_coords * 1.5) * 0.25;
}
fn tap(t: texture_2d<f32>, s: sampler, uv: vec2<f32>) -> vec4<f32> {
    let d = vec2<f32>(textureDimensions(t));
    return textureSample(t, s, uv) * 0.5 + textureGather(2, t, s, uv.yx) * 0.25 + textureSampleLevel(t, s, uv * 0.5, 1.0) * 0.125
        + vec4(d.x / 4096.0, d.y / 4096.0, 0.0, 0.0);
}
fn twice(t: texture_2d<f32>, s: sampler, uv: vec2<f32>) -> vec4<f32> {
    return tap(t, s, uv) * 0.5 + tap(t, s, uv.yx) * 0.25;"""),
        tex_shader(f"""    let i = u32(base_params.plane_id);
    return ({_tap("textures[i + 1u]", "input.tex_coords")} * 0.5 + {_tap("textures[i + 1u]", "(input.tex_coords).yx")} * 0.25) * 0.5
        + {_tap("textures[i]", "input.tex_coords * 1.5")} * 0.25;""")),
    "alias": (
        tex_shader("""    let w = Arr3(0.5, 0.25, 0.125);
    let c: V4 = textureSample(textures[U(base_params.plane_id)], sampler_, input.tex_coords);
    return c * pick(w, U(base_params.plane_id)) + V4(F(0.0), 0.0, 0.0, 0.0625);
}
alias V4 = vec4<F>;
alias F = f32;
alias Arr3 = array<F, 3>;
alias U = u32;
fn pick(a: Arr3, k: U) -> F {
    return a[k];""").replace("var textures: binding_array<texture_2d<f32>, 16>;", "var textures: Tex;\nalias Tex = binding_array<texture_2d<f32>, 16>;"),
        tex_shader("""    let w = array<f32, 3>(0.5, 0.25, 0.125);
    let c: vec4<f32> = textureSample(textures[u32(base_params.plane_id)], sampler_, input.tex_coords);
    return c * pick(w, u32(base_params.plane_id)) + vec4<f32>(f32(0.0), 0.0, 0.0, 0.0625);
}
fn pick(a: array<f32, 3>, k: u32) -> f32 {
    return a[k];""")),
    "hexadecimal floats, const_assert and diagnostic": (
        "diagnostic(off, derivative_uniformity);\n" + tex_shader("""    const_assert 0x10 == 16;
    let c = textureSample(textures[u32(base_params.plane_id)], sampler_, input.tex_coords * 0x1.8p0 - vec2(0x.4p0));
    return c * 0x1p-1f + vec4(0x1.8p-3, 0x.1p0, 0X1P-4f, 0x1.0p-2);
}
const_assert 0x1.8p1 == 3.0;
@diagnostic(off, derivative_uniformity)
fn unused() {"""),
        tex_shader("""    let c = textureSample(textures[u32(base_params.plane_id)], sampler_, input.tex_coords * 1.5 - vec2(0.25));
    return c * 0.5f + vec4(0.1875, 0.0625, 0.0625f, 0.25);""")),
    "fs_main struct result": (
        HEADER + """struct FragmentOutput { @location(0) color: vec4<f32> }
@fragment
fn fs_main(input: VertexOutput) -> FragmentOutput {
    var o: FragmentOutput;
    o.color = textureSample(textures[u32(base_params.plane_id)], sampler_, input.tex_coords) * 0.5;
    if (input.tex_coords.x > 0.75) { discard; }
    return o;
}
""",
        tex_shader("""    let c = textureSample(textures[u32(base_params.plane_id)], sampler_, input.tex_coords) * 0.5;
    if (input.tex_coords.x > 0.75) { discard; }
    return c;""")),
    # every vs_main and fs_main invocation starts from the initial value: the counters read 1 in each vertex, and in
    # each fragment of the three planes (alpha 0 adds every plane's value to the pixel)
    "per-invocation reset": (
        tex_shader("""    let k = bump();
    return vec4(f32(k) * 0.125, input.tex_coords.x * 0.25, f32(fcount) * 0.0625, 0.0);
}
var<private> vcount: i32;
var<private> fcount = 0u;
fn bump() -> u32 {
    fcount++;
    return fcount;""", vs="""@vertex
fn vs_main(input: VertexInput) -> VertexOutput {
    var output: VertexOutput;
    vcount += 1;
    output.position = vec4(input.position * f32(vcount), 1.0);
    output.tex_coords = input.tex_coords * f32(vcount);
    return output;
}
"""),
        tex_shader("    return vec4(0.125, input.tex_coords.x * 0.25, 0.0625, 0.0);", vs="""@vertex
fn vs_main(input: VertexInput) -> VertexOutput {
    var output: VertexOutput;
    output.position = vec4(input.position * 1.0, 1.0);
    output.tex_coords = input.tex_coords * 1.0;
    return output;
}
""")),
    # WGSL evaluates operands left to right.  A private PRNG drawn several times in one constructor, builtin, texture
    # builtin, compound assignment (whose right side writes the left) and indexed assignment, against the same draws
    # sequenced by lets
    "evaluation order": (tex_shader(ORDER_SEED + """    let v = vec2(rand(), rand());
    let m = mix(rand(), rand(), 0.25);
    let q = mat2x2<f32>(rand(), rand(), rand(), rand());
    acc += bump();
    arr[ri()] = rand();
    let c = textureSampleLevel(textures[ri()], sampler_, vec2(rand(), rand()), rand());
    let g = textureGather(1, textures[ri()], sampler_, vec2(rand(), rand()));""" + ORDER_OUT) + ORDER_PRE,
                         tex_shader(ORDER_SEED + """    let r0 = rand();
    let r1 = rand();
    let v = vec2(r0, r1);
    let r2 = rand();
    let r3 = rand();
    let m = mix(r2, r3, 0.25);
    let r4 = rand();
    let r5 = rand();
    let r6 = rand();
    let r7 = rand();
    let q = mat2x2<f32>(r4, r5, r6, r7);
    let old = acc;
    let b = bump();
    acc = old + b;
    let i = ri();
    let r8 = rand();
    arr[i] = r8;
    let t0 = ri();
    let r9 = rand();
    let r10 = rand();
    let r11 = rand();
    let c = textureSampleLevel(textures[t0], sampler_, vec2(r9, r10), r11);
    let t1 = ri();
    let r12 = rand();
    let r13 = rand();
    let g = textureGather(1, textures[t1], sampler_, vec2(r12, r13));""" + ORDER_OUT) + ORDER_PRE),
}


def test_equivalent_shaders_register():
    r = host()
    for name, (a, b) in EQUIVALENT.items():
        r.register_wgsl_shader(name + " with", a)
        r.register_wgsl_shader(name + " without", b)


def _draw(p, sid, src, param=None):
    p.r.register_wgsl_shader(sid, src)
    p.r.update_scene("output_1", s.Resolution(W, H), RGBA,
                     SH(shader_id=sid, shader_param=param, width=W, height=H, children=[IN(input_id=k) for k in INPUTS]))
    return np.asarray(p.r.render(s.FrameSet(frames=p.frames(0.25), pts=0.25)).frames["output_1"].data.planes[0]).copy()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", TW.MODES)
@pytest.mark.parametrize("name", sorted(EQUIVALENT))
def test_construct_renders_as_without_it(name, mode):
    p = TW.Pair(out=(W, H), fmt=RGBA, mode=mode, inputs=INPUTS)
    with_it, without = EQUIVALENT[name]
    a, b = _draw(p, "with", with_it), _draw(p, "without", without)
    assert b.any()
    bad = np.argwhere((a != b).any(axis=-1))
    assert bad.size == 0, (name, bad[:5].tolist(), a[tuple(bad[0])].tolist(), b[tuple(bad[0])].tolist())


@pytest.mark.gpu
@pytest.mark.parametrize("mode", TW.MODES)
def test_layout_attributes_read_the_restated_offsets(mode):
    a, b, size = layout_shaders()
    pu, praw = layout_params(size)
    p = TW.Pair(out=(W, H), fmt=RGBA, mode=mode, inputs=INPUTS)
    got, exp = _draw(p, "attrs", a, pu), _draw(p, "raw", b, praw)
    assert len(np.unique(exp[..., 0])) > 8   # the reads differ from field to field
    assert np.array_equal(got, exp)


# ---- GPU: the oracle ------------------------------------------------------------------------------------------------
# two taps through a helper taking a texture and the sampler; its private weight halves at every call (WGSL evaluates
# the two calls left to right) and the private count of taps reaches fs_main's result
ORACLE_SRC = tex_shader("""    let t = textures[base_params.plane_id];
    let s = sampler_;
    let c = tap(t, s, input.tex_coords) + tap(textures[2], s, input.tex_coords.yx);
    return c + vec4(f32(taps) * 0.0625, 0.0, 0.0, 0.0625);
}
var<private> weight: f32 = 0.5;
var<private> taps: u32;
fn tap(t: texture_2d<f32>, s: sampler, uv: vec2<f32>) -> vec4<f32> {
    taps += 1u;
    weight = weight * 0.5;
    return textureSample(t, s, uv) * weight;""")
ORACLE_RESTATED = IDENTITY_VS + SAMPLE + FS + r'''
    float w = 0.5f;
    unsigned taps = 0;
    float4 k[2];
    const int idx[2] = {b.plane_id, 2};
    const float uv[2][2] = {{tc[0], tc[1]}, {tc[1], tc[0]}};
    for (int j = 0; j < 2; j++) {
        taps += 1;
        w = w * 0.5f;
        const float4 c = S(t, idx[j], uv[j][0], uv[j][1]);
        k[j] = make_float4(c.x * w, c.y * w, c.z * w, c.w * w);
    }
    out = make_float4((k[0].x + k[1].x) + (float)taps * 0.0625f, (k[0].y + k[1].y) + 0.0f, (k[0].z + k[1].z) + 0.0f,
                      (k[0].w + k[1].w) + 0.0625f);
    return true; }'''


@pytest.mark.gpu
@pytest.mark.parametrize("mode", TW.MODES)
def test_texture_parameters_and_private_state_match_oracle(mode):
    p = Pair(out=(W, H), fmt=RGBA, mode=mode, inputs=INPUTS)
    p.register_wgsl("taps", None, src=ORACLE_SRC, restated=ORACLE_RESTATED)
    p.update(SH(shader_id="taps", width=W, height=H, children=[IN(input_id=k) for k in INPUTS]))
    p.render_check(0.25, "texture parameters and private state")
