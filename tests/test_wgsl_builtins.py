"""WGSL builtins in registered shaders (smr_register_wgsl_shader): the numeric, bit, packing and texture builtins beyond
the first subset, translated by smelter_b200/csrc/wgsl.cpp to the wb_* functions of wgsl_rt.cuh.

The numpy restatements below are the specification, written from the rules of DESIGN.md's "WGSL builtins" list.  CPU
(host-only handle): every newly accepted builtin registers, misuses answer SMR_ERR_INVALID_ARGUMENT with a position, and
every builtin still refused answers SMR_ERR_UNSUPPORTED and names itself.  GPU: each builtin evaluated by a probe shader
on edge inputs and hashed inputs, every result byte against numpy; the hyperbolics within a tolerance; the texture
builtins against textureSample and against hand-written restatements on tests/wgsl_oracle_shim.h.
"""
import ctypes as C
import math
from fractions import Fraction

import numpy as np
import pytest

import smelter_b200 as s
from tests import oracle_shader, oracle_wgsl
from tests import test_web_view_component as TW
from tests.test_wgsl_shader import HEADER, Pair, host, status, with_fs

IN, SH, P = s.InputStreamComponent, s.ShaderComponent, s.ShaderParam
RGBA = TW.RGBA
f32 = np.float32


def fbits(x):
    return int(np.array([x], np.float32).view(np.uint32)[0])


def bitsf(b):
    return np.array([b & 0xFFFFFFFF], np.uint32).view(np.float32)[0]


# ---- CPU ------------------------------------------------------------------------------------------------------------
V2, V3, V4 = "vec2(0.25, -0.5)", "vec3(0.25, -0.5, 0.75)", "vec4(0.25, -0.5, 0.75, 1.0)"
T0 = "textures[0], sampler_"
ACCEPTED = {
    "saturate": "let r = saturate(1.5) + saturate(vec2(0.5, 2.0)).x;",
    "degrees": "let r = degrees(1.0) + degrees(vec3<f32>(1.0)).y;",
    "radians": "let r = radians(90.0) + radians(vec4<f32>(1.0)).w;",
    "fma": "let r = fma(1.0, 2.0, 3.0) + fma(vec2(1.0), vec2(2.0), vec2(3.0)).x;",
    "ldexp": "let r = ldexp(1.5, 3) + ldexp(vec2(1.0), vec2<i32>(1, -2)).y;",
    "frexp": "let q = frexp(3.0); let v = frexp(vec3(1.0, 2.0, 3.0)); let r = q.fract + f32(q.exp) + v.fract.z + f32(v.exp.x);",
    "modf": "let q = modf(-2.5); let v = modf(vec4<f32>(1.5)); let r = q.fract + q.whole + v.whole.x + v.fract.w;",
    "determinant": "let r = determinant(mat2x2<f32>(1.0, 2.0, 3.0, 4.0)) + determinant(mat3x3<f32>()) + determinant(mat4x4<f32>());",
    "faceForward": f"let r = faceForward({V3}, {V3}, {V3}).x;",
    "reflect": f"let r = reflect({V2}, {V2}).x + reflect({V4}, {V4}).w;",
    "refract": f"let r = refract({V3}, {V3}, 0.5).y;",
    "quantizeToF16": "let r = quantizeToF16(0.1) + quantizeToF16(vec2(0.1, 0.2)).y;",
    "sinh": "let r = sinh(0.5);", "cosh": "let r = cosh(0.5);", "tanh": "let r = tanh(vec2(0.5)).x;",
    "asinh": "let r = asinh(0.5);", "acosh": "let r = acosh(1.5);", "atanh": "let r = atanh(0.5);",
    "countOneBits": "let r = f32(countOneBits(7u) + u32(countOneBits(-1)) + countOneBits(vec2(3u, 1u)).x);",
    "countLeadingZeros": "let r = f32(countLeadingZeros(7u)) + f32(countLeadingZeros(vec3<i32>(1)).z);",
    "countTrailingZeros": "let r = f32(countTrailingZeros(8u)) + f32(countTrailingZeros(vec4<i32>(1)).z);",
    "reverseBits": "let r = f32(reverseBits(8u)) + f32(reverseBits(vec2<i32>(1)).y);",
    "firstTrailingBit": "let r = f32(firstTrailingBit(8u)) + f32(firstTrailingBit(-4));",
    "firstLeadingBit": "let r = f32(firstLeadingBit(8u)) + f32(firstLeadingBit(vec2<i32>(-4, 5)).x);",
    "extractBits": "let r = f32(extractBits(0xF0u, 4u, 4u)) + f32(extractBits(vec3<i32>(-1), 1u, 3u).y);",
    "insertBits": "let r = f32(insertBits(0u, 3u, 4u, 2u)) + f32(insertBits(vec2<i32>(1), vec2<i32>(2), 4u, 2u).x);",
    "dot4U8Packed": "let r = f32(dot4U8Packed(0x01020304u, 0x01010101u));",
    "dot4I8Packed": "let r = f32(dot4I8Packed(0xFF020304u, 0x01010101u));",
    "pack4x8snorm": f"let r = f32(pack4x8snorm({V4}));",
    "pack4x8unorm": f"let r = f32(pack4x8unorm({V4}));",
    "pack2x16snorm": f"let r = f32(pack2x16snorm({V2}));",
    "pack2x16unorm": f"let r = f32(pack2x16unorm({V2}));",
    "pack2x16float": f"let r = f32(pack2x16float({V2}));",
    "unpack4x8snorm": "let r = unpack4x8snorm(0x7F80FF01u).x;",
    "unpack4x8unorm": "let r = unpack4x8unorm(0x7F80FF01u).w;",
    "unpack2x16snorm": "let r = unpack2x16snorm(0x7FFF8000u).y;",
    "unpack2x16unorm": "let r = unpack2x16unorm(123u).x;",
    "unpack2x16float": "let r = unpack2x16float(0x3C00u).x;",
    "textureSampleLevel": f"let r = textureSampleLevel({T0}, input.tex_coords, 0.0).x;",
    "textureSampleBias": f"let r = textureSampleBias({T0}, input.tex_coords, 1.0).x;",
    "textureSampleGrad": f"let r = textureSampleGrad({T0}, input.tex_coords, vec2(0.1), vec2(0.0)).x;",
    "textureSampleBaseClampToEdge": f"let r = textureSampleBaseClampToEdge({T0}, input.tex_coords).x;",
    "textureGather": f"const c = 2u; let r = textureGather(1, {T0}, input.tex_coords).x + textureGather(c, {T0}, input.tex_coords).w;",
    "textureDimensions": "let r = f32(textureDimensions(textures[1], 3).x + textureDimensions(textures[0], 0u).y);",
    "textureNumLevels": "let r = f32(textureNumLevels(textures[0]));",
}
# the builtins still refused: derivatives, textureLoad, comparison, storage and layer / sample queries, atomics, arrayLength,
# barriers, workgroupUniformLoad, subgroups, f16 and ptr
STILL_REFUSED = ["dpdx", "dpdy", "fwidth", "dpdxCoarse", "dpdyCoarse", "dpdxFine", "dpdyFine", "fwidthCoarse", "fwidthFine",
                 "textureLoad", "textureSampleCompare", "textureSampleCompareLevel", "textureGatherCompare", "textureStore",
                 "textureNumLayers", "textureNumSamples", "atomicLoad", "atomicStore", "atomicAdd", "atomicSub", "atomicMax",
                 "atomicMin", "atomicAnd", "atomicOr", "atomicXor", "atomicExchange", "atomicCompareExchangeWeak",
                 "arrayLength", "workgroupBarrier", "storageBarrier", "textureBarrier", "workgroupUniformLoad", "subgroupAdd",
                 "subgroupBroadcast", "f16", "ptr"]


@pytest.mark.parametrize("name", sorted(ACCEPTED))
def test_builtin_registers(name):
    host().register_wgsl_shader(name, with_fs(ACCEPTED[name] + "\n    return vec4(r);"))


def test_builtins_in_module_constants_and_vertex_stage_register():
    """a call in a const declaration is evaluated where it is used, as `const k = sqrt(2.0);` is; textureSampleLevel,
    textureSampleGrad and textureSampleBaseClampToEdge are allowed in vs_main and in the functions it calls"""
    src = HEADER.replace("output.position = vec4(input.position, 1.0);",
                         "output.position = vec4(input.position, 1.0) + vp();") + r'''
const k = degrees(1.0);
const m = vec2<u32>(countOneBits(7u), reverseBits(1u));
fn vp() -> vec4<f32> {
    return textureSampleLevel(textures[0], sampler_, vec2(0.5), 0.0) * 0.0 + textureSampleGrad(textures[1], sampler_, vec2(0.5), vec2(0.0), vec2(0.0))
        * 0.0 + textureSampleBaseClampToEdge(textures[2], sampler_, vec2(0.25)) * 0.0;
}
@fragment
fn fs_main(input: VertexOutput) -> @location(0) vec4<f32> {
    const j = saturate(2.0);
    return vec4(k * j, f32(m.x), 0.0, 1.0);
}
'''
    host().register_wgsl_shader("consts", src)


VS_BIAS = HEADER.replace("output.position = vec4(input.position, 1.0);",
                         "output.position = vec4(input.position, 1.0) + biased();") + r'''
fn biased() -> vec4<f32> {
    return textureSampleBias(textures[0], sampler_, vec2(0.5), 1.0) * 0.0;
}
@fragment
fn fs_main(input: VertexOutput) -> @location(0) vec4<f32> { return vec4(1.0); }
'''
MISUSES = {   # (source, the text at the position the refusal names)
    "textureGather component 4": (with_fs("let r = textureGather(4, textures[0], sampler_, input.tex_coords);\n    return r;"), "4, textures"),
    "textureGather non-const component": (with_fs("let c = 1;\n    return textureGather(c, textures[0], sampler_, input.tex_coords);"), "c, textures"),
    "extractBits on f32": (with_fs("let r = extractBits(1.5f, 0u, 4u);\n    return vec4(r);"), "extractBits"),
    "pack4x8unorm on vec3": (with_fs("let r = pack4x8unorm(vec3(0.5, 0.5, 0.5));\n    return vec4(f32(r));"), "pack4x8unorm"),
    "textureSampleBias in vs_main": (VS_BIAS, "textureSampleBias"),
}


def _line_col(src, needle):
    i = src.index(needle)
    return f"{src.count(chr(10), 0, i) + 1}:{i - (src.rfind(chr(10), 0, i) + 1) + 1}"


@pytest.mark.parametrize("name", sorted(MISUSES))
def test_misuse_is_invalid_with_a_position(name):
    src, at = MISUSES[name]
    st, msg = status(host(), src)
    assert st == 1, msg
    assert "WGSL " + _line_col(src, at) + ":" in msg, (msg, _line_col(src, at))


@pytest.mark.parametrize("name", STILL_REFUSED)
def test_still_refused_builtins_are_named(name):
    st, msg = status(host(), with_fs(f"let r = {name}(1.0);\n    return vec4(1.0);"))
    assert st == 5, msg
    assert f"unsupported: {name}" in msg, msg


def test_textureSample_offset_overloads_stay_out_of_scope():
    for call in ("textureSampleLevel(textures[0], sampler_, input.tex_coords, 0.0, vec2<i32>(1, 0))",
                 "textureGather(0, textures[0], sampler_, input.tex_coords, vec2<i32>(1, 0))"):
        st, msg = status(host(), with_fs(f"return {call};"))
        assert st == 5 and "with an offset" in msg, msg


# ---- numpy restatements: the rules, one function per builtin -------------------------------------------------------
def round_f32(q):
    """an exact rational rounded to f32 (nearest, ties to even; subnormals and overflow as IEEE 754)"""
    if q == 0:
        return f32(0.0)
    sign, q = (-1 if q < 0 else 1), abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if Fraction(2) ** e > q:
        e -= 1
    e = max(e, -126)                               # subnormals share the smallest normal exponent's spacing
    scaled = q / Fraction(2) ** (e - 23)           # the integer significand, before rounding
    m = scaled.numerator // scaled.denominator
    rem = scaled - m
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and m % 2):
        m += 1
    v = Fraction(m) * Fraction(2) ** (e - 23)
    if v >= Fraction(2) ** 128:
        return f32(sign * np.inf)
    return f32(sign * float(v))


def fma_f32(a, b, c):
    a, b, c = f32(a), f32(b), f32(c)
    if not (np.isfinite(a) and np.isfinite(b) and np.isfinite(c)):
        return f32(float(a) * float(b) + float(c))
    p, r = Fraction(float(a)) * Fraction(float(b)), Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    if r == 0:   # an exact zero: -0 only when the product and the addend are both -0
        neg = math.copysign(1, float(a)) * math.copysign(1, float(b)) < 0 and math.copysign(1, float(c)) < 0 and p == 0
        return f32(-0.0 if neg else 0.0)
    return round_f32(r)


def fmax(a, b):   # wb_max: fmaxf, NaN gives the other operand, -0 < +0
    a, b = f32(a), f32(b)
    if np.isnan(a):
        return b
    if np.isnan(b):
        return a
    if a == b == 0:
        return a if math.copysign(1, a) > 0 else b
    return a if a > b else b


def fmin(a, b):
    a, b = f32(a), f32(b)
    if np.isnan(a):
        return b
    if np.isnan(b):
        return a
    if a == b == 0:
        return a if math.copysign(1, a) < 0 else b
    return a if a < b else b


def ldexp_f32(x, e):
    x = f32(x)
    if not np.isfinite(x) or x == 0:
        return x
    e = max(-400, min(400, e))   # beyond this every f32 scales to 0 or infinity either way
    return round_f32(Fraction(float(x)) * Fraction(2) ** e)


def det(a):
    """cofactor expansion along the first column, terms added left to right, in f32; a[r][c]"""
    n = len(a)
    if n == 1:
        return f32(a[0][0])
    acc = None
    for i in range(n):
        minor = [row[1:] for r, row in enumerate(a) if r != i]
        t = f32(f32(a[i][0]) * det(minor))
        acc = t if i == 0 else f32(acc - t) if i % 2 else f32(acc + t)
    return acc


def dot(a, b):
    acc = f32(f32(a[0]) * f32(b[0]))
    for x, y in zip(a[1:], b[1:]):
        acc = f32(acc + f32(f32(x) * f32(y)))
    return acc


def reflect(e1, e2):
    k = f32(f32(2.0) * dot(e2, e1))
    return [f32(f32(x) - f32(k * f32(y))) for x, y in zip(e1, e2)]


def refract(e1, e2, e3):
    e3 = f32(e3)
    d = dot(e2, e1)
    k = f32(f32(1.0) - f32(f32(e3 * e3) * f32(f32(1.0) - f32(d * d))))
    if k < 0:
        return [f32(0.0)] * len(e1)
    sc = f32(f32(e3 * d) + f32(np.sqrt(k)))
    return [f32(f32(e3 * f32(x)) - f32(sc * f32(y))) for x, y in zip(e1, e2)]


def face_forward(e1, e2, e3):
    return list(e1) if dot(e2, e3) < 0 else [f32(-f32(x)) for x in e1]


def to_f16_bits(x):   # f32 -> f16, nearest even
    return int(np.array([f32(x)], np.float32).astype(np.float16).view(np.uint16)[0])


def from_f16_bits(h):
    return f32(np.array([h], np.uint16).view(np.float16)[0])


def i32(v):
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v >> 31 else v


def clz(v):
    return 32 - (v & 0xFFFFFFFF).bit_length()


def ctz(v):
    v &= 0xFFFFFFFF
    return 32 if v == 0 else (v & -v).bit_length() - 1


def first_leading_i32(v):
    v = i32(v)
    u = ~v & 0xFFFFFFFF if v < 0 else v
    return -1 if u == 0 else u.bit_length() - 1


def extract_bits(e, off, cnt, signed):
    o = min(off, 32)
    c = min(cnt, 32 - o)
    if c == 0:
        return 0
    v = ((e & 0xFFFFFFFF) >> o) & ((1 << c) - 1)
    return v - (1 << c) if signed and v >> (c - 1) else v


def insert_bits(e, nb, off, cnt):
    o = min(off, 32)
    c = min(cnt, 32 - o)
    if c == 0:
        return e & 0xFFFFFFFF
    mask = ((1 << c) - 1) << o
    return ((e & ~mask) | ((nb << o) & mask)) & 0xFFFFFFFF


def pack(vals, lo, scale, width):
    r = 0
    for i, x in enumerate(vals):
        q = int(np.floor(f32(f32(0.5) + f32(f32(scale) * fmin(1.0, fmax(lo, x))))))
        r |= (q & ((1 << width) - 1)) << (i * width)
    return r


def unpack(v, width, signed, scale):
    out = []
    for i in range(32 // width):
        b = (v >> (i * width)) & ((1 << width) - 1)
        if signed:
            b = b - (1 << width) if b >> (width - 1) else b
            out.append(fmax(f32(f32(b) / f32(scale)), -1.0))
        else:
            out.append(f32(f32(b) / f32(scale)))
    return out


# ---- GPU probes -----------------------------------------------------------------------------------------------------
# A probe shader evaluates one builtin per pixel: column x takes its arguments from the edge table (x < NT) or from a hash
# of x; row y writes component y of the result, four bytes from the least significant, as f32(k) / 255.0 (CpuOptimized
# stores that byte back exactly).  Arguments: a_k the raw u32 bits, f_k the f32 (the table's bits, or a hashed value in
# [-2, 2)), s_k a small u32 (the table's value, or a hash below 40), h_k(j) further hashed f32s.
NT, NCOL = 64, 128
PROBE = r'''
struct U { t: array<vec4<u32>, 64>, }
@group(1) @binding(0) var<uniform> u: U;
fn hash(v: u32) -> u32 {
    var h = v * 747796405u + 2891336453u;
    h = ((h >> ((h >> 28u) + 4u)) ^ h) * 277803737u;
    return (h >> 22u) ^ h;
}
fn fh(i: u32) -> f32 { return f32(hash(i) >> 8u) / 16777216.0 * 4.0 - 2.0; }
fn raw(x: u32, k: u32) -> u32 { if x < 64u { return u.t[x][k]; } return hash(x * 4u + k); }
fn flt(x: u32, k: u32) -> f32 { if x < 64u { return bitcast<f32>(u.t[x][k]); } return fh(x * 4u + k); }
fn small(x: u32, k: u32) -> u32 { if x < 64u { return u.t[x][k]; } return hash(x * 4u + k) % 40u; }
fn fb(v: f32) -> u32 { return bitcast<u32>(v); }
fn ib(v: i32) -> u32 { return bitcast<u32>(v); }
fn probe(x: u32) -> vec4<u32> {
    let a0 = raw(x, 0u); let a1 = raw(x, 1u); let a2 = raw(x, 2u); let a3 = raw(x, 3u);
    let f0 = flt(x, 0u); let f1 = flt(x, 1u); let f2 = flt(x, 2u); let f3 = flt(x, 3u);
    let s0 = small(x, 0u); let s1 = small(x, 1u); let s2 = small(x, 2u); let s3 = small(x, 3u);
    let i0 = bitcast<i32>(a0); let i1 = bitcast<i32>(a1);
    return EXPR;
}
'''


def probe_src(expr):
    return with_fs(r'''
    let x = u32(input.position.x);
    let y = u32(input.position.y);
    let v = probe(x)[y];
    return vec4(f32(v & 255u) / 255.0, f32((v >> 8u) & 255u) / 255.0, f32((v >> 16u) & 255u) / 255.0, f32(v >> 24u) / 255.0);''',
                   PROBE.replace("EXPR", expr))


def _hash(v):
    h = (v * 747796405 + 2891336453) & 0xFFFFFFFF
    h = (((h >> ((h >> 28) + 4)) ^ h) * 277803737) & 0xFFFFFFFF
    return (h >> 22) ^ h


def fh(i):
    return f32(f32(f32(_hash(i) >> 8) / f32(16777216.0)) * f32(4.0)) - f32(2.0)


class Args:
    """column x's arguments, as the probe computes them"""

    def __init__(self, table, x):
        t = (table[x] if x < len(table) else [0, 0, 0, 0]) if x < NT else None   # the uniform is zero-padded
        self.x = x
        self.a = [t[k] if t else _hash(x * 4 + k) for k in range(4)]
        self.f = [bitsf(t[k]) if t else fh(x * 4 + k) for k in range(4)]
        self.s = [t[k] if t else _hash(x * 4 + k) % 40 for k in range(4)]
        self.i = [i32(v) for v in self.a]

    def h(self, n, j):
        return fh(self.x * n + j)


def B(v):   # a result as its u32 bits
    return fbits(v) if isinstance(v, (float, np.floating)) else int(v) & 0xFFFFFFFF


def vec_u(parts):
    return "vec4<u32>(" + ", ".join(parts + ["0u"] * (4 - len(parts))) + ")"


def vec_of(v, n, cast):   # the components of a vecN expression as vec4<u32>: cast "fb" (f32), "ib" (i32) or "" (u32)
    return vec_u([f"{cast}(({v}).{'xyzw'[k]})" for k in range(n)])


ZF = [0.0, -0.0, 1.0, -1.0, 0.5, -0.5, 1e-45, -1e-45, 1.1754942e-38, 3.4028235e38, -3.4028235e38, np.inf, -np.inf, np.nan,
      2.5, -2.5, 100.75, -7.25, 3.0, 1e-3]
INTS = [0, 1, 0xFFFFFFFF, 0x80000000, 0x7FFFFFFF, 0x00010000, 0x80000001, 0xF0F0F0F0, 0x12345678, 0xFFFF0000, 2, 0x40000000]


def ftable(vals, k=4):
    vals = [fbits(f32(v)) for v in vals]
    return [[vals[(i + j * 7) % len(vals)] for j in range(k)] for i in range(len(vals))]


def itable(vals):
    return [[vals[(i + j * 5) % len(vals)] for j in range(4)] for i in range(len(vals))]


BITOPS = [(0, 0), (0, 31), (0, 32), (0, 33), (31, 1), (31, 2), (32, 0), (32, 5), (33, 1), (1, 31), (1, 32), (5, 27),
          (16, 16), (0xFFFFFFFF, 5), (5, 0xFFFFFFFF), (31, 0), (0, 1), (12, 0), (31, 32), (33, 33)]
BITS_TABLE = [[INTS[i % len(INTS)], INTS[(i * 3 + 1) % len(INTS)], o, c] for i, (o, c) in enumerate(BITOPS)]
ONE = np.nextafter(f32(1.0), f32(2.0))
PACK_F = [1.0, -1.0, ONE, -ONE, 0.5, -0.5, 0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, 2.0, -2.0, 0.25, 0.75,
          f32(1.5) / f32(255.0), f32(0.5) / f32(127.0), 0.999, -0.999]
F16_EDGE = [65504.0, 65520.0, np.nextafter(f32(65520.0), f32(0.0)), 65519.0, -65520.0, 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11,
            2.0 ** -25, 3 * 2.0 ** -25, 2.0 ** -24, 2.0 ** -14, 2.0 ** -15 + 2.0 ** -26, 1e-45, -0.0, 0.0, np.inf, -np.inf,
            6.1e-5, 1.0 / 3.0, 1e6]
UNPACK = [0x0, 0xFFFFFFFF, 0x80808080, 0x7F7F7F7F, 0x01FF807F, 0x80007FFF, 0x7C00FC00, 0x00017BFF, 0x03FF8001, 0x3C00BC00,
          0xFBFF0400, 0x12345678, 0x7E000000]


def _f(fn):   # a scalar f32 -> f32 rule, per column
    return lambda A: [[B(fn(A.f[0]))]]


PROBES = {   # name: (WGSL expression giving vec4<u32>, rows, edge table, numpy rule: Args -> rows of u32)
    "saturate": (vec_u(["fb(saturate(f0))"]), 1, ftable(ZF + [1.5, -3.0]), _f(lambda x: fmin(fmax(x, 0.0), 1.0))),
    "saturate vec4": (vec_of("saturate(vec4(f0, f1, f2, f3))", 4, "fb"), 4, ftable(ZF),
                      lambda A: [[B(fmin(fmax(A.f[k], 0.0), 1.0))] for k in range(4)]),
    "degrees": (vec_u(["fb(degrees(f0))"]), 1, ftable(ZF), _f(lambda x: f32(f32(x) * bitsf(0x42652EE1)))),
    "radians": (vec_u(["fb(radians(f0))"]), 1, ftable(ZF), _f(lambda x: f32(f32(x) * bitsf(0x3C8EFA35)))),
    "fma": (vec_u(["fb(fma(f0, f1, f2))"]), 1, ftable(ZF + [1.0 + 2.0 ** -23, -(1.0 + 2.0 ** -22), 2.0 ** -24]),
            lambda A: [[B(fma_f32(*A.f[:3]))]]),
    "fma vec3": (vec_of("fma(vec3(f0, f1, f2), vec3(f1, f2, f0), vec3(f2, f0, f3))", 3, "fb"), 3,
                 ftable(ZF), lambda A: [[B(fma_f32(A.f[k], A.f[(k + 1) % 3], [A.f[2], A.f[0], A.f[3]][k]))] for k in range(3)]),
    "ldexp": (vec_u(["fb(ldexp(f0, select(i1, i32(s2) - 20, x >= 64u)))"]), 1,
              [[fbits(f32(v)), e & 0xFFFFFFFF, 0, 0] for v, e in [(1.0, 0), (1.5, 127), (1.5, 128), (1.0, -149), (1.0, -150),
                                                                  (3.0, -151), (1.0, 0x7FFFFFFF), (1.0, -0x80000000), (1e-45, 149),
                                                                  (1e-45, -1), (-0.0, 5), (np.inf, -5), (0.75, -126), (1.75, -149),
                                                                  (3.4028235e38, 1), (-2.5, -140)]],
              lambda A: [[B(ldexp_f32(A.f[0], A.i[1] if A.x < NT else A.s[2] - 20))]]),
    "ldexp vec2": (vec_of("ldexp(vec2(f0, f1), vec2(i32(s2) - 20, 3 - i32(s3)))", 2, "fb"), 2,
                   [[fbits(f32(1.5)), fbits(f32(-1e-45)), 150, 1], [fbits(f32(2.0)), fbits(f32(3.0)), 0, 40]],
                   lambda A: [[B(ldexp_f32(A.f[0], A.s[2] - 20))], [B(ldexp_f32(A.f[1], 3 - A.s[3]))]]),
    "frexp": ("vec4<u32>(fb(frexp(f0).fract), ib(frexp(f0).exp), 0u, 0u)", 2,
              ftable([v for v in ZF if np.isfinite(v)] + [1e-40, -3e-39, 0.49999997]),
              lambda A: [[B(np.frexp(f32(A.f[0]))[0])], [B(int(np.frexp(f32(A.f[0]))[1]))]]),
    "frexp vec2": ("vec4<u32>(fb(frexp(vec2(f0, f1)).fract.x), fb(frexp(vec2(f0, f1)).fract.y), ib(frexp(vec2(f0, f1)).exp.x), ib(frexp(vec2(f0, f1)).exp.y))", 4,
                   ftable([v for v in ZF if np.isfinite(v)]),
                   lambda A: [[B(np.frexp(f32(A.f[k]))[0])] for k in range(2)] + [[B(int(np.frexp(f32(A.f[k]))[1]))] for k in range(2)]),
    "modf": ("vec4<u32>(fb(modf(f0).fract), fb(modf(f0).whole), 0u, 0u)", 2, ftable(ZF),
             lambda A: [[B(f32(f32(A.f[0]) - np.trunc(f32(A.f[0]))))], [B(np.trunc(f32(A.f[0])))]]),
    "modf vec4": (vec_of("modf(vec4(f0, f1, f2, f3)).fract", 4, "fb"), 4, ftable(ZF),
                  lambda A: [[B(f32(f32(A.f[k]) - np.trunc(f32(A.f[k]))))] for k in range(4)]),
    "quantizeToF16": (vec_u(["fb(quantizeToF16(f0))"]), 1, ftable(F16_EDGE + [np.nan]),
                      _f(lambda x: from_f16_bits(to_f16_bits(x)))),
    "quantizeToF16 vec2": (vec_of("quantizeToF16(vec2(f0, f1))", 2, "fb"), 2, ftable(F16_EDGE),
                           lambda A: [[B(from_f16_bits(to_f16_bits(A.f[k])))] for k in range(2)]),
    "countOneBits": ("vec4<u32>(countOneBits(a0), ib(countOneBits(i1)), 0u, 0u)", 2, itable(INTS),
                     lambda A: [[bin(A.a[0]).count("1")], [bin(A.a[1]).count("1")]]),
    "countOneBits vec4": ("countOneBits(vec4(a0, a1, a2, a3))", 4, itable(INTS), lambda A: [[bin(A.a[k]).count("1")] for k in range(4)]),
    "countLeadingZeros": ("vec4<u32>(countLeadingZeros(a0), ib(countLeadingZeros(i1)), 0u, 0u)", 2, itable(INTS),
                          lambda A: [[clz(A.a[0])], [clz(A.a[1])]]),
    "countTrailingZeros": ("vec4<u32>(countTrailingZeros(a0), ib(countTrailingZeros(i1)), 0u, 0u)", 2, itable(INTS),
                           lambda A: [[ctz(A.a[0])], [ctz(A.a[1])]]),
    "reverseBits": ("vec4<u32>(reverseBits(a0), ib(reverseBits(i1)), 0u, 0u)", 2, itable(INTS),
                    lambda A: [[int(f"{A.a[0]:032b}"[::-1], 2)], [int(f"{A.a[1]:032b}"[::-1], 2)]]),
    "reverseBits vec3 i32": (vec_of("reverseBits(vec3(i0, i1, bitcast<i32>(a2)))", 3, "ib"), 3, itable(INTS),
                             lambda A: [[int(f"{A.a[k]:032b}"[::-1], 2)] for k in range(3)]),
    "firstTrailingBit": ("vec4<u32>(firstTrailingBit(a0), ib(firstTrailingBit(i1)), 0u, 0u)", 2, itable(INTS),
                         lambda A: [[0xFFFFFFFF if A.a[0] == 0 else ctz(A.a[0])], [0xFFFFFFFF if A.a[1] == 0 else ctz(A.a[1])]]),
    "firstLeadingBit": ("vec4<u32>(firstLeadingBit(a0), ib(firstLeadingBit(i1)), 0u, 0u)", 2, itable(INTS),
                        lambda A: [[0xFFFFFFFF if A.a[0] == 0 else A.a[0].bit_length() - 1], [first_leading_i32(A.a[1])]]),
    "extractBits": ("vec4<u32>(extractBits(a0, s2, s3), ib(extractBits(i1, s2, s3)), 0u, 0u)", 2, BITS_TABLE,
                    lambda A: [[extract_bits(A.a[0], A.s[2], A.s[3], False)], [extract_bits(A.a[1], A.s[2], A.s[3], True)]]),
    "extractBits vec2 i32": (vec_of("extractBits(vec2(i0, i1), s2, s3)", 2, "ib"), 2, BITS_TABLE,
                             lambda A: [[extract_bits(A.a[k], A.s[2], A.s[3], True)] for k in range(2)]),
    "insertBits": ("vec4<u32>(insertBits(a0, a1, s2, s3), ib(insertBits(i1, i0, s2, s3)), 0u, 0u)", 2, BITS_TABLE,
                   lambda A: [[insert_bits(A.a[0], A.a[1], A.s[2], A.s[3])], [insert_bits(A.a[1], A.a[0], A.s[2], A.s[3])]]),
    "insertBits vec2 u32": ("vec4<u32>(insertBits(vec2(a0, a1), vec2(a1, a0), s2, s3), 0u, 0u)", 2, BITS_TABLE,
                            lambda A: [[insert_bits(A.a[k], A.a[1 - k], A.s[2], A.s[3])] for k in range(2)]),
    "dot4U8Packed": (vec_u(["dot4U8Packed(a0, a1)"]), 1, itable(INTS),
                     lambda A: [[sum(((A.a[0] >> i) & 255) * ((A.a[1] >> i) & 255) for i in range(0, 32, 8))]]),
    "dot4I8Packed": (vec_u(["ib(dot4I8Packed(a0, a1))"]), 1, itable(INTS),
                     lambda A: [[sum(i32(((A.a[0] >> i) & 255) << 24) // 2 ** 24 * (i32(((A.a[1] >> i) & 255) << 24) // 2 ** 24)
                                     for i in range(0, 32, 8))]]),
    "pack4x8snorm": (vec_u(["pack4x8snorm(vec4(f0, f1, f2, f3))"]), 1, ftable(PACK_F), lambda A: [[pack(A.f, -1.0, 127.0, 8)]]),
    "pack4x8unorm": (vec_u(["pack4x8unorm(vec4(f0, f1, f2, f3))"]), 1, ftable(PACK_F), lambda A: [[pack(A.f, 0.0, 255.0, 8)]]),
    "pack2x16snorm": (vec_u(["pack2x16snorm(vec2(f0, f1))"]), 1, ftable(PACK_F), lambda A: [[pack(A.f[:2], -1.0, 32767.0, 16)]]),
    "pack2x16unorm": (vec_u(["pack2x16unorm(vec2(f0, f1))"]), 1, ftable(PACK_F), lambda A: [[pack(A.f[:2], 0.0, 65535.0, 16)]]),
    "pack2x16float": (vec_u(["pack2x16float(vec2(f0, f1))"]), 1, ftable(F16_EDGE),
                      lambda A: [[to_f16_bits(A.f[0]) | (to_f16_bits(A.f[1]) << 16)]]),
    "unpack4x8snorm": (vec_of("unpack4x8snorm(a0)", 4, "fb"), 4, itable(UNPACK), lambda A: [[B(v)] for v in unpack(A.a[0], 8, True, 127.0)]),
    "unpack4x8unorm": (vec_of("unpack4x8unorm(a0)", 4, "fb"), 4, itable(UNPACK), lambda A: [[B(v)] for v in unpack(A.a[0], 8, False, 255.0)]),
    "unpack2x16snorm": (vec_of("unpack2x16snorm(a0)", 2, "fb"), 2, itable(UNPACK),
                        lambda A: [[B(v)] for v in unpack(A.a[0], 16, True, 32767.0)]),
    "unpack2x16unorm": (vec_of("unpack2x16unorm(a0)", 2, "fb"), 2, itable(UNPACK),
                        lambda A: [[B(v)] for v in unpack(A.a[0], 16, False, 65535.0)]),
    "unpack2x16float": (vec_of("unpack2x16float(a0)", 2, "fb"), 2, itable(UNPACK),
                        lambda A: [[B(from_f16_bits(A.a[0] & 0xFFFF))], [B(from_f16_bits(A.a[0] >> 16))]]),
}


def _vecs(n, first):
    return ", ".join(f"vec{n}(" + ", ".join(f"fh(x * 16u + {first + k * n + j}u)" for j in range(n)) + ")" for k in range(3))


for _n in (2, 3, 4):
    PROBES[f"determinant mat{_n}"] = (
        vec_u([f"fb(determinant(mat{_n}x{_n}<f32>(" + ", ".join(f"fh(x * 16u + {j}u)" for j in range(_n * _n)) + ")))"]), 1, [],
        (lambda n: lambda A: [[B(det([[A.h(16, c * n + r) for c in range(n)] for r in range(n)]))]])(_n))
# vector rules on three hashed vec3s (e1, e2, e3), and refract's ratio
_E = lambda A, k: [A.h(16, 3 * k + j) for j in range(3)]
_V = lambda k: f"vec3(fh(x * 16u + {3 * k}u), fh(x * 16u + {3 * k + 1}u), fh(x * 16u + {3 * k + 2}u))"
PROBES["reflect"] = (vec_of(f"reflect({_V(0)}, {_V(1)})", 3, "fb"), 3, [],
                     lambda A: [[B(v)] for v in reflect(_E(A, 0), _E(A, 1))])
PROBES["refract"] = (vec_of(f"refract({_V(0)}, {_V(1)} * 0.5, fh(x * 16u + 9u) * 0.5)", 3, "fb"), 3, [],
                     lambda A: [[B(v)] for v in refract(_E(A, 0), [f32(v * f32(0.5)) for v in _E(A, 1)], f32(A.h(16, 9) * f32(0.5)))])
PROBES["faceForward"] = (vec_of(f"faceForward({_V(0)}, {_V(1)}, {_V(2)})", 3, "fb"), 3, [],
                         lambda A: [[B(v)] for v in face_forward(_E(A, 0), _E(A, 1), _E(A, 2))])


def _table_param(table):
    rows = [list(r) + [0] * (4 - len(r)) for r in table] + [[0, 0, 0, 0]] * (NT - len(table))
    return P.struct([("t", P.list([P.list([P.u32(int(v) & 0xFFFFFFFF) for v in r]) for r in rows]))])


def expected(rule, table, rows):
    """the rule's u32 result bits, (rows, NCOL); numpy's overflow and NaN warnings are the rules' own infinities and NaNs"""
    with np.errstate(all="ignore"):
        cols = [rule(Args(table, x)) for x in range(NCOL)]
    return np.array([[B(c[y][0]) for c in cols] for y in range(rows)], np.uint64).astype(np.uint32)


@pytest.fixture(scope="module")
def cpu_renderer():
    return s.Renderer(s.RendererOptions(rendering_mode=s.RenderingMode.CpuOptimized))


def run_probe(r, sid, expr, rows, table):
    r.register_wgsl_shader(sid, probe_src(expr))
    r.update_scene("output_1", s.Resolution(NCOL, rows), RGBA,
                   SH(shader_id=sid, shader_param=_table_param(table), width=NCOL, height=rows))
    px = np.asarray(r.render(s.FrameSet(frames={}, pts=0.0)).frames["output_1"].data.planes[0]).astype(np.uint32)
    return px[..., 0] | (px[..., 1] << 8) | (px[..., 2] << 16) | (px[..., 3] << 24)


def test_probe_restatements_cover_edge_tables():
    """runs without a GPU: every probe's rule evaluates on every column, and each edge table fits the uniform"""
    for name, (expr, rows, table, rule) in PROBES.items():
        assert len(table) <= NT, name
        exp = expected(rule, table, rows)
        assert exp.shape == (rows, NCOL), name
    assert fma_f32(1.0 + 2.0 ** -23, 1.0 + 2.0 ** -23, -1.0) == f32(2.0 ** -22 + 2.0 ** -46)
    assert round_f32(Fraction(3, 2 ** 151)) == f32(2.0 ** -149) and round_f32(Fraction(1, 2 ** 150)) == f32(0.0)
    assert round_f32(Fraction(3, 2 ** 150)) == f32(2.0 ** -148) and round_f32(Fraction(2 ** 128)) == f32(np.inf)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(PROBES))
def test_builtin_bit_exact(cpu_renderer, name):
    expr, rows, table, rule = PROBES[name]
    got = run_probe(cpu_renderer, "probe " + name, expr, rows, table)
    exp = expected(rule, table, rows)
    nan = lambda v: np.isnan(v.view(np.float32))
    float_result = not any(k in name for k in ("Bits", "Bit", "dot4", "pack", "count")) or name.startswith("unpack")
    same = (got == exp) | ((nan(got) & nan(exp)) if float_result else False)   # a NaN result: any NaN
    bad = np.argwhere(~same)
    assert bad.size == 0, [(int(y), int(x), Args(table, int(x)).a, hex(got[y, x]), hex(exp[y, x])) for y, x in bad[:8]]


HYPER = {"sinh": (np.sinh, -10.0, 10.0), "cosh": (np.cosh, -10.0, 10.0), "tanh": (np.tanh, -10.0, 10.0),
         "asinh": (np.arcsinh, -100.0, 100.0), "acosh": (np.arccosh, 1.0, 100.0), "atanh": (np.arctanh, -0.999, 0.999)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(HYPER))
def test_hyperbolics_within_tolerance(cpu_renderer, name):
    """as test_transcendental_shaders_within_tolerance: CUDA's functions against float64, within a few ulp"""
    fn, lo, hi = HYPER[name]
    xs = np.linspace(lo, hi, NT * 4, dtype=np.float64).astype(np.float32)
    for c in range(4):   # 64 arguments of the range from the table, 64 hashed ones in [-2, 2) (some outside the domain)
        table = [[fbits(v), 0, 0, 0] for v in xs[c * NT:(c + 1) * NT]]
        got = run_probe(cpu_renderer, f"hyper {name} {c}", vec_u([f"fb({name}(f0))"]), 1, table)[0].view(np.float32).astype(np.float64)
        x = np.array([Args(table, k).f[0] for k in range(NCOL)], np.float32).astype(np.float64)
        with np.errstate(invalid="ignore", divide="ignore"):
            exp = fn(x)
        both_nan = np.isnan(got) & np.isnan(exp)
        err = np.abs(got - exp)
        ok = both_nan | (got == exp) | (err <= 4 * 2.0 ** -23 * np.abs(exp)) | (err <= 2.0 ** -24)
        assert ok.all(), (name, x[~ok][:5], got[~ok][:5], exp[~ok][:5])


# ---- textures -------------------------------------------------------------------------------------------------------
# Two children, an NV12 input and a translucent RGBA8 input (640 x 360 each), drawn by a Shader root smaller and larger
# than them, in both modes.  The restatements run on tests/wgsl_oracle_shim.h; wo_vs receives the textures through
# orc_render_wgsl_vs, which hands them to the shim's rasteriser unchanged.
TEX_INPUTS = ("nv12_1", "rgba_2")
SIZES = {"down": (320, 180), "up": (960, 540)}
IDENTITY_VS = HEADER[HEADER.index("@vertex"):HEADER.index("struct BaseShaderParameters")]


def tex_shader(fs_body, vs=IDENTITY_VS):
    return HEADER.replace(IDENTITY_VS, vs) + "\n@fragment\nfn fs_main(input: VertexOutput) -> @location(0) vec4<f32> {\n" + fs_body + "\n}\n"


UV = "    let uv = input.tex_coords * 1.25 - vec2(0.1, 0.05);\n"
SAMPLES = {   # the same read, written with each textureSample variant
    "textureSample": "textureSample(textures[i], sampler_, uv)",
    "textureSampleLevel": "textureSampleLevel(textures[i], sampler_, uv, 2.5)",
    "textureSampleBias": "textureSampleBias(textures[i], sampler_, uv, -1.0)",
    "textureSampleGrad": "textureSampleGrad(textures[i], sampler_, uv, vec2(0.3, 0.0), vec2(0.0, 0.7))",
}


def sample_variant(call):
    return tex_shader("    let i = u32(base_params.plane_id);\n" + UV + "    return " + call + " * 0.75;")


VS_PRE = r'''
static smr_textures vs_tex;   // the children, for wo_vs
extern "C" void orc_render_wgsl(int, int, int, float, const void *, const uint8_t *const *, const int *, const int *, int, uint8_t *);
extern "C" void orc_render_wgsl_vs(int W, int H, int mode, float time, const void *params, const uint8_t *const *tex,
                                   const int *tw, const int *th, int n, uint8_t *out) {
    vs_tex = smr_textures{tex, tw, th, (unsigned)n, mode};
    orc_render_wgsl(W, H, mode, time, params, tex, tw, th, n, out);
}
#define WO_NVARY 2
static const int wo_interp[2] = {0, 0};
/* textureGather: NC-6's footprint, clamped to the edge; x = (u0, v1), y = (u1, v1), z = (u1, v0), w = (u0, v0) */
static float4 G(const smr_textures &t, int c, int i, float u, float v) {
    if ((unsigned)i >= t.count || !t.tex[i]) return make_float4(0, 0, 0, 0);
    int x0, x1, y0, y1;
    float fx, fy;
    tap(u, t.w[i], &x0, &x1, &fx);
    tap(v, t.h[i], &y0, &y1, &fy);
    const float *lut = t.mode == 0 && c < 3 ? dec : u8n;
    const uint8_t *p = t.tex[i];
    const int w = t.w[i];
    return make_float4(lut[p[((size_t)y1 * w + x0) * 4 + c]], lut[p[((size_t)y1 * w + x1) * 4 + c]],
                       lut[p[((size_t)y0 * w + x1) * 4 + c]], lut[p[((size_t)y0 * w + x0) * 4 + c]]);
}
/* textureSampleBaseClampToEdge: each coordinate clamped to [0.5 / dim, 1 - 0.5 / dim]; the empty view is 1 x 1 */
static float4 BC(const smr_textures &t, int i, float u, float v) {
    const bool live = (unsigned)i < t.count && t.tex[i];
    const float lu = 0.5f / (float)(live ? t.w[i] : 1), lv = 0.5f / (float)(live ? t.h[i] : 1);
    return t.sample((unsigned)i, make_float2(fminf(fmaxf(u, lu), 1.0f - lu), fminf(fmaxf(v, lv), 1.0f - lv)));
}
'''
ID_VS = r'''
static void wo_vs(const wo_base &, const void *, const float *p, const float *tc, float *pos, float *vary) {
    pos[0] = p[0]; pos[1] = p[1]; pos[2] = p[2]; pos[3] = 1.0f; vary[0] = tc[0]; vary[1] = tc[1];
}
'''
FS = "static bool wo_fs(const wo_base &b, const void *, const smr_textures &t, const float *, const float *tc, float4 &out) {\n"
GATHER = tex_shader(UV + r'''    let g0 = textureGather(0, textures[0], sampler_, uv);
    let g1 = textureGather(1u, textures[0], sampler_, uv);
    const three = 3;
    let g3 = textureGather(three, textures[1], sampler_, uv.yx);
    let g2 = textureGather(2, textures[base_params.plane_id + 1], sampler_, uv);
    let c = textureSampleBaseClampToEdge(textures[1], sampler_, uv);
    let d = textureSampleBaseClampToEdge(textures[0], sampler_, input.tex_coords * 3.0 - vec2(1.0));
    return vec4(g0.x * 0.5 + g1.w * 0.5, g0.y * 0.5 + g0.z * 0.5, (g3.x + g3.y + g3.z + g3.w) * 0.25, 1.0) * 0.25
        + g2 * 0.125 + c * 0.25 + d * 0.25;''')
GATHER_RESTATED = VS_PRE + ID_VS + FS + r'''
    const float u = tc[0] * 1.25f - 0.1f, v = tc[1] * 1.25f - 0.05f;
    const float4 g0 = G(t, 0, 0, u, v), g1 = G(t, 1, 0, u, v), g3 = G(t, 3, 1, v, u), g2 = G(t, 2, b.plane_id + 1, u, v);
    const float4 c = BC(t, 1, u, v), d = BC(t, 0, tc[0] * 3.0f - 1.0f, tc[1] * 3.0f - 1.0f);
    const float a[4] = {g0.x * 0.5f + g1.w * 0.5f, g0.y * 0.5f + g0.z * 0.5f, (((g3.x + g3.y) + g3.z) + g3.w) * 0.25f, 1.0f};
    const float g[4] = {g2.x, g2.y, g2.z, g2.w}, cc[4] = {c.x, c.y, c.z, c.w}, dd[4] = {d.x, d.y, d.z, d.w};
    float o[4];
    for (int k = 0; k < 4; k++) o[k] = ((a[k] * 0.25f + g[k] * 0.125f) + cc[k] * 0.25f) + dd[k] * 0.25f;
    out = make_float4(o[0], o[1], o[2], o[3]);
    return true; }'''
# vs_main moves each vertex by a textureSampleLevel of child 0 and a textureSampleGrad of child 1
VS_SAMPLE = r'''@vertex
fn vs_main(input: VertexInput) -> VertexOutput {
    var output: VertexOutput;
    let s = textureSampleLevel(textures[0], sampler_, input.tex_coords * 0.5 + vec2(0.25), 0.0);
    let q = textureSampleGrad(textures[1], sampler_, input.tex_coords.yx, vec2(1.0), vec2(1.0));
    output.position = vec4(input.position.xy * (0.5 + s.x * 0.5) + vec2(s.y - 0.5, q.z - 0.5) * 0.25, 0.0, 1.0);
    output.tex_coords = input.tex_coords;
    return output;
}
'''
VS_SHADER = tex_shader("    return textureSample(textures[u32(base_params.plane_id)], sampler_, input.tex_coords) * 0.75;", VS_SAMPLE)
VS_RESTATED = VS_PRE + r'''
static void wo_vs(const wo_base &, const void *, const float *p, const float *tc, float *pos, float *vary) {
    const float4 s = vs_tex.sample(0, make_float2(tc[0] * 0.5f + 0.25f, tc[1] * 0.5f + 0.25f));
    const float4 q = vs_tex.sample(1, make_float2(tc[1], tc[0]));
    const float k = 0.5f + s.x * 0.5f;
    pos[0] = p[0] * k + (s.y - 0.5f) * 0.25f; pos[1] = p[1] * k + (q.z - 0.5f) * 0.25f; pos[2] = 0.0f; pos[3] = 1.0f;
    vary[0] = tc[0]; vary[1] = tc[1];
}
''' + FS + r'''
    const float4 s = t.sample((unsigned)b.plane_id, make_float2(tc[0], tc[1]));
    out = make_float4(s.x * 0.75f, s.y * 0.75f, s.z * 0.75f, s.w * 0.75f);
    return true; }'''


def render_vs(restatement, W, H, children, pts=0.0, params=b"", mode=0):
    """oracle_wgsl.render through orc_render_wgsl_vs, so that wo_vs can sample the children"""
    L = oracle_wgsl.lib(restatement)
    L.orc_render_wgsl_vs.argtypes = L.orc_render_wgsl.argtypes
    out = np.zeros((H, W, 4), np.uint8)
    kids = [None if c is None else np.ascontiguousarray(c, np.uint8) for c in children]
    ptrs = (C.c_void_p * max(1, len(kids)))(*[None if c is None else c.ctypes.data for c in kids])
    cw = (C.c_int * max(1, len(kids)))(*[1 if c is None else c.shape[1] for c in kids])
    ch = (C.c_int * max(1, len(kids)))(*[1 if c is None else c.shape[0] for c in kids])
    pb = C.create_string_buffer(bytes(params), max(1, len(params)))
    L.orc_render_wgsl_vs(W, H, int(mode), float(oracle_shader.time_of(pts)), pb if params else None, ptrs, cw, ch, len(kids),
                         out.ctypes.data)
    return out


class TexPair(Pair):
    """the WGSL test's pair, its shaders drawn through orc_render_wgsl_vs"""

    def leaf_texture(self, c, frames, live, pts=0.0):
        if isinstance(c, SH) and c.shader_id in self.wgsl:
            kids = [self.leaf_texture(k, frames, live, pts) for k in c.children]
            return render_vs(self.wgsl[c.shader_id][0], int(c.width), int(c.height), kids, pts, b"", self.m)
        return super().leaf_texture(c, frames, live, pts)


def test_texture_shaders_register_and_restatements_build():
    """runs without a GPU: the texture shaders translate and compile; their restatements build and draw"""
    r = host()
    for name, call in SAMPLES.items():
        r.register_wgsl_shader(name, sample_variant(call))
    r.register_wgsl_shader("gather", GATHER)
    r.register_wgsl_shader("vs", VS_SHADER)
    px = TW.page(37, 23, 4)
    for m in (0, 1):
        assert render_vs(GATHER_RESTATED, 40, 30, [px, px], mode=m).any()
        assert render_vs(VS_RESTATED, 40, 30, [px, px], mode=m).any()


def _tex_scene(sid, size):
    return SH(shader_id=sid, width=size[0], height=size[1], children=[IN(input_id=k) for k in TEX_INPUTS])


@pytest.mark.gpu
@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("mode", TW.MODES)
def test_sample_level_bias_grad_are_texture_sample(mode, size):
    """a node texture has one level: every variant gives textureSample's bytes, through the same view"""
    W, H = SIZES[size]
    p = Pair(out=(W, H), fmt=RGBA, mode=mode, inputs=TEX_INPUTS)
    got = {}
    for name, call in SAMPLES.items():
        p.r.register_wgsl_shader(name, sample_variant(call))
        p.r.update_scene("output_1", s.Resolution(W, H), RGBA, _tex_scene(name, (W, H)))
        got[name] = np.asarray(p.r.render(s.FrameSet(frames=p.frames(0.25), pts=0.25)).frames["output_1"].data.planes[0]).copy()
    assert got["textureSample"][..., 3].any()
    for name in SAMPLES:
        assert np.array_equal(got[name], got["textureSample"]), name


@pytest.mark.gpu
@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("mode", TW.MODES)
def test_gather_and_clamp_to_edge_match_oracle(mode, size):
    p = TexPair(out=SIZES[size], fmt=RGBA, mode=mode, inputs=TEX_INPUTS)
    p.register_wgsl("gather", None, src=GATHER, restated=GATHER_RESTATED)
    p.update(_tex_scene("gather", SIZES[size]))
    p.render_check(0.25, "gather")


@pytest.mark.gpu
@pytest.mark.parametrize("size", sorted(SIZES))
@pytest.mark.parametrize("mode", TW.MODES)
def test_vertex_stage_sampling_matches_oracle(mode, size):
    p = TexPair(out=SIZES[size], fmt=RGBA, mode=mode, inputs=TEX_INPUTS)
    p.register_wgsl("vs", None, src=VS_SHADER, restated=VS_RESTATED)
    p.update(_tex_scene("vs", SIZES[size]))
    p.render_check(0.25, "vertex sampling")
