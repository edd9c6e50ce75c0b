"""smr_set_input_color on the H100: every reader of input YUV converts with the input's matrix and range, byte for byte
against the colour oracle `tests/input_color_oracle.c` (DESIGN.md NC-13), and an input left at the default converts as before.

- the composite's 1:1 reader over the joint byte space of every YUV format, for BT.709 / BT.601 x limited / full;
- every fused-kernel instantiation with a BT.601 source (and the interleaved sources at full range), as the library
  lists them (smr_debug_fused_variants), with the same kernel choice as the BT.709 child of the same geometry;
- one tick that mixes matrices and ranges on k_resample_tma3 with direct tiles and on k_resample_tma0: one launch per
  (kernel, source class, range, matrix) key;
- the composite's fast readers (FAST_HALF, FAST_IDENT), rotated and masked layers and the generic reader;
- defaults, and explicit settings equal to a format's own rule, give the bytes of a handle that never made the call;
- a setting changed between ticks, an input registered again, deinterlacing with BT.601, RGB inputs.
"""
import numpy as np
import pytest

import smelter_b200 as s
from smelter_b200 import _ffi as F
from oracle import oracle as orc
from tests import input_color_oracle as ico
from tests.test_color_conversion_space import yuv420_block_triples
from tests.test_gpu_color_conversion import interleaved_frame, reader_frames, run_one, yuv_frame
from tests.parity import to_oracle_layout
from tests.test_gpu_composite_classes import child
from tests.test_gpu_fused_variants import (ALIGNED, REGISTRY, Job, fused_variants, make_frame, mismatch_report, render,
                                           scene_of)

pytestmark = pytest.mark.gpu

GPU, CPU = s.RenderingMode.GpuOptimized, s.RenderingMode.CpuOptimized
RGBA, YUV = s.OutputFrameFormat.RgbaWgpuTexture, s.OutputFrameFormat.PlanarYuv420Bytes
OUTPUT_ID = "output_1"
BT709, BT601 = s.YuvMatrix.BT709, s.YuvMatrix.BT601
LIMITED, FULL = s.YuvRange.Limited, s.YuvRange.Full


# ------------------------------------------------------------------------------------------------
# the oracle with a colour setting per input
# ------------------------------------------------------------------------------------------------
def effective(frame, color):
    """(full_range, oracle matrix) a frame converts with under color = (matrix, range) (DEFAULT: the format's rule)"""
    m, r = color
    fr = (frame.data.kind == "PlanarYuvJ420") if r == s.YuvRange.Default else r == FULL
    return int(fr), 1 if m == BT601 else 0


def node_texture_color(frame, color=(s.YuvMatrix.Default, s.YuvRange.Default)):
    d = frame.data
    w, h = frame.resolution.width, frame.resolution.height
    fr, m = effective(frame, color)
    if d.kind in ("PlanarYuv420", "PlanarYuvJ420"):
        return ico.yuv_planar_to_rgba(*d.planes, w, h, w // 2, h // 2, fr, m)
    if d.kind == "PlanarYuv422":
        return ico.yuv_planar_to_rgba(*d.planes, w, h, w // 2, h, fr, m)
    if d.kind == "PlanarYuv444":
        return ico.yuv_planar_to_rgba(*d.planes, w, h, w, h, fr, m)
    if d.kind in ("InterleavedUyvy422", "InterleavedYuyv422"):
        return ico.interleaved422_to_rgba(d.planes[0], w, h, d.kind == "InterleavedYuyv422", fr, m)
    if d.kind == "Nv12":
        return ico.nv12_to_rgba(d.planes[0], d.planes[1], w, h, fr, m)
    from tests.parity import node_texture
    return node_texture(frame)


def oracle_layers(layers, frames, ids, colors, root, out_res, fmt, mode):
    rgba = orc.render_layout_node(root[0], root[1], [to_oracle_layout(l) for l in layers],
                                  [node_texture_color(frames[i], colors.get(i, (0, 0))) for i in ids], mode=int(mode))
    w, h = out_res
    if fmt == RGBA:
        return [rgba.reshape(h, w * 4)]
    return list(orc.rgba_to_yuv_planar_scaled(rgba, w, h, w // 2, h // 2))


def first_diff(got, exp, what):
    got, exp = np.asarray(got).reshape(np.shape(exp)), np.asarray(exp)
    if not np.array_equal(got, exp):
        d = np.argwhere(got != exp)
        raise AssertionError(f"{what}: {len(d)} bytes differ; first at {tuple(d[0])}: got {got[tuple(d[0])]} expected "
                             f"{exp[tuple(d[0])]}")


def colored_renderer(colors, mode=GPU):
    r = s.Renderer(s.RendererOptions(rendering_mode=mode))
    for i, c in colors.items():
        r.register_input(i)
        r.set_input_color(i, *c)
    r.set_profiling(True)
    return r


SETTINGS = [(BT709, LIMITED), (BT709, FULL), (BT601, LIMITED), (BT601, FULL)]
SETTING_IDS = ["709-limited", "709-full", "601-limited", "601-full"]


# ------------------------------------------------------------------------------------------------
# 1. the joint byte space through the composite's 1:1 reader
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("color", SETTINGS, ids=SETTING_IDS)
@pytest.mark.parametrize("kind", ["yuv", "yuvj", "nv12", "yuv422", "yuv444", "uyvy", "yuyv"])
def test_passthrough_every_tuple(kind, color):
    """every (Y, U, V) of the format's reader frames shown 1:1 as the only opaque child of a GpuOptimized RGBA root: the
    composite converts it with the input's setting (one composite launch, no k_convert, no fused resample) and, as
    encode(decode(b)) == b, its bytes are the oracle's node texture"""
    for name, fr in reader_frames(kind):
        w, h = fr.resolution.width, fr.resolution.height
        ls = [child(0, 0.0, 0.0, float(w), float(h), w, h)]
        r = colored_renderer({"a": color})
        got = run_one(ls, {"a": fr}, ["a"], (w, h), (w, h), RGBA, r)
        kt = r.kernel_times()
        assert kt["composite"][1] == 1 and kt["convert"][1] == 0 and kt["resample_fused"][1] == 0, (kind, name, kt)
        info = r.debug_composite_layers()
        assert info[0]["tex_matrix"] == color[0], info[0]
        first_diff(got[0], node_texture_color(fr, color), f"{kind} {name} {color}")
        r.close()


# ------------------------------------------------------------------------------------------------
# 2. / 3. every fused-kernel instantiation with BT.601, and the same kernel choice as BT.709
# ------------------------------------------------------------------------------------------------
def color_registry():
    """one (REGISTRY entry, (matrix, range)) per colour instantiation; DEFAULT keeps the entry's format rule"""
    R = []
    for e in REGISTRY:
        R.append((e, (BT601, s.YuvRange.Default)))
        if e.kernel == "tma_int" and e.fmt == "nv12":
            R.append((e, (BT601, FULL)))
        if e.fmt in ("uyvy", "yuyv"):
            R.append((e, (BT601, FULL)))
            R.append((e, (BT709, FULL)))
    return R


COLOR_REGISTRY = color_registry()


def key_of(e, color, compiled):
    """the launch key of entry e's job under `color`: a kernel compiled for one range runs a full-range source at range 1,
    any other reads the range per job (0)"""
    fr = (1 if e.fmt == "yuvj" else 0) if color[1] == s.YuvRange.Default else int(color[1] == FULL)
    key = (e.kernel, e.ratio, e.window, e.box, e.src_class, 1 if color[0] == BT601 else 0)
    return key + (fr if key + (1,) in compiled else 0,)


def test_color_registry_covers_every_new_compiled_variant():
    """every instantiation a BT.601 source (or an interleaved source at full range) reaches has a scene"""
    compiled = set(fused_variants())
    have = {key_of(e, c, compiled) for e, c in COLOR_REGISTRY}
    want = {k for k in compiled if k[5] == 1 or (k[0] == "ldg" and k[6] == 1)}
    assert len(want) == 56, sorted(want)
    assert want <= have, f"instantiations without a scene: {sorted(want - have)}"


def oracle_color_planes(jobs, frames, colors, out_format):
    W, H, ids, ls, _ = scene_of(jobs)
    rgba = orc.render_layout_node(W, H, [to_oracle_layout(l) for l in ls],
                                  [node_texture_color(frames[i], colors[i]) for i in ids], mode=GPU)
    if out_format == RGBA:
        return (rgba,)
    return orc.rgba_to_yuv_planar_scaled(rgba, W, H, W // 2, H // 2)


@pytest.mark.parametrize("case", COLOR_REGISTRY, ids=[f"{e.name}-{'601' if c[0] == BT601 else '709'}-{c[1]}"
                                                      for e, c in COLOR_REGISTRY])
def test_fused_variant(case):
    """the scene with the setting takes the kernel, ratio, window, box and direct decision of the same scene at BT.709
    and the format's range (only `matrix` and `full_range` differ), and its RGBA equals the oracle's, for extreme and
    smooth content"""
    e, color = case
    jobs = [Job("input_1", e.crop, e.dst)]
    for content in ("extreme", "smooth"):
        frame = make_frame(e.fmt, content, 3, *e.src)
        ra, rb = colored_renderer({"input_1": color}), s.Renderer()
        got = render(ra, jobs, {"input_1": frame}, RGBA)
        ref = render(rb, jobs, {"input_1": frame}, RGBA)
        fa, fb = ra.debug_fused_jobs(), rb.debug_fused_jobs()
        assert len(fa) == len(fb) == 1, (fa, fb)
        fr, m = effective(frame, color)
        assert fa[0]["matrix"] == (2 if m else 1) and fa[0]["full_range"] == fr, fa[0]
        assert fb[0]["matrix"] == 1
        same = {k: (fa[0][k], fb[0][k]) for k in fa[0] if k not in ("matrix", "full_range") and fa[0][k] != fb[0][k]}
        assert not same, (e.name, same)
        for k, v in e.expect().items():
            if k != "full_range":
                assert fa[0][k] == v, (e.name, k, fa[0][k], v)
        rep = mismatch_report(got, oracle_color_planes(jobs, {"input_1": frame}, {"input_1": color}, RGBA), jobs, fa)
        assert rep is None, f"{e.name} {color} {content}: {rep}"
        if m and content == "extreme":
            assert not np.array_equal(got[0], ref[0])
        ra.close()
        rb.close()


# ------------------------------------------------------------------------------------------------
# 4. one tick that mixes matrices and ranges
# ------------------------------------------------------------------------------------------------
def test_mixed_tick():
    """BT.709-limited, BT.601-limited and BT.601-full NV12 children at 4:1 (k_resample_tma3, direct tiles into a planar
    4:2:0 output) and BT.709 / BT.601 planar 4:2:0 children at 1.5:1 (k_resample_tma0): the output equals the oracle, and
    the fused kernel runs once per (kernel, source class, range, matrix) key -- five launches"""
    colors = {"a": (BT709, LIMITED), "b": (BT601, LIMITED), "c": (BT601, FULL), "d": (BT709, LIMITED), "e": (BT601, LIMITED)}
    frames = {i: make_frame("nv12", "extreme", k, 1920, 1080) for k, i in enumerate("abc")}
    frames.update({i: make_frame("yuv", "extreme", 5 + k, 960, 540) for k, i in enumerate("de")})
    ids = list("abcde")
    ls = [child(k, 512.0 * k, 0.0, 480.0, 270.0, 1920, 1080) for k in range(3)]
    ls += [child(3 + k, 656.0 * k, 272.0, 640.0, 360.0, 960, 540) for k in range(2)]
    root = (1536, 640)
    r = colored_renderer(colors)
    from tests.test_gpu_fused_variants import fill_input
    import torch
    keep = []
    arr = (F.InputFrame * len(ids))()
    for k, i in enumerate(ids):
        fill_input(arr[k], i, frames[i], ALIGNED, keep)
    r.set_layouts(OUTPUT_ID, s.Resolution(*root), YUV, root, ids, ls)
    planes = [np.zeros(sh, np.uint8) for sh in ((root[1], root[0]), (root[1] // 2, root[0] // 2), (root[1] // 2, root[0] // 2))]
    outs = (F.OutputFrame * 1)()
    ob = OUTPUT_ID.encode()
    outs[0].output_id, outs[0].mem_kind = ob, F.MEM_HOST
    for p, a in enumerate(planes):
        outs[0].planes[p] = a.ctypes.data
    torch.cuda.synchronize()
    r.render_raw(0, arr, len(ids), outs, 1)
    fused = r.debug_fused_jobs()
    kinds = sorted((j["kernel"], j["src_class"], j["full_range"], j["matrix"]) for j in fused)
    assert kinds == sorted([("tma_int", 1, 0, 1), ("tma_int", 1, 0, 2), ("tma_int", 1, 1, 2), ("tma_any", 0, 0, 1),
                            ("tma_any", 0, 0, 2)]), kinds
    assert any(j["direct"] for j in fused if j["kernel"] == "tma_int") and r.stats()["last_render_direct_tiles"] > 0, fused
    assert r.kernel_times()["resample_fused"][1] == 5, r.kernel_times()
    exp = oracle_layers(ls, frames, ids, colors, root, root, YUV, GPU)
    for p, (g, e) in enumerate(zip(planes, exp)):
        first_diff(g, e, f"mixed tick plane {p}")
    r.close()


# ------------------------------------------------------------------------------------------------
# 5. the composite's readers
# ------------------------------------------------------------------------------------------------
def composite_case(name):
    """(layers, frames, ids, root, mode, fast bits the probe layer 0 must have)"""
    (y, u, v), _ = yuv420_block_triples(1)
    y, u, v = (np.ascontiguousarray(p[:512, :1024]) if p is y else np.ascontiguousarray(p[:256, :512]) for p in (y, u, v))
    if name == "half":   # cfg2's shape: CpuOptimized, a 4:2:0 child at exactly half its size
        fr = {"a": yuv_frame("nv12", y, u, v)}
        return [child(0, 0.0, 0.0, 512.0, 256.0, 1024, 512)], fr, ["a"], (512, 256), CPU, 32
    if name == "ident":
        fr = {"a": yuv_frame("yuv", y, u, v)}
        return [child(0, 8.0, 4.0, 1024.0, 512.0, 1024, 512)], fr, ["a"], (1040, 520), GPU, 1
    if name == "rotated":
        fr = {"a": yuv_frame("nv12", y, u, v)}
        return [child(0, 40.0, 30.0, 700.0, 350.0, 1024, 512, rotation=17.0)], fr, ["a"], (800, 420), CPU, 0
    if name == "masked":
        fr = {"a": yuv_frame("yuv", y, u, v)}
        return [child(0, 0.0, 0.0, 1024.0, 512.0, 1024, 512, radius=(40, 10, 0, 60),
                      masks=[((30, 30, 30, 30), 20.0, 20.0, 900.0, 400.0)])], fr, ["a"], (1024, 512), GPU, 0
    kind = name.split("-")[1]   # generic reader: scaled 4:2:2 / 4:4:4 / UYVY / YUYV children drawn by the layout shader
    if kind in ("uyvy", "yuyv"):
        t = np.empty((512, 512, 4), np.uint8)
        t[..., 0], t[..., 1], t[..., 2], t[..., 3] = y[:, 0::2], u.repeat(2, 0), y[:, 1::2], v.repeat(2, 0)
        fr = {"a": interleaved_frame(t, kind == "yuyv")}
    elif kind == "yuv422":
        fr = {"a": yuv_frame(kind, y, u.repeat(2, 0), v.repeat(2, 0))}
    else:
        fr = {"a": yuv_frame(kind, y, np.ascontiguousarray(y[:, ::-1]), np.ascontiguousarray(y[::-1]))}
    return [child(0, 3.0, 2.0, 700.0, 333.0, 1024, 512)], fr, ["a"], (720, 340), CPU, 0


COMPOSITE_CASES = ["half", "ident", "rotated", "masked", "generic-yuv422", "generic-yuv444", "generic-uyvy", "generic-yuyv"]


@pytest.mark.parametrize("color", [(BT601, LIMITED), (BT601, FULL)], ids=["601-limited", "601-full"])
@pytest.mark.parametrize("name", COMPOSITE_CASES)
def test_composite_readers(name, color):
    ls, frames, ids, root, mode, fast = composite_case(name)
    r = colored_renderer({"a": color}, mode)
    got = run_one(ls, frames, ids, root, root, RGBA, r)
    kt = r.kernel_times()
    assert kt["resample_fused"][1] == 0, (name, kt)
    info = r.debug_composite_layers()
    assert info[0]["tex_matrix"] == BT601 and (info[0]["fast"] & fast) == fast, info[0]
    first_diff(got[0], oracle_layers(ls, frames, ids, {"a": color}, root, root, RGBA, mode)[0], f"{name} {color}")
    r.close()


@pytest.mark.parametrize("fmt", [RGBA, YUV], ids=["rgba", "yuv420"])
@pytest.mark.parametrize("kind", ["nv12", "yuyv"])
def test_passthrough_root(kind, fmt):
    """a BT.601 input as the scene's root, to RGBA at its size and to 4:2:0 at its size and scaled to another output size"""
    (y, u, v), _ = yuv420_block_triples(2)
    y, u, v = np.ascontiguousarray(y[:360, :640]), np.ascontiguousarray(u[:180, :320]), np.ascontiguousarray(v[:180, :320])
    if kind == "nv12":
        fr = yuv_frame(kind, y, u, v)
    else:
        t = np.empty((360, 320, 4), np.uint8)
        t[..., 0], t[..., 1], t[..., 2], t[..., 3] = y[:, 0::2], u.repeat(2, 0), y[:, 1::2], v.repeat(2, 0)
        fr = interleaved_frame(t, True)
    for out in ((640, 360),) if fmt == RGBA else ((640, 360), (320, 180)):   # an RGBA root keeps the input's size
        r = s.Renderer()
        r.register_input("a")
        r.set_input_color("a", BT601, LIMITED)
        ref = s.Renderer()
        for rr in (r, ref):
            rr.register_input("a")
            rr.update_scene("out", s.Resolution(*out), fmt, s.InputStreamComponent(input_id="a"))
        got = [np.array(p) for p in r.render(s.FrameSet(frames={"a": fr}, pts=0.0)).frames["out"].data.planes]
        node = node_texture_color(fr, (BT601, LIMITED))
        if fmt == RGBA and out == (640, 360):
            first_diff(got[0], node, f"{kind} root rgba")
        elif fmt == YUV:
            w, h = out
            exp = orc.rgba_to_yuv_planar_scaled(node, w, h, w // 2, h // 2)
            for p, (g, e) in enumerate(zip(got, exp)):
                first_diff(g, e, f"{kind} root yuv {out} plane {p}")
        base = [np.array(p) for p in ref.render(s.FrameSet(frames={"a": fr}, pts=0.0)).frames["out"].data.planes]
        assert not np.array_equal(got[0], base[0])
        r.close()
        ref.close()


# ------------------------------------------------------------------------------------------------
# 6. defaults change nothing
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["fused_4to1_direct", "one_to_one", "generic_422"])
def test_defaults_are_unchanged(name):
    """{DEFAULT, DEFAULT}, and an explicit setting equal to each format's own rule, give the bytes and launches of a handle
    that never made the call (two ticks each)"""
    from tests.test_deinterlace import random_planes
    from tests.test_gpu_deinterlace import make_handle, render_scene, scene_inputs
    _, _, _, ins = scene_inputs(name)
    content = {i: random_planes(fmt, w, h, n + 70) for n, (i, (fmt, w, h)) in enumerate(ins.items())}
    ref = make_handle(name)
    want = [render_scene(ref, name, content, k * 0.04) for k in range(2)]
    launches = ref.stats()["last_render_kernel_launches"]
    ref.close()
    for setting in ("default", "own rule"):
        r = make_handle(name)
        for i, (fmt, _, _) in ins.items():
            if setting == "default":
                r.set_input_color(i, s.YuvMatrix.Default, s.YuvRange.Default)
            else:
                r.set_input_color(i, BT709, FULL if fmt == F.FRAME_PLANAR_YUVJ420 else LIMITED)
        for k in range(2):
            got = render_scene(r, name, content, k * 0.04)
            for p, (g, wnt) in enumerate(zip(got, want[k])):
                assert np.array_equal(g, wnt), (name, setting, k, p)
        assert r.stats()["last_render_kernel_launches"] == launches
        r.close()


def test_registry_defaults_are_unchanged():
    """every fused-registry scene (J420 at BT.709 full, the others at BT.709 limited) is byte-identical to no call"""
    for e in REGISTRY:
        frame = make_frame(e.fmt, "extreme", 9, *e.src)
        jobs = [Job("input_1", e.crop, e.dst)]
        color = (BT709, FULL if e.fmt == "yuvj" else LIMITED)
        ra, rb = colored_renderer({"input_1": color}), s.Renderer()
        a, b = render(ra, jobs, {"input_1": frame}, RGBA), render(rb, jobs, {"input_1": frame}, RGBA)
        assert np.array_equal(a[0], b[0]), e.name
        ra.close()
        rb.close()


# ------------------------------------------------------------------------------------------------
# 7. lifetime and combinations
# ------------------------------------------------------------------------------------------------
def one_tick(r, frame, out, wait=True, planes=None):
    keep = []
    from tests.test_gpu_composite_classes import host_input
    arr = (F.InputFrame * 1)()
    host_input(arr[0], "a", frame, keep)
    outs = (F.OutputFrame * 1)()
    ob = OUTPUT_ID.encode()
    outs[0].output_id, outs[0].mem_kind = ob, F.MEM_HOST
    outs[0].planes[0] = planes.ctypes.data
    r.render_raw(0, arr, 1, outs, 1, wait=wait)
    return keep


def test_setting_changed_between_ticks_in_flight():
    """two ticks in flight on one handle: the first planned at BT.601, the second at BT.709; each keeps its own"""
    (y, u, v), _ = yuv420_block_triples(3)
    fr = yuv_frame("nv12", np.ascontiguousarray(y[:256, :512]), np.ascontiguousarray(u[:128, :256]),
                   np.ascontiguousarray(v[:128, :256]))
    ls = [child(0, 0.0, 0.0, 512.0, 256.0, 512, 256)]
    r = s.Renderer()
    r.register_input("a")
    r.set_layouts(OUTPUT_ID, s.Resolution(512, 256), RGBA, (512, 256), ["a"], ls)
    o1, o2 = np.zeros(512 * 256 * 4, np.uint8), np.zeros(512 * 256 * 4, np.uint8)
    r.set_input_color("a", BT601, LIMITED)
    k1 = one_tick(r, fr, OUTPUT_ID, wait=False, planes=o1)
    r.set_input_color("a", BT709, LIMITED)
    k2 = one_tick(r, fr, OUTPUT_ID, wait=False, planes=o2)
    r.wait()
    r.wait()
    del k1, k2
    for o, c in ((o1, (BT601, LIMITED)), (o2, (BT709, LIMITED))):
        first_diff(o, oracle_layers(ls, {"a": fr}, ["a"], {"a": c}, (512, 256), (512, 256), RGBA, GPU)[0], f"tick {c}")
    r.close()


def test_reregistered_input_returns_to_the_default():
    (y, u, v), _ = yuv420_block_triples(0)
    fr = yuv_frame("yuv", np.ascontiguousarray(y[:256, :512]), np.ascontiguousarray(u[:128, :256]),
                   np.ascontiguousarray(v[:128, :256]))
    ls = [child(0, 0.0, 0.0, 512.0, 256.0, 512, 256)]
    r = s.Renderer()
    r.register_input("a")
    r.set_input_color("a", BT601, FULL)
    a = run_one(ls, {"a": fr}, ["a"], (512, 256), (512, 256), RGBA, r)[0]
    first_diff(a, oracle_layers(ls, {"a": fr}, ["a"], {"a": (BT601, FULL)}, (512, 256), (512, 256), RGBA, GPU)[0], "601")
    r.unregister_input("a")
    b = run_one(ls, {"a": fr}, ["a"], (512, 256), (512, 256), RGBA, r)[0]
    first_diff(b, oracle_layers(ls, {"a": fr}, ["a"], {}, (512, 256), (512, 256), RGBA, GPU)[0], "default again")
    r.close()


def test_deinterlace_with_bt601():
    """FIELD deinterlacing runs on the bytes, then the BT.601 conversion: the tick equals a handle that is fed the
    deinterlaced planes and the same colour setting"""
    from tests.test_deinterlace import FIELD, TOP, deinterlace_plane, random_planes
    planes = random_planes(F.FRAME_NV12, 640, 360, 77)
    di = [deinterlace_plane(p, FIELD, TOP) for p in planes]
    mk = lambda ps: s.Frame(s.FrameData.Nv12(s.NvPlanes(ps[0], np.asarray(ps[1]).reshape(180, 320, 2))), s.Resolution(640, 360))
    out = []
    for deint, ps in ((True, planes), (False, di)):
        r = s.Renderer()
        r.register_input("a")
        r.set_input_color("a", BT601, LIMITED)
        if deint:
            r.set_input_deinterlace("a", s.DeinterlaceMode.Field, s.FieldOrder.TopFirst)
        r.update_scene("out", s.Resolution(320, 180), YUV, s.InputStreamComponent(input_id="a"))
        out.append([np.array(p) for p in r.render(s.FrameSet(frames={"a": mk(ps)}, pts=0.0)).frames["out"].data.planes])
        r.close()
    for p, (g, e) in enumerate(zip(*out)):
        first_diff(g, e, f"deinterlaced plane {p}")


@pytest.mark.parametrize("kind", ["bgra", "argb", "rgba"])
def test_rgb_inputs_ignore_the_setting(kind):
    from tests.test_gpu_color_conversion import rgb_frame
    rng = np.random.default_rng(5)
    rgba = rng.integers(0, 256, (180, 320, 4), dtype=np.uint8)
    rgba[..., 3] = 255
    fr = rgb_frame(kind, rgba)
    ls = [child(0, 0.0, 0.0, 200.0, 100.0, 320, 180)]
    a = run_one(ls, {"a": fr}, ["a"], (200, 100), (200, 100), RGBA, colored_renderer({"a": (BT601, FULL)}))[0]
    b = run_one(ls, {"a": fr}, ["a"], (200, 100), (200, 100), RGBA, s.Renderer())[0]
    assert np.array_equal(a, b)
