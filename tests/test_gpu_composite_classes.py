"""Every fast class of the composite (k_composite_p / k_composite_multi) against the oracle, byte for byte.

Inside a layer's interior bars the composite replaces the fragment shader with a fast class -- FAST_CONST, FAST_LUT,
FAST_HALF, FAST_SAMPLE, FAST_IDENT, FAST_OPAQUE occlusion -- and outside them its general path shades the pixels a warp
gathers (cooperatively, or each lane its own when a warp has more than 160).  Each scene here is built with `set_layouts`
so that one probe layer gets one class and sub-branch on purpose; smr_debug_composite_layers confirms which.  Scenes are
crossed with both rendering modes, RGBA / planar 4:2:0 / NV12 output (the fused K10 / K11 stores) plus a 4:2:2 output
through k_output, and with one output (k_composite_p) against many layers or two outputs (k_composite_multi).  Content
is the extreme content of the fused-resample tests: every code, 0 / 255 runs.

The second half covers caller-owned device output planes at every alignment: bytes equal the host-output run and the
oracle, guard bytes around each plane stay untouched, and RGBA8 planes that are not 4-byte aligned are refused before
any kernel runs.
"""
from dataclasses import dataclass
from typing import Callable, Dict, Optional

import numpy as np
import pytest

import smelter_b200 as s
from smelter_b200 import _ffi as F
from smelter_b200.renderer import _FRAME_KIND
from tests.parity import OUTPUT_ID, node_texture, to_oracle_layout
from tests.test_gpu_fused_variants import extreme_plane, make_frame, plane_list

GPU, CPU = s.RenderingMode.GpuOptimized, s.RenderingMode.CpuOptimized
RGBA, YUV, NV12 = s.OutputFrameFormat.RgbaWgpuTexture, s.OutputFrameFormat.PlanarYuv420Bytes, s.OutputFrameFormat.Nv12WgpuTexture
YUV422 = F.OUT_PLANAR_YUV422
IDENT, CONST, LUT, OPAQUE, SAMPLE, HALF = 1, 2, 4, 8, 16, 32
NAN = float("nan")
# root: width = 2 (mod 4), height = 2 (mod 16), two 128 x 16 tiles across and four down
W, H = 258, 66


def rgba_frame(seed, w, h, translucent=0.0, one_translucent=False):
    """premultiplied RGBA8 with extreme colour bytes; alpha 255 except a share `translucent` of texels (or one texel)"""
    rng = np.random.default_rng(seed)
    t = np.empty((h, w, 4), np.uint8)
    for c in range(3):
        t[..., c] = extreme_plane(rng, w, h)
    t[..., 3] = 255
    if translucent:
        a = rng.integers(0, 256, (h, w)).astype(np.uint8)
        sel = rng.random((h, w)) < translucent
        t[..., 3][sel] = a[sel]
    if one_translucent:
        t[h // 2, w // 2, 3] = 17
    t[..., :3] = np.minimum(t[..., :3], t[..., 3:4])   # premultiplied: colour <= alpha
    return s.Frame(s.FrameData.Rgba8(t), s.Resolution(w, h))


def layout(type, left, top, width, height, child=0, color=(0, 0, 0, 0), radius=(0, 0, 0, 0), border=0.0,
           border_color=(0, 0, 0, 0), masks=(), rotation=0.0, crop=None, blur=0.0):
    l = F.RenderLayout()
    l.type, l.left, l.top, l.width, l.height, l.rotation_degrees = type, left, top, width, height, rotation
    l.child_index = child
    l.color, l.border_color = F.Rgba(*color), F.Rgba(*border_color)
    l.border_radius[:] = list(radius)
    l.border_width, l.blur_radius = border, blur
    if crop is not None:
        l.crop_left, l.crop_top, l.crop_width, l.crop_height = crop
    l.masks_len = len(masks)
    for i, (r, t, le, w, h) in enumerate(masks):
        l.masks[i].radius[:] = list(r)
        l.masks[i].top, l.masks[i].left, l.masks[i].width, l.masks[i].height = t, le, w, h
    return l


def child(k, left, top, w, h, src_w, src_h, **kw):
    return layout(0, left, top, w, h, child=k, crop=(0.0, 0.0, float(src_w), float(src_h)), **kw)


def colour(left, top, w, h, rgba, **kw):
    return layout(1, left, top, w, h, color=rgba, **kw)


# ------------------------------------------------------------------------------------------------
# the registry: one scene per fast class and sub-branch
# ------------------------------------------------------------------------------------------------
@dataclass
class Scene:
    name: str
    build: Callable                 # (dx, dy) -> (layers, {input id: frame}, [input ids])
    probe: int                      # index (among drawn layers) of the layer whose class is checked
    fast: int                       # bits the probe must have
    not_fast: int = 0               # bits it must not have
    modes: tuple = (GPU, CPU)
    device_inputs: Optional[Dict[str, tuple]] = None   # input id -> per-plane pitch mod 16 (device planes)
    probe_check: Optional[Callable] = None             # extra check of the probe's hook record


def background(ids, frames):
    """an opaque YUV child under everything, so that translucent layers blend over varying bytes"""
    frames["bg"] = make_frame("yuv", "extreme", 5, W, H)
    ids.append("bg")
    return child(len(ids) - 1, 0.0, 0.0, float(W), float(H), W, H)


def sc_const(dx, dy):
    ids, fr = [], {}
    bg = background(ids, fr)
    return [bg, colour(3.0 + dx, 1.0 + dy, 200.0, 60.0, (200, 40, 90, 255), radius=(6, 0, 11, 3))], fr, ids


def sc_lut(n):
    def build(dx, dy):
        ids, fr = [], {}
        ls = [background(ids, fr)]
        for k in range(n):
            ls.append(colour(2.0 + dx + 3 * k, 1.0 + dy + k, 180.0, 50.0, (30 * k, 60, 110, 100 + 30 * k), radius=(4, 4, 4, 4)))
        return ls, fr, ids
    return build


def sc_half(fmt):
    def build(dx, dy):
        fr = {"a": make_frame(fmt, "extreme", 11, 2 * 128, 2 * 32)}
        # the layer at an even position: its pixel (x, y) takes texels (2 (x - left), 2 (y - top)); the guard of the
        # packed path needs 2 <= texel x and texel x + 9 <= W - 1 -- blocks at texel x 0, 2 and W - 10 sit on its edges
        return [child(0, 2.0 * dx, 2.0 * dy, 128.0, 32.0, 256, 64)], fr, ["a"]
    return build


def sc_sample_rgba(dx, dy):   # GpuOptimized: a child resampled 1.5:1 by the fused kernel (opaque RGBA8), fractional size
    fr = {"a": make_frame("nv12", "extreme", 12, 1280, 720)}
    return [child(0, -300.25 + dx, -200.5 + dy, 852.4, 480.4, 1280, 720)], fr, ["a"]


def sc_sample_yuv(fmt):   # CpuOptimized: the layout shader's own bilinear scaling of a YUV child
    def build(dx, dy):
        fr = {"a": make_frame(fmt, "extreme", 13, 160, 90)}
        return [child(0, 1.5 + dx, 0.25 + dy, 211.0, 61.5, 160, 90)], fr, ["a"]
    return build


def sc_ident_yuv(fmt):
    def build(dx, dy):
        fr = {"a": make_frame(fmt, "extreme", 14, 200, 60)}
        return [child(0, float(2 * dx), float(2 * dy), 200.0, 60.0, 200, 60)], fr, ["a"]
    return build


def sc_ident_rgba(translucent=0.0, one=False):
    def build(dx, dy):
        ids, fr = [], {}
        ls = [background(ids, fr)]
        fr["a"] = rgba_frame(15, 200, 60, translucent, one)
        ids.append("a")
        ls.append(child(1, float(4 + dx), float(2 + dy), 200.0, 60.0, 200, 60))
        return ls, fr, ids
    return build


def sc_occlusion(dx, dy):
    ids, fr = [], {}
    ls = [background(ids, fr)]
    ls.append(colour(10.0, 5.0, 100.0, 40.0, (10, 200, 30, 160), radius=(5, 5, 5, 5)))
    ls.append(colour(0.0 + dx, 0.0 + dy, 240.0, 62.0, (90, 10, 200, 255)))   # opaque: hides both below in its bars
    ls.append(colour(20.5, 10.5, 50.0, 20.0, (200, 200, 30, 90)))
    return ls, fr, ids


def sc_dense(dx, dy):   # a rotated child: every covered pixel runs the fragment shader, most warps > 160 pixels
    fr = {"a": make_frame("yuv", "extreme", 16, 160, 90)}
    return [child(0, 30.0 + dx, -40.0 + dy, 200.0, 150.0, 160, 90, rotation=45.0)], fr, ["a"]


def sc_coop(dx, dy):    # rounded corners, a border and a mask: thin bands of general pixels
    ids, fr = [], {}
    ls = [background(ids, fr)]
    ls.append(colour(4.0 + dx, 3.0 + dy, 230.0, 58.0, (40, 90, 200, 255), radius=(9, 20, 2, 14), border=1.001,
                     border_color=(250, 250, 0, 255), masks=[((3, 3, 3, 3), 1.0, 1.0, 250.0, 64.0)]))
    return ls, fr, ids


REGISTRY = [
    Scene("const", sc_const, 1, CONST | OPAQUE),
    *[Scene(f"lut{n}", sc_lut(n), n, LUT) for n in (1, 4)],
    Scene("lut5", sc_lut(5), 5, LUT),   # the fifth translucent layer of a tile has no table: the general path
    Scene("half_nv12_pairs", sc_half("nv12"), 0, HALF | SAMPLE, modes=(CPU,), device_inputs={"a": (0, 0)}),
    Scene("half_nv12_rows", sc_half("nv12"), 0, HALF | SAMPLE, modes=(CPU,), device_inputs={"a": (0, 2)}),
    Scene("half_planar", sc_half("yuv"), 0, HALF | SAMPLE, modes=(CPU,)),
    Scene("sample_rgba", sc_sample_rgba, 0, SAMPLE | OPAQUE, not_fast=HALF, modes=(GPU,),
          probe_check=lambda L: L["tex_kind"] == 1),
    *[Scene(f"sample_{f}", sc_sample_yuv(f), 0, SAMPLE | OPAQUE, not_fast=HALF, modes=(CPU,)) for f in ("yuv", "nv12")],
    *[Scene(f"ident_{f}_quad", sc_ident_yuv(f), 0, IDENT | OPAQUE, modes=(CPU,)) for f in ("yuv", "nv12")],
    Scene("ident_rgba_vec", sc_ident_rgba(), 1, IDENT, probe_check=lambda L: L["tex_kind"] == 1),
    Scene("ident_rgba_translucent", sc_ident_rgba(0.3), 1, IDENT),
    Scene("ident_rgba_one_translucent", sc_ident_rgba(0.0, True), 1, IDENT),
    Scene("occlusion", sc_occlusion, 2, CONST | OPAQUE),
    Scene("dense", sc_dense, 0, 0, not_fast=IDENT | SAMPLE, probe_check=lambda L: L["rotated"] == 1),
    Scene("coop", sc_coop, 1, CONST | OPAQUE),
]
SCENES = {sc.name: sc for sc in REGISTRY}


def test_registry_names_every_fast_class():
    bits = 0
    for sc in REGISTRY:
        bits |= sc.fast
    assert bits == IDENT | CONST | LUT | OPAQUE | SAMPLE | HALF
    assert {"lut5", "dense", "coop", "half_nv12_rows", "ident_rgba_one_translucent"} <= set(SCENES)


# ------------------------------------------------------------------------------------------------
# running a scene and its oracle
# ------------------------------------------------------------------------------------------------
def device_input(arr_entry, iid, frame, pitch_mods, keep):
    """frame planes in device memory, plane p's pitch = (row bytes rounded up to 16) + pitch_mods[p]"""
    import torch
    b = iid.encode()
    keep.append(b)
    arr_entry.input_id, arr_entry.format = b, _FRAME_KIND[frame.data.kind]
    arr_entry.width, arr_entry.height, arr_entry.pts_ns = frame.resolution.width, frame.resolution.height, 0
    for pi, p in enumerate(plane_list(frame)):
        rows, rb = p.shape
        pitch = (rb + 15) // 16 * 16 + pitch_mods[pi]
        buf = torch.zeros(pitch * rows + 64, dtype=torch.uint8, device="cuda:0")
        buf[:pitch * rows].view(rows, pitch)[:, :rb] = torch.from_numpy(p).to("cuda:0")
        keep.append(buf)
        arr_entry.planes[pi], arr_entry.pitch[pi], arr_entry.mem_kind = buf.data_ptr(), pitch, F.MEM_DEVICE


def host_input(arr_entry, iid, frame, keep):
    b = iid.encode()
    keep.append(b)
    arr_entry.input_id, arr_entry.format = b, _FRAME_KIND[frame.data.kind]
    arr_entry.width, arr_entry.height, arr_entry.pts_ns = frame.resolution.width, frame.resolution.height, 0
    for pi, p in enumerate(plane_list(frame)):
        keep.append(p)
        arr_entry.planes[pi], arr_entry.pitch[pi], arr_entry.mem_kind = p.ctypes.data, 0, F.MEM_HOST


def plane_shapes(fmt, w, h):
    return {RGBA: [(h, w * 4)], YUV: [(h, w), (h // 2, w // 2), (h // 2, w // 2)], NV12: [(h, w), (h // 2, w)],
            YUV422: [(h, w), (h, w // 2), (h, w // 2)]}[fmt]


def oracle_out(layers, frames, ids, root, out_res, fmt, mode):
    from oracle import oracle as orc
    rgba = orc.render_layout_node(root[0], root[1], [to_oracle_layout(l) for l in layers], [node_texture(frames[i]) for i in ids],
                                  mode=int(mode))
    w, h = out_res
    if fmt == RGBA:
        return [rgba.reshape(h, w * 4)]
    if fmt == NV12:
        y, uv = orc.rgba_to_nv12_scaled(rgba, w, h)
        return [y, uv.reshape(h // 2, w)]
    cw, ch = w // 2, (h if fmt == YUV422 else h // 2)
    return list(orc.rgba_to_yuv_planar_scaled(rgba, w, h, cw, ch))


def run(outputs, frames, ids, mode, device_inputs=None, renderer=None):
    """one tick; outputs: [(output id, layers, root (w, h), out (w, h), format, out planes or None)] where out planes
    None means host planes.  -> (host numpy planes per output, renderer)"""
    import torch
    r = renderer or s.Renderer(s.RendererOptions(rendering_mode=mode))
    for i in ids:
        r.register_input(i)
    keep = []
    arr = (F.InputFrame * max(1, len(ids)))()
    for k, i in enumerate(ids):
        if device_inputs and i in device_inputs:
            device_input(arr[k], i, frames[i], device_inputs[i], keep)
        else:
            host_input(arr[k], i, frames[i], keep)
    outs = (F.OutputFrame * len(outputs))()
    host = []
    for k, (oid, layers, root, out_res, fmt, dev_planes) in enumerate(outputs):
        r.set_layouts(oid, s.Resolution(*out_res), fmt, root, ids, layers)
        b = oid.encode()
        keep.append(b)
        outs[k].output_id = b
        if dev_planes is None:
            planes = [np.zeros(sh, np.uint8) for sh in plane_shapes(fmt, *out_res)]
            outs[k].mem_kind = F.MEM_HOST
            for p, a in enumerate(planes):
                outs[k].planes[p] = a.ctypes.data
            host.append(planes)
        else:
            outs[k].mem_kind = F.MEM_DEVICE
            for p, (ptr, pitch) in enumerate(dev_planes):
                outs[k].planes[p], outs[k].pitch[p] = ptr, pitch
            host.append(None)
    torch.cuda.synchronize()
    r.render_raw(0, arr, len(ids), outs, len(outputs))
    torch.cuda.synchronize()
    return host, r


def first_mismatch(got, exp, layer_recs, fmt):
    """None when equal; else the plane, pixel, the 128 x 16 tile and the topmost layer whose box holds the pixel"""
    for p, (g, e) in enumerate(zip(got, exp)):
        if np.array_equal(g, e):
            continue
        n = int(np.count_nonzero(g != e))
        y, xb = (int(v) for v in np.argwhere(g != e)[0])
        x = xb // 4 if fmt == RGBA else xb
        if p > 0:   # chroma: the top-left luma pixel of its block
            x, y = (x // 2 if fmt == NV12 else x) * 2, y * (1 if fmt == YUV422 else 2)
        hit = [L for L in layer_recs if L["box"][0] <= x < L["box"][1] and L["box"][2] <= y < L["box"][3]]
        top = hit[-1] if hit else None
        who = "no layer" if top is None else f"layer {top['layer']} (fast {top['fast']:#x}, box {top['box']})"
        return (f"plane {p}: {n} bytes differ; first at byte ({xb}, {y}) = pixel ({x}, {y}), tile ({x // 128}, {y // 16}), "
                f"{who}: got {g[y, xb]} expected {e[y, xb]}")
    return None


FORMATS = [RGBA, YUV, NV12]
MANY = 100   # more layers than k_composite_p's parameter block holds


def padding(n):
    """n tiny translucent colour layers in the bottom-right corner (each covers pixels, so each is drawn)"""
    return [colour(W - 6.0 + (k % 5), H - 6.0 + (k // 5) % 5, 1.0, 1.0, (k % 256, 50, 9, 40)) for k in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["p", "multi_layers", "multi_outputs"])
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("mode", [GPU, CPU], ids=["gpu_mode", "cpu_mode"])
@pytest.mark.parametrize("name", [sc.name for sc in REGISTRY])
def test_fast_class(name, mode, fmt, kernel):
    sc = SCENES[name]
    if mode not in sc.modes:
        pytest.skip("the class is not reachable in this mode")
    for dx, dy in ((0, 0), (1, 1), (3, 0)) if kernel == "p" else ((2, 1),):
        layers, frames, ids = sc.build(dx, dy)
        probe = sc.probe
        if kernel == "multi_layers":
            layers = layers + padding(MANY)
        outputs = [(OUTPUT_ID, layers, (W, H), (W, H), fmt, None)]
        if kernel == "multi_outputs":
            outputs.append(("output_2", layers, (W, H), (W, H), RGBA if fmt != RGBA else NV12, None))
        got, r = run(outputs, frames, ids, mode, sc.device_inputs)
        recs = r.debug_composite_layers()
        what = f"{name} {mode} fmt={fmt} {kernel} offset=({dx},{dy})"
        expect_kernel = "p" if kernel == "p" else "multi"
        assert recs and all(L["kernel"] == expect_kernel for L in recs), (what, {L["kernel"] for L in recs})
        for k, (oid, ls, root, out_res, f, _) in enumerate(outputs):
            mine = [L for L in recs if L["job"] == k]
            L = mine[probe]
            assert L["fast"] & sc.fast == sc.fast and not L["fast"] & sc.not_fast, (what, L)
            assert sc.probe_check is None or sc.probe_check(L), (what, L)
            exp = oracle_out(ls, frames, ids, root, out_res, f, mode)
            rep = first_mismatch(got[k], exp, mine, f)
            assert rep is None, f"{what} output {oid}: {rep}"


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [GPU, CPU], ids=["gpu_mode", "cpu_mode"])
def test_output_422_through_k_output(mode):
    """root != output size: the composite writes an RGBA8 frame and k_output resamples it to 4:2:2"""
    layers, frames, ids = sc_coop(1, 1)
    got, r = run([(OUTPUT_ID, layers, (W, H), (200, 50), YUV422, None)], frames, ids, mode)
    recs = r.debug_composite_layers()
    assert recs and all(L["out_format"] == -1 for L in recs)
    rep = first_mismatch(got[0], oracle_out(layers, frames, ids, (W, H), (200, 50), YUV422, mode), recs, YUV422)
    assert rep is None, rep


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("mode", [GPU, CPU], ids=["gpu_mode", "cpu_mode"])
def test_values_from_outside_the_program(mode, fmt):
    """NaN / infinite / huge radii, border widths and mask fields, and positions near the 1e7 cut-off: the composite
    draws what the oracle draws (no interior is claimed where the fragment is not bare)."""
    ids, fr = [], {}
    ls = [background(ids, fr)]
    specs = [dict(radius=(-1e9, 0, 0, 0)), dict(radius=(-1e8, 0, 0, 0)), dict(radius=(NAN, 0, 0, 0)),
             dict(radius=(0, 0, float("-inf"), 0)), dict(border=NAN, border_color=(0, 250, 0, 255)),
             dict(border=0.999, border_color=(0, 250, 0, 255)), dict(border=1.0, border_color=(0, 250, 0, 255)),
             dict(masks=[((0, 0, 0, 0), 0.0, 0.0, NAN, 60.0)]), dict(masks=[((NAN, 0, 0, 0), 0.0, 0.0, 300.0, 60.0)]),
             dict(radius=(1e30, 0, 0, 0))]
    for k, kw in enumerate(specs):
        ls.append(colour(2.0 + 25 * k, 2.0 + (k % 3), 24.0, 50.0, (200, 20 * k, 60, 255 if k % 2 else 180), **kw))
    ls.append(colour(-1e7 + 3.0, 55.0, 1e7, 9.0, (20, 90, 200, 255), radius=(2, 2, 2, 2)))
    got, r = run([(OUTPUT_ID, ls, (W, H), (W, H), fmt, None)], fr, ids, mode)
    recs = r.debug_composite_layers()
    rep = first_mismatch(got[0], oracle_out(ls, fr, ids, (W, H), (W, H), fmt, mode), recs, fmt)
    assert rep is None, rep


# ------------------------------------------------------------------------------------------------
# caller-owned device output planes
# ------------------------------------------------------------------------------------------------
GUARD = 64
PLACEMENTS = [(0, 0), (1, 0), (2, 2), (4, 4), (8, 8), (0, 1), (0, 2), (4, 0), (8, 4), (1, 8)]   # (base, pitch mod 16)


def device_planes(fmt, w, h, base, pm):
    """-> (planes [(ptr, pitch)], buffers, [(rows, row bytes, pitch)]) with GUARD bytes of 0xA5 around each plane"""
    import torch
    planes, bufs, geo = [], [], []
    for rows, rb in plane_shapes(fmt, w, h):
        pitch = (rb + 15) // 16 * 16 + pm
        buf = torch.full((GUARD + base + pitch * rows + GUARD,), 0xA5, dtype=torch.uint8, device="cuda:0")
        planes.append((buf.data_ptr() + GUARD + base, pitch))
        bufs.append(buf)
        geo.append((rows, rb, pitch))
    return planes, bufs, geo


def read_back(bufs, geo, base):
    """the planes' bytes, and whether every byte outside them (guards, row padding) still holds 0xA5"""
    out, intact = [], True
    for buf, (rows, rb, pitch) in zip(bufs, geo):
        a = buf.cpu().numpy()
        body = a[GUARD + base:GUARD + base + pitch * rows].reshape(rows, pitch)
        out.append(body[:, :rb].copy())
        rest = np.concatenate([a[:GUARD + base], a[GUARD + base + pitch * rows:], body[:, rb:].reshape(-1)])
        intact = intact and bool(np.all(rest == 0xA5))
    return out, intact


def path_scene(path, fmt):
    """-> (layers, frames, ids, root, out size) for one writer of the output planes"""
    if path == "direct":   # a 4:1 child 1:1 in the frame: the fused resample kernel writes its direct tiles
        fr = {"a": make_frame("yuv", "extreme", 21, 1280, 720)}
        return [child(0, 0.0, 0.0, 320.0, 180.0, 1280, 720)], fr, ["a"], (320, 180), (320, 180)
    ids, fr = [], {}
    ls = [background(ids, fr), colour(5.0, 3.0, 200.0, 50.0, (20, 200, 90, 170), radius=(7, 7, 7, 7))]
    if path == "composite":
        return ls, fr, ids, (W, H), (W, H)
    if path == "k_output":
        return ls, fr, ids, (W, H), (W - 2, H + 2)
    return ls, fr, ids, (0, 0), (W, H)   # k_fill: an empty root


PATHS = ["composite", "k_output", "fill", "direct"]


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("fmt", [RGBA, YUV, NV12, YUV422])
def test_device_output_planes(fmt, path):
    if path == "direct" and fmt not in (YUV, NV12):
        pytest.skip("direct tiles write fused 4:2:0 / NV12 output only")
    if path == "composite" and fmt == YUV422:
        pytest.skip("4:2:2 output always goes through k_output")
    layers, frames, ids, root, out_res = path_scene(path, fmt)
    if path == "k_output" and fmt == RGBA:
        pytest.skip("RGBA output must match the root size")
    w, h = out_res
    ref, r0 = run([(OUTPUT_ID, layers, root, out_res, fmt, None)], frames, ids, s.RenderingMode.GpuOptimized)
    ref = ref[0]
    if path == "direct":
        assert r0.stats()["last_render_direct_tiles"] > 0
    if path != "fill":
        rep = first_mismatch(ref, oracle_out(layers, frames, ids, root, out_res, fmt, GPU), r0.debug_composite_layers(), fmt)
        assert rep is None, rep
    for base, pm in PLACEMENTS:
        planes, bufs, geo = device_planes(fmt, w, h, base, pm)
        r = s.Renderer()
        refused = fmt == RGBA and ((base | pm) & 3) != 0
        what = f"{path} fmt={fmt} base+{base} pitch%16={pm}"
        if refused:
            with pytest.raises(s.RenderSceneError) as e:
                run([(OUTPUT_ID, layers, root, out_res, fmt, planes)], frames, ids, GPU, renderer=r)
            assert e.value.status == 1, what   # SMR_ERR_INVALID_ARGUMENT
            assert "4-byte aligned" in r._err(), (what, r._err())
            assert r.stats()["kernel_launches"] == 0, what
            _, intact = read_back(bufs, geo, base)
            assert intact, what
            continue
        run([(OUTPUT_ID, layers, root, out_res, fmt, planes)], frames, ids, GPU, renderer=r)
        got, intact = read_back(bufs, geo, base)
        assert intact, f"{what}: bytes outside the planes were written"
        for p, (g, e) in enumerate(zip(got, ref)):
            assert np.array_equal(g, e), f"{what}: plane {p} differs from the host-output run"
        if path == "direct":
            assert r.stats()["last_render_direct_tiles"] == (r0.stats()["last_render_direct_tiles"] if (base | pm) % 2 == 0 else 0), what
