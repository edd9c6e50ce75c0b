"""Shared parity harness: run a scene through the product (C ABI -> sm_90a kernels) and through the
CPU oracle on the same inputs, return both outputs.  Test infrastructure (imports oracle/)."""
import numpy as np

import smelter_b200 as s
from oracle import oracle as orc
from tests import layout_ref as LR

OUTPUT_ID = "output_1"


def leaf_inputs(comp):
    """DFS order of InputStream leaves == node children order (scene/layout.rs:95-103)."""
    if isinstance(comp, s.InputStreamComponent):
        return [comp.input_id]
    if isinstance(comp, s.RescalerComponent):
        return leaf_inputs(comp.child) if comp.child is not None else []
    out = []
    for c in getattr(comp, "children", []):
        out += leaf_inputs(c)
    return out


def to_oracle_layout(l):
    masks = [(tuple(l.masks[i].radius), l.masks[i].top, l.masks[i].left, l.masks[i].width, l.masks[i].height)
             for i in range(l.masks_len)]
    return orc.make_layout(l.type, l.top, l.left, l.width, l.height, l.rotation_degrees, tuple(l.border_radius),
                           (l.color.r, l.color.g, l.color.b, l.color.a),
                           (l.border_color.r, l.border_color.g, l.border_color.b, l.border_color.a),
                           l.border_width, l.blur_radius, l.child_index,
                           (l.crop_top, l.crop_left, l.crop_width, l.crop_height), masks)


class TrackedRenderer(s.Renderer):
    """A Renderer whose scene updates are mirrored into the INDEPENDENT layout engine (tests/layout_ref.py), so that the
    oracle is fed layouts the product did not compute (and the product's own are checked against them)."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.ref_scenes = {}

    def update_scene(self, output_id, resolution, out_format, scene):
        super().update_scene(output_id, resolution, out_format, scene)
        st = self.ref_scenes.get(output_id)
        if st is None or (st.out_w, st.out_h) != (resolution.width, resolution.height):
            st = self.ref_scenes[output_id] = LR.StatefulScene(resolution.width, resolution.height)
        st.update_scene(scene)


def from_ref_layout(l):
    kind = {"child": orc.LAYOUT_TEXTURE, "color": orc.LAYOUT_COLOR, "shadow": orc.LAYOUT_BOX_SHADOW}[l.kind]
    masks = [(tuple(float(x) for x in m.radius.tup()), float(m.top), float(m.left), float(m.width), float(m.height)) for m in l.masks]
    crop = (0, 0, 0, 0) if l.crop is None else (float(l.crop.top), float(l.crop.left), float(l.crop.width), float(l.crop.height))
    return orc.make_layout(kind, float(l.top), float(l.left), float(l.width), float(l.height), float(l.rotation),
                           tuple(float(x) for x in l.border_radius.tup()), l.color, l.border_color, float(l.border_width),
                           float(l.blur_radius), max(l.index, 0), crop, masks)


def layouts_equal(prod, ref):
    """field-for-field, bit-for-bit as f32, of the product's flattened layouts and the independent ones"""
    import numpy as np
    if len(prod) != len(ref):
        return f"{len(prod)} layouts, independent engine has {len(ref)}"
    kinds = {0: "child", 1: "color", 2: "shadow"}
    eq = lambda a, b: np.float32(a) == np.float32(b) or (np.isnan(np.float32(a)) and np.isnan(np.float32(b)))
    for i, (p, r) in enumerate(zip(prod, ref)):
        if kinds[p.type] != r.kind:
            return f"layout {i}: kind {kinds[p.type]} vs {r.kind}"
        pairs = [(p.top, r.top), (p.left, r.left), (p.width, r.width), (p.height, r.height), (p.rotation_degrees, r.rotation)]
        pairs += list(zip(p.border_radius, r.border_radius.tup()))
        if r.kind == "shadow":
            pairs.append((p.blur_radius, r.blur_radius))
        else:
            pairs.append((p.border_width, r.border_width))
        if r.kind == "child":
            pairs += [(p.crop_top, r.crop.top), (p.crop_left, r.crop.left), (p.crop_width, r.crop.width), (p.crop_height, r.crop.height)]
            if p.child_index != r.index:
                return f"layout {i}: child index {p.child_index} vs {r.index}"
        if p.masks_len != len(r.masks):
            return f"layout {i}: {p.masks_len} masks vs {len(r.masks)}"
        for k in range(p.masks_len):
            m, q = p.masks[k], r.masks[k]
            pairs += list(zip(m.radius, q.radius.tup())) + [(m.top, q.top), (m.left, q.left), (m.width, q.width), (m.height, q.height)]
        if not all(eq(a, b) for a, b in pairs):
            return f"layout {i} ({r.kind}): {[(float(a), float(b)) for a, b in pairs if not eq(a, b)][:4]}"
    return None


def node_texture(frame: s.Frame):
    """K1/K2/K4 through the oracle."""
    d = frame.data
    w, h = frame.resolution.width, frame.resolution.height
    if d.kind == "PlanarYuv420":
        return orc.yuv420_to_rgba(*d.planes, w, h)
    if d.kind == "PlanarYuvJ420":
        return orc.yuv420_to_rgba(*d.planes, w, h, full_range=True)
    if d.kind == "PlanarYuv422":
        return orc.yuv_planar_to_rgba(*d.planes, w, h, w // 2, h)
    if d.kind == "PlanarYuv444":
        return orc.yuv_planar_to_rgba(*d.planes, w, h, w, h)
    if d.kind in ("InterleavedUyvy422", "InterleavedYuyv422"):
        return orc.interleaved422_to_rgba(d.planes[0], w, h, d.kind == "InterleavedYuyv422")
    if d.kind == "Nv12":
        return orc.nv12_to_rgba(d.planes[0], d.planes[1], w, h)
    if d.kind == "Bgra":
        return orc.bgra_to_rgba(d.planes[0], w, h)
    if d.kind == "Argb":
        return orc.argb_to_rgba(d.planes[0], w, h)
    if d.kind == "Rgba8":
        return np.ascontiguousarray(d.planes[0], np.uint8).reshape(h, w, 4)
    raise ValueError(d.kind)


def oracle_output(renderer, scene, frames, resolution, out_format, mode, pts, live_inputs=None):
    """Expected output planes from the oracle, fed with the layouts the product flattened."""
    live = frames if live_inputs is None else {k: v for k, v in frames.items() if k in live_inputs}
    if isinstance(scene, s.InputStreamComponent):
        fr = live.get(scene.input_id)
        if fr is None:
            return black(resolution, out_format)
        rgba = node_texture(fr)
    else:
        layouts, (rw, rh) = renderer.debug_layouts(OUTPUT_ID, pts)
        ref = getattr(renderer, "ref_scenes", {}).get(OUTPUT_ID)
        if ref is not None:   # layouts from the independent engine; the product's must be identical
            res = {k: (f.resolution.width, f.resolution.height) for k, f in live.items()}
            ref_layouts, ref_root = ref.layouts(pts, res)
            assert (rw, rh) == ref_root, f"root resolution {(rw, rh)} vs independent engine {ref_root}"
            d = layouts_equal(layouts, ref_layouts)
            assert d is None, f"product layouts differ from the independent engine: {d}"
        if rw == 0 or rh == 0:
            return black(resolution, out_format)
        nodes = [node_texture(live[i]) if i in live else None for i in leaf_inputs(scene)]
        layouts = [from_ref_layout(l) for l in ref_layouts] if ref is not None else [to_oracle_layout(l) for l in layouts]
        rgba = orc.render_layout_node(rw, rh, layouts, nodes, mode=mode, max_layouts=renderer.opts.max_layouts_count)
    W, H = resolution.width, resolution.height
    if out_format == s.OutputFrameFormat.RgbaWgpuTexture:
        assert rgba.shape[:2] == (H, W)
        return (rgba,)
    if out_format == s.OutputFrameFormat.Nv12WgpuTexture:
        return orc.rgba_to_nv12_scaled(rgba, W, H)
    cw, ch = chroma_size(out_format, W, H)
    return orc.rgba_to_yuv_planar_scaled(rgba, W, H, cw, ch)


def chroma_size(out_format, W, H):
    """texture/planar_yuv.rs:64-83"""
    if out_format == s.OutputFrameFormat.PlanarYuv422Bytes:
        return W // 2, H
    if out_format == s.OutputFrameFormat.PlanarYuv444Bytes:
        return W, H
    return W // 2, H // 2


def black(resolution, out_format):
    W, H = resolution.width, resolution.height
    y, u, v = orc.rgb_to_yuv_bytes(0, 0, 0)
    if out_format == s.OutputFrameFormat.RgbaWgpuTexture:
        return (np.zeros((H, W, 4), np.uint8),)
    if out_format == s.OutputFrameFormat.Nv12WgpuTexture:
        uv = np.empty((H // 2, W // 2, 2), np.uint8)
        uv[..., 0], uv[..., 1] = u, v
        return (np.full((H, W), y, np.uint8), uv)
    cw, ch = chroma_size(out_format, W, H)
    return (np.full((H, W), y, np.uint8), np.full((ch, cw), u, np.uint8), np.full((ch, cw), v, np.uint8))


def product_planes(frame: s.Frame):
    return tuple(np.asarray(p) for p in frame.data.planes)


def run_case(scene, frames, resolution=s.Resolution(640, 360), out_format=s.OutputFrameFormat.PlanarYuv420Bytes,
             mode=s.RenderingMode.GpuOptimized, pts=0.0, renderer=None, updates=None, max_layouts=100):
    """frames: {input_id: Frame}.  Returns (product planes, oracle planes, renderer)."""
    r = renderer or TrackedRenderer(s.RendererOptions(rendering_mode=mode, max_layouts_count=max_layouts))
    if renderer is None:
        for iid in frames:
            r.register_input(iid)
        r.update_scene(OUTPUT_ID, resolution, out_format, scene)
    fs = s.FrameSet(frames=dict(frames), pts=pts)
    out = r.render(fs)
    got = product_planes(out.frames[OUTPUT_ID])
    timeout = r.opts.stream_fallback_timeout
    live = {k for k, f in frames.items() if not (max(pts - timeout, 0.0) > f.pts)}
    exp = oracle_output(r, scene, frames, resolution, out_format, mode, pts, live_inputs=live)
    return got, exp, r


def assert_identical(got, exp, what=""):
    assert len(got) == len(exp)
    for i, (g, e) in enumerate(zip(got, exp)):
        g = np.asarray(g).reshape(np.asarray(e).shape)
        if not np.array_equal(g, e):
            d = np.abs(g.astype(int) - np.asarray(e).astype(int))
            idx = np.unravel_index(np.argmax(d), d.shape)
            raise AssertionError(f"{what} plane {i}: {np.count_nonzero(d)} / {d.size} bytes differ, max |d|={d.max()} "
                                 f"at {idx}: got {g[idx]} expected {np.asarray(e)[idx]}")


def yuv_frame(planes, w, h, pts=0.0):
    y, u, v = planes
    return s.Frame(s.FrameData.PlanarYuv420(s.YuvPlanes(y, u, v)), s.Resolution(w, h), pts)


def nv12_frame(planes, w, h, pts=0.0):
    y, u, v = planes
    uv = np.stack([u, v], axis=-1)
    return s.Frame(s.FrameData.Nv12(s.NvPlanes(y, uv)), s.Resolution(w, h), pts)


def wide_chroma_frame(kind, seed, w, h, pts=0.0):
    """seeded frame in one of the non-4:2:0 input formats (FrameData::{PlanarYuv422, PlanarYuv444,
    InterleavedUyvy422, InterleavedYuyv422}); smooth luma ramp + noise so that scaling has something to filter"""
    rng = np.random.default_rng(seed)
    xx, yy = np.meshgrid(np.arange(w), np.arange(h))
    y = (16 + ((xx * 3 + yy * 5 + seed * 7) % 200) * 0.9 + rng.integers(0, 20, (h, w))).astype(np.uint8)
    cw = w if kind == "PlanarYuv444" else w // 2
    u = rng.integers(16, 241, (h, cw), dtype=np.uint8)
    v = rng.integers(16, 241, (h, cw), dtype=np.uint8)
    if kind == "PlanarYuv422":
        d = s.FrameData.PlanarYuv422(s.YuvPlanes(y, u, v))
    elif kind == "PlanarYuv444":
        d = s.FrameData.PlanarYuv444(s.YuvPlanes(y, u, v))
    else:
        t = np.empty((h, w // 2, 4), np.uint8)
        if kind == "InterleavedUyvy422":
            t[..., 0], t[..., 1], t[..., 2], t[..., 3] = u, y[:, 0::2], v, y[:, 1::2]
            d = s.FrameData.InterleavedUyvy422(t)
        else:
            t[..., 0], t[..., 1], t[..., 2], t[..., 3] = y[:, 0::2], u, y[:, 1::2], v
            d = s.FrameData.InterleavedYuyv422(t)
    return s.Frame(d, s.Resolution(w, h), pts)
