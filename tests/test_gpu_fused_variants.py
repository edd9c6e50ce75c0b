"""Every compiled instantiation of the fused resample (K1/K2 + both Lanczos passes in one kernel) against the oracle.

`Renderer::try_fused_resample` picks one of three kernels for each resampled YUV child -- `k_resample_tma3<S, SRC>`
(integer ratio 2 / 4, TMA-staged), `k_resample_tma0<SRC, WINDOW, BOX>` (any ratio <= 4, TMA-staged, optionally box-reduced
2:1 on the fly) and `k_resample_fused_int<S, SRC>` (LDG-staged) -- from the ratio, crop offset, tap window, box level,
source format, destination width parity and plane alignment.  Each case here builds its scene with `set_layouts`, whose
crop rectangle sets each axis's scale and offset directly, asks `debug_fused_jobs` which variant ran, and compares the
RGBA output byte for byte with the oracle fed the same layouts.  The children are opaque and sit at integer positions, so
the output bytes are the fused kernel's bytes.

- `REGISTRY`: one scene per reachable (kernel, ratio or window, box, source class) instantiation, for k_resample_tma3
  also per source range and per vertical path (`v_same`).  `test_registry_covers_every_compiled_variant` reads the set of
  instantiations from the library (`smr_debug_fused_variants`) and fails when one has no scene.
- Geometry edges of each kernel family on planar and NV12 sources: the last strip, tiny and odd sizes, sources smaller
  than one TMA box, tiles that end at the image edge, crop offsets, two crops of one input.
- Content that hits every byte code in each plane, with runs of alternating 0 / 255 across strip and tile boundaries.
- Device planes at several base and pitch alignments: TMA and LDG kernels on the same frame give the same bytes, and
  planes the kernels cannot read are refused before anything is launched.
- Direct tiles (the fused kernel writing output YUV itself) in a launch whose partition cuts the second job at odd rows.
"""
import ctypes as C
from dataclasses import dataclass, field
from typing import Optional, Tuple

import numpy as np
import pytest

import smelter_b200 as s
from smelter_b200 import _ffi as F
from smelter_b200.renderer import _FRAME_KIND
from tests import harness
from tests.parity import OUTPUT_ID, node_texture, to_oracle_layout

YUV = s.OutputFrameFormat.PlanarYuv420Bytes
NV12 = s.OutputFrameFormat.Nv12WgpuTexture
RGBA = s.OutputFrameFormat.RgbaWgpuTexture
FRAME_KIND = {"yuv": "PlanarYuv420", "yuvj": "PlanarYuvJ420", "nv12": "Nv12", "uyvy": "InterleavedUyvy422",
              "yuyv": "InterleavedYuyv422"}
SRC_CLASS = {"yuv": 0, "yuvj": 0, "nv12": 1, "uyvy": 2, "yuyv": 3}
# source columns where strips or TMA tiles of some variant begin: 4:1 strips (58 columns), 2:1 strips (122 columns),
# 64-column strips, 272-pixel luma tiles on 16-pixel steps
BOUNDARY_PERIODS = (232, 244, 128, 256)


# ------------------------------------------------------------------------------------------------
# content
# ------------------------------------------------------------------------------------------------
def extreme_plane(rng, w, h, scale=1):
    """Random bytes; runs of alternating 0 / 255 (a checkerboard, the largest Lanczos overshoot on both axes) 16 pixels
    wide across every strip / tile boundary column and across every 32-row TMA chunk boundary; then all 256 codes at
    random positions.  `scale` = 2 for a 4:2:0 chroma plane (boundaries at half the luma coordinates)."""
    p = rng.integers(0, 256, (h, w), dtype=np.uint8)
    xs, ys = np.arange(w), np.arange(h)
    cols = np.zeros(w, bool)
    for per in BOUNDARY_PERIODS:
        per //= scale
        cols |= np.abs(((xs + per // 2) % per) - per // 2) < 8 // scale + 1
    rows = np.abs(((ys + 16 // scale) % (32 // scale)) - 16 // scale) < 4
    checker = ((xs[None, :] + ys[:, None]) & 1).astype(np.uint8) * 255
    band = cols[None, :] | rows[:, None]
    p[band] = checker[band]
    n = min(w * h, 256)   # a plane of fewer than 256 bytes gets a random subset of the codes
    p.reshape(-1)[rng.permutation(w * h)[:n]] = rng.permutation(256)[:n].astype(np.uint8) if n < 256 else np.arange(256)
    return p


def planes_of(content, seed, w, h, cw, ch):
    """(y, u, v): luma w x h, chroma cw x ch (cw = w / 2; ch = h / 2 or h).  content: "extreme" or "smooth"."""
    if content == "extreme":
        rng = np.random.default_rng(seed)
        sc = 2 if ch < h else 1
        return extreme_plane(rng, w, h), extreme_plane(rng, cw, ch, sc), extreme_plane(rng, cw, ch, sc)
    if ch < h:
        return harness.smooth_yuv420(seed, w, h)
    y, u, v = harness.smooth_yuv420(seed, w, 2 * h)   # chroma of a 2h-row 4:2:0 frame: h x w / 2
    return y[:h], u, v


def make_frame(fmt, content, seed, w, h):
    il = fmt in ("uyvy", "yuyv")
    y, u, v = planes_of(content, seed, w, h, w // 2, h if il else h // 2)
    res = s.Resolution(w, h)
    if fmt == "nv12":
        return s.Frame(s.FrameData.Nv12(s.NvPlanes(y, np.stack([u, v], axis=-1))), res)
    if fmt in ("yuv", "yuvj"):
        return s.Frame(s.FrameData(FRAME_KIND[fmt], (y, u, v)), res)
    t = np.empty((h, w // 2, 4), np.uint8)
    if fmt == "uyvy":
        t[..., 0], t[..., 1], t[..., 2], t[..., 3] = u, y[:, 0::2], v, y[:, 1::2]
    else:
        t[..., 0], t[..., 1], t[..., 2], t[..., 3] = y[:, 0::2], u, y[:, 1::2], v
    return s.Frame(s.FrameData(FRAME_KIND[fmt], (t,)), res)


def test_extreme_content_hits_every_code():
    rng = np.random.default_rng(1)
    for w, h, sc in ((1280, 720, 1), (640, 360, 2), (48, 12, 2)):
        p = extreme_plane(rng, w, h, sc)
        assert len(np.unique(p)) == 256, (w, h)
        assert np.count_nonzero(p == 0) > 20 and np.count_nonzero(p == 255) > 20


# ------------------------------------------------------------------------------------------------
# scenes: children side by side on one root, each at an integer position, opaque, no rounding
# ------------------------------------------------------------------------------------------------
@dataclass
class Job:
    input_id: str
    crop: Tuple[float, float, float, float]   # left, top, width, height in source pixels
    dst: Tuple[int, int]


def scene_of(jobs, gap=2):
    """-> (W, H, child ids, [RenderLayout], x offset of each job).  An even gap keeps every child on even columns."""
    ids = []
    for j in jobs:
        if j.input_id not in ids:
            ids.append(j.input_id)
    xs, x = [], 0
    for j in jobs:
        xs.append(x)
        x += j.dst[0] + gap
    W, H = max(x - gap, 2), max(max(j.dst[1] for j in jobs), 1)
    ls = []
    for j, x0 in zip(jobs, xs):
        l = F.RenderLayout()
        l.type, l.left, l.top, l.width, l.height = 0, float(x0), 0.0, float(j.dst[0]), float(j.dst[1])
        l.child_index = ids.index(j.input_id)
        l.crop_left, l.crop_top, l.crop_width, l.crop_height = (float(c) for c in j.crop)
        ls.append(l)
    return W, H, ids, ls, xs


def oracle_planes(jobs, frames, out_format, mode=s.RenderingMode.GpuOptimized):
    from oracle import oracle as orc
    W, H, ids, ls, _ = scene_of(jobs)
    rgba = orc.render_layout_node(W, H, [to_oracle_layout(l) for l in ls], [node_texture(frames[i]) for i in ids], mode=mode)
    if out_format == RGBA:
        return (rgba,)
    if out_format == NV12:
        return orc.rgba_to_nv12_scaled(rgba, W, H)
    return orc.rgba_to_yuv_planar_scaled(rgba, W, H, W // 2, H // 2)


# ------------------------------------------------------------------------------------------------
# running a scene: host frames (tightly packed uploads) or device planes at a chosen base offset and pitch
# ------------------------------------------------------------------------------------------------
@dataclass
class Placement:
    base: int = 0          # byte offset of every plane from a 512-byte aligned allocation
    pitch_mod: int = 0     # pitch = (row bytes rounded up to 16) + pitch_mod
    chroma_base: Optional[int] = None   # NV12 / planar chroma planes' own offset (default: `base`)


def plane_list(frame):
    d = frame.data
    if d.kind == "Nv12":
        return [np.ascontiguousarray(d.planes[0]), np.ascontiguousarray(d.planes[1]).reshape(d.planes[1].shape[0], -1)]
    if d.kind.startswith("Interleaved"):
        t = np.ascontiguousarray(d.planes[0])
        return [t.reshape(t.shape[0], -1)]
    return [np.ascontiguousarray(p) for p in d.planes]


def fill_input(arr_entry, iid, frame, placement, keep):
    import torch
    b = iid.encode()
    keep.append(b)
    a = arr_entry
    a.input_id, a.format = b, _FRAME_KIND[frame.data.kind]
    a.width, a.height, a.pts_ns = frame.resolution.width, frame.resolution.height, 0
    for pi, p in enumerate(plane_list(frame)):
        if placement is None:
            keep.append(p)
            a.planes[pi], a.pitch[pi], a.mem_kind = p.ctypes.data, 0, F.MEM_HOST
            continue
        rows, rb = p.shape
        pitch = (rb + 15) // 16 * 16 + placement.pitch_mod
        base = placement.base if pi == 0 or placement.chroma_base is None else placement.chroma_base
        buf = torch.zeros(base + pitch * rows + 64, dtype=torch.uint8, device="cuda:0")
        buf[base:base + pitch * rows].view(rows, pitch)[:, :rb] = torch.from_numpy(p).to("cuda:0")
        keep.append(buf)
        a.planes[pi], a.pitch[pi], a.mem_kind = buf.data_ptr() + base, pitch, F.MEM_DEVICE


def render(r, jobs, frames, out_format=RGBA, placements=None):
    """one tick of the scene on renderer r (inputs registered here): -> output planes (host numpy)"""
    import torch
    W, H, ids, ls, _ = scene_of(jobs)
    for i in ids:
        r.register_input(i)
    r.set_layouts(OUTPUT_ID, s.Resolution(W, H), out_format, (W, H), ids, ls)
    keep = []
    arr = (F.InputFrame * len(ids))()
    for k, i in enumerate(ids):
        fill_input(arr[k], i, frames[i], (placements or {}).get(i), keep)
    sizes = (C.c_size_t * 3)()
    assert F.lib().smr_output_plane_sizes(W, H, out_format, C.byref(sizes)) == 0
    outs = [np.zeros(sizes[p], np.uint8) if sizes[p] else None for p in range(3)]
    out = (F.OutputFrame * 1)()
    ob = OUTPUT_ID.encode()
    out[0].output_id, out[0].mem_kind = ob, F.MEM_HOST
    for p in range(3):
        if outs[p] is not None:
            out[0].planes[p] = outs[p].ctypes.data
    torch.cuda.synchronize()
    r.render_raw(0, arr, len(ids), out, 1)
    if out_format == RGBA:
        return (outs[0].reshape(H, W, 4),)
    if out_format == NV12:
        return (outs[0].reshape(H, W), outs[1].reshape(H // 2, W // 2, 2))
    return (outs[0].reshape(H, W), outs[1].reshape(H // 2, W // 2), outs[2].reshape(H // 2, W // 2))


def mismatch_report(got, exp, jobs, fused):
    """None when equal; else where the first differing byte is: the job, and for RGBA its column, strip, row and 8-row group"""
    _, _, _, _, xs = scene_of(jobs)
    for pi, (g, e) in enumerate(zip(got, exp)):
        g = np.asarray(g).reshape(np.asarray(e).shape)
        if np.array_equal(g, e):
            continue
        n = int(np.count_nonzero(g != e))
        idx = np.argwhere(g != e)[0]
        if len(got) > 1:
            return f"plane {pi}: {n} bytes differ, first at {tuple(idx)}: got {g[tuple(idx)]} expected {e[tuple(idx)]}"
        y, x = int(idx[0]), int(idx[1])
        k = max(i for i, x0 in enumerate(xs) if x0 <= x)
        col = x - xs[k]
        info = fused[k] if k < len(fused) else {}
        sc = info.get("strip_cols") or 64
        return (f"{n} bytes differ; first at job {k} ({info.get('kernel')}, {jobs[k]}), column {col}, strip {col // sc}, row {y}, "
                f"8-row group {y // 8}: got {g[y, x]} expected {e[y, x]}")
    return None


def check(jobs, frames, out_format=RGBA, placements=None, expect=None, renderer=None, what=""):
    """render + oracle + hook; expect: per job a dict of fields the job's hook record must have (None: no check)"""
    r = renderer or s.Renderer()
    got = render(r, jobs, frames, out_format, placements)
    fused = r.debug_fused_jobs()
    if expect is not None:
        assert len(fused) == len(expect), (what, fused)
        for k, (e, f) in enumerate(zip(expect, fused)):
            if e is None:
                continue
            diff = {key: (f[key], v) for key, v in e.items() if f[key] != v}
            assert not diff, f"{what}: job {k} ran {f}, expected {e} (got, expected) {diff}"
    rep = mismatch_report(got, oracle_planes(jobs, frames, out_format), jobs, fused)
    assert rep is None, f"{what}: {rep}"
    return got, fused, r


# ------------------------------------------------------------------------------------------------
# the registry: one scene per reachable instantiation
# ------------------------------------------------------------------------------------------------
@dataclass
class Entry:
    name: str
    kernel: str              # "tma_int", "tma_any", "ldg"
    ratio: int               # template ratio (0: any)
    window: int              # k_resample_tma0 window slots, else 0
    box: int
    fmt: str                 # frame format key (FRAME_KIND)
    src: Tuple[int, int]
    crop: Tuple[float, float, float, float]
    dst: Tuple[int, int]
    v_same: Optional[int] = None

    @property
    def src_class(self):
        return SRC_CLASS[self.fmt]

    @property
    def full_range(self):
        return 1 if self.fmt == "yuvj" else 0

    def expect(self):
        e = {"kernel": self.kernel, "ratio": self.ratio, "window": self.window, "box": self.box, "src_class": self.src_class,
             "full_range": self.full_range}
        if self.v_same is not None:
            e["v_same"] = self.v_same
        return e


def full(w, h):
    return (0.0, 0.0, float(w), float(h))


def _registry():
    R = []
    # k_resample_tma3: 4:1 from 1280 x 720, 2:1 from 640 x 360; v_same = 0: the same ratio vertically with a fractional
    # offset, which fills the ring exactly (4:1: 28 + 25 + 1 == kTmaRing4, 2:1: 14 + 13 + 1 == kTmaRing2)
    for S in (4, 2):
        w, h = 640 * S // 2, 360 * S // 2
        for fmt in ("yuv", "yuvj", "nv12"):
            R.append(Entry(f"tma3-{S}-{fmt}-vsame", "tma_int", S, 0, 0, fmt, (w, h), full(w, h), (w // S, h // S), 1))
            R.append(Entry(f"tma3-{S}-{fmt}-voff", "tma_int", S, 0, 0, fmt, (w, h), (0.0, 0.37, float(w), float(S * 179)),
                           (w // S, 179), 0))
    # k_resample_tma0 without box: (window, scale, source, destination); widths multiples of 32 keep every plane's rows
    # 16-byte aligned when uploaded tightly packed
    tma0 = [(20, "1.5", (480, 270), full(480, 270), (320, 180)),
            (20, "0.5", (160, 90), full(160, 90), (320, 180)),
            (20, "2+0.5", (640, 360), (0.5, 0.5, 636.0, 356.0), (318, 178)),
            (25, "3", (960, 540), full(960, 540), (320, 180)),
            (29, "3.25", (832, 572), full(832, 572), (256, 176)),
            (33, "3.75", (960, 660), full(960, 660), (256, 176)),
            (33, "3.9", (1248, 702), full(1248, 702), (320, 180))]   # vertically ceil(7 * 3.9) + 25 + 1 == 54: ring full
    tma0_box = [(20, "4.2", (672, 378), full(672, 378), (160, 90)),
                (25, "6", (960, 540), full(960, 540), (160, 90)),
                (29, "6.5", (832, 572), full(832, 572), (128, 88)),
                (33, "8", (1280, 720), full(1280, 720), (160, 90)),
                (33, "7.5", (960, 660), full(960, 660), (128, 88))]
    for box, rows in ((0, tma0), (1, tma0_box)):
        for win, sc, src, crop, dst in rows:
            for fmt in ("yuv", "nv12"):
                R.append(Entry(f"tma0-w{win}-box{box}-{sc}-{fmt}", "tma_any", 0, win, box, fmt, src, crop, dst))
    # k_resample_fused_int on planar / NV12: widths whose tightly packed rows are not 16-byte aligned (planar chroma:
    # not a multiple of 32; NV12: not of 16) keep the TMA kernels out
    ldg = {("yuv", 2): (656, 368), ("nv12", 2): (648, 360), ("yuv", 3): (1008, 540), ("nv12", 3): (1002, 540),
           ("yuv", 4): (1296, 720), ("nv12", 4): (1288, 720)}
    for (fmt, S), (w, h) in ldg.items():
        R.append(Entry(f"ldg-{S}-{fmt}", "ldg", S, 0, 0, fmt, (w, h), full(w, h), (w // S, h // S)))
    for fmt in ("yuv", "nv12"):
        # any ratio: an odd destination width (no TMA kernel), and 4:1 with a crop offset (window 34 > 33)
        R.append(Entry(f"ldg-0-odd-{fmt}", "ldg", 0, 0, 0, fmt, (640, 360), full(640, 360), (321, 181)))
        R.append(Entry(f"ldg-0-4off-{fmt}", "ldg", 0, 0, 0, fmt, (1280, 720), (0.5, 0.0, 1272.0, 720.0), (318, 180)))
    for fmt in ("uyvy", "yuyv"):
        for S, sc, (w, h) in ((2, "2", (640, 360)), (3, "3", (960, 540)), (4, "4", (1280, 720)), (0, "1.5", (480, 270))):
            R.append(Entry(f"ldg-{S}-{fmt}", "ldg", S, 0, 0, fmt, (w, h), full(w, h), (int(w / float(sc)), int(h / float(sc)))))
    return R


REGISTRY = _registry()


FUSED_KERNEL = {F.FUSED_LDG: "ldg", F.FUSED_TMA_INT: "tma_int", F.FUSED_TMA_ANY: "tma_any"}


def fused_variants():
    """(kernel, ratio, window, box, src_class, matrix, launch range) of every fused kernel instantiation the library
    compiles (smr_debug_fused_variants, no device needed), one per launch key; matrix 1 is BT.601"""
    L, n = F.lib(), C.c_uint32()
    assert L.smr_debug_fused_variants(None, 0, C.byref(n)) == 0
    arr = (F.FusedVariantInfo * n.value)()
    assert L.smr_debug_fused_variants(arr, n.value, C.byref(n)) == 0 and n.value == len(arr)
    return [(FUSED_KERNEL[v.kernel], v.ratio, v.window, v.box, v.src_class, int(v.matrix == F.MATRIX_BT601), v.range)
            for v in arr]


def launchable_instantiations():
    """The (kernel, ratio, window, box, src_class) template instantiations the library compiles"""
    return {v[:5] for v in fused_variants()}


def test_registry_covers_every_compiled_variant():
    """36 kernels: k_resample_tma3 <2|4, planar|NV12>, k_resample_tma0 <planar|NV12, 20|25|29|33, box 0|1>,
    k_resample_fused_int <2|3|4|0, planar|NV12|UYVY|YUYV>; k_resample_tma3 also on both source ranges (NV12 is limited
    only) and both vertical paths.  The library compiles 96 distinct instantiations in all."""
    variants = fused_variants()
    assert len(variants) == len(set(variants)) == 96, sorted(variants)
    inst = launchable_instantiations()
    assert len(inst) == 36, sorted(inst)
    have = {(e.kernel, e.ratio, e.window, e.box, e.src_class) for e in REGISTRY}
    assert inst <= have, f"instantiations without a registry scene: {sorted(inst - have)}"
    assert have <= inst, f"registry scenes for kernels that are not compiled: {sorted(have - inst)}"
    tma3 = {(e.ratio, e.src_class, e.full_range, e.v_same) for e in REGISTRY if e.kernel == "tma_int"}
    assert tma3 == {(S, sc, fr, vs) for S in (2, 4) for sc, fr in ((0, 0), (0, 1), (1, 0)) for vs in (0, 1)}
    assert len({e.name for e in REGISTRY}) == len(REGISTRY)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", REGISTRY, ids=lambda e: e.name)
def test_registry_variant(entry):
    """the scene selects its variant, and the RGBA bytes equal the oracle's for extreme and for smooth content"""
    r = s.Renderer()
    for k, content in enumerate(("extreme", "smooth")):
        fr = {"input_1": make_frame(entry.fmt, content, 17 + k, *entry.src)}
        check([Job("input_1", entry.crop, entry.dst)], fr, expect=[entry.expect()], renderer=r, what=f"{entry.name} {content}")


# ------------------------------------------------------------------------------------------------
# geometry edges of each family, planar and NV12
# ------------------------------------------------------------------------------------------------
ALIGNED = Placement(0, 0)      # device planes with 16-byte aligned rows: the TMA kernels can take them
MISALIGNED = Placement(8, 8)   # 8 bytes off: no tensor map, the LDG kernel


def first_tap(scale, offset, o):
    """first source pixel of output coordinate o (k_weights, in f32)"""
    f = np.float32
    c = f(offset) + (f(o) + f(0.5)) * f(scale)
    d = c - f(0.5)
    return int(np.ceil(d - f(3.0) * f(max(scale, 1.0))))


def family_job(family, dw, dh, crop_left=0.0, crop_top=0.0, src_w=None):
    """(source size, crop, destination, placement, expected kernel) of a `family` job with destination dw x dh:
    tma3 at 4:1, tma0 at 2:1 with a 0.5 horizontal offset, ldg at 4:1 on 8-byte offset device planes"""
    pad_x, pad_y = 2 * int(np.ceil(crop_left)), 2 * int(np.ceil(crop_top))   # the crop stays inside the source
    if family == "tma0":
        cw, ch = 2.0 * dw, 2.0 * dh
        w, h = src_w or int(cw) + 2 + pad_x, int(ch) + 2 + pad_y
        return (w, h), (0.5 + crop_left, crop_top, cw, ch), (dw, dh), ALIGNED, "tma_any"
    cw, ch = 4.0 * dw, 4.0 * dh
    w, h = src_w or int(cw) + pad_x, int(ch) + pad_y
    return (w, h), (crop_left, crop_top, cw, ch), (dw, dh), ALIGNED if family == "tma3" else MISALIGNED, \
        "tma_int" if family == "tma3" else "ldg"


def run_family(family, fmt, geoms, what, content="extreme", expect_kernel=True):
    """one tick with one job per geometry (dw, dh[, crop_left, crop_top]) of `family` on `fmt` frames"""
    jobs, frames, places, expect = [], {}, {}, []
    for k, g in enumerate(geoms):
        src, crop, dst, pl, kern = family_job(family, *g)
        iid = f"input_{k}"
        frames[iid] = make_frame(fmt, content, 300 + k, *src)
        places[iid] = pl
        jobs.append(Job(iid, crop, dst))
        expect.append({"kernel": kern} if expect_kernel else None)
    return check(jobs, frames, placements=places, expect=expect, what=f"{family} {fmt} {what}")


FAMILIES = ["tma3", "tma0", "ldg"]
FMTS = ["yuv", "nv12"]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("family", FAMILIES)
def test_destination_widths(family, fmt):
    """a last strip of 2 columns, a destination 2 columns wide, fewer than 32 column pairs"""
    last2 = {"tma3": 58 * 3 + 2, "tma0": None, "ldg": 64 * 2 + 2}[family]
    if last2 is None:   # tma0 at 2:1: the job's own strip width
        _, fused, _ = run_family(family, fmt, [(200, 24)], "probe strip width")
        last2 = fused[0]["strip_cols"] + 2
    _, fused, _ = run_family(family, fmt, [(last2, 40), (2, 24), (40, 30)], "widths")
    assert fused[0]["dst"][0] % fused[0]["strip_cols"] == 2, fused[0]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("family", FAMILIES)
def test_destination_heights(family, fmt):
    """1, 2, 3, 7, 9 output rows, in one launch (the partition cuts the 9-row job's strip between blocks)"""
    run_family(family, fmt, [(120, h) for h in (1, 2, 3, 7, 9)], "heights")


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("family", FAMILIES)
def test_partition_cuts_a_strip(family, fmt):
    """one strip, 250 rows: every partition over more than one block cuts it mid-job; a second job in the same launch"""
    run_family(family, fmt, [(40, 250), (250, 77)], "cut strips")


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("family", FAMILIES)
def test_source_smaller_than_a_tma_box(family, fmt):
    """4:1 from 96 x 24 (tma0: 2:1 from 50 x 26): narrower than a 272-pixel luma box and shorter than a 32-row chunk, a
    25-tap window clamped at both ends; at 4:1 with v_same the vertical fast path falls back to one_row"""
    run_family(family, fmt, [(24, 6), (12, 4)], "tiny source")


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("family", ["tma3", "tma0"])
def test_tile_ends_at_the_right_edge(family, fmt):
    """source widths where the last strip's 272-pixel luma tile ends exactly at, 2 pixels before, or 2 pixels beyond the
    right image edge (the crop is narrower than the source, so the source width is free)"""
    geoms = []
    for slack in (0, -2, 2):
        if family == "tma3":
            dw, strip = 58 * 2 + 40, 58 * 2
            x0 = first_tap(4.0, 0.0, strip)
        else:
            dw, strip = 150, 64 * 2
            x0 = first_tap(2.0, 0.5, strip) & ~1
        xt = x0 & ~15
        W = xt + 272 + slack
        crop_w = (4 if family == "tma3" else 2) * dw
        assert W >= crop_w + 2 and W % 2 == 0, (W, crop_w)
        geoms.append((dw, 40, 0.0, 0.0, W))
    _, fused, _ = run_family(family, fmt, geoms, "tile at the edge")
    if family == "tma0":
        assert fused[0]["strip_cols"] == 64, fused[0]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("family", FAMILIES)
def test_crop_offsets(family, fmt):
    """left only, top only and both, integral (8.0) and fractional (0.37); an offset may move the job to another kernel
    (a horizontal offset at 4:1 widens the window past 33 slots), so only the bytes are checked"""
    geoms = [(100, 40, l, t) for l, t in ((8.0, 0.0), (0.0, 8.0), (8.0, 8.0), (0.37, 0.0), (0.0, 0.37), (0.37, 0.37))]
    run_family(family, fmt, geoms, "crop offsets", expect_kernel=False)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FMTS)
def test_two_crops_of_one_input(fmt):
    """two different crops of one input next to a full showing, all 4:1 without a horizontal offset: three jobs of one
    k_resample_tma3 launch, the cropped two on its second vertical path (integral vertical offsets)"""
    w, h = 1280, 720
    fr = {"input_1": make_frame(fmt, "extreme", 41, w, h)}
    jobs = [Job("input_1", full(w, h), (320, 180)), Job("input_1", (0.0, 128.0, 512.0, 288.0), (128, 72)),
            Job("input_1", (0.0, 360.0, 640.0, 360.0), (160, 90))]
    r = s.Renderer()
    r.set_profiling(True)
    check(jobs, fr, placements={"input_1": ALIGNED}, renderer=r, what="two crops",
          expect=[{"kernel": "tma_int", "v_same": v} for v in (1, 0, 0)])
    assert r.kernel_times()["resample_fused"][1] == 1, r.kernel_times()


# ------------------------------------------------------------------------------------------------
# the byte range: both ranges in one launch, and the non-fused readers of the same frames
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["tma_any", "ldg"])
def test_mixed_range_launch(kernel):
    """k_resample_tma0 and k_resample_fused_int read the range per job: limited and full-range planar jobs share a launch"""
    w, h, dst = (480, 270, (320, 180)) if kernel == "tma_any" else (1296, 720, (324, 180))
    fr = {"input_1": make_frame("yuv", "extreme", 51, w, h), "input_2": make_frame("yuvj", "extreme", 52, w, h),
          "input_3": make_frame("yuv", "smooth", 53, w, h)}
    jobs = [Job(i, full(w, h), dst) for i in fr]
    r = s.Renderer()
    r.set_profiling(True)
    _, fused, _ = check(jobs, fr, renderer=r, expect=[{"kernel": kernel, "full_range": f} for f in (0, 1, 0)], what="ranges")
    assert r.kernel_times()["resample_fused"][1] == 1, r.kernel_times()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["yuv", "yuvj", "nv12"])
def test_extreme_bytes_outside_the_fused_kernels(fmt):
    """the same content through the other K1 / K2 readers: a pass-through child (the composite's yuv_quad), CpuOptimized
    at exactly half size (FAST_HALF), and the generic resample passes after k_convert (5:1 by 2:1 has no fused kernel)"""
    w, h = 640, 360
    fr = {"input_1": make_frame(fmt, "extreme", 61, w, h)}
    check([Job("input_1", full(w, h), (w, h))], fr, expect=[], what="pass-through")
    check([Job("input_1", full(w, h), (w, h))], fr, out_format=NV12, expect=[], what="pass-through NV12")
    r = s.Renderer(s.RendererOptions(rendering_mode=s.RenderingMode.CpuOptimized))
    got = render(r, [Job("input_1", full(w, h), (w // 2, h // 2))], fr)
    exp = oracle_planes([Job("input_1", full(w, h), (w // 2, h // 2))], fr, RGBA, mode=s.RenderingMode.CpuOptimized)
    assert mismatch_report(got, exp, [Job("input_1", full(w, h), (w // 2, h // 2))], []) is None, "FAST_HALF"
    r = s.Renderer()
    r.set_profiling(True)
    check([Job("input_1", full(w, h), (w // 5, h // 2))], fr, expect=[], renderer=r, what="generic passes")
    kt = r.kernel_times()
    assert kt["convert"][1] == 1 and kt["resample_fused"][1] == 0, kt


# ------------------------------------------------------------------------------------------------
# device planes: alignment
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["yuv", "nv12"])
def test_device_plane_alignments_agree(fmt):
    """one frame at base + 0 / 2 / 8 with pitch = 0 / 2 / 8 (mod 16): base + 0 with a 16-byte pitch takes the TMA kernel, every
    other placement the LDG kernel; all match the oracle and one another (the TMA and LDG kernels checked against each
    other, independently of the oracle).  4:1 and 1.5:1 jobs in each tick."""
    w, h = 1280, 720
    fr = {"input_1": make_frame(fmt, "extreme", 71, w, h)}
    jobs = [Job("input_1", full(w, h), (320, 180)), Job("input_1", full(w, h), (852, 480))]
    seen = {}
    for base in (0, 2, 8):
        for pm in (0, 2, 8):
            tma = base == 0 and pm == 0
            exp = [{"kernel": "tma_int"}, {"kernel": "tma_any"}] if tma else [{"kernel": "ldg", "ratio": 4}, {"kernel": "ldg", "ratio": 0}]
            got, _, _ = check(jobs, fr, placements={"input_1": Placement(base, pm)}, expect=exp, what=f"base+{base} pitch%16={pm}")
            seen[(base, pm)] = got[0]
    ref = seen[(0, 0)]
    for k, g in seen.items():
        assert np.array_equal(g, ref), f"placement {k} differs from the TMA run"


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["yuv", "yuvj", "nv12"])
@pytest.mark.parametrize("where", ["luma pointer", "luma pitch", "chroma pointer", "chroma pitch"])
def test_odd_device_planes_are_refused(fmt, where):
    """4:2:0 luma and NV12 chroma are read two bytes at a time: an odd pointer or pitch is SMR_ERR_INVALID_ARGUMENT before
    any kernel runs.  Planar U / V are read byte by byte and may sit anywhere."""
    import torch
    w, h = 640, 360
    frame = make_frame(fmt, "smooth", 81, w, h)
    planes = plane_list(frame)
    keep = []
    arr = (F.InputFrame * 1)()
    fill_input(arr[0], "input_1", frame, Placement(0, 0), keep)
    p = 0 if where.startswith("luma") else 1
    rows, rb = planes[p].shape
    odd_pitch = (rb + 15) // 16 * 16 + 1
    buf = torch.zeros(1 + odd_pitch * rows + 64, dtype=torch.uint8, device="cuda:0")
    if where.endswith("pointer"):
        buf[1:1 + rows * rb].view(rows, rb)[:] = torch.from_numpy(planes[p]).to("cuda:0")
        arr[0].planes[p], arr[0].pitch[p] = buf.data_ptr() + 1, rb
    else:
        buf[:odd_pitch * rows].view(rows, odd_pitch)[:, :rb] = torch.from_numpy(planes[p]).to("cuda:0")
        arr[0].planes[p], arr[0].pitch[p] = buf.data_ptr(), odd_pitch
    r = s.Renderer()
    r.register_input("input_1")
    W, H, ids, ls, _ = scene_of([Job("input_1", full(w, h), (320, 180))])
    r.set_layouts(OUTPUT_ID, s.Resolution(W, H), RGBA, (W, H), ids, ls)
    out = (F.OutputFrame * 1)()
    o = np.zeros((H, W, 4), np.uint8)
    ob = OUTPUT_ID.encode()
    out[0].output_id, out[0].mem_kind, out[0].planes[0] = ob, F.MEM_HOST, o.ctypes.data
    torch.cuda.synchronize()
    st = F.lib().smr_render(r._h, 0, arr, 1, out, 1)
    launches = r.stats()["kernel_launches"]
    if fmt != "nv12" and p == 1:   # the U plane: no rule
        assert st == F.SMR_OK, r._err()
        assert mismatch_report((o,), oracle_planes([Job("input_1", full(w, h), (320, 180))], {"input_1": frame}, RGBA),
                               [Job("input_1", full(w, h), (320, 180))], r.debug_fused_jobs()) is None
        return
    assert st == 1, (st, r._err())
    assert "2-byte aligned" in r._err()
    assert launches == 0 and r.debug_fused_jobs() == []


# ------------------------------------------------------------------------------------------------
# direct tiles in a launch that cuts the second job at odd rows
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("out_format", [YUV, NV12])
def test_direct_tiles_after_an_odd_height_job(out_format, monkeypatch):
    """Two 4:1 children in one k_resample_tma3 launch.  The first (in layer order) has an odd height and an odd number of
    58-column strips, so its row total is odd and the partition's 2-row shares cut the second job at odd rows; a job cut
    at an odd row cannot emit whole row pairs and goes back to the composite.  Bytes equal the oracle and the run with
    direct tiles off; the hook's `direct` agrees with the direct-tile count."""
    fr = {"input_1": make_frame("yuv", "extreme", 91, 4 * 174, 4 * 101), "input_2": make_frame("yuv", "smooth", 92, 1280, 720)}
    pl = {"input_1": ALIGNED, "input_2": ALIGNED}
    second = Job("input_2", full(1280, 720), (320, 180))
    # alone, the second child (even size, even position, wholly inside the frame) writes its direct tiles itself
    _, fused, r = check([second], fr, out_format=out_format, placements=pl, expect=[{"kernel": "tma_int", "v_same": 1}],
                        what="direct, alone")
    assert fused[0]["direct"] == 1 and r.stats()["last_render_direct_tiles"] > 0, (fused, r.stats())
    # after 3 strips x 101 rows of the first child the partition's 2-row shares end on odd rows of the second
    jobs = [Job("input_1", full(4 * 174, 4 * 101), (174, 101)), second]
    got, fused, r = check(jobs, fr, out_format=out_format, placements=pl,
                          expect=[{"kernel": "tma_int", "v_same": 1}, {"kernel": "tma_int", "v_same": 1}], what="direct")
    assert fused[0]["strip_cols"] == 58 and (174 // 58) * 101 % 2 == 1
    n_direct = r.stats()["last_render_direct_tiles"]
    assert fused[0]["direct"] == 0 and fused[1]["direct"] == 0, fused   # the second job was sent back to the composite
    assert n_direct == 0, n_direct
    monkeypatch.setenv("SMR_DIRECT_K11", "0")
    got0, fused0, r0 = check(jobs, fr, out_format=out_format, placements=pl, what="no direct")
    assert r0.stats()["last_render_direct_tiles"] == 0 and not any(f["direct"] for f in fused0)
    for a, b in zip(got, got0):
        assert np.array_equal(a, b), "direct tiles differ from the composite path"
