"""Every YUV <-> RGB converter of the kernels over the joint byte space, byte for byte against the oracle.

The content is that of `tests/test_color_conversion_space.py` (every (Y, U, V) triple, every interpolated 4:2:0 chroma
value with every luma, every (r, g, b) colour per texel and as a constant 2 x 2 block, the near-tie tuples), and where a
path is a pure conversion its bytes are also held to the float64 tie rule of that file.  Each test proves which path ran
(kernel classes launched, the fused variant, direct tiles), so none can pass by taking another one.

Readers (K1-K4): `node_texture` through `smr_preprocess_frame` (k_preprocess, every input kind, both modes, host frames
and pitched device frames), the composite's 1:1 reader and `yuv_quad` on a pass-through root, and the fused resample
kernels on constant blocks of every near-tie triple.
Writers (K10/K11): the composite's fused output stage (W1) and `k_output` (W3) on every colour, the fused kernel's direct
tiles (W2) against W1, `k_fill`, and `premultiply_store` over every (channel, alpha) pair.
"""
import numpy as np
import pytest

import smelter_b200 as s
from smelter_b200 import _ffi as F
from smelter_b200.renderer import _FRAME_KIND
from oracle import oracle as orc
from tests.parity import node_texture
from tests.test_color_conversion_space import (N, SIDE, constant_blocks, interleaved_all_triples, interleaved_planes, k1_frame_420, k1_rgb, k10_uv, k10_y,
                                               near_tie_rgb, near_tie_yuv, rgb_all_triples, rgb_block_triples, tie_rule,
                                               to_yuv, yuv420_block_triples, yuv420_chroma_sums, yuv444_all_triples)
from tests.test_gpu_composite_classes import GUARD, child, host_input, oracle_out
from tests.test_gpu_fused_variants import ALIGNED, MISALIGNED, Job, check, full

pytestmark = pytest.mark.gpu

GPU, CPU = s.RenderingMode.GpuOptimized, s.RenderingMode.CpuOptimized
RGBA, YUV, NV12 = s.OutputFrameFormat.RgbaWgpuTexture, s.OutputFrameFormat.PlanarYuv420Bytes, s.OutputFrameFormat.Nv12WgpuTexture
YUV422, YUV444 = F.OUT_PLANAR_YUV422, F.OUT_PLANAR_YUV444
OUTPUT_ID = "output_1"


# ------------------------------------------------------------------------------------------------
# frames
# ------------------------------------------------------------------------------------------------
def yuv_frame(kind, y, u, v):
    h, w = y.shape
    if kind == "nv12":
        d = s.FrameData.Nv12(s.NvPlanes(y, np.stack([u, v], axis=-1)))
    else:
        d = s.FrameData({"yuv": "PlanarYuv420", "yuvj": "PlanarYuvJ420", "yuv422": "PlanarYuv422",
                         "yuv444": "PlanarYuv444"}[kind], (y, u, v))
    return s.Frame(d, s.Resolution(w, h))


def interleaved_frame(t, yuyv):
    h, tw, _ = t.shape
    return s.Frame(s.FrameData("InterleavedYuyv422" if yuyv else "InterleavedUyvy422", (t,)), s.Resolution(2 * tw, h))


def rgb_frame(kind, rgba):
    h, w, _ = rgba.shape
    if kind == "bgra":
        return s.Frame(s.FrameData("Bgra", (np.ascontiguousarray(rgba[..., [2, 1, 0, 3]]),)), s.Resolution(w, h))
    if kind == "argb":
        return s.Frame(s.FrameData("Argb", (np.ascontiguousarray(rgba[..., [3, 0, 1, 2]]),)), s.Resolution(w, h))
    return s.Frame(s.FrameData.Rgba8(rgba), s.Resolution(w, h))


def reader_frames(kind):
    """-> [(name, frame)] whose content covers the kind's joint space (the coverage is asserted by the generators' tests
    in test_color_conversion_space.py and re-asserted here where it is cheap)"""
    if kind == "yuv444":
        (y, u, v), n = yuv444_all_triples()
        assert n == N
        return [("all triples", yuv_frame(kind, y, u, v))]
    if kind in ("yuv", "yuvj", "nv12", "yuv422"):
        out = []
        seen = np.zeros(N, bool)
        for part in range(4):
            (y, u, v), cov = yuv420_block_triples(part)
            seen |= cov
            if kind == "yuv422":   # each chroma row twice: the same horizontal taps, no vertical interpolation
                u, v = np.repeat(u, 2, 0), np.repeat(v, 2, 0)
            out.append((f"blocks {part}", yuv_frame(kind, y, u, v)))
        assert np.all(seen)
        (y, u, v), cov = yuv420_chroma_sums()
        assert cov["u"] == cov["v"] == 256 * 4081
        if kind == "yuv422":
            u, v = np.repeat(u, 2, 0), np.repeat(v, 2, 0)
        out.append(("chroma sums", yuv_frame(kind, y, u, v)))
        if kind != "yuv422":   # odd sizes: the NC-6 odd-size branch of node_texture
            out.append(("odd 1023 x 511", yuv_frame(kind, np.ascontiguousarray(y[:511, :1023]),
                                                    np.ascontiguousarray(u[:255, :511]), np.ascontiguousarray(v[:255, :511]))))
        return out
    if kind in ("uyvy", "yuyv"):
        t, n = interleaved_all_triples(kind == "yuyv")
        assert n == N
        return [("all triples", interleaved_frame(t, kind == "yuyv"))]
    rgba, n = rgb_all_triples()
    assert n == N
    return [("all colours", rgb_frame(kind, rgba))]


def device_frame(arr_entry, frame, keep, extra=32):
    """the frame's planes in device memory, each row's pitch `extra` bytes past its length rounded up to 16"""
    import torch
    b = b"_"
    keep.append(b)
    arr_entry.input_id, arr_entry.format = b, _FRAME_KIND[frame.data.kind]
    arr_entry.width, arr_entry.height, arr_entry.pts_ns = frame.resolution.width, frame.resolution.height, 0
    for pi, p in enumerate(frame.data.planes):
        p = np.ascontiguousarray(p)
        p = p.reshape(p.shape[0], -1)
        rows, rb = p.shape
        pitch = (rb + 15) // 16 * 16 + extra
        buf = torch.zeros(pitch * rows + 64, dtype=torch.uint8, device="cuda:0")
        buf[:pitch * rows].view(rows, pitch)[:, :rb] = torch.from_numpy(p).to("cuda:0")
        keep.append(buf)
        arr_entry.planes[pi], arr_entry.pitch[pi], arr_entry.mem_kind = buf.data_ptr(), pitch, F.MEM_DEVICE


def preprocess(r, frame, device):
    """smr_preprocess_frame at the source size (k_preprocess kind 0: node_texture at every pixel) -> (rgba, launches)"""
    import torch
    keep = []
    arr = (F.InputFrame * 1)()
    if device:
        device_frame(arr[0], frame, keep)
    else:
        host_input(arr[0], "_", frame, keep)
    w, h = frame.resolution.width, frame.resolution.height
    out = np.empty((h, w, 4), np.uint8)
    torch.cuda.synchronize()
    before = r.stats()["kernel_launches"]
    st = F.lib().smr_preprocess_frame(r._h, arr, 0, 0, out.ctypes.data, 0, F.MEM_HOST)
    assert st == F.SMR_OK, r._err()
    return out, r.stats()["kernel_launches"] - before


def out_shapes(fmt, w, h):
    """(rows, row bytes) of each output plane (out_plane_layout: chroma w / 2 x h / 2, w / 2 x h or w x h, rounded down)"""
    return {RGBA: [(h, w * 4)], YUV: [(h, w), (h // 2, w // 2), (h // 2, w // 2)], NV12: [(h, w), (h // 2, 2 * (w // 2))],
            YUV422: [(h, w), (h, w // 2), (h, w // 2)], YUV444: [(h, w), (h, w), (h, w)]}[fmt]


def run_one(layers, frames, ids, root, out_res, fmt, renderer, dev_planes=None):
    """one tick of one output (host planes, or device planes [(ptr, pitch)]) -> host planes (None for device output)"""
    import torch
    r = renderer
    for i in ids:
        r.register_input(i)
    keep = []
    arr = (F.InputFrame * max(1, len(ids)))()
    for k, i in enumerate(ids):
        host_input(arr[k], i, frames[i], keep)
    r.set_layouts(OUTPUT_ID, s.Resolution(*out_res), fmt, root, ids, layers)
    outs = (F.OutputFrame * 1)()
    b = OUTPUT_ID.encode()
    outs[0].output_id = b
    planes = None
    if dev_planes is None:
        planes = [np.zeros(sh, np.uint8) for sh in out_shapes(fmt, *out_res)]
        outs[0].mem_kind = F.MEM_HOST
        for p, a in enumerate(planes):
            outs[0].planes[p] = a.ctypes.data
    else:
        outs[0].mem_kind = F.MEM_DEVICE
        for p, (ptr, pitch) in enumerate(dev_planes):
            outs[0].planes[p], outs[0].pitch[p] = ptr, pitch
    torch.cuda.synchronize()
    r.render_raw(0, arr, len(ids), outs, 1)
    torch.cuda.synchronize()
    return planes


def first_diff(got, exp, what):
    assert np.shape(got) == np.shape(exp), (what, np.shape(got), np.shape(exp))
    if np.array_equal(got, exp):
        return
    d = np.argwhere(got != exp)
    i = tuple(d[0])
    raise AssertionError(f"{what}: {len(d)} bytes differ; first at {i}: got {got[i]} expected {exp[i]}")


# ------------------------------------------------------------------------------------------------
# readers
# ------------------------------------------------------------------------------------------------
READER_KINDS = ["yuv", "yuvj", "nv12", "yuv422", "yuv444", "uyvy", "yuyv", "bgra", "argb", "rgba"]


@pytest.mark.parametrize("kind", READER_KINDS)
def test_node_texture_every_tuple(kind):
    """R1 / R2 / R3 directly: k_preprocess at source size is node_texture for every pixel.  Both modes, host frames and
    device frames whose pitch exceeds the row.  k_preprocess has no kernel class of its own: each call must launch exactly
    one kernel and leave every profiled class at zero launches (no k_convert, composite, fused resample or k_output).
    Bytes equal the oracle; the conversion being pure, they also meet the float64 tie rule (4:2:0 / J420 / NV12 with the
    exactly interpolated chroma, 4:4:4 / UYVY / YUYV texel by texel).  Every run's bytes equal the oracle's, so the tie rule
    is applied once per frame, to those bytes."""
    for name, fr in reader_frames(kind):
        exp = node_texture(fr)
        for mode in (GPU, CPU):
            r = s.Renderer(s.RendererOptions(rendering_mode=mode))
            r.set_profiling(True)
            for device in (False, True):
                what = f"{kind} {name} {mode} {'device' if device else 'host'}"
                got, launches = preprocess(r, fr, device)
                assert launches == 1, (what, launches)
                first_diff(got, exp, what)
            assert all(n == 0 for _, n in r.kernel_times().values()), (kind, name, r.kernel_times())
        w, h = fr.resolution.width, fr.resolution.height
        if kind in ("yuv", "yuvj", "nv12") and w % 2 == 0:
            y, u, v = (fr.data.planes[0], fr.data.planes[1][..., 0], fr.data.planes[1][..., 1]) if kind == "nv12" \
                else fr.data.planes
            for r0 in range(0, h, 512):
                rows = np.arange(r0, min(r0 + 512, h))
                for c, e in enumerate(k1_frame_420((np.asarray(y), np.asarray(u), np.asarray(v)), kind == "yuvj", rows)):
                    tie_rule(exp[rows, :, c], e, f"{kind} {name} {'rgb'[c]}")
        elif kind in ("yuv444", "uyvy", "yuyv"):
            if kind == "yuv444":
                y, u, v = fr.data.planes
            else:
                y, u, v = interleaved_planes(np.asarray(fr.data.planes[0]), kind == "yuyv")
            for r0 in range(0, SIDE, 512):
                sl = slice(r0, r0 + 512)
                for c, e in enumerate(k1_rgb(y[sl] / 255.0, u[sl] / 255.0, v[sl] / 255.0, False)):
                    tie_rule(exp[sl, :, c], e, f"{kind} {'rgb'[c]}")


def passthrough(frame, mode, fmt=RGBA, out_res=None, root=None):
    """the frame as the only child, 1:1 on a root of its size -> (output planes, renderer)"""
    w, h = frame.resolution.width, frame.resolution.height
    root = root or (w, h)
    ls = [child(0, 0.0, 0.0, float(root[0]), float(root[1]), w, h)]
    r = s.Renderer(s.RendererOptions(rendering_mode=mode))
    r.set_profiling(True)
    return run_one(ls, {"a": frame}, ["a"], root, out_res or root, fmt, r), ls, r


@pytest.mark.parametrize("kind", ["yuv", "yuvj", "nv12", "yuv422", "yuv444", "uyvy", "yuyv"])
def test_composite_reader_passthrough(kind):
    """R4 and the composite's 1:1 reader: the frames as a pass-through root to RGBA.  The composite converts the frame
    itself (no k_convert, no k_output, no fused resample) and its bytes equal the oracle's"""
    for name, fr in reader_frames(kind):
        for mode in (GPU, CPU):
            got, ls, r = passthrough(fr, mode)
            kt = r.kernel_times()
            what = f"{kind} {name} {mode}"
            assert kt["composite"][1] == 1 and kt["convert"][1] == 0 and kt["output"][1] == 0 \
                and kt["resample_fused"][1] == 0, (what, kt)
            w, h = fr.resolution.width, fr.resolution.height
            first_diff(got[0], oracle_out(ls, {"a": fr}, ["a"], (w, h), (w, h), RGBA, mode)[0], what)


def test_sample_node_bilinear():
    """sample_node's bilinear branch (CpuOptimized: the layout shader scales a YUV child itself): children of the
    chroma-sum frame scaled by 3 / 4 and 5 / 4, and by exactly 1 / 2, where the four taps of every pixel are one
    chroma-aligned quad and yuv_quad converts them; no fused resample and no k_convert run"""
    (y, u, v), _ = yuv420_chroma_sums()
    for kind in ("yuv", "yuvj", "nv12"):
        fr = yuv_frame(kind, np.ascontiguousarray(y[:1024, :1024]), np.ascontiguousarray(u[:512, :512]),
                       np.ascontiguousarray(v[:512, :512]))
        ls = [child(0, 0.0, 0.0, 768.0, 768.0, 1024, 1024), child(0, 770.0, 0.0, 512.0, 512.0, 1024, 1024),
              child(0, 0.0, 770.0, 1280.0, 1280.0, 1024, 1024)]
        root = (2050, 2050)
        r = s.Renderer(s.RendererOptions(rendering_mode=CPU))
        r.set_profiling(True)
        got = run_one(ls, {"a": fr}, ["a"], root, root, RGBA, r)
        kt = r.kernel_times()
        assert kt["composite"][1] == 1 and kt["resample_fused"][1] == 0 and kt["convert"][1] == 0, kt
        first_diff(got[0], oracle_out(ls, {"a": fr}, ["a"], root, root, RGBA, CPU)[0], f"{kind} scaled children")


# ------------------------------------------------------------------------------------------------
# fused resample kernels: constant blocks of every near-tie triple
# ------------------------------------------------------------------------------------------------
SLICE_CHROMA = (0, 16, 128, 240, 255)


def slice_triples():
    """the (Y, V) slices at U in SLICE_CHROMA and the (Y, U) slices at V in SLICE_CHROMA: index Y | U << 8 | V << 16"""
    a = np.arange(65536, dtype=np.int64)
    out = [(a & 255) | (c << 8) | ((a >> 8) << 16) for c in SLICE_CHROMA]
    out += [(a & 255) | ((a >> 8) << 8) | (c << 16) for c in SLICE_CHROMA]
    return np.unique(np.concatenate(out))


def block_frames(kind, triples, B, side=SIDE):
    """4:2:0 / NV12 / UYVY / YUYV frames of side x side luma in which each triple gets one constant B x B block (the
    last frame's spare blocks repeat the first triple) -> [(frame, triple index per block (nb, nb))]"""
    nb = side // B
    per = nb * nb
    out = []
    for k in range(0, len(triples), per):
        t = np.full(per, triples[0], np.int64)
        t[:len(triples[k:k + per])] = triples[k:k + per]
        t = t.reshape(nb, nb)
        Y, U, V = (t & 255).astype(np.uint8), ((t >> 8) & 255).astype(np.uint8), (t >> 16).astype(np.uint8)
        y = np.repeat(np.repeat(Y, B, 0), B, 1)
        if kind in ("uyvy", "yuyv"):
            u, v = np.repeat(np.repeat(U, B, 0), B // 2, 1), np.repeat(np.repeat(V, B, 0), B // 2, 1)
            tx = np.empty((side, side // 2, 4), np.uint8)
            if kind == "uyvy":
                tx[..., 0], tx[..., 1], tx[..., 2], tx[..., 3] = u, y[:, 0::2], v, y[:, 1::2]
            else:
                tx[..., 0], tx[..., 1], tx[..., 2], tx[..., 3] = y[:, 0::2], u, y[:, 1::2], v
            out.append((interleaved_frame(tx, kind == "yuyv"), t))
        else:
            u, v = np.repeat(np.repeat(U, B // 2, 0), B // 2, 1), np.repeat(np.repeat(V, B // 2, 0), B // 2, 1)
            out.append((yuv_frame(kind, y, u, v), t))
    return out


def interior(n_out, scale, offset, B):
    """(n_out,) bool: output coordinates whose Lanczos footprint (plus one pixel for the chroma taps) lies inside one
    B-pixel block"""
    o = np.arange(n_out, dtype=np.float64)
    c = offset + (o + 0.5) * scale - 0.5
    first, last = np.ceil(c - 3.0 * scale) - 1, np.floor(c + 3.0 * scale) + 1
    return (np.floor(first / B) == np.floor(last / B)) & (first >= 0)


def check_block_interiors(got, t, scale, offset, B, full_range, what):
    """every interior output byte is within 1 of the float64 K1 byte of its block's triple (the f16 ring of pass 1
    allows no tighter bound)"""
    h, w = got.shape[:2]
    ix, iy = interior(w, scale, offset, B), interior(h, scale, 0.0, B)
    bx = ((offset + (np.arange(w) + 0.5) * scale) // B).astype(int)
    by = (((np.arange(h) + 0.5) * scale) // B).astype(int)
    tt = t[np.clip(by, 0, t.shape[0] - 1)][:, np.clip(bx, 0, t.shape[1] - 1)]
    exact = k1_rgb((tt & 255) / 255.0, ((tt >> 8) & 255) / 255.0, (tt >> 16) / 255.0, full_range)
    m = iy[:, None] & ix[None, :]
    per_block = np.zeros(t.shape, np.int64)
    yy, xx = np.nonzero(m)
    np.add.at(per_block, (np.clip(by, 0, t.shape[0] - 1)[yy], np.clip(bx, 0, t.shape[1] - 1)[xx]), 1)
    assert np.all(per_block >= 1), (what, int(np.count_nonzero(per_block == 0)))   # every block has an interior pixel
    for c, e in enumerate(exact):
        d = np.abs(got[..., c].astype(int) - np.rint(e).astype(int))
        assert d[m].max() <= 1, f"{what}: channel {'rgb'[c]} off by {d[m].max()} inside a block"


FUSED = [  # (name, frame kind, source range, scale, crop offset, block side, placement, expected kernel)
    ("tma3-2-limited", "yuv", 0, 2, 0.0, 16, ALIGNED, {"kernel": "tma_int", "ratio": 2, "full_range": 0}),
    ("tma3-2-full", "yuvj", 1, 2, 0.0, 16, ALIGNED, {"kernel": "tma_int", "ratio": 2, "full_range": 1}),
    ("tma3-4-limited", "yuv", 0, 4, 0.0, 32, ALIGNED, {"kernel": "tma_int", "ratio": 4, "full_range": 0}),
    ("tma3-4-full", "yuvj", 1, 4, 0.0, 32, ALIGNED, {"kernel": "tma_int", "ratio": 4, "full_range": 1}),
    ("tma3-4-nv12", "nv12", 0, 4, 0.0, 32, ALIGNED, {"kernel": "tma_int", "ratio": 4, "src_class": 1}),
    ("tma0-2+0.5", "yuv", 0, 2, 0.5, 16, ALIGNED, {"kernel": "tma_any"}),
    ("ldg-2-planar", "yuv", 0, 2, 0.0, 16, MISALIGNED, {"kernel": "ldg", "ratio": 2, "src_class": 0}),
    ("ldg-2-nv12", "nv12", 0, 2, 0.0, 16, MISALIGNED, {"kernel": "ldg", "ratio": 2, "src_class": 1}),
    ("ldg-2-uyvy", "uyvy", 0, 2, 0.0, 16, None, {"kernel": "ldg", "ratio": 2, "src_class": 2}),
    ("ldg-2-yuyv", "yuyv", 0, 2, 0.0, 16, None, {"kernel": "ldg", "ratio": 2, "src_class": 3}),
]


@pytest.mark.parametrize("case", FUSED, ids=[c[0] for c in FUSED])
def test_fused_near_tie_blocks(case):
    """R5 / R6 / R7: every triple of near_tie_yuv(range) (and, for k_resample_tma3 at 2:1 on limited range, the (Y, V)
    / (Y, U) slices at U or V in {0, 16, 128, 240, 255}) as a constant block wide enough for whole Lanczos footprints; the fused variant is asserted per frame, the
    whole frame equals the oracle and block interiors are within 1 of the float64 K1 byte"""
    name, kind, fr_, S, off, B, place, expect = case
    triples = np.flatnonzero(near_tie_yuv(fr_))
    if name == "tma3-2-limited":   # the slices take eleven 4096 x 4096 frames: one kernel and range carries them
        triples = np.union1d(triples, slice_triples())
    if kind in ("uyvy", "yuyv", "nv12"):
        assert fr_ == 0   # NV12 and the interleaved kinds are limited range
    seen = np.zeros(N, bool)
    for k, (frame, t) in enumerate(block_frames(kind, triples, B)):
        seen[t.ravel()] = True
        w = h = SIDE
        crop = (off, 0.0, float(w) - 2 * S if off else float(w), float(h))
        dst = (int(crop[2] // S), h // S)
        pl = {"input_1": place} if place is not None else None
        got, fused, _ = check([Job("input_1", crop, dst)], {"input_1": frame}, placements=pl, expect=[expect],
                              what=f"{name} frame {k}")
        check_block_interiors(got[0], t, float(S), off, B, fr_, f"{name} frame {k}")
    assert np.all(seen[triples])
    print(f"\n{name}: {len(triples)} triples ({int(near_tie_yuv(fr_).sum())} near ties)")


# ------------------------------------------------------------------------------------------------
# writers
# ------------------------------------------------------------------------------------------------
def writer_frames():
    """the every-colour frame and the four constant-block frames (every colour as a 2 x 2 block)"""
    rgba, n = rgb_all_triples()
    assert n == N
    yield "all colours", rgba
    seen = np.zeros(N, bool)
    for p in range(4):
        rgba, cov = rgb_block_triples(p)
        seen |= cov
        yield f"blocks {p}", rgba
    assert np.all(seen)


@pytest.mark.parametrize("fmt", [YUV, NV12], ids=["yuv420", "nv12"])
def test_composite_writer_every_colour(fmt):
    """W1: an opaque RGBA8 root passed through to 4:2:0 / NV12 -- Y' per texel over every colour and the 2 x 2 mean
    chroma of every constant-block colour, written by the composite itself (no k_output); equal to the oracle and, the
    pass-through being a pure conversion, to the float64 K10/K11 bytes under the tie rule"""
    for name, rgba in writer_frames():
        fr = rgb_frame("rgba", rgba)
        got, ls, r = passthrough(fr, GPU, fmt)
        kt = r.kernel_times()
        assert kt["composite"][1] == 1 and kt["output"][1] == 0, (name, kt)
        y = got[0]
        u, v = (got[1][..., 0::2], got[1][..., 1::2]) if fmt == NV12 else (got[1], got[2])
        if fmt == NV12:
            ey, euv = orc.rgba_to_nv12(rgba)
            eu, ev = euv[..., 0], euv[..., 1]
        else:
            ey, eu, ev = orc.rgba_to_yuv420(rgba)
        for g, e, c in ((y, ey, "y"), (u, eu, "u"), (v, ev, "v")):
            first_diff(np.asarray(g).reshape(e.shape), e, f"{name} {c}")
        f = rgba[..., :3] / 255.0
        tie_rule(y, k10_y(f[..., 0], f[..., 1], f[..., 2]), f"{name} Y'")
        m = [(f[0::2, 0::2, c] + f[0::2, 1::2, c] + f[1::2, 0::2, c] + f[1::2, 1::2, c]) / 4.0 for c in range(3)]
        xu, xv = k10_uv(*m)
        tie_rule(np.asarray(u).reshape(xu.shape), xu, f"{name} U'")
        tie_rule(np.asarray(v).reshape(xv.shape), xv, f"{name} V'")


def check_output(rgba, fmt, out_res, what):
    fr = rgb_frame("rgba", rgba)
    h, w = rgba.shape[:2]
    got, ls, r = passthrough(fr, GPU, fmt, out_res=out_res)
    kt = r.kernel_times()
    assert kt["output"][1] == 1, (what, kt)
    root = oracle_out(ls, {"a": fr}, ["a"], (w, h), (w, h), RGBA, GPU)[0].reshape(h, w, 4)
    cw, ch = {YUV: (out_res[0] // 2, out_res[1] // 2), YUV422: (out_res[0] // 2, out_res[1]), YUV444: out_res}[fmt]
    exp = orc.rgba_to_yuv_planar_scaled(root, out_res[0], out_res[1], cw, ch)
    for p, (g, e) in enumerate(zip(got, exp)):
        first_diff(g, e, f"{what} plane {p}")
    return got


@pytest.mark.parametrize("fmt", [YUV444, YUV422], ids=["yuv444", "yuv422"])
def test_output_writer_every_colour(fmt):
    """W3 (k_output, NC-6u sample at each target texel) at 1:1: 4:4:4 and 4:2:2 outputs of the every-colour frame and of
    the four constant-block frames, so every colour's chroma is written as a texel (4:4:4) and as a horizontal pair mean
    (4:2:2); equal to the oracle and, the path being a pure conversion, to the float64 K10/K11 bytes under the tie rule"""
    for name, rgba in writer_frames():
        got = check_output(rgba, fmt, (SIDE, SIDE), f"{name} {fmt}")
        f = rgba[..., :3] / 255.0
        tie_rule(got[0], k10_y(f[..., 0], f[..., 1], f[..., 2]), f"{name} Y'")
        if fmt == YUV422:   # chroma texel x samples at luma 2x + 1: the mean of pixels 2x and 2x + 1
            f = (f[:, 0::2] + f[:, 1::2]) / 2.0
        eu, ev = k10_uv(f[..., 0], f[..., 1], f[..., 2])
        tie_rule(got[1], eu, f"{name} U'")
        tie_rule(got[2], ev, f"{name} V'")


@pytest.mark.parametrize("case", ["odd", "rescaled"])
def test_output_writer_sizes(case):
    """W3 at an odd 4:2:0 output size and from a root of another size; the composite writes RGBA8, k_output converts it"""
    rgba, _ = rgb_all_triples()
    if case == "odd":
        rgba = np.ascontiguousarray(rgba[:1023, :2047])
        check_output(rgba, YUV, (2047, 1023), case)
    else:
        check_output(np.ascontiguousarray(rgba[:1024, :2048]), YUV, (1500, 700), case)


def k1_image_near_ties():
    """the near-tie colours (near_tie_rgb) that K1 reaches, and one limited-range (Y, U, V) triple that reaches each
    -> (triples, number of reachable near-tie colours, size of K1's image)"""
    (y, u, v), _ = yuv444_all_triples()
    rgb = orc.yuv_planar_to_rgba(y, u, v, SIDE, SIDE, SIDE, SIDE).reshape(-1, 4)
    col = rgb[:, 0].astype(np.int64) | (rgb[:, 1].astype(np.int64) << 8) | (rgb[:, 2].astype(np.int64) << 16)
    tri = y.reshape(-1).astype(np.int64) | (u.reshape(-1).astype(np.int64) << 8) | (v.reshape(-1).astype(np.int64) << 16)
    near, _ = near_tie_rgb()
    image, first = np.unique(col, return_index=True)
    hit = near[image]
    return tri[first[hit]], int(hit.sum()), len(image)


def test_direct_tiles_against_composite(monkeypatch):
    """W2 against W1: 4:1 constant YUV blocks whose K1 bytes are near-tie colours of K10 / K11, rendered to 4:2:0 by the
    fused kernel's direct tiles and, with SMR_DIRECT_K11=0, by the composite; the two sets of planes are identical and
    equal to the oracle.

    W2's input is the fused resample's output, so only colours in K1's image can reach it: 2 327 of the near-tie colours.
    Which of them arrive as constant 2 x 2 blocks is counted from an RGBA render of the same frames (the f16 ring of
    pass 1 moves many block interiors by one step): 756 on an H100, asserted as at least 700.  Of the 20 constant-block
    colours whose bytes change when the three terms of to_u / to_v are reversed, one, (223, 0, 116), is in K1's image, and
    it does not arrive as a block, so that reversal in emit_yuv_2x2 cannot show in this test: W2 is held to W1 and to the
    oracle on what the fused kernel can deliver, not over the whole constant-block space."""
    triples, n_reach, n_image = k1_image_near_ties()
    near, _ = near_tie_rgb()
    arrived = np.zeros(N, bool)
    jobs = [Job("input_1", full(SIDE, SIDE), (SIDE // 4, SIDE // 4))]
    frames = block_frames("yuv", triples, 32)
    for frame, _ in frames:
        rgba, _, _ = check(jobs, {"input_1": frame}, placements={"input_1": ALIGNED}, expect=[{"kernel": "tma_int"}],
                           what="RGBA")
        arrived |= constant_blocks(rgba[0])
    n_arrived = int(np.count_nonzero(arrived & near))
    print(f"\nK1 image: {n_image} colours, {n_reach} of them near-tie colours of K10 / K11, {n_arrived} arrive as 2 x 2 blocks")
    print(f"(223, 0, 116) arrives as a block: {bool(arrived[223 | (116 << 16)])}")
    assert n_reach == 2327 and n_arrived >= 700, (n_reach, n_arrived)
    for k, (frame, _) in enumerate(frames):
        monkeypatch.delenv("SMR_DIRECT_K11", raising=False)
        got, fused, r = check(jobs, {"input_1": frame}, out_format=YUV, placements={"input_1": ALIGNED},
                              expect=[{"kernel": "tma_int", "ratio": 4}], what=f"direct {k}")
        assert fused[0]["direct"] == 1 and r.stats()["last_render_direct_tiles"] > 0, (fused, r.stats())
        monkeypatch.setenv("SMR_DIRECT_K11", "0")
        got0, fused0, r0 = check(jobs, {"input_1": frame}, out_format=YUV, placements={"input_1": ALIGNED},
                                 what=f"composite {k}")
        assert r0.stats()["last_render_direct_tiles"] == 0 and not any(f["direct"] for f in fused0)
        for p, (a, b) in enumerate(zip(got, got0)):
            first_diff(a, b, f"frame {k} plane {p}: direct tiles vs composite")


@pytest.mark.parametrize("fmt", [RGBA, YUV, NV12, YUV422, YUV444], ids=["rgba", "yuv420", "nv12", "yuv422", "yuv444"])
def test_fill(fmt):
    """k_fill: a scene with nothing to draw, at even and odd sizes, into host planes and into device planes with odd
    pitches and guard bytes; every byte is RGBColor::to_yuv of black (float64, rounded) or 0 for RGBA"""
    import torch
    ey, eu, ev = (int(np.rint(c)) for c in to_yuv(0, 0, 0))
    for w, h in ((64, 36), (65, 37)):
        want = [np.zeros(sh, np.uint8) for sh in out_shapes(fmt, w, h)] if fmt == RGBA else \
            [np.full(sh, val, np.uint8) for sh, val in zip(out_shapes(fmt, w, h), (ey, eu, ev))]
        if fmt == NV12:
            want[1][:, 0::2], want[1][:, 1::2] = eu, ev
        for pm in (None, 1, 3):
            r = s.Renderer()
            r.set_profiling(True)
            what = f"{w}x{h} pitch+{pm}"
            if pm is None:
                got = run_one([], {}, [], (0, 0), (w, h), fmt, r)
            else:
                if fmt == RGBA:
                    pm = 4 * pm   # RGBA8 planes must be 4-byte aligned
                bufs, planes = [], []
                for rows, rb in out_shapes(fmt, w, h):
                    pitch = rb + pm
                    buf = torch.full((GUARD + pitch * rows + GUARD,), 0xA5, dtype=torch.uint8, device="cuda:0")
                    bufs.append((buf, rows, rb, pitch))
                    planes.append((buf.data_ptr() + GUARD, pitch))
                run_one([], {}, [], (0, 0), (w, h), fmt, r, dev_planes=planes)
                got = []
                for buf, rows, rb, pitch in bufs:
                    a = buf.cpu().numpy()
                    body = a[GUARD:GUARD + pitch * rows].reshape(rows, pitch)
                    got.append(body[:, :rb].copy())
                    assert np.all(a[:GUARD] == 0xA5) and np.all(a[GUARD + pitch * rows:] == 0xA5) \
                        and np.all(body[:, rb:] == 0xA5), f"{what}: bytes outside the planes were written"
            kt = r.kernel_times()
            assert kt["fill"][1] >= 1 and kt["composite"][1] == 0, (what, kt)
            for p, (g, e) in enumerate(zip(got, want)):
                first_diff(np.asarray(g).reshape(e.shape), e, f"{what} plane {p}")


def eotf(c):
    return np.where(c <= 0.04045, c / 12.92, ((c + 0.055) / 1.055) ** 2.4)


def oetf(x):
    return np.where(x <= 0.0031308, x * 12.92, 1.055 * np.power(np.maximum(x, 0.0031308), 1 / 2.4) - 0.055)


@pytest.mark.parametrize("mode", [GPU, CPU], ids=["gpu_mode", "cpu_mode"])
def test_premultiply_every_pair(mode):
    """premultiply_store (k_preprocess kind 2) over every (channel, alpha) pair: equal to the oracle, and to a float64
    premultiply-then-encode under the tie rule (GpuOptimized: sRGB decode, multiply, the ideal encode whose thresholds
    are eotf_f64((k + .5) / 255); CpuOptimized: c a / 255)"""
    c, a = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    rgba = np.empty((256, 256, 4), np.uint8)
    rgba[..., 0], rgba[..., 1], rgba[..., 2], rgba[..., 3] = c, 255 - c, c, a
    r = s.Renderer(s.RendererOptions(rendering_mode=mode))
    before = r.stats()["kernel_launches"]
    got = r.premultiply_rgba8(rgba)
    assert r.stats()["kernel_launches"] - before == 1
    first_diff(got, orc.add_premultiplied_alpha(rgba, int(mode)), f"{mode} premultiply")
    am = np.maximum(rgba[..., 3] / 255.0, 0.00001)
    for ch in range(3):
        x = rgba[..., ch] / 255.0
        e = oetf(np.clip(eotf(x) * am, 0, 1)) * 255.0 if mode == GPU else np.clip(x * am, 0, 1) * 255.0
        tie_rule(got[..., ch], e, f"{mode} channel {ch}")
    assert np.array_equal(got[..., 3], rgba[..., 3])
