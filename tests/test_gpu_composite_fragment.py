"""The composite's general fragment path (`shade` / `shade_blend`) against the oracle, byte for byte, at every branch edge.

The scenes are those of `tests/fragment_ref.py`, where `tests/test_composite_fragment_space.py` holds the oracle to a
float64 restatement of apply_layouts.wgsl: corner radii with `dist == 0` exact, both border ramps on both kinds of
layer, 1 to 21 masks and the `mask_alpha < 0.01` cut, box shadows from blur 0 to 40, rotations, fractional and exact
crops, coordinates near 3000.  Here each is built with `set_layouts` (the probe over a 1:1 background child holding every
byte) and crossed with both rendering modes, RGBA and NV12 output, and both composite kernels:
  * k_composite_p: the background and the probe;
  * k_composite_multi: more layers than k_composite_p's parameter block holds, with the probe after the 40 layers each
    tile keeps in shared memory, so the general path reads the probe from global memory.

Proof of path: every pixel where the oracle's fragment is not the bare colour or sample (ramps, borders, masks,
shadows) must lie outside the probe's interior bars when it has a fast class, and outside the per-pixel shortcut of
`shade_blend`; so it ran through `shade`.  `test_gathers` checks that the cooperative warp gather and the per-lane
gather (more than 160 pixels of one warp) both run.  Two scenes are left to the CPU test: the one without a child (an
input without a frame cannot be fed to one tick here) and the one with 21 masks (a render layout holds at most 20).
"""
import ctypes as C
import functools

import numpy as np
import pytest

import smelter_b200 as s
from smelter_b200 import _ffi as F
from tests import fragment_ref as R
from tests.parity import OUTPUT_ID, to_oracle_layout
from tests.test_gpu_composite_classes import colour, first_mismatch, layout, oracle_out, run

GPU, CPU = s.RenderingMode.GpuOptimized, s.RenderingMode.CpuOptimized
RGBA, NV12 = s.OutputFrameFormat.RgbaWgpuTexture, s.OutputFrameFormat.Nv12WgpuTexture
FAST_CLASSES = 1 | 2 | 4 | 16 | 32     # IDENT, CONST, LUT, SAMPLE, HALF: the classes that skip the fragment path in the bars
SM_LAYERS = 40                         # kernels.cu: layers of a tile kept in shared memory
PARAM_LAYERS = 96                      # kCompositeParamLayers
SCENES = {sc.name: sc for sc in R.SCENES
          if (sc.probe.type != R.TEXTURE or sc.probe.tex is not None) and len(sc.probe.masks) <= R.MAX_MASKS}


def frame(t):
    return s.Frame(s.FrameData.Rgba8(t), s.Resolution(t.shape[1], t.shape[0]))


def probe_layout(p):
    crop = p.crop if p.crop is not None else (0.0, 0.0, 0.0, 0.0)
    return layout(p.type, p.left, p.top, p.width, p.height, child=1 if p.type == R.TEXTURE else 0, color=p.color,
                  radius=p.radius, border=p.border, border_color=p.border_color, masks=p.masks, rotation=p.rotation,
                  crop=crop, blur=p.blur)


def padding(n, W, H):
    """n tiny translucent colour layers in the bottom-right corner, each covering pixels"""
    return [colour(W - 6.0 + (k % 5), H - 6.0 + (k // 5) % 5, 1.0, 1.0, (k % 256, 50, 9, 40)) for k in range(n)]


def build(sc, kernel):
    """-> (layers, frames, ids, index of the probe)"""
    frames = {"bg": frame(R.background(sc.W, sc.H))}
    ids = ["bg"]
    if sc.probe.tex is not None:
        frames["tex"] = frame(sc.probe.tex)
        ids.append("tex")
    bg = layout(0, 0.0, 0.0, float(sc.W), float(sc.H), child=0, crop=(0.0, 0.0, float(sc.W), float(sc.H)))
    under = [bg] * (1 if kernel == "p" else SM_LAYERS + 1)
    layers = under + [probe_layout(sc.probe)]
    if kernel == "multi":
        layers += padding(PARAM_LAYERS + 1 - len(layers), sc.W, sc.H)
    return layers, frames, ids, len(under)


@functools.lru_cache(maxsize=None)
def covered(name):
    """pixels the probe covers (NC-7; ambiguous snaps included)"""
    sc = SCENES[name]
    a = R.evaluate(sc.probe, R.background(sc.W, sc.H), R.GPU_OPTIMIZED)
    return a.covered | a.cover_ambiguous


def shortcut_and_bars(L, W, H):
    """smr_debug_interior: (shortcut (H, W) bool, [bar boxes])"""
    box = (C.c_int32 * 12)()
    sc = np.zeros((H, W), np.uint8)
    assert F.lib().smr_debug_interior(C.byref(L), W, H, C.byref(box), sc.ctypes.data_as(C.c_void_p)) == 0
    return sc.astype(bool), [tuple(box[4:8]), tuple(box[8:12])]


def in_bars(bars, W, H):
    m = np.zeros((H, W), bool)
    for x0, x1, y0, y1 in bars:
        if x0 < x1 and y0 < y1:
            m[max(y0, 0):max(y1, 0), max(x0, 0):max(x1, 0)] = True
    return m


def warp_totals(need):
    """pixels each warp (one 128 x 2 strip of a 128 x 16 tile) sends to the general path"""
    H, W = need.shape
    p = np.zeros(((H + 1) // 2 * 2, (W + 127) // 128 * 128), np.int64)
    p[:H, :W] = need
    return p.reshape(p.shape[0] // 2, 2, p.shape[1] // 128, 128).sum(axis=(1, 3))


def need_map(rec, cov, W, H):
    """the probe's pixels its warps gather: covered pixels of the 4 x 2 thread blocks it does not handle as a fast class"""
    need = cov.copy()
    if rec["fast"] & FAST_CLASSES:
        box = rec["box"]
        for x0, x1, y0, y1 in (box[4:8], box[8:12]):
            bx0, by0 = (max(x0, 0) + 3) // 4 * 4, (max(y0, 0) + 1) // 2 * 2     # blocks wholly inside the bar
            bx1, by1 = x1 // 4 * 4, y1 // 2 * 2
            if bx0 < bx1 and by0 < by1:
                need[by0:by1, bx0:bx1] = False
    return need


def check_path(sc, layers, probe, rec, mode):
    """every non-bare pixel of the probe went through `shade`; -> the warp totals of its gather"""
    L = layers[probe]
    W, H = sc.W, sc.H
    cov = covered(sc.name)
    bare = orc_bare(L, W, H, mode)
    claimed = cov & ~bare
    assert claimed.sum() > 0, (sc.name, "no pixel of the probe needs the fragment path")
    shortcut, bars = shortcut_and_bars(L, W, H)
    shaded = cov & ~shortcut
    if rec["fast"] & FAST_CLASSES:
        shaded &= ~in_bars(bars, W, H)
    assert not (claimed & ~shaded).any(), (sc.name, rec, int((claimed & ~shaded).sum()))
    return warp_totals(need_map(rec, cov, W, H))


def orc_bare(L, W, H, mode):
    from oracle import oracle as orc
    return orc.bare_map(W, H, to_oracle_layout(L), mode=int(mode))


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["p", "multi"])
@pytest.mark.parametrize("fmt", [RGBA, NV12], ids=["rgba", "nv12"])
@pytest.mark.parametrize("mode", [GPU, CPU], ids=["gpu_mode", "cpu_mode"])
@pytest.mark.parametrize("name", list(SCENES))
def test_fragment_path(name, mode, fmt, kernel):
    sc = SCENES[name]
    layers, frames, ids, probe = build(sc, kernel)
    assert (len(layers) > PARAM_LAYERS) == (kernel == "multi")
    got, r = run([(OUTPUT_ID, layers, (sc.W, sc.H), (sc.W, sc.H), fmt, None)], frames, ids, mode)
    recs = r.debug_composite_layers()
    what = f"{name} {mode} fmt={fmt} {kernel}"
    assert len(recs) == len(layers) and all(L["kernel"] == kernel for L in recs), (what, {L["kernel"] for L in recs})
    totals = check_path(sc, layers, probe, recs[probe], mode)
    assert totals.sum() > 0, what
    rep = first_mismatch(got[0], oracle_out(layers, frames, ids, (sc.W, sc.H), (sc.W, sc.H), fmt, mode), recs, fmt)
    assert rep is None, f"{what}: {rep}"


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [GPU, CPU], ids=["gpu_mode", "cpu_mode"])
def test_gathers(mode):
    """a warp with more than 160 probe pixels shades them lane by lane; one with fewer gathers them cooperatively.
    Which gather a warp takes is not observed on the device: `need_map` / `warp_totals` model the kernel's rule
    (kernels.cu: a 4 x 2 thread block leaves the general path only when it lies wholly inside an interior bar of a
    fast layer; a warp with more than 5 * 32 such pixels shades per lane).  A change to that rule must change them."""
    kinds = set()
    for name in ("rotated_45", "border_color_4.0"):
        sc = SCENES[name]
        layers, frames, ids, probe = build(sc, "p")
        got, r = run([(OUTPUT_ID, layers, (sc.W, sc.H), (sc.W, sc.H), RGBA, None)], frames, ids, mode)
        recs = r.debug_composite_layers()
        t = check_path(sc, layers, probe, recs[probe], mode)
        kinds |= {"lane"} if (t > 160).any() else set()
        kinds |= {"coop"} if ((t > 0) & (t <= 160)).any() else set()
        rep = first_mismatch(got[0], oracle_out(layers, frames, ids, (sc.W, sc.H), (sc.W, sc.H), RGBA, mode), recs, RGBA)
        assert rep is None, f"{name} {mode}: {rep}"
    assert kinds == {"lane", "coop"}, kinds
