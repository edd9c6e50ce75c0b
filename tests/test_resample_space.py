"""The oracle's Lanczos3 resampler (`orc_resample`) against the float64 restatement in tests/resample_ref.py.

Every resample kernel is held byte for byte to `orc_resample`, which was written alongside them.  Here the oracle is
held to a restatement of resampler.rs, resample.wgsl and downsample.wgsl written from those sources alone, under the
acceptance rule of `resample_ref` (its docstring derives the tie window).  The plan is compared too: the oracle's
`plan_passes` and `predecimate_levels` against the restatement's.

- `CATALOGUE`: crops and sizes at every edge of the plan, the box pass and the kernel pass, each on several contents
  (random, smooth, 0 / 255 extremes in every channel, a translucent constant, alpha ramps).
  `test_catalogue_covers_every_edge` fails when an edge has no case.
- The scenes of the fused-kernel and generic-pass registries, on the oracle's own conversion of each case's input.
"""
from dataclasses import dataclass
from typing import Tuple

import numpy as np
import pytest

from oracle import oracle as orc
from tests import resample_ref as R

ALL = ("extreme", "random", "smooth", "constant", "alpha")


@dataclass
class Case:
    name: str
    src: Tuple[int, int]
    crop: Tuple[float, float, float, float]    # left, top, width, height
    dst: Tuple[int, int]
    contents: Tuple[str, ...] = ALL


def full(w, h):
    return (0.0, 0.0, float(w), float(h))


def _catalogue():
    C = []
    # plan outcomes: no pass; one pass carrying a positive, negative or past-the-edge perp_offset; separable
    C.append(Case("direct", (48, 36), (3.0, 2.0, 40.0, 30.0), (40, 30), ("extreme",)))
    for p in (5.0, -3.0, 30.0, 60.0, -40.0):
        C.append(Case(f"one-pass-h-perp{p:+.0f}", (64, 48), (1.5, p, 50.0, 30.0), (37, 30)))
        C.append(Case(f"one-pass-v-perp{p:+.0f}", (48, 64), (p, 2.5, 30.0, 44.0), (30, 27)))
    C.append(Case("two-pass-h-first", (96, 64), full(96, 64), (40, 30)))
    C.append(Case("two-pass-v-first", (160, 90), full(160, 90), (80, 44)))
    C.append(Case("two-pass-tie", (120, 90), full(120, 90), (80, 60)))
    # as_direct's 0.001, just inside and just outside, on offset and on length, on each axis
    for o, l in ((0.0009, 40.0), (0.0011, 40.0), (0.0, 40.0009), (0.0, 40.0011), (0.0, 39.9991), (0.0, 39.9989)):
        C.append(Case(f"near-direct-h-{o}-{l}", (48, 48), (o, 2.0, l, 30.0), (40, 30), ("extreme", "random")))
        C.append(Case(f"near-direct-v-{o}-{l}", (48, 48), (2.0, o, 30.0, l), (30, 40), ("extreme", "random")))
    # scales
    C.append(Case("scale-0.4", (40, 30), full(40, 30), (100, 75)))
    C.append(Case("scale-1-fractional", (48, 36), (0.25, 0.5, 40.0, 30.0), (40, 30)))
    C.append(Case("scale-1.5", (96, 60), full(96, 60), (64, 40)))
    C.append(Case("scale-2", (128, 80), full(128, 80), (64, 40)))
    C.append(Case("scale-2.5", (160, 100), full(160, 100), (64, 40)))
    C.append(Case("scale-3", (192, 120), full(192, 120), (64, 40)))
    C.append(Case("scale-3.5", (224, 140), full(224, 140), (64, 40)))
    C.append(Case("scale-4", (256, 160), full(256, 160), (64, 40)))
    C.append(Case("scale-4+eps", (208, 60), (0.0, 0.0, 200.01, 60.0), (50, 37)))
    C.append(Case("scale-8", (400, 60), full(400, 60), (50, 37)))
    C.append(Case("scale-8+eps", (410, 60), (0.0, 0.0, 400.02, 60.0), (50, 37)))
    C.append(Case("scale-16", (800, 60), full(800, 60), (50, 37)))
    C.append(Case("scale-20", (1000, 60), full(1000, 60), (50, 40)))
    # box levels, on sources that are not a multiple of the factor
    C.append(Case("box-1-0", (203, 40), full(203, 40), (40, 20)))
    C.append(Case("box-0-1", (40, 203), full(40, 203), (20, 40)))
    C.append(Case("box-1-1", (245, 183), full(245, 183), (40, 30)))
    C.append(Case("box-2-2", (402, 302), full(402, 302), (40, 30)))
    C.append(Case("box-3-0", (1003, 61), full(1003, 61), (50, 40)))
    # box levels with crop offsets: on_reduced_source divides them by the factor
    C.append(Case("box-1-1-offset", (245, 183), (10.5, -6.25, 220.0, 170.0), (40, 30)))
    C.append(Case("box-2-0-offset", (700, 60), (37.0, 3.5, 600.0, 50.0), (50, 37)))
    # crops hanging over each edge, negative offsets
    for c in ((-10.0, -7.0, 60.0, 40.0), (20.0, 15.0, 50.0, 40.0), (-30.5, 10.0, 40.0, 30.0), (10.0, -25.25, 30.0, 36.0),
              (-100.0, -100.0, 400.0, 300.0)):
        C.append(Case(f"over-edge-{c[0]}-{c[1]}", (48, 32), c, (30, 19)))
    # destinations of 1, sources of 1
    C.append(Case("dst-1-wide", (40, 30), full(40, 30), (1, 30)))
    C.append(Case("dst-1-high", (40, 30), full(40, 30), (40, 1)))
    C.append(Case("dst-1x1", (40, 30), full(40, 30), (1, 1)))
    C.append(Case("src-1xN", (1, 50), full(1, 50), (3, 20)))
    C.append(Case("src-Nx1", (50, 1), full(50, 1), (20, 3)))
    # crop offsets past 4096 on a 16 384-wide source
    for c, d in (((7000.3, 1.5, 300.0, 6.0), (200, 5)), ((4096.5, 0.0, 600.0, 12.0), (400, 12)),
                 ((12000.7, 0.25, 100.0, 10.0), (333, 13)), ((16000.0, 0.0, 800.0, 12.0), (200, 12)),
                 ((9000.5, 2.0, 64.0, 8.0), (64, 8))):
        C.append(Case(f"far-{c[0]}", (16384, 16), c, d, ("extreme", "random")))
    # full-size frames
    C.append(Case("1920x1080-960x540", (1920, 1080), full(1920, 1080), (960, 540), ("random",)))
    C.append(Case("3840x2160-crop-960x540", (3840, 2160), (1000.5, 600.25, 1920.0, 1080.0), (960, 540), ("extreme",)))
    return C


CATALOGUE = _catalogue()


def run(src8, crop, dst, what):
    """the oracle against the restatement, plan and bytes; -> Verdict (None when both find the crop direct)"""
    ev = R.evaluate(src8, crop, dst)
    got = orc.resample(src8, *crop, *dst)
    left, top, cw, ch = (float(np.float32(c)) for c in crop)
    assert orc.plan_passes(left, top, cw, ch, *dst) == (ev.plan.direct if ev else []), what
    if ev is None:
        assert got is None, what
        return None
    assert (orc.predecimate_levels(cw, dst[0]), orc.predecimate_levels(ch, dst[1])) == ev.plan.levels, what
    return R.assert_rule(got, ev, what)


@pytest.mark.parametrize("case", CATALOGUE, ids=lambda c: c.name)
def test_catalogue(case):
    for k, kind in enumerate(case.contents):
        src8 = R.content(kind, *case.src, seed=100 + k)
        vd = run(src8, case.crop, case.dst, f"{case.name} {kind}")
        if vd is None:
            continue
        print(f"{case.name} {kind}: {vd.line()}")
        if kind == "constant":
            got = orc.resample(src8, *case.crop, *case.dst)
            assert vd.off_rint == 0 and (got == src8[0, 0]).all(), case.name


def scale_bins(s):
    out = set()
    for lo, hi, name in ((0, 1, "<1"), (1, 2, "(1,2)"), (2, 3, "(2,3)"), (3, 4, "(3,4)"), (16, np.inf, ">16")):
        if lo < s < hi:
            out.add(name)
    for v in (1.0, 2.0, 3.0, 4.0, 8.0, 16.0):
        if s == v:
            out.add(str(v))
        if v in (4.0, 8.0) and v < s < v * 1.001:
            out.add(f"{v}+eps")
    return out


def test_catalogue_covers_every_edge():
    seen = set()
    for c in CATALOGUE:
        pl = R.plan(c.src, c.crop, c.dst)
        seen.add(pl.shape())
        maps = R.axis_mappings(c.crop, c.dst)
        for p in pl.passes:
            if len(pl.passes) == 1:
                span = c.src[1 - p.axis]
                edge = "neg" if p.perp_offset < 0 else "past" if p.perp_offset + p.dst[1 - p.axis] > span else \
                    "pos" if p.perp_offset > 0 else "0"
                seen.add(("perp", "hv"[p.axis], edge))
        for m in maps:
            if pl.passes and m.as_direct() is None:
                for b in scale_bins(m.scale):
                    seen.add(("scale", b))
                if m.scale == 1.0 and m.offset % 1:
                    seen.add(("scale", "1-fractional"))
            d = abs(np.float32(m.length) - np.float32(m.dst))
            o = abs(np.float32(m.offset) - np.float32(R.f32_round(m.offset)))
            for what, dist in (("length", d), ("offset", o)):
                if 0 < dist < 0.001 and max(d, o) == dist:
                    seen.add(("near-direct", "hv"[m.axis], what, "inside"))
                if 0.001 <= dist < 0.0012 and max(d, o) == dist:
                    seen.add(("near-direct", "hv"[m.axis], what, "outside"))
        if pl.passes:
            seen.add(("levels", pl.levels))
            if pl.box and (c.src[0] % pl.box[0][0] or c.src[1] % pl.box[0][1]):
                seen.add("box-not-a-multiple")
            if max(pl.levels) >= 3 and min(pl.levels) == 0:
                seen.add("level>=3-one-axis")
        left, top, w, h = c.crop
        for cond, e in ((left < 0, "left"), (top < 0, "top"), (left + w > c.src[0], "right"), (top + h > c.src[1], "bottom")):
            if cond:
                seen.add(("over", e))
        if c.dst[0] == 1:
            seen.add("dst-w-1")
        if c.dst[1] == 1:
            seen.add("dst-h-1")
        if c.src[0] == 1:
            seen.add("src-1xN")
        if c.src[1] == 1:
            seen.add("src-Nx1")
        if c.src[0] >= 16384 and left >= 4096 and "extreme" in c.contents:
            seen.add("far-extreme")
        for kind in c.contents:
            seen.add(("content", kind))
    need = {"none", "one-pass-h", "one-pass-v", "two-pass-h-first", "two-pass-v-first"}
    need |= {("perp", a, e) for a in "hv" for e in ("pos", "neg", "past")}
    need |= {("near-direct", a, w, s) for a in "hv" for w in ("length", "offset") for s in ("inside", "outside")}
    need |= {("scale", b) for b in ("<1", "1-fractional", "(1,2)", "2.0", "(2,3)", "3.0", "(3,4)", "4.0", "4.0+eps", "8.0",
                                    "8.0+eps", "16.0", ">16")}
    need |= {("levels", l) for l in ((0, 0), (1, 0), (0, 1), (1, 1), (2, 2))}
    need |= {"box-not-a-multiple", "level>=3-one-axis", "dst-w-1", "dst-h-1", "src-1xN", "src-Nx1", "far-extreme"}
    need |= {("over", e) for e in ("left", "top", "right", "bottom")}
    need |= {("content", k) for k in ALL}
    assert need <= seen, sorted(map(str, need - seen))
    # a tie of the two scales goes horizontal first
    assert R.plan((120, 90), full(120, 90), (80, 60)).passes[0].axis == R.HORIZONTAL


# ------------------------------------------------------------------------------------------------
# the GPU registries' scenes, on the CPU
# ------------------------------------------------------------------------------------------------
def fused_registry():
    from tests.test_gpu_fused_variants import REGISTRY
    return REGISTRY


def generic_registry():
    from tests.test_gpu_generic_resample import REGISTRY
    return REGISTRY


@pytest.mark.parametrize("entry", fused_registry(), ids=lambda e: e.name)
def test_fused_registry_scene(entry):
    """the oracle's resample of the oracle's conversion of the case's input (K1 / K2 / K3 are held to float64 by
    tests/test_color_conversion_space.py)"""
    from tests.parity import node_texture
    from tests.test_gpu_fused_variants import make_frame
    src8 = node_texture(make_frame(entry.fmt, "extreme", 17, *entry.src))
    vd = run(src8, entry.crop, entry.dst, entry.name)
    print(f"{entry.name}: {vd.line()}")


@pytest.mark.parametrize("case", generic_registry(), ids=lambda c: c.name)
def test_generic_registry_scene(case):
    from tests.parity import node_texture
    from tests.test_gpu_generic_resample import frames_of
    fr = frames_of(case, "extreme", 900)
    done = set()
    for j in case.jobs:
        key = (j.input_id, j.crop, j.dst)
        if key in done:
            continue
        done.add(key)
        vd = run(node_texture(fr[j.input_id]), j.crop, j.dst, f"{case.name} {j}")
        print(f"{case.name} {j.crop} -> {j.dst}: {vd.line()}")
