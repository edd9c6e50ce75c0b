"""The composite's interior proof against the oracle, without a GPU.

Inside a layer's two interior bars the composite replaces the fragment shader with a fast class (constant bytes, a blend
table, the bare sample or texel), and outside them its general path takes a per-pixel shortcut past the shader.  Both are
only right where the oracle's fragment is the bare colour or sample: every alpha factor exactly 1, no border colour.
smr_debug_interior reports the bars and the shortcut the library computes for one layout (the very function the kernel
runs); oracle.bare_map reports where the oracle's fragment is bare.  Seeded random layouts -- radii, border widths, masks
and positions at their edges, NaN and infinities included -- must never claim a pixel the oracle does not paint bare.
"""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import oracle as orc
from smelter_b200 import _ffi as F

NAN, INF = float("nan"), float("inf")
W, H = 200, 112

RADII = [0.0, 0.5, 3.0, 10.0, 37.25, -1.0, -10.0, -1e3, 1e6, -1e6, 1e8, -1e8, -1e9, 1e30, -1e30, INF, -INF, NAN]
BORDERS = [0.0, 0.5, 0.999, 1.0, 1.0001, 2.5, 7.0, NAN, INF, -INF]


def interior(layout, w=W, h=H):
    """(box[12], shortcut (h, w) bool) of smr_debug_interior"""
    box = (C.c_int32 * 12)()
    sc = np.zeros((h, w), np.uint8)
    assert F.lib().smr_debug_interior(C.byref(layout), w, h, C.byref(box), sc.ctypes.data_as(C.c_void_p)) == 0
    return list(box), sc.astype(bool)


def bare(layout, w=W, h=H, mode=orc.MODE_GPU_OPTIMIZED):
    return orc.bare_map(w, h, orc.Layout.from_buffer_copy(bytes(layout)), mode)


def make(type=1, left=0.0, top=0.0, width=W, height=H, radius=(0, 0, 0, 0), border_width=0.0, masks=(), rotation=0.0,
         blur=0.0):
    """masks: [(radius4, top, left, width, height)]"""
    L = F.RenderLayout()
    L.type = type
    L.left, L.top, L.width, L.height = left, top, width, height
    L.rotation_degrees = rotation
    L.border_radius[:] = list(radius)
    L.color = F.Rgba(200, 30, 60, 255)
    L.border_color = F.Rgba(10, 220, 40, 255)
    L.border_width, L.blur_radius = border_width, blur
    L.crop_width, L.crop_height = width, height
    L.masks_len = len(masks)
    for i, (r, t, l, w, h) in enumerate(masks):
        L.masks[i].radius[:] = list(r)
        L.masks[i].top, L.masks[i].left, L.masks[i].width, L.masks[i].height = t, l, w, h
    return L


def bars_of(box):
    return [box[4:8], box[8:12]]


def describe(L):
    masks = [(tuple(L.masks[i].radius), L.masks[i].top, L.masks[i].left, L.masks[i].width, L.masks[i].height)
             for i in range(L.masks_len)]
    return (f"type={L.type} left={L.left!r} top={L.top!r} w={L.width!r} h={L.height!r} rot={L.rotation_degrees!r} "
            f"radius={tuple(L.border_radius)} border={L.border_width!r} masks={masks}")


def check(L):
    """asserts the bars and the shortcut lie inside the oracle's bare pixels; returns (box, shortcut, bare)"""
    box, sc = interior(L)
    b = bare(L)
    for x0, x1, y0, y1 in bars_of(box):
        if x0 < x1 and y0 < y1:
            bad = np.argwhere(~b[y0:y1, x0:x1])
            assert len(bad) == 0, (f"bar [{x0},{x1})x[{y0},{y1}) claims {len(bad)} non-bare pixels, first (x, y) = "
                                   f"{(x0 + bad[0][1], y0 + bad[0][0])}: {describe(L)}")
    bad = np.argwhere(sc & ~b)
    assert len(bad) == 0, f"shortcut claims {len(bad)} non-bare pixels, first (x, y) = {tuple(bad[0][::-1])}: {describe(L)}"
    return box, sc, b


def pick(rng, values, p_special):
    return values[rng.integers(len(values))] if rng.random() < p_special else float(rng.choice([0.0, 2.0, 5.5, 12.0]))


def random_layout(rng):
    kind = rng.random()
    big = rng.random() < 0.1
    if big:   # positions near the 1e7 cut-off; the layer still reaches into the frame
        left = -1e7 + float(rng.uniform(0, 4096))
        top = -1e7 + float(rng.uniform(0, 4096)) if rng.random() < 0.5 else float(rng.uniform(-8, 8))
        width = 1e7 - float(rng.uniform(-4096, 0)) if left < -1e6 else float(rng.uniform(20, 400))
        width = min(width, 1e7)
        height = 1e7 if top < -1e6 else float(rng.uniform(20, 200))
    else:
        left, top = float(rng.uniform(-40, W - 20)), float(rng.uniform(-30, H - 10))
        if rng.random() < 0.5:
            left, top = round(left), round(top)
        width, height = float(rng.uniform(4, 260)), float(rng.uniform(4, 150))
    special = rng.random() < 0.5   # else ordinary radii and border widths
    radius = [pick(rng, RADII, 0.4 if special else 0.0) for _ in range(4)]
    border = BORDERS[rng.integers(len(BORDERS) if special else 7)] if rng.random() < 0.6 else float(rng.uniform(0, 9))
    masks = []
    for _ in range(int(rng.integers(0, 21)) if rng.random() < 0.6 else 0):
        ml, mt = float(rng.uniform(left - 20, left + width * 0.5)), float(rng.uniform(top - 20, top + height * 0.5))
        mw, mh = float(rng.uniform(10, width + 60)), float(rng.uniform(10, height + 60))
        if big and rng.random() < 0.5:
            ml, mw = left - float(rng.uniform(0, 10)), width + 20.0
        mr = [pick(rng, RADII, 0.2 if special else 0.0) for _ in range(4)]
        if special and rng.random() < 0.03:   # a non-finite mask field
            field = int(rng.integers(4))
            vals = [mt, ml, mw, mh]
            vals[field] = [NAN, INF, -INF][rng.integers(3)]
            mt, ml, mw, mh = vals
        masks.append((mr, mt, ml, mw, mh))
    rotation = 0.0
    if rng.random() < 0.05:
        rotation = float(rng.choice([90.0, 45.0, 0.01, 180.0]))
    type_ = 1 if kind < 0.5 else (0 if kind < 0.95 else 2)
    return make(type_, left, top, width, height, radius, border, masks, rotation, blur=4.0 if type_ == 2 else 0.0)


def test_random_layouts_claim_only_bare_pixels():
    rng = np.random.default_rng(20261015)
    n, with_bars, with_special = 4000, 0, 0
    for _ in range(n):
        L = random_layout(rng)
        box, sc, b = check(L)
        if any(x0 < x1 and y0 < y1 for x0, x1, y0, y1 in bars_of(box)):
            with_bars += 1
        if not all(math.isfinite(v) and abs(v) < 1e5 for v in list(L.border_radius) + [L.border_width]):
            with_special += 1
    # the property is not vacuous: many layouts keep an interior, many carry the values the proof must refuse
    assert with_bars > n // 5, with_bars
    assert with_special > n // 4, with_special


@pytest.mark.parametrize("radius, border, expect_bars", [
    ((-1e8, 0, 0, 0), 0.0, True),
    ((-1e9, 0, 0, 0), 0.0, False),
    ((-INF, 0, 0, 0), 0.0, False),
    ((NAN, 0, 0, 0), 0.0, False),
    ((0, 0, NAN, 0), 0.0, False),
    ((0, 0, 0, 0), NAN, False),
    ((0, 0, 0, 0), INF, False),
    ((0, 0, 0, 0), -INF, False),
    ((1e30, 0, 0, 0), 0.0, False),
    ((0, 0, 0, 0), 0.999, True),
    ((0, 0, 0, 0), 1.0, True),
    ((0, 0, 0, 0), 1.001, True),
])
def test_values_from_outside_the_program(radius, border, expect_bars):
    """The 200 x 100 opaque colour layer of the bug report: a huge negative, infinite or NaN radius and a NaN border width
    once left pixels inside the bars that the oracle paints transparent, in the border colour or blended."""
    for type_ in (1, 0):
        L = make(type_, 0.0, 0.0, 200.0, 100.0, radius, border)
        box, sc, b = check(L)
        has = any(x0 < x1 and y0 < y1 for x0, x1, y0, y1 in bars_of(box))
        if not expect_bars:
            assert not has and not sc.any(), describe(L)


def test_non_finite_mask_field_gives_no_interior():
    for field in range(4):
        for v in (NAN, INF, -INF):
            m = [0.0, 0.0, 200.0, 100.0]
            m[field] = v
            L = make(1, 0.0, 0.0, 200.0, 100.0, masks=[((0, 0, 0, 0), *m)])
            box, sc, b = check(L)
            assert box[4:] == [0] * 8 and not sc.any(), describe(L)
    L = make(1, 0.0, 0.0, 200.0, 100.0, masks=[((0, NAN, 0, 0), 0.0, 0.0, 200.0, 100.0)])
    box, sc, b = check(L)
    assert box[4:] == [0] * 8 and not sc.any()


def test_ordinary_layouts_keep_their_interior():
    """The fix must not empty the bars of ordinary layers: a 300 x 200 layer with radius 10 and two masks keeps most of
    its pixels in the bars, and the shortcut finds nearly every bare pixel."""
    w, h = 320, 224
    masks = [((4, 4, 4, 4), 10.0, 5.0, 290.0, 190.0), ((0, 0, 0, 0), -5.0, 0.0, 320.0, 230.0)]
    for type_ in (1, 0):
        for border in (0.0, 2.0):
            L = make(type_, 6.0, 12.0, 300.0, 200.0, (10, 10, 10, 10), border, masks)
            box, sc = interior(L, w, h)
            b = bare(L, w, h)
            in_bars = np.zeros((h, w), bool)
            for x0, x1, y0, y1 in bars_of(box):
                in_bars[y0:y1, x0:x1] = True
            assert not (in_bars & ~b).any() and not (sc & ~b).any()
            assert in_bars.sum() >= 0.8 * b.sum(), (in_bars.sum(), b.sum())
            assert sc.sum() >= 0.9 * b.sum(), (sc.sum(), b.sum())


def test_interior_rule_is_unchanged_for_integral_layouts():
    """Bars of ordinary layers follow the same edges as before: 2 px margin, a corner square of r + 2, the border's
    width + 1 on top (these bars decide fast classes and direct tiles, which must not move)."""
    L = make(1, 10.0, 20.0, 100.0, 60.0, (8, 8, 8, 8))
    box, _ = interior(L)
    assert box == [10, 110, 20, 80, 20, 100, 22, 78, 12, 108, 30, 70]
    L = make(0, 10.0, 20.0, 100.0, 60.0, (0, 0, 0, 0), 3.0)
    box, _ = interior(L)
    assert box == [10, 110, 20, 80, 16, 104, 26, 74, 16, 104, 26, 74]


def test_rotated_and_box_shadow_layers_have_no_interior():
    for L in (make(1, 10.0, 10.0, 100.0, 60.0, rotation=0.01), make(2, 10.0, 10.0, 100.0, 60.0, blur=3.0)):
        box, sc = interior(L)
        assert box[:4] != [0, 0, 0, 0] and box[4:] == [0] * 8 and not sc.any()
