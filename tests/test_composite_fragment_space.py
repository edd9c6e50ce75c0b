"""The oracle's composite fragment stage against a float64 restatement of apply_layouts.wgsl, at every branch edge.

The oracle (`oracle/smelter_oracle.c`, `fragment` / `rounded_rect_sdf` / `quad_covers` / `blend_store`) and the kernel
(`smelter_b200/csrc/kernels.cu`, `shade`) are twins, and every other composite test compares one with the other.  Here
the oracle is held to `tests/fragment_ref.py`, which restates the reference shader from its source alone: the vertex
stage as its matrix chain, the rasteriser on float64 vertices snapped to 1/256 px (NC-7), `roundedRectSDF` and `fs_main`
branch for branch with WGSL's `smoothstep` and `mix`, NC-6's sampler, `convert_to_shader_color` and the premultiplied
blend through the target's view (NC-3 / NC-4 in GpuOptimized, NC-1 / NC-2 in CpuOptimized).

Each scene is one probe layer over a background texture holding every byte value in every channel, drawn 1:1, so the
blend meets every destination byte.  Both rendering modes are run.

Acceptance rule.  The oracle computes in f32, the restatement in float64, and the SDF ramps turn a coordinate rounding
into a value change of up to 1.5 per pixel, so a fixed tie window does not fit.  Instead each pixel gets its own bound:
  * eps = 4 ulp (f32) of the largest coordinate the layer meets.  The restatement is evaluated at the pixel centre and
    at the centre moved by -eps, 0, +eps in x and in y (nine points); every point's blended value, widened by
    VALUE_SLACK (2e-6, the f32 rounding of the colour products and the blend) and stored, gives a byte, and the
    oracle's byte must lie between the least and the greatest of them.  Where an axis of an unrotated layer is
    computed exactly in f32 (positions and half sizes multiples of 1/256 below 2^14), the SDFs' corner-radius selects
    keep the centre's side of that axis, so `dist.x == 0` / `dist.y == 0` are held to the reference's choice; where
    both axes are, `edge > bw / 2` is decided at the centre too, off the corner arcs (no square root, so f32 computes
    the edge exactly there).
  * A pixel is ambiguous when its NC-7 coverage changes with a vertex snap taken within eps, or when its branch
    (`edge > bw / 2`, `mask_alpha < 0.01`) differs between the nine points.  Coverage-ambiguous pixels may hold
    either the destination or the layer's bytes; branch-ambiguous ones the bytes of either branch.
  * Each scene asserts the number of covered, ambiguous, per-branch and ramp pixels (the ramp pixels have a smoothstep
    factor strictly between 0 and 1), and that the ambiguous ones stay under `max_ambiguous` of the covered ones, so
    the check can neither excuse everything nor stop reaching the edge it is there for.
"""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import fragment_ref as R

MODES = [R.GPU_OPTIMIZED, R.CPU_OPTIMIZED]
SCENES = {sc.name: sc for sc in R.SCENES}

# pixels per scene: covered, ambiguous, and per branch of fs_main (see the module docstring)
EXPECTED = {
    "corners": dict(covered=24000, ambiguous=0, plain=24000, ramp=350),
    "corners_pill": dict(covered=12000, ambiguous=0, plain=12000, ramp=318),
    "corners_over": dict(covered=12000, ambiguous=0, plain=12000, ramp=321),
    "corners_over_tall": dict(covered=12000, ambiguous=0, plain=12000, ramp=307),
    "corners_zero": dict(covered=13500, ambiguous=0, plain=13500, ramp=239),
    "border_color_0.999": dict(covered=45180, ambiguous=0, plain=45180, ramp=603),
    "border_texture_0.999": dict(covered=41040, ambiguous=0, plain=41040, ramp=643),
    "border_color_1.0": dict(covered=45180, ambiguous=0, inner=44463, outer=717, ramp=1437),
    "border_texture_1.0": dict(covered=41040, ambiguous=0, inner=40283, outer=757, ramp=1442),
    "border_color_1.5": dict(covered=45180, ambiguous=0, inner=44448, outer=732, ramp=1430),
    "border_texture_1.5": dict(covered=41040, ambiguous=0, inner=40267, outer=773, ramp=1435),
    "border_color_4.0": dict(covered=45180, ambiguous=0, inner=43367, outer=1813, ramp=1419),
    "border_texture_4.0": dict(covered=41040, ambiguous=0, inner=39307, outer=1733, ramp=1418),
    "border_color_10.0": dict(covered=45180, ambiguous=0, inner=40903, outer=4277, ramp=1374),
    "border_texture_10.0": dict(covered=41040, ambiguous=1, inner=36965, outer=4074, ramp=1380),
    "masks_1": dict(covered=75900, ambiguous=0, plain=75900, ramp=1569),
    "masks_2": dict(covered=75900, ambiguous=0, plain=75900, ramp=1542),
    "masks_20": dict(covered=75900, ambiguous=0, plain=75900, ramp=1086),
    "masks_21": dict(covered=75900, ambiguous=0, plain=75900, ramp=1086),
    "mask_cut_0": dict(covered=20000, ambiguous=0, masked_out=7000, inner=12288, outer=712, ramp=100),
    "mask_cut_1": dict(covered=20000, ambiguous=0, masked_out=7000, inner=12288, outer=712, ramp=100),
    "mask_cut_2": dict(covered=20000, ambiguous=0, masked_out=7000, inner=12288, outer=712, ramp=100),
    "mask_cut_3": dict(covered=20000, ambiguous=0, masked_out=6900, inner=12384, outer=716, ramp=100),
    "mask_cut_4": dict(covered=20000, ambiguous=0, masked_out=6900, inner=12384, outer=716, ramp=100),
    "mask_cut_5": dict(covered=20000, ambiguous=0, masked_out=6900, inner=12384, outer=716, ramp=100),
    "shadow_0.0": dict(covered=30800, ambiguous=0, shadow=30800, ramp=0),
    "shadow_0.25": dict(covered=30940, ambiguous=0, shadow=30940, ramp=258),
    "shadow_1.0": dict(covered=31524, ambiguous=0, shadow=31524, ramp=699),
    "shadow_7.5": dict(covered=36425, ambiguous=0, shadow=36425, ramp=4940),
    "shadow_40.0": dict(covered=66000, ambiguous=0, shadow=66000, ramp=27724),
    "shadow_rotated": dict(covered=26325, ambiguous=0, shadow=26325, ramp=4370),
    "rotated_0.001": dict(covered=17710, ambiguous=0, inner=16537, outer=1173, ramp=869),
    "rotated_30": dict(covered=17695, ambiguous=0, inner=16528, outer=1167, ramp=782),
    "rotated_45": dict(covered=17706, ambiguous=0, inner=16479, outer=1227, ramp=909),
    "rotated_90": dict(covered=17871, ambiguous=0, inner=16678, outer=1193, ramp=1022),
    "rotated_-90": dict(covered=17871, ambiguous=0, inner=16677, outer=1194, ramp=1018),
    "rotated_180": dict(covered=17710, ambiguous=0, inner=16541, outer=1169, ramp=874),
    "rotated_270": dict(covered=17871, ambiguous=0, inner=16677, outer=1194, ramp=1018),
    "rotated_360": dict(covered=17710, ambiguous=0, inner=16537, outer=1173, ramp=869),
    "rotated_texture_30": dict(covered=20499, ambiguous=1, inner=19947, outer=551, ramp=852),
    "rotated_90_top_left": dict(covered=6000, ambiguous=0, plain=6000, ramp=159),
    "texture_fractional_crop": dict(covered=68731, ambiguous=0, plain=68731, ramp=560),
    "texture_exact_texels": dict(covered=3072, ambiguous=0, plain=3072, ramp=28),
    "texture_missing_child": dict(covered=30000, ambiguous=9, inner=28203, outer=1788, ramp=1025),
    "precision_3000": dict(covered=12341, ambiguous=0, inner=11605, outer=736, ramp=1325),
}


def oracle_layout(p, child):
    crop = (0.0, 0.0, 0.0, 0.0) if p.crop is None else (p.crop[1], p.crop[0], p.crop[2], p.crop[3])
    return orc.make_layout(p.type, p.top, p.left, p.width, p.height, p.rotation, p.radius, p.color, p.border_color,
                           p.border, p.blur, child, crop, list(p.masks))


def background_layout(W, H):
    return orc.make_layout(R.TEXTURE, 0.0, 0.0, float(W), float(H), crop=(0.0, 0.0, float(W), float(H)), child_index=0)


def oracle_scene(sc, mode):
    bg = R.background(sc.W, sc.H)
    out = orc.apply_layouts(sc.W, sc.H, [background_layout(sc.W, sc.H), oracle_layout(sc.probe, 1)], [bg, sc.probe.tex],
                            mode=mode)
    return bg, out


def check(sc, mode, got, bg):
    """the acceptance rule: -> Allowed; raises on the first byte outside its bound"""
    a = R.evaluate(sc.probe, bg, mode)
    g = got.astype(np.int64)
    bad = (g < a.lo) | (g > a.hi)
    if bad.any():
        y, x, c = (int(v) for v in np.argwhere(bad)[0])
        raise AssertionError(f"{sc.name} mode {mode}: {int(bad.any(-1).sum())} pixels outside the bound; first ({x}, {y}) "
                             f"channel {c}: got {g[y, x, c]}, allowed [{a.lo[y, x, c]}, {a.hi[y, x, c]}], branch "
                             f"{R.BRANCH_NAMES.get(int(a.branch[y, x]), 'outside')}, eps {a.eps:.3g}")
    return a


@pytest.mark.parametrize("mode", MODES)
def test_background_is_the_destination(mode):
    """the background layer alone reproduces its texture byte for byte, so it is the destination every probe meets"""
    bg = R.background(384, 256)
    out = orc.apply_layouts(384, 256, [background_layout(384, 256)], [bg], mode=mode)
    assert np.array_equal(out, bg)
    for c in range(4):
        assert len(np.unique(bg[..., c])) == 256


@pytest.mark.parametrize("mode", MODES, ids=["gpu_mode", "cpu_mode"])
@pytest.mark.parametrize("name", list(SCENES))
def test_fragment_against_restatement(name, mode):
    sc = SCENES[name]
    bg, got = oracle_scene(sc, mode)
    a = check(sc, mode, got, bg)
    print(name, a.counts)
    assert a.counts["ambiguous"] <= sc.max_ambiguous * a.counts["covered"], a.counts
    assert a.counts == EXPECTED[name], a.counts


def test_catalogue_reaches_every_branch():
    """across the catalogue: every branch of fs_main, ramps, a masked-out pixel with mask_alpha strictly between 0 and
    .01, and more than 20 masks"""
    seen = set()
    for name, c in EXPECTED.items():
        seen |= {k for k in c if k not in ("covered", "ambiguous", "ramp") and c[k] > 0}
    assert seen == set(R.BRANCH_NAMES.values())
    p = SCENES["mask_cut_0"].probe
    geo = R.Geometry(p, 256, 128)
    _, br, ma = R.fragment(p, R.GPU_OPTIMIZED, geo, np.array([150.5]), np.array([50.5]))
    assert br[0] == R.MASKED_OUT and 0.0 < ma[0] < 0.01
    assert len(SCENES["masks_21"].probe.masks) > R.MAX_MASKS
