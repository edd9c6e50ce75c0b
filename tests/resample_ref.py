"""Float64 restatement of the Lanczos3 resampler, written from the reference's sources alone.

The reference resamples a child whose crop is not a whole-texel 1:1 copy (`ResampledChild::render`,
smelter-render/src/transformations/layout/resampler.rs:305-378):
  * `axis_mappings` (:381-396) gives each axis a mapping: crop offset, crop length, destination length, and
    `scale = crop_len / dst_len` in f32 (:51-53).
  * `predecimate_levels` (:56-58) is `ceil(log2(scale / KERNEL_BUDGET))`, floored at 0 (`f32::max(NaN, 0) = 0`), cast
    saturating to u32 and capped at MAX_PREDECIMATE_LEVELS (:19, :23).  Levels other than (0, 0) run one box pass
    (downsample.wgsl:28-41) of 2^lx x 2^ly texels per output texel into a div_ceil-sized Rgba16Float texture, source
    coordinates clamped to the texture; `on_reduced_source` (:60-67) divides the offset and the length by the factor.
  * `plan_passes` (:123-145) on the reduced mappings: an axis whose length is within 0.001 of its destination and whose
    offset is within 0.001 of `f32::round(offset)` (`as_direct`, :71-75, `is_same_px`, :398-400) gets no pass of its
    own; its rounded offset rides on the other axis's pass as `perp_offset`.  Two such axes need no resampler at all.
    Otherwise both axes get a pass, the larger scale first (a tie goes horizontal first).
  * Each kernel pass is resample.wgsl's `fs_main` (:31-88): `center = offset + (o + 0.5) scale - 0.5` (:46),
    `first = ceil(center - support)` and `taps = ceil(2 support) + 1` with `support = 3 max(scale, 1)` (:43-48), the
    source index clamped to [0, dim - 1] (:72) and the perpendicular coordinate `p + perp_offset` clamped too (:36-40),
    Lanczos3 weights `sinc(x) sinc(x / 3)` at `x = (first + t - center) / max(scale, 1)`: 1 below 1e-5, 0 from 3 on
    (:64-71), and the sum divided by the weight sum (:87).  A pass before the last renders into Rgba16Float
    (`pipeline_f16`, :221); the last renders into the child's texture through `default_view_format` (wgpu/ctx.rs:52-58),
    which in the only mode with a resampler (layout_renderer.rs:22-27: GpuOptimized) is Rgba8UnormSrgb.
  * The source is a node texture read through the same sRGB view: colour channels decoded with the sRGB EOTF, alpha
    as b / 255.  The last pass stores colour as 255 oetf(clamp01(v)) and alpha as 255 clamp01(v), each rounded.

Here every one of those steps is float64 and vectorised; the weights are the exact sinc product (the shader's f32
rotation recurrence is bounded separately, by `test_oracle_weights_are_lanczos3`), f16 storage is numpy's
round-to-nearest-even conversion from float64, and nothing is shared with `oracle/` or the kernels.  `evaluate` returns
each final byte's value before rounding, with the plan.

Acceptance rule (`judge`), used by tests/test_resample_space.py (the oracle) and tests/test_gpu_resample_space.py (the
kernels).  A byte must equal rint(v); it may be the other neighbour of a rounding tie, and then differs by exactly 1,
only where v lies within T of that tie.  T = T_ARITH + T_geom.

T_ARITH = 1/32 LSB covers the contract's f32 arithmetic against float64 on the final value:
  * weights: each f32 weight is within 2^-19 / min(|x|, 1) of the sinc product (`test_oracle_weights_are_lanczos3`),
    a few 1e-6 of the linear value once normalised;
  * the f32 accumulation of at most 25 products and the division by the weight sum: a few f32 ulps, below 1e-6.
  The largest slope from a linear value to an output byte is the sRGB OETF's linear segment, 255 x 12.92 = 3295 LSB
  per unit, so together they stay under 0.02 LSB; 1/32 keeps a margin of 1.5.
An f16 intermediate is different: where its f32 value and its float64 value straddle an f16 rounding tie, the two
store neighbouring f16 values, one f16 ulp apart (2^-11 of the value), and the next pass carries that step to the
byte with the texel's weight -- up to 0.055 LSB for a bright texel of weight 1, more for a dark output.  A fixed
window would have to be twice as wide everywhere for the few bytes this touches, so the step is accounted where it
happens instead: every intermediate texel whose float64 value lies within F16_TIE = 2^-16 of an f16 tie may hold
either neighbour, and the pass after it widens each output by sum(|weight| x that step).  2^-16 is 2.5 times the
largest difference found between the oracle's f32 intermediate and the float64 one (5.9e-6, on 0 / 255 content at
scale 1.99, where thirteen weights' f32 errors add up on texels of 0 and 1).

T_geom covers the shader computing `center` in f32: at most a few ulps of the largest source coordinate the pass
meets, a phase error that 0 / 255 content turns into up to half an LSB of a bright byte at coordinates near 16 384,
and several LSB of a dark one (the OETF is steepest there).  Each pass's centres are also evaluated moved by -eps and
+eps, eps = EPS_ULPS f32 ulps of that coordinate (3 evaluations for one pass, 9 for two), and a byte may lie anywhere
in the hull of those values, widened by the f16 band and by T_ARITH.  A texel of the intermediate whose shifted
values round to different f16 values joins the band with that difference, since the contract's run may round it
either way whatever its neighbours do.  The extra evaluations are skipped when a first-order bound on their effect,
eps x max |dv/dcenter|, stays under T_ARITH: then T_geom is that bound itself.

Each scene must also keep the share of bytes that T_ARITH alone excuses -- bytes that differ from rint(v) although
the whole range [vmin, vmax] rounds to rint(v), v not at an exact tie -- at or below MAX_OFF_RINT_SHARE, so that the
tie window cannot silently excuse a kernel that is wrong everywhere.  (Where the range itself straddles a tie, the
centre's f32 phase decides the byte, and far from the origin on 0 / 255 content that is a few percent of the bytes.)

On the oracle's 354 scenes (16.4 million bytes) 1 878 bytes differ from rint(v), none of them by T_ARITH alone; the
largest share off rint outside the scenes far from the origin is 1.4e-3.  The kernels' 189 scenes on an H100 (14.1
million bytes) give 792, none by T_ARITH alone, at most 8.0e-4 of a scene.
"""
import math
from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import numpy as np
from scipy import sparse

f32 = np.float32

KERNEL_BUDGET = 4.0              # resampler.rs:19
MAX_PREDECIMATE_LEVELS = 16      # resampler.rs:23
SAME_PX = f32(0.001)             # resampler.rs:399
HORIZONTAL, VERTICAL = 0, 1      # resampler.rs:36-39

T_ARITH = 1.0 / 32               # LSB; derivation in the module docstring
EPS_ULPS = 2                     # centre shift, in f32 ulps of the pass's largest source coordinate
MAX_OFF_RINT_SHARE = 1e-3        # per scene
SRGB_SLOPE = 255.0 * 12.92       # the largest d(byte) / d(linear) of the final store
F16_TIE = 2.0 ** -16             # an f16 intermediate this close to an f16 tie may round either way (docstring)
EXACT_TIE = 1e-5                 # LSB: 0 / 255 content averaged evenly lands on ties, give or take f16 storage


# ------------------------------------------------------------------------------------------------
# the host side: mappings and the plan (resampler.rs)
# ------------------------------------------------------------------------------------------------
def f32_round(x):
    """f32::round: half away from zero"""
    x = float(x)
    return math.copysign(math.floor(abs(x) + 0.5), x)


def is_same_px(a, b):
    return bool(abs(f32(a) - f32(b)) < SAME_PX)


@dataclass(frozen=True)
class AxisMapping:
    axis: int
    offset: float      # f32 values
    length: float
    dst: int

    @property
    def scale(self):
        return float(f32(self.length) / f32(self.dst))

    def predecimate_levels(self):
        q = f32(self.scale) / f32(KERNEL_BUDGET)
        with np.errstate(all="ignore"):
            lg = f32(math.log2(q)) if q > 0 else (f32(-math.inf) if q == 0 else f32(math.nan))  # f32::log2
        l = float(np.ceil(lg))
        l = l if l > 0.0 else 0.0               # f32::max(NaN, 0) == 0
        lv = 0xFFFFFFFF if l >= 4294967296.0 else int(l)   # saturating `as u32`
        return min(lv, MAX_PREDECIMATE_LEVELS)

    def on_reduced_source(self, levels):
        fac = f32(1 << levels)
        return AxisMapping(self.axis, float(f32(self.offset) / fac), float(f32(self.length) / fac), self.dst)

    def as_direct(self):
        r = f32_round(self.offset)
        if is_same_px(self.length, float(self.dst)) and is_same_px(self.offset, r):
            return int(r)
        return None


def axis_mappings(crop, dst):
    """crop = (left, top, width, height), as f32"""
    left, top, w, h = (float(f32(c)) for c in crop)
    return AxisMapping(HORIZONTAL, left, w, dst[0]), AxisMapping(VERTICAL, top, h, dst[1])


def plan_passes(mappings):
    """-> None (direct) or [(mapping, perp_offset), ...] in execution order"""
    hm, vm = mappings
    hd, vd = hm.as_direct(), vm.as_direct()
    if hd is not None and vd is not None:
        return None
    if vd is not None:
        return [(hm, vd)]
    if hd is not None:
        return [(vm, hd)]
    if f32(vm.scale) > f32(hm.scale):
        return [(vm, 0), (hm, 0)]
    return [(hm, 0), (vm, 0)]


def taps_of(scale):
    """resample.wgsl:43-48, in f32 as the shader computes it (and as the host sizes its tables)"""
    k = max(f32(scale), f32(1.0))
    return int(np.ceil(f32(2.0) * (f32(3.0) * k))) + 1


@dataclass
class Pass:
    stage: str                 # "first" / "last"
    axis: int
    scale: float
    offset: float
    perp_offset: int
    taps: int
    src: Tuple[int, int]
    dst: Tuple[int, int]

    @property
    def dst_f16(self):
        return int(self.stage != "last")


@dataclass
class Plan:
    levels: Tuple[int, int]
    direct: Optional[List[Tuple[int, int]]]      # plan_passes on the crop itself: [(axis, perp_offset)], [] when direct
    box: Optional[Tuple[Tuple[int, int], Tuple[int, int], Tuple[int, int]]]   # (factor, src, dst) of the box pass
    passes: List[Pass] = field(default_factory=list)

    def stages(self):
        """the stages in debug_resample_stages' fields (without the source kind)"""
        out = []
        if self.box:
            (fx, fy), src, dst = self.box
            out.append(dict(stage="box", axis=-1, box_fx=fx, box_fy=fy, taps=0, perp_offset=0, src=src, dst=dst, dst_f16=1))
        for p in self.passes:
            out.append(dict(stage=p.stage, axis=p.axis, box_fx=1, box_fy=1, taps=p.taps, perp_offset=p.perp_offset,
                            src=p.src, dst=p.dst, dst_f16=p.dst_f16))
        return out

    def shape(self):
        if not self.passes:
            return "none"
        if len(self.passes) == 1:
            return f"one-pass-{'hv'[self.passes[0].axis]}"
        return f"two-pass-{'hv'[self.passes[0].axis]}-first"


def plan(src_size, crop, dst):
    """ResampledChild::render's plan for a src_size = (w, h) texture; passes == [] when the crop is direct"""
    maps = axis_mappings(crop, dst)
    top = plan_passes(maps)
    levels = tuple(m.predecimate_levels() for m in maps)
    pl = Plan(levels, [] if top is None else [(m.axis, p) for m, p in top], None)
    if top is None:
        return pl
    cur = tuple(src_size)
    if levels != (0, 0):
        fx, fy = 1 << levels[0], 1 << levels[1]
        red = (-(-cur[0] // fx), -(-cur[1] // fy))       # div_ceil
        pl.box = ((fx, fy), cur, red)
        cur = red
    res = plan_passes(tuple(m.on_reduced_source(l) for m, l in zip(maps, levels)))
    assert res is not None, "box reduction leaves a residual scale"   # resampler.rs:343-344
    for i, (m, perp) in enumerate(res):
        last = i == len(res) - 1
        d = tuple(dst) if last else ((dst[0], cur[1]) if m.axis == HORIZONTAL else (cur[0], dst[1]))   # output_size
        pl.passes.append(Pass("last" if last else "first", m.axis, m.scale, m.offset, perp, taps_of(m.scale), cur, d))
        cur = d
    return pl


# ------------------------------------------------------------------------------------------------
# the device side: load, box, kernel pass, store
# ------------------------------------------------------------------------------------------------
def srgb_eotf(c):
    c = np.asarray(c, np.float64)
    return np.where(c <= 0.04045, c / 12.92, ((c + 0.055) / 1.055) ** 2.4)


def srgb_oetf(y):
    """the inverse of srgb_eotf"""
    y = np.asarray(y, np.float64)
    return np.where(y <= 0.04045 / 12.92, y * 12.92, 1.055 * np.power(np.maximum(y, 0.0), 1.0 / 2.4) - 0.055)


DECODE = srgb_eotf(np.arange(256) / 255.0)


def load(src8):
    """an RGBA8 node texture through the sRGB view: (h, w, 4) float64 linear colour, unorm alpha"""
    src8 = np.asarray(src8, np.uint8)
    out = np.empty(src8.shape, np.float64)
    out[..., :3] = DECODE[src8[..., :3]]
    out[..., 3] = src8[..., 3] / 255.0
    return out


def to_f16(v):
    """Rgba16Float store: round to nearest even"""
    return np.asarray(v, np.float64).astype(np.float16).astype(np.float64)


def box_pass(lin, fx, fy):
    """downsample.wgsl:28-41: the mean of fx x fy texels from (x fx, y fy), coordinates clamped to the texture (only
    the upper clamp can bind); the mean in float64, before storage"""
    h, w = lin.shape[:2]
    rw, rh = -(-w // fx), -(-h // fy)
    a = np.pad(lin, ((0, 0), (0, rw * fx - w), (0, 0)), mode="edge").reshape(h, rw, fx, 4).sum(axis=2)
    a = np.pad(a, ((0, rh * fy - h), (0, 0), (0, 0)), mode="edge").reshape(rh, fy, rw, 4).sum(axis=1)
    return a / float(fx * fy)


def lanczos3(x):
    ax = np.abs(x)
    return np.where(ax < 1e-5, 1.0, np.where(ax < 3.0, np.sinc(x) * np.sinc(x / 3.0), 0.0))


def lanczos3_slope(x):
    """d/dx of sinc(x) sinc(x / 3) (0 at the ends of the support, where the shader's weight jumps to 0 by a value of
    the order of 1e-16)"""
    def dsinc(u):
        with np.errstate(all="ignore"):
            d = (np.cos(np.pi * u) - np.sinc(u)) / u
        return np.where(np.abs(u) < 1e-8, 0.0, d)
    return np.where(np.abs(x) < 3.0, dsinc(x) * np.sinc(x / 3.0) + np.sinc(x) * dsinc(x / 3.0) / 3.0, 0.0)


def pass_weights(p, delta=0.0):
    """(first tap index (n_out, taps), normalised weights (n_out, taps), sum over taps of |d weight / d center|) of
    every output coordinate of pass p, the centres moved by delta"""
    n_out = p.dst[p.axis]
    k = max(p.scale, 1.0)
    center = p.offset + (np.arange(n_out) + 0.5) * p.scale - 0.5 + delta
    first = np.ceil(center - 3.0 * k)
    pos = first[:, None] + np.arange(p.taps)[None, :]
    x = (pos - center[:, None]) / k
    w = lanczos3(x)
    ws = w.sum(axis=1, keepdims=True)
    dw = -lanczos3_slope(x) / k
    slope = (np.abs(dw).sum(1) + np.abs(w).sum(1) * np.abs(dw.sum(1)) / np.abs(ws[:, 0])) / np.abs(ws[:, 0])
    return pos.astype(np.int64), w / ws, slope


def pass_matrix(p, n_src, delta=0.0):
    """pass p's normalised weights as a sparse (n_out, n_src) matrix, source indices clamped (a clamped texel's weights
    summed)"""
    pos, w, _ = pass_weights(p, delta)
    n_out = pos.shape[0]
    rows = np.repeat(np.arange(n_out), pos.shape[1])
    return sparse.csr_matrix((w.ravel(), (rows, np.clip(pos, 0, n_src - 1).ravel())), shape=(n_out, n_src))


def kernel_pass(src, p, delta=0.0, m=None):
    """one resample.wgsl pass over src (h, w, 4) float64: -> (dst_h, dst_w, 4) float64, before storage"""
    h, wd = src.shape[:2]
    tw, th = p.dst
    if p.axis == HORIZONTAL:
        m = pass_matrix(p, wd, delta) if m is None else m
        rows = src[np.clip(np.arange(th) + p.perp_offset, 0, h - 1)]
        return (m @ rows.transpose(1, 0, 2).reshape(wd, th * 4)).reshape(tw, th, 4).transpose(1, 0, 2)
    m = pass_matrix(p, h, delta) if m is None else m
    cols = src[:, np.clip(np.arange(tw) + p.perp_offset, 0, wd - 1)]
    return (m @ cols.reshape(h, tw * 4)).reshape(th, tw, 4)


def store(v):
    """the last pass through the sRGB view: each byte's value before rounding"""
    v = np.clip(v, 0.0, 1.0)
    out = np.empty_like(v)
    out[..., :3] = 255.0 * srgb_oetf(v[..., :3])
    out[..., 3] = 255.0 * v[..., 3]
    return out


def ulp32(x):
    x = max(abs(float(x)), 2.0 ** -126)
    return 2.0 ** (math.floor(math.log2(x)) - 23)


def pass_eps(p):
    """EPS_ULPS f32 ulps of the largest source coordinate the pass's centre computation meets"""
    length = p.scale * p.dst[p.axis]
    return EPS_ULPS * ulp32(max(abs(p.offset), abs(p.offset + length), length, 1.0))


def f16_band(y):
    """the distance to the other f16 neighbour where y (float64, before storage) lies within F16_TIE of an f16 rounding
    tie, else 0: how far the stored value may move when the contract's f32 value rounds the other way"""
    y16 = np.asarray(y, np.float64).astype(np.float16)
    up = np.nextafter(y16, np.float16(np.inf)).astype(np.float64)
    dn = np.nextafter(y16, np.float16(-np.inf)).astype(np.float64)
    c = y16.astype(np.float64)
    near_up = np.abs(y - (c + up) / 2.0) < F16_TIE
    near_dn = np.abs(y - (c + dn) / 2.0) < F16_TIE
    return np.where(near_up, up - c, 0.0) + np.where(near_dn, c - dn, 0.0)


@dataclass
class Evaluation:
    plan: Plan
    v: np.ndarray        # (dst_h, dst_w, 4) float64: each byte's value before rounding
    vmin: np.ndarray     # the bytes' range: the centre-shifted evaluations and the f16 band (or v -+ t_geom)
    vmax: np.ndarray
    t_geom: float        # the first-order bound of the centre shift's effect, LSB
    hull: bool           # whether the shifted evaluations were run


def evaluate(src8, crop, dst, shifts=True):
    """the restatement of ResampledChild::render on an RGBA8 node texture: None when the crop is direct"""
    pl = plan((src8.shape[1], src8.shape[0]), crop, dst)
    if not pl.passes:
        return None
    lin = load(src8)
    band = np.zeros_like(lin)
    if pl.box:
        (fx, fy), _, _ = pl.box
        red = box_pass(lin, fx, fy)
        lin, band = to_f16(red), f16_band(red)
    ps = pl.passes
    eps = [pass_eps(p) for p in ps]
    mats = [pass_matrix(p, p.src[p.axis]) for p in ps]
    # first-order bound of the centre shifts: a pass moves its output by eps sum|dw / dcenter| (max - min) / 2 of its
    # source; a later pass carries that through its weights (at most sum |w|)
    mid = None if len(ps) == 1 else kernel_pass(lin, ps[0], m=mats[0])
    srcs = [lin] if mid is None else [lin, to_f16(mid)]
    g = 0.0
    for i, (p, s) in enumerate(zip(ps, srcs)):
        gi = eps[i] * float(pass_weights(p)[2].max()) * float(s.max() - s.min()) / 2.0
        for q in ps[i + 1:]:
            gi *= float(np.abs(pass_weights(q)[1]).sum(1).max())
        g += gi
    t_geom = 2.0 * SRGB_SLOPE * g        # x 2: the bound is first order
    hull = shifts and t_geom >= T_ARITH
    d_first = (-eps[0], 0.0, eps[0]) if hull and mid is not None else (0.0,)
    d_last = (-eps[-1], 0.0, eps[-1]) if hull else (0.0,)
    if mid is None:
        sources = {0.0: lin}
    else:
        # the f16 band of the intermediate over every shift of its centres; the box pass's band carried through
        mids = {d: mid if d == 0.0 else kernel_pass(lin, ps[0], d) for d in d_first}
        ylo, yhi = np.minimum.reduce(list(mids.values())), np.maximum.reduce(list(mids.values()))
        # a texel whose shifted values round to different f16 values may hold either in the contract's run, whichever
        # its neighbours hold: the hull alone moves all texels together
        band = kernel_pass(band, ps[0], m=abs(mats[0])) + np.maximum(f16_band(ylo), f16_band(yhi)) + \
            (to_f16(yhi) - to_f16(ylo))
        sources = {d: to_f16(m) for d, m in mids.items()}
    band = kernel_pass(band, ps[-1], m=abs(mats[-1]))
    lin_out = kernel_pass(sources[0.0], ps[-1], m=mats[-1])
    lo, hi = lin_out.copy(), lin_out.copy()
    for d1, src in sources.items():
        for d2 in d_last:
            if d1 == 0.0 and d2 == 0.0:
                continue
            o = kernel_pass(src, ps[-1], d2)
            np.minimum(lo, o, out=lo)
            np.maximum(hi, o, out=hi)
    v = store(lin_out)
    if hull:
        return Evaluation(pl, v, store(lo - band), store(hi + band), t_geom, True)
    return Evaluation(pl, v, store(lin_out - band) - t_geom, store(lin_out + band) + t_geom, t_geom, False)


# ------------------------------------------------------------------------------------------------
# the acceptance rule
# ------------------------------------------------------------------------------------------------
@dataclass
class Verdict:
    n: int                 # bytes
    off_rint: int          # bytes != rint(v), v not at a tie
    unexplained: int       # off-rint bytes whose range [vmin, vmax] lies on one side of the tie: T_ARITH alone excuses them
    at_tie: int            # bytes whose v is a tie (both neighbours are rint(v)): 0 / 255 content averaged evenly
    bad: int               # bytes outside the rule
    worst_tie: float       # the largest |v - tie| of an off-rint byte, LSB
    worst_excess: float    # the largest distance from an off-rint byte's tie to the hull [vmin, vmax], LSB
    hull_width: float      # the largest vmax - vmin, LSB
    first_bad: str

    @property
    def share(self):
        return self.unexplained / max(self.n, 1)

    def line(self):
        return (f"{self.n} bytes, {self.off_rint} off rint, {self.unexplained} of them by T_ARITH alone (share {self.share:.2e}), "
                f"{self.at_tie} at a tie, worst tie distance "
                f"{self.worst_tie:.4f} LSB, worst excess over the hull {self.worst_excess:.4f} LSB, hull width "
                f"{self.hull_width:.4f} LSB")


def rint(v):
    return np.floor(v + 0.5)


def judge(got, ev):
    """got: (dst_h, dst_w, 4) uint8 bytes of the resampled child; ev: evaluate()'s result"""
    g = np.asarray(got).astype(np.float64)
    assert g.shape == ev.v.shape, (g.shape, ev.v.shape)
    r = rint(ev.v)
    lo, hi = rint(ev.vmin - T_ARITH), rint(ev.vmax + T_ARITH)
    bad = (g < lo) | (g > hi) | (np.abs(g - r) > 1)
    at_tie = np.abs(ev.v - np.floor(ev.v) - 0.5) < EXACT_TIE    # both neighbours are rint(v)
    off = (g != r) & ~at_tie
    unexplained = off & (rint(ev.vmin) == rint(ev.vmax))        # the range of v does not reach the tie
    tie = (g + r) / 2.0
    worst_tie = float(np.abs(ev.v - tie)[off].max()) if off.any() else 0.0
    excess = np.maximum(np.where(g < r, ev.vmin - tie, tie - ev.vmax), 0.0)
    worst_excess = float(excess[off].max()) if off.any() else 0.0
    first = ""
    if bad.any():
        y, x, c = (int(i) for i in np.argwhere(bad)[0])
        first = (f"first at ({x}, {y}) channel {c}: got {int(g[y, x, c])}, v {ev.v[y, x, c]:.4f}, hull "
                 f"[{ev.vmin[y, x, c]:.4f}, {ev.vmax[y, x, c]:.4f}], allowed [{int(lo[y, x, c])}, {int(hi[y, x, c])}]")
    return Verdict(int(g.size), int(off.sum()), int(unexplained.sum()), int(at_tie.sum()), int(bad.sum()), worst_tie, worst_excess,
                   float((ev.vmax - ev.vmin).max()), first)


def assert_rule(got, ev, what):
    vd = judge(got, ev)
    assert vd.bad == 0, f"{what}: {vd.bad} bytes outside the rule ({vd.line()}); {vd.first_bad}"
    assert vd.share <= MAX_OFF_RINT_SHARE, f"{what}: off-rint share {vd.share:.2e} > {MAX_OFF_RINT_SHARE} ({vd.line()})"
    return vd


# ------------------------------------------------------------------------------------------------
# content
# ------------------------------------------------------------------------------------------------
def content(kind, w, h, seed):
    """(h, w, 4) uint8 node texture.  random: uniform bytes; smooth: a few low-frequency waves per channel; extreme: 0 /
    255 checkers, column and row stripes and random 0 / 255 bits, a different arrangement in each channel, alpha
    included, one texel in ten flipped so that the patterns repeat no value exactly; constant: one translucent colour; alpha: random colour over an alpha ramp from 0 to 255 along both axes."""
    rng = np.random.default_rng(seed)
    ys, xs = np.mgrid[0:h, 0:w]
    if kind == "random":
        return rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    if kind == "smooth":
        out = np.empty((h, w, 4), np.uint8)
        for c in range(4):
            f = rng.uniform(0.002, 0.05, (3, 2))
            ph = rng.uniform(0, 2 * np.pi, 3)
            v = sum(np.sin(2 * np.pi * (f[i, 0] * xs + f[i, 1] * ys) + ph[i]) for i in range(3)) / 3.0
            out[..., c] = np.rint(127.5 + 127.5 * v).astype(np.uint8)
        return out
    if kind == "extreme":
        patterns = [(xs + ys) & 1, xs & 1, ys & 1, rng.integers(0, 2, (h, w)), ((xs >> 1) + ys) & 1]
        out = np.empty((h, w, 4), np.uint8)
        for c in range(4):
            # the texture in 3 x 3 regions, each channel drawing its patterns in a different order
            reg = (3 * ys // max(h, 1)) * 3 + 3 * xs // max(w, 1)
            pick = (reg + 2 * c) % len(patterns)
            ch = np.choose(pick, patterns) ^ (rng.random((h, w)) < 0.1)   # one texel in ten flipped: no exact period
            out[..., c] = (ch * 255).astype(np.uint8)
        return out
    if kind == "constant":
        return np.broadcast_to(np.array([37, 200, 128, 97], np.uint8), (h, w, 4)).copy()
    if kind == "alpha":
        out = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        out[..., 3] = np.rint(255.0 * (xs / max(w - 1, 1) + ys / max(h - 1, 1)) / 2.0).astype(np.uint8)
        return out
    raise ValueError(kind)
