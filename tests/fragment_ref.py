"""Float64 restatement of the composite's fragment stage, written from the reference's layout shader alone.

`apply_layouts.wgsl` (smelter-render/src/transformations/layout) draws one quad per layout: `vs_main` (:174-235) places it
with `vertices_transformation_matrix` (:127-157) and interpolates `center_position` / `tex_coords`; `fs_main` (:258-377)
turns them into a premultiplied colour with `roundedRectSDF` (:246-256), WGSL's `smoothstep` and `mix`; the pipeline
blends it with PREMULTIPLIED_ALPHA_BLENDING (wgpu/common_pipeline.rs:125) through the target's view.  What the reference
leaves to wgpu and the GPU is the project's numeric contract (DESIGN.md section 3): NC-1 / NC-3 fetches, NC-2 / NC-4 stores,
NC-6's sampler and NC-7's rasteriser.  Everything here is float64 and vectorised over pixels; nothing is shared with
`oracle/smelter_oracle.c` or the kernels.

`evaluate` answers, per pixel of a probe layer drawn over a known destination, which bytes the contract allows and which
branch of `fs_main` the pixel takes; the per-pixel error bound it uses is described in
`tests/test_composite_fragment_space.py`.  The scene catalogue at the end is shared with `tests/test_gpu_composite_fragment.py`.
"""
import itertools
from dataclasses import dataclass, field
from typing import Optional, Tuple

import numpy as np

GPU_OPTIMIZED, CPU_OPTIMIZED = 0, 1
TEXTURE, COLOR, BOX_SHADOW = 0, 1, 2
MAX_MASKS = 20          # params.rs:15 MAX_MASKS_COUNT: masks past the 20th are dropped (params.rs:284-305)
VALUE_SLACK = 2e-6      # f32 arithmetic of the contract on a value in [0, 1] (colour products, fma blend): ~17 ulp of 1.0

# branch codes of fs_main, per covered pixel
OUTSIDE, PLAIN, MASKED_OUT, INNER, OUTER, SHADOW = 0, 1, 2, 3, 4, 5
BRANCH_NAMES = {PLAIN: "plain", MASKED_OUT: "masked_out", INNER: "inner", OUTER: "outer", SHADOW: "shadow"}


# ------------------------------------------------------------------------------------------------
# colours and views
# ------------------------------------------------------------------------------------------------
def srgb_to_linear(c):
    """wgpu/utils.rs:74-81 (`<`), on c in [0, 1]; also the sRGB view's decode (NC-3), which agrees on every byte"""
    c = np.asarray(c, np.float64)
    return np.where(c < 0.04045, c / 12.92, ((c + 0.055) / 1.055) ** 2.4)


def shader_color(rgba, mode):
    """convert_to_shader_color, wgpu/utils.rs:51-71: premultiplied, linear in GpuOptimized"""
    a = rgba[3] / 255.0
    if mode == GPU_OPTIMIZED:
        rgb = [a * float(srgb_to_linear(c / 255.0)) for c in rgba[:3]]
    else:
        rgb = [a * c / 255.0 for c in rgba[:3]]
    return np.array(rgb + [a])


BYTES = np.arange(256) / 255.0
DECODE = {GPU_OPTIMIZED: (srgb_to_linear(BYTES), BYTES), CPU_OPTIMIZED: (BYTES, BYTES)}   # (colour, alpha) per byte
SRGB_THRESHOLDS = srgb_to_linear((np.arange(255) + 0.5) / 255.0)                          # NC-4, float64


def clamp01(x):
    """the render target's clamp of a fragment output; NaN -> 0 (the contract's clamp)"""
    return np.where(np.isnan(x), 0.0, np.clip(x, 0.0, 1.0))


def store(x, mode, alpha):
    """NC-4 (sRGB colour channels in GpuOptimized: thresholds at or below x) or NC-2 (rint of 255 x)"""
    x = clamp01(x)
    if mode == GPU_OPTIMIZED and not alpha:
        return np.searchsorted(SRGB_THRESHOLDS, x, side="right")
    return np.rint(x * 255.0).astype(np.int64)


# ------------------------------------------------------------------------------------------------
# WGSL builtins
# ------------------------------------------------------------------------------------------------
def smoothstep(e0, e1, x):
    """WGSL smoothstep: t = clamp((x - e0) / (e1 - e0)); a zero-width ramp divides by zero and its NaN clamps to 0"""
    with np.errstate(all="ignore"):
        t = clamp01((x - e0) / (e1 - e0))
    return t * t * (3.0 - 2.0 * t)


def mix(a, b, t):
    return a * (1.0 - t) + b * t


def rounded_rect_sdf(dist_x, dist_y, size, radius, sel_x=None, sel_y=None):
    """roundedRectSDF, apply_layouts.wgsl:246-256; radius = [top-left, top-right, bottom-right, bottom-left].
    sel_x / sel_y: the distances the two `select`s test (default: dist itself)."""
    qx, qy, r = _sdf_q(dist_x, dist_y, size, radius, sel_x, sel_y)
    return np.minimum(np.maximum(qx, qy), 0.0) + np.hypot(np.maximum(qx, 0.0), np.maximum(qy, 0.0)) - r


def _sdf_q(dist_x, dist_y, size, radius, sel_x=None, sel_y=None):
    """roundedRectSDF's q and the corner radius r.x it selects"""
    sel_x = dist_x if sel_x is None else sel_x
    sel_y = dist_y if sel_y is None else sel_y
    hx, hy = size[0] / 2.0, size[1] / 2.0
    r_x = np.where(sel_x < 0.0, radius[0], radius[1])     # select(radius.yz, radius.xw, dist.x < 0.0)
    r_y = np.where(sel_x < 0.0, radius[3], radius[2])
    r = np.where(sel_y < 0.0, r_y, r_x)                  # r.x = select(r.x, r.y, dist.y < 0.0)
    return np.abs(dist_x) - hx + r, np.abs(dist_y) - hy + r, r


# ------------------------------------------------------------------------------------------------
# the probe layer
# ------------------------------------------------------------------------------------------------
@dataclass
class Probe:
    """one layout as LayoutInfo + Texture/Color/BoxShadowParams carry it (apply_layouts.wgsl:17-74)"""
    type: int
    left: float
    top: float
    width: float
    height: float
    rotation: float = 0.0
    radius: Tuple[float, float, float, float] = (0.0, 0.0, 0.0, 0.0)
    color: Tuple[int, int, int, int] = (0, 0, 0, 0)
    border_color: Tuple[int, int, int, int] = (0, 0, 0, 0)
    border: float = 0.0
    blur: float = 0.0
    crop: Optional[Tuple[float, float, float, float]] = None    # (left, top, width, height) in texels
    masks: tuple = ()                                           # ((radius4), top, left, width, height)
    tex: Optional[np.ndarray] = None                            # (h, w, 4) uint8 node texture; None: no child


def quad_params(p):
    """vs_main's (left, top, width, height) of the drawn quad: a box shadow grows by blur_radius (:215-229)"""
    if p.type == BOX_SHADOW:
        return p.left - p.blur, p.top - p.blur, p.width + 2.0 * p.blur, p.height + 2.0 * p.blur
    return p.left, p.top, p.width, p.height


def scale_matrix(sx, sy):
    return np.diag([sx, sy, 1.0, 1.0])


def translation_matrix(tx, ty):
    m = np.eye(4)
    m[0, 3], m[1, 3] = tx, ty
    return m


def rotation_matrix(deg):
    a = np.radians(deg)
    c, s = np.cos(a), np.sin(a)
    m = np.eye(4)
    m[0, 0], m[1, 0], m[0, 1], m[1, 1] = c, s, -s, c     # columns (c, s), (-s, c): :95-106
    return m


def vertices_transformation_matrix(left, top, width, height, rotation, W, H):
    """apply_layouts.wgsl:127-157"""
    to_pixels_x, to_pixels_y = W / 2.0, H / 2.0
    s_pix = scale_matrix(to_pixels_x * (width / W), to_pixels_y * (height / H))
    s_clip = scale_matrix(1.0 / to_pixels_x, 1.0 / to_pixels_y)
    t = translation_matrix(-(W / 2.0) + (left + width / 2.0), H / 2.0 - (top + height / 2.0))
    return s_clip @ t @ rotation_matrix(rotation) @ s_pix


# plane.rs:11-28: the quad's clip-space positions and texture coordinates
QUAD_POS = np.array([[1.0, -1.0], [1.0, 1.0], [-1.0, 1.0], [-1.0, -1.0]])


class Geometry:
    """the quad on screen: framebuffer position = A @ position + b, with the viewport transform of a W x H target"""

    def __init__(self, p, W, H):
        ql, qt, qw, qh = quad_params(p)
        m = vertices_transformation_matrix(ql, qt, qw, qh, p.rotation, W, H)
        vp = np.array([[W / 2.0, 0.0], [0.0, -H / 2.0]])      # clip -> framebuffer: ((x + 1) W / 2, (1 - y) H / 2)
        self.A = vp @ m[:2, :2]
        self.b = vp @ m[:2, 3] + np.array([W / 2.0, H / 2.0])
        self.Ainv = np.linalg.inv(self.A)
        self.size = (qw, qh)
        self.verts = QUAD_POS @ self.A.T + self.b             # framebuffer vertices, float64

    def varyings(self, X, Y):
        """-> center_position (x, y) and tex_coords (u, v) interpolated at framebuffer point (X, Y)"""
        px = self.Ainv[0, 0] * (X - self.b[0]) + self.Ainv[0, 1] * (Y - self.b[1])
        py = self.Ainv[1, 0] * (X - self.b[0]) + self.Ainv[1, 1] * (Y - self.b[1])
        # affine interpolation of plane.rs's attributes: tex = ((x + 1) / 2, (1 - y) / 2)
        return px / 2.0 * self.size[0], py / 2.0 * self.size[1], (px + 1.0) / 2.0, (1.0 - py) / 2.0


def coverage(verts256, X, Y):
    """NC-7 on snapped vertices (integer 1/256 px): edge functions around the quad, top-left rule for e == 0.
    X, Y: pixel centres in 1/256 px."""
    # order the quad clockwise on screen (y down): positive signed area in this orientation
    v = verts256
    area = sum(v[i][0] * v[(i + 1) % 4][1] - v[(i + 1) % 4][0] * v[i][1] for i in range(4))
    if area < 0:
        v = v[::-1]
    inside = np.ones(np.broadcast(X, Y).shape, bool)
    for i in range(4):
        (x0, y0), (x1, y1) = v[i], v[(i + 1) % 4]
        dx, dy = x1 - x0, y1 - y0
        e = dx * (Y - y0) - dy * (X - x0)
        top_left = dy < 0 or (dy == 0 and dx > 0)
        inside &= (e > 0) | ((e == 0) & top_left)
    return inside


def f32_ulp(x):
    return 2.0 ** (np.floor(np.log2(max(abs(x), 1.0))) - 23)


def exact_axis(*vals):
    """every value a multiple of 1/256 below 2^14: f32 sums and differences of them and of pixel centres are exact"""
    return all(abs(v) < 2 ** 14 and float(v) * 256.0 == np.rint(float(v) * 256.0) for v in vals)


# ------------------------------------------------------------------------------------------------
# fs_main
# ------------------------------------------------------------------------------------------------
def sample(p, mode, u, v):
    """textureSample through NC-6 (8-bit weights, clamp to edge) of the node texture's view: NC-3 colour in
    GpuOptimized, NC-1 otherwise, NC-1 alpha; a layout without a child samples the 1x1 transparent view"""
    if p.tex is None:
        return np.zeros(u.shape + (4,))
    th, tw = p.tex.shape[:2]
    cl, ct, cw, ch = p.crop
    # texture_coord_transformation_matrix, :159-172: translation(crop / dim) * scale(crop_size / dim)
    tx = u * (cw / tw) + cl / tw
    ty = v * (ch / th) + ct / th

    def taps(t, dim):
        c = t * dim - 0.5
        fl = np.floor(c)
        w = np.rint((c - fl) * 256.0) / 256.0
        return np.clip(fl, 0, dim - 1).astype(np.int64), np.clip(fl + 1, 0, dim - 1).astype(np.int64), w

    x0, x1, wx = taps(tx, tw)
    y0, y1, wy = taps(ty, th)
    col, alp = DECODE[mode]
    out = np.empty(u.shape + (4,))
    for c in range(4):
        lut = alp if c == 3 else col
        t = lut[p.tex[..., c]]
        out[..., c] = ((t[y0, x0] * (1 - wx) + t[y0, x1] * wx) * (1 - wy) + (t[y1, x0] * (1 - wx) + t[y1, x1] * wx) * wy)
    return out


def fragment(p, mode, geo, X, Y, sel=None, exact=False):
    """fs_main at framebuffer point (X, Y) -> (premultiplied colour (..., 4), branch code, mask_alpha).
    sel: the point (X, Y) at which the SDFs' radius selects are decided (default: the point itself).
    exact: both axes of the layer are computed exactly in f32 and sel is the pixel centre; then `edge > bw / 2` is
    decided at sel wherever the SDF there needs no square root (off the corner arcs), as f32 computes it exactly."""
    SX, SY = (X, Y) if sel is None else sel
    cx, cy, u, v = geo.varyings(X, Y)
    scx, scy, _, _ = geo.varyings(SX, SY)
    mask_alpha = np.ones(np.shape(X))
    for m in p.masks[:MAX_MASKS]:
        r, mt, ml, mw, mh = m
        d = rounded_rect_sdf(ml + mw / 2.0 - X, mt + mh / 2.0 - Y, (mw, mh), r, ml + mw / 2.0 - SX, mt + mh / 2.0 - SY)
        mask_alpha = mask_alpha * smoothstep(-0.5, 0.5, -d)
    edge = -rounded_rect_sdf(cx, cy, (p.width, p.height), p.radius, scx, scy)
    ma = mask_alpha[..., None]
    branch = np.zeros(np.shape(X), np.int64)
    if p.type == BOX_SHADOW:
        color = shader_color(p.color, mode)
        a = smoothstep(-p.blur / 2.0, p.blur / 2.0, edge)[..., None] * ma
        branch[:] = SHADOW
        return color * a, branch, mask_alpha
    content = sample(p, mode, u, v) if p.type == TEXTURE else np.broadcast_to(shader_color(p.color, mode), np.shape(X) + (4,))
    border = shader_color(p.border_color, mode)
    bw = p.border
    if bw < 1.0:
        branch[:] = PLAIN
        return content * smoothstep(-0.5, 0.5, edge)[..., None] * ma, branch, mask_alpha
    inner = edge > bw / 2.0
    if exact:
        qx, qy, _ = _sdf_q(scx, scy, (p.width, p.height), p.radius)
        on_arc = (qx > 0.0) & (qy > 0.0)
        inner = np.where(on_arc, inner, -rounded_rect_sdf(scx, scy, (p.width, p.height), p.radius) > bw / 2.0)
    if p.type == TEXTURE:
        ba = smoothstep(bw - 0.5, bw + 0.5, edge)
    else:
        ba = smoothstep(bw, bw + 1.0, edge)
    src_inner = mix(border, content, ba[..., None]) * ma
    src_outer = border * smoothstep(-0.5, 0.5, edge)[..., None] * ma
    src = np.where(inner[..., None], src_inner, src_outer)
    branch[:] = np.where(inner, INNER, OUTER)
    if p.type == TEXTURE:
        cut = mask_alpha < 0.01
        src = np.where(cut[..., None], 0.0, src)
        branch[cut] = MASKED_OUT
    return src, branch, mask_alpha


# ------------------------------------------------------------------------------------------------
# one probe over a destination: the bytes the contract allows
# ------------------------------------------------------------------------------------------------
@dataclass
class Allowed:
    lo: np.ndarray              # (h, w, 4) least allowed byte
    hi: np.ndarray              # (h, w, 4) greatest allowed byte
    covered: np.ndarray         # (h, w) certainly covered
    cover_ambiguous: np.ndarray  # (h, w) covered or not depending on a vertex snap within eps
    branch: np.ndarray          # (h, w) branch at the pixel centre (OUTSIDE where not covered)
    branch_ambiguous: np.ndarray  # (h, w) covered pixels whose branch changes within eps
    ramp: np.ndarray            # (h, w) covered pixels whose smoothstep factor is strictly between 0 and 1
    eps: float
    counts: dict = field(default_factory=dict)


def coordinate_eps(p, W, H):
    """4 ulp (f32) of the largest coordinate the layer's arithmetic meets"""
    ql, qt, qw, qh = quad_params(p)
    mags = [ql, qt, ql + qw, qt + qh, W, H] + [v for m in p.masks[:MAX_MASKS] for v in (m[1], m[2], m[1] + m[4], m[2] + m[3])]
    return 4.0 * f32_ulp(max(abs(v) for v in mags))


def evaluate(p, dst, mode):
    """dst: (H, W, 4) uint8 destination.  -> Allowed"""
    H, W = dst.shape[:2]
    geo = Geometry(p, W, H)
    eps = coordinate_eps(p, W, H)
    # the pixels that can be touched: the quad's bounding box and a margin
    x0 = int(max(np.floor(geo.verts[:, 0].min()) - 2, 0)); x1 = int(min(np.ceil(geo.verts[:, 0].max()) + 2, W))
    y0 = int(max(np.floor(geo.verts[:, 1].min()) - 2, 0)); y1 = int(min(np.ceil(geo.verts[:, 1].max()) + 2, H))
    lo = dst.astype(np.int64).copy()
    hi = lo.copy()
    covered = np.zeros((H, W), bool)
    amb_cov = np.zeros((H, W), bool)
    branch_map = np.zeros((H, W), np.int64)
    amb_br = np.zeros((H, W), bool)
    ramp_map = np.zeros((H, W), bool)
    if x0 >= x1 or y0 >= y1:
        return Allowed(lo, hi, covered, amb_cov, branch_map, amb_br, ramp_map, eps)
    ys, xs = np.mgrid[y0:y1, x0:x1]
    # NC-7: every snap a vertex can take within eps; a pixel covered under some and not under others is ambiguous
    snaps = [sorted({int(np.rint((v + s * eps) * 256.0)) for s in (-1, 0, 1)}) for v in geo.verts.reshape(-1)]
    X256, Y256 = xs * 256 + 128, ys * 256 + 128
    cov_any = np.zeros(xs.shape, bool)
    cov_all = np.ones(xs.shape, bool)
    for choice in itertools.product(*snaps):
        c = coverage([(choice[2 * i], choice[2 * i + 1]) for i in range(4)], X256, Y256)
        cov_any |= c
        cov_all &= c
    # fs_main at the centre moved by up to eps; the SDFs' radius selects keep the centre's side of an axis whose
    # coordinates the f32 arithmetic computes exactly (there dist == 0 is exact, and the reference's choice is defined)
    ql, qt, qw, qh = quad_params(p)
    unrot = p.rotation == 0.0
    ex = unrot and exact_axis(ql, qw / 2.0) and all(exact_axis(m[2], m[3] / 2.0) for m in p.masks[:MAX_MASKS])
    ey = unrot and exact_axis(qt, qh / 2.0) and all(exact_axis(m[1], m[4] / 2.0) for m in p.masks[:MAX_MASKS])
    pcx, pcy = xs + 0.5, ys + 0.5
    dstf = np.empty(xs.shape + (4,))
    col, alp = DECODE[mode]
    d = dst[y0:y1, x0:x1].astype(np.int64)
    for c in range(4):
        dstf[..., c] = (alp if c == 3 else col)[d[..., c]]
    vmin = np.full(xs.shape + (4,), np.inf)
    vmax = np.full(xs.shape + (4,), -np.inf)
    branches = []
    centre_branch, centre_ramp = None, None
    for ox in (-1, 0, 1):
        for oy in (-1, 0, 1):
            X, Y = pcx + ox * eps, pcy + oy * eps
            sel = (pcx if ex else X, pcy if ey else Y)
            src, br, ma = fragment(p, mode, geo, X, Y, sel, ex and ey)
            src = clamp01(src)
            val = src + dstf * (1.0 - src[..., 3:4])          # PREMULTIPLIED_ALPHA_BLENDING
            vmin = np.minimum(vmin, val)
            vmax = np.maximum(vmax, val)
            branches.append(br)
            if ox == 0 and oy == 0:
                centre_branch = br
                centre_ramp = ramp_of(p, mode, geo, X, Y, sel, br)
    lo_b = np.stack([store(vmin[..., c] - VALUE_SLACK, mode, c == 3) for c in range(4)], -1)
    hi_b = np.stack([store(vmax[..., c] + VALUE_SLACK, mode, c == 3) for c in range(4)], -1)
    amb = cov_any & ~cov_all
    sl = (slice(y0, y1), slice(x0, x1))
    lo[sl] = np.where(cov_all[..., None], lo_b, np.where(amb[..., None], np.minimum(lo_b, d), d))
    hi[sl] = np.where(cov_all[..., None], hi_b, np.where(amb[..., None], np.maximum(hi_b, d), d))
    covered[sl] = cov_all
    amb_cov[sl] = amb
    branch_map[sl] = np.where(cov_all, centre_branch, OUTSIDE)
    amb_br[sl] = cov_all & np.any([b != centre_branch for b in branches], axis=0)
    ramp_map[sl] = cov_all & centre_ramp
    a = Allowed(lo, hi, covered, amb_cov, branch_map, amb_br, ramp_map, eps)
    certain = covered & ~amb_br
    a.counts = {"covered": int(covered.sum()), "ambiguous": int((amb_cov | amb_br).sum())}
    for code, name in BRANCH_NAMES.items():
        n = int((certain & (branch_map == code)).sum())
        if n:
            a.counts[name] = n
    a.counts["ramp"] = int((certain & ramp_map).sum())
    return a


def ramp_of(p, mode, geo, X, Y, sel, br):
    """covered pixels whose fragment's smoothstep factors (edge ramp, border ramp, mask, blur) are not all 0 or 1"""
    cx, cy, _, _ = geo.varyings(X, Y)
    scx, scy, _, _ = geo.varyings(*sel)
    edge = -rounded_rect_sdf(cx, cy, (p.width, p.height), p.radius, scx, scy)
    _, _, ma = fragment(p, mode, geo, X, Y, sel, False)
    if p.type == BOX_SHADOW:
        f = smoothstep(-p.blur / 2.0, p.blur / 2.0, edge)
    elif p.border >= 1.0:
        f = np.where(br == INNER, smoothstep(p.border - 0.5, p.border + 0.5, edge) if p.type == TEXTURE
                     else smoothstep(p.border, p.border + 1.0, edge), smoothstep(-0.5, 0.5, edge))
    else:
        f = smoothstep(-0.5, 0.5, edge)
    frac = lambda t: (t > 0.0) & (t < 1.0)
    return frac(f) | frac(ma)


# ------------------------------------------------------------------------------------------------
# the scene catalogue: one probe layer over a background that holds every byte in every channel
# ------------------------------------------------------------------------------------------------
def rgba_content(seed, w, h):
    """premultiplied RGBA8 (colour <= alpha) holding every byte value in every channel"""
    rng = np.random.default_rng(seed)
    t = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    t[..., :3] = np.minimum(t[..., :3], t[..., 3:4])
    t[: h // 2, : w // 4, 3] = 255          # an opaque corner: texels that replace the destination
    return t


def probe_texture(seed, w, h):
    """rgba_content with a 16 x 16 block of texels that have colour but zero alpha: a source the blend must still add"""
    t = rgba_content(seed, w, h)
    t[h // 2:h // 2 + 16, w // 2:w // 2 + 16, :3] |= 1
    t[h // 2:h // 2 + 16, w // 2:w // 2 + 16, 3] = 0
    return t


@dataclass
class Scene:
    name: str
    probe: Probe
    W: int = 384
    H: int = 256
    max_ambiguous: float = 0.02     # ambiguous pixels, as a share of the covered ones


TEX = probe_texture(7, 96, 64)
FULL = (0.0, 0.0, 96.0, 64.0)
RADII = (12.0, 4.0, 20.0, 8.0)
BORDER_RGBA = (250, 200, 20, 170)


def _masks(n):
    """n rounded masks, each a little smaller and further in than the last, so that they overlap in part"""
    return tuple(((6.0 + k, 2.0 * k, 10.0, 3.0 + k % 4), 20.25 + 2.0 * k, 30.5 + 3.0 * k, 300.0 - 7.0 * k, 200.0 - 5.0 * k)
                 for k in range(n))


def _catalogue():
    sc = []
    C, T, B = COLOR, TEXTURE, BOX_SHADOW
    col = (200, 40, 90, 180)
    # corners: the centre on a pixel centre (dist.x == 0 and dist.y == 0 exactly)
    sc.append(Scene("corners", Probe(C, 91.5, 67.5, 200.0, 120.0, radius=(3.0, 11.0, 27.0, 0.0), color=col)))
    sc.append(Scene("corners_pill", Probe(C, 91.5, 97.5, 200.0, 60.0, radius=(30.0, 30.0, 30.0, 30.0), color=col)))
    sc.append(Scene("corners_over", Probe(C, 91.5, 97.5, 200.0, 60.0, radius=(45.0, 38.0, 31.0, 52.0), color=col)))
    # the same, transposed: radii above half the width make the select at dist.x == 0 visible (at dist.y == 0 above)
    sc.append(Scene("corners_over_tall", Probe(C, 161.5, 27.5, 60.0, 200.0, radius=(45.0, 38.0, 31.0, 52.0), color=col)))
    sc.append(Scene("corners_zero", Probe(C, 40.25, 30.75, 150.0, 90.0, color=col)))
    # borders: translucent border colours, fractional positions, both ramps and both sides of edge = bw / 2
    for bw in (0.999, 1.0, 1.5, 4.0, 10.0):
        sc.append(Scene(f"border_color_{bw}", Probe(C, 20.3, 15.6, 250.5, 180.25, radius=RADII, color=col,
                                                    border_color=BORDER_RGBA, border=bw)))
        sc.append(Scene(f"border_texture_{bw}", Probe(T, 30.7, 20.1, 240.25, 170.5, radius=RADII, border_color=BORDER_RGBA,
                                                      border=bw, crop=FULL, tex=TEX)))
    # masks: the first 20 count, the 21st (which would hide nearly everything) does not
    for n in (1, 2, 20):
        sc.append(Scene(f"masks_{n}", Probe(C, 10.5, 8.25, 330.0, 230.0, radius=RADII, color=col, masks=_masks(n))))
    sc.append(Scene("masks_21", Probe(C, 10.5, 8.25, 330.0, 230.0, radius=RADII, color=col,
                                      masks=_masks(20) + (((2.0, 2.0, 2.0, 2.0), 100.0, 100.0, 20.0, 20.0),))))
    # a bordered texture layer whose mask's right edge steps across the place where mask_alpha crosses 0.01 at the
    # pixel centres x = 150.5: the edge at 150 + f puts them at mask_alpha = smoothstep(0, 1, f), here .0029, .0064,
    # .0087, .0112, .0174 and .0248 -- the cut is pinned to (.0087, .0112]
    for k, f in enumerate((2 / 64, 3 / 64, 3.5 / 64, 4 / 64, 5 / 64, 6 / 64)):
        m = ((0.0, 0.0, 0.0, 0.0), 0.0, 0.0, 150.0 + f, 128.0)
        sc.append(Scene(f"mask_cut_{k}", Probe(T, 20.0, 10.0, 200.0, 100.0, border_color=BORDER_RGBA, border=4.0, crop=FULL,
                                               tex=TEX, masks=(m,)), W=256, H=128))
    # box shadows: the quad grows by blur_radius, the SDF keeps the ungrown size
    for blur in (0.0, 0.25, 1.0, 7.5, 40.0):
        sc.append(Scene(f"shadow_{blur}", Probe(B, 70.5, 50.25, 220.0, 140.0, radius=RADII, color=(10, 20, 30, 150),
                                                blur=blur)))
    sc.append(Scene("shadow_rotated", Probe(B, 90.5, 60.25, 180.0, 120.0, rotation=30.0, radius=RADII, color=(10, 20, 30, 150),
                                            blur=7.5)))
    # rotation, with a border and radii
    for deg in (1e-3, 30.0, 45.0, 90.0, -90.0, 180.0, 270.0, 360.0):
        sc.append(Scene(f"rotated_{deg:g}", Probe(C, 110.3, 70.6, 160.5, 110.25, rotation=deg, radius=RADII, color=col,
                                                  border_color=BORDER_RGBA, border=4.0)))
    sc.append(Scene("rotated_texture_30", Probe(T, 100.3, 60.6, 170.5, 120.25, rotation=30.0, radius=RADII,
                                                border_color=BORDER_RGBA, border=1.5, crop=(5.5, 3.25, 80.0, 50.5), tex=TEX)))
    # an integral box rotated by 90 degrees: on screen its edges run through pixel centres (x 120.5 / 180.5, y 70.5 / 170.5)
    sc.append(Scene("rotated_90_top_left", Probe(C, 100.5, 90.5, 100.0, 60.0, rotation=90.0, color=col)))
    # texture: bilinear taps everywhere, one texel per pixel, no child
    sc.append(Scene("texture_fractional_crop", Probe(T, 15.5, 12.25, 310.5, 220.75, radius=RADII, crop=(3.3, 2.7, 40.6, 30.2),
                                                     tex=TEX)))
    sc.append(Scene("texture_exact_texels", Probe(T, 40.0, 30.0, 64.0, 48.0, radius=(5.0, 5.0, 5.0, 5.0),
                                                  crop=(8.0, 4.0, 64.0, 48.0), tex=TEX)))
    sc.append(Scene("texture_missing_child", Probe(T, 25.5, 18.5, 200.0, 150.0, radius=RADII, border_color=BORDER_RGBA,
                                                   border=4.0, crop=FULL, tex=None)))
    # precision: coordinates near 3000 on a 4096-wide target
    sc.append(Scene("precision_3000", Probe(C, 3000.37, 5.3, 300.4, 40.6, radius=(6.0, 9.0, 3.0, 12.0), color=col,
                                            border_color=BORDER_RGBA, border=2.0), W=4096, H=64))
    return sc


SCENES = _catalogue()


def background(W, H):
    return rgba_content(3, W, H)
