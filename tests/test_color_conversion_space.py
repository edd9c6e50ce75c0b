"""The oracle's colour converters over their whole joint byte space, against a float64 restatement of the reference shaders.

A converted byte depends on a tuple, not on one plane: r on (Y, V), b on (Y, U), g on (Y, U, V), and Y' on (r, g, b).  Each
tuple has its own rounding boundary, so a converter that evaluates its f32 expression in a different order, or with one
coefficient or clamp wrong, differs from the contract on a few tuples only -- the ones whose exact value lies near a
rounding tie.  Random frames, or frames that fill each plane independently, almost never contain them.

The frames here contain every tuple.  Each converter of `oracle/smelter_oracle.c` (K1/K2 planar, 4:2:0, J420 and NV12,
K3 UYVY / YUYV, K10/K11 planar and NV12, the black fill) is fed them, and every byte it writes must equal `rint` of the
float64 value of the WGSL expression, except where that value lies within TIE_DELTA (10^-3 LSB) of a rounding tie, where
it may differ by exactly 1: an f32 evaluation may round a near-tie either way, nothing else.  The restatement below is
written from the shaders alone (cited per function), with the coefficients as the WGSL has them; the sampler is the
contract's NC-6u (an 8-bit texel filter with 8-bit weights, exact) evaluated in integers.

The content generators and the restatement are shared with `tests/test_gpu_color_conversion.py`, which holds the kernels
to the same bytes.  Every generator reports the tuples it covers and every test asserts that coverage, so the content
cannot shrink silently.
"""
import functools

import numpy as np
import pytest

from oracle import oracle as orc

TIE_DELTA = 1e-3          # LSB: the f32 contract may round a float64 value this close to a tie either way
N = 1 << 24               # (Y, U, V) triples, (r, g, b) colours
SIDE = 4096               # one frame of 2^24 texels
CHUNK = 512               # rows per numpy slice (keeps the float64 temporaries near 100 MB)

KY = 0.85882352941        # (235 - 16) / 255, as written in the shaders
KC = 0.87843137254        # (240 - 16) / 255


# ------------------------------------------------------------------------------------------------
# float64 restatement of the reference shaders
# ------------------------------------------------------------------------------------------------
def k1_rgb(y, u, v, full_range):
    """K1/K2/K3 at sampled values y, u, v in [0, 1] -> exact r, g, b in byte units (clamped, times 255).
    planar_yuv_to_rgba.wgsl:45-57 (limited: pixel_format 0; full: 1), nv12_to_rgba.wgsl:37-47,
    interleaved_uyvy_to_rgba.wgsl:51-61 and interleaved_yuyv_to_rgba.wgsl:51-61 (always limited)."""
    y, u, v = (np.asarray(a, np.float64) for a in (y, u, v))
    if not full_range:
        y = np.clip((y - (16.0 / 255.0)) / 0.85882352941, 0.0, 1.0)
        u = np.clip((u - (16.0 / 255.0)) / 0.87843137254, 0.0, 1.0)
        v = np.clip((v - (16.0 / 255.0)) / 0.87843137254, 0.0, 1.0)
    r = y + 1.5748 * (v - 0.5)
    g = y - 0.1873 * (u - 0.5) - 0.4681 * (v - 0.5)
    b = y + 1.8556 * (u - 0.5)
    return tuple(np.clip(c, 0.0, 1.0) * 255.0 for c in (r, g, b))


def k10_y(r, g, b):
    """K10/K11 luma at sampled r, g, b in [0, 1] -> exact Y' in byte units.  rgba_to_yuv.wgsl:36-38 (plane 0),
    rgba_to_nv12.wgsl:31-33 (fs_main_y), clamp at :53 / :33."""
    y = r * 0.2126 + g * 0.7152 + b * 0.0722
    return np.clip((y * 0.85882352941) + (16.0 / 255.0), 0.0, 1.0) * 255.0


def k10_uv(r, g, b):
    """K10/K11 chroma -> exact (U', V') in byte units.  rgba_to_yuv.wgsl:41-48 (planes 1, 2), rgba_to_nv12.wgsl:44-51."""
    u = r * -0.1146 + g * -0.3854 + b * 0.5
    v = r * 0.5 + g * -0.4542 + b * -0.0458
    return (np.clip(((u + 0.5) * 0.87843137254) + (16.0 / 255.0), 0.0, 1.0) * 255.0,
            np.clip(((v + 0.5) * 0.87843137254) + (16.0 / 255.0), 0.0, 1.0) * 255.0)


def to_yuv(r, g, b):
    """RGBColor::to_yuv (scene/types.rs:28-42), the black fill's colour, with its Rust literals -> exact bytes (Y, U, V)"""
    r, g, b = (np.asarray(c, np.float64) / 255.0 for c in (r, g, b))
    y = r * 0.2126 + g * 0.7152 + b * 0.0722
    u = r * -0.1146 + g * -0.3854 + b * 0.5
    v = r * 0.5 + g * -0.4542 + b * -0.0458
    return (np.clip((y * 0.858_823_54) + (16.0 / 255.0), 0.0, 1.0) * 255.0,
            np.clip(((u + 0.5) * 0.878_431_4) + (16.0 / 255.0), 0.0, 1.0) * 255.0,
            np.clip(((v + 0.5) * 0.878_431_4) + (16.0 / 255.0), 0.0, 1.0) * 255.0)


def tie_distance(e):
    """distance in LSB of the exact byte value e from the nearest rounding tie k + .5"""
    return np.abs(e - np.floor(e) - 0.5)


def tie_rule(got, exact, what, delta=TIE_DELTA):
    """Every byte equals rint(exact), or differs from it by exactly 1 where exact lies within delta of a tie.
    -> the number of bytes that differ from rint(exact) (all of them near-ties)."""
    got = np.asarray(got).astype(np.int16)
    want = np.rint(exact).astype(np.int16)
    diff = got != want
    bad = diff & ~((np.abs(got - want) == 1) & (tie_distance(exact) < delta))
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} bytes break the tie rule; first at {i}: got {got[i]}, float64 "
                             f"{exact[i]!r} (rint {want[i]}, {tie_distance(exact)[i]:.3g} LSB from a tie)")
    return int(diff.sum())


# ------------------------------------------------------------------------------------------------
# the NC-6u sampler, exactly: what each output pixel of a converter reads
# ------------------------------------------------------------------------------------------------
def half_taps(n_out, n_in):
    """(i0, i1, w1 in 1/4 units) of the linear sampler at pixel centres of n_out = 2 * n_in: c = (o + .5) / 2 - .5, so the
    weights are .25 / .75 (exact in 8 bits) and the taps clamp at both ends"""
    c = (np.arange(n_out) + 0.5) / 2.0 - 0.5
    i0 = np.floor(c).astype(np.int64)
    w1 = np.rint((c - i0) * 4).astype(np.int64)
    return np.clip(i0, 0, n_in - 1), np.clip(i0 + 1, 0, n_in - 1), w1


def upsample2_sum16(p, rows):
    """4:2:0 chroma plane p (ch x cw) sampled at the luma pixel centres of `rows`: 16 x the interpolated value, an integer
    in [0, 16 * 255] (a + 3b + 3c + 9d over the 2 x 2 neighbourhood)"""
    ch, cw = p.shape
    x0, x1, wx = half_taps(2 * cw, cw)
    y0, y1, wy = half_taps(2 * ch, ch)
    y0, y1, wy = y0[rows], y1[rows], wy[rows]
    p = p.astype(np.int64)
    r0 = p[y0][:, x0] * (4 - wx) + p[y0][:, x1] * wx
    r1 = p[y1][:, x0] * (4 - wx) + p[y1][:, x1] * wx
    return r0 * (4 - wy)[:, None] + r1 * wy[:, None]


def mean2x2_sum4(p):
    """a w x h plane sampled at the centres of its (w / 2) x (h / 2) chroma texels: 4 x the 2 x 2 mean, an integer"""
    p = p.astype(np.int64)
    return p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2]


# ------------------------------------------------------------------------------------------------
# content generators
# ------------------------------------------------------------------------------------------------
def _index_planes():
    """(a, b, c): 4096 x 4096 planes in which (a, b, c) runs over every byte triple exactly once"""
    x = np.arange(SIDE, dtype=np.int64)[None, :]
    y = np.arange(SIDE, dtype=np.int64)[:, None]
    a = np.broadcast_to(x & 255, (SIDE, SIDE)).astype(np.uint8)
    b = np.broadcast_to(y & 255, (SIDE, SIDE)).astype(np.uint8)
    c = ((x >> 8) + 16 * (y >> 8)).astype(np.uint8)
    return a, b, c


def triple_index(a, b, c):
    return a.astype(np.int64) | (b.astype(np.int64) << 8) | (c.astype(np.int64) << 16)


def coverage(mask):
    """a 2^24 bitmap -> number of tuples set"""
    return int(np.count_nonzero(mask))


def yuv444_all_triples():
    """4:4:4 planes (y, u, v), 4096 x 4096, in which pixel (x, y) holds one of the 2^24 (Y, U, V) triples, each once.
    -> (planes, number of distinct triples)"""
    y, u, v = _index_planes()
    seen = np.zeros(N, bool)
    seen[triple_index(y, u, v).ravel()] = True
    return (y, u, v), coverage(seen)


@functools.lru_cache(maxsize=4)
def yuv420_block_triples(part):
    """4:2:0 planes (y, u, v) of 4096 x 4096 in which every (U, V) pair is a constant 2 x 2 chroma block (one 4 x 4 luma
    block).  With the .25 / .75 taps the four inner luma pixels (4j + 1, 4j + 2 on both axes) sample only their own block,
    so they see exactly (U, V); the 16 blocks of a pair in one part carry its 64 luma values 64 part .. 64 part + 63 on
    those pixels, and the four parts carry all 256.  The outer luma pixels repeat the block's values.
    -> (planes, bitmap of the (Y, U, V) triples whose chroma the frame delivers exactly)"""
    nb = SIDE // 4                                              # 1024 x 1024 blocks
    by, bx = np.meshgrid(np.arange(nb), np.arange(nb), indexing="ij")
    k = (by & 3) * 4 + (bx & 3)                                 # block k of 16 for its pair
    U, V = (bx >> 2).astype(np.uint8), (by >> 2).astype(np.uint8)
    u = np.repeat(np.repeat(U, 2, 0), 2, 1)
    v = np.repeat(np.repeat(V, 2, 0), 2, 1)
    # luma of block (by, bx) at in-block (r, c): inner pixel (1 + i, 1 + j) gets 64 part + 4 k + 2 i + j, the ring the
    # value of its nearest inner pixel
    ir = np.array([0, 0, 1, 1])                                  # in-block row -> inner row index
    Yb = 64 * part + 4 * k[:, :, None, None] + 2 * ir[None, None, :, None] + ir[None, None, None, :]
    y = Yb.transpose(0, 2, 1, 3).reshape(SIDE, SIDE).astype(np.uint8)
    return (y, u, v), exact_chroma_triples((y, u, v))


def exact_chroma_triples(planes):
    """bitmap of the (Y, U, V) triples the 4:2:0 frame delivers at pixels whose interpolated chroma is a whole byte"""
    y, u, v = planes
    seen = np.zeros(N, bool)
    for r0 in range(0, y.shape[0], CHUNK):
        rows = np.arange(r0, min(r0 + CHUNK, y.shape[0]))
        su, sv = upsample2_sum16(u, rows), upsample2_sum16(v, rows)
        ok = (su % 16 == 0) & (sv % 16 == 0)
        seen[triple_index(y[rows][ok], (su[ok] // 16), (sv[ok] // 16))] = True
    return seen


@functools.lru_cache(maxsize=1)
def yuv420_chroma_sums():
    """4:2:0 planes (y, u, v), 4096 x 4096, in which the interpolated chroma 16 c = n (n = a + 3b + 3c + 9d over a 2 x 2
    chroma neighbourhood) takes every value 0 .. 4080 with every Y, on both channels.  Vertical variation is needed for
    the values that are not multiples of 4.  Block b of the 1024 x 1024 4 x 4 luma blocks targets its inner pixel
    (4j + 2, 4i + 2), whose weight 9 falls on the block's chroma texel (2j + 1, 2i + 1): Y = b mod 256, n_u = b div 256 and
    n_v = (1031 n_u + 7 Y) mod 4081, a permutation of n_u for each Y, so (Y, n_u, n_v) also samples g's joint space.
    The other pixels see other sums; all of them are checked.
    -> (planes, {"u": bitmap of (Y, n_u), "v": bitmap of (Y, n_v), "uv": number of distinct (Y, n_u, n_v)})"""
    nb = SIDE // 4
    b = np.arange(nb * nb, dtype=np.int64) % (256 * 4081)
    Y, nu = b % 256, b // 256
    nv = (1031 * nu + 7 * Y) % 4081

    def split(n):   # a + 3 (b + c) + 9 d = n with each term a byte
        d = np.minimum(255, n // 9)
        rem = n - 9 * d
        bc = np.minimum(510, rem // 3)
        a = rem - 3 * bc
        return a, bc // 2, bc - bc // 2, d

    def plane(n):
        a, bb, cc, d = (t.reshape(nb, nb) for t in split(n))
        p = np.empty((2 * nb, 2 * nb), np.int64)
        p[0::2, 0::2], p[0::2, 1::2], p[1::2, 0::2], p[1::2, 1::2] = a, bb, cc, d
        assert p.min() >= 0 and p.max() <= 255
        return p.astype(np.uint8)

    u, v = plane(nu), plane(nv)
    y = np.repeat(np.repeat(Y.reshape(nb, nb).astype(np.uint8), 4, 0), 4, 1)
    cov_u, cov_v = np.zeros(256 * 4081, bool), np.zeros(256 * 4081, bool)
    seen = set()
    rows = np.arange(2, SIDE, 4)
    su, sv = upsample2_sum16(u, rows)[:, 2::4], upsample2_sum16(v, rows)[:, 2::4]
    yy = y[rows][:, 2::4].astype(np.int64)
    cov_u[yy.ravel() * 4081 + su.ravel()] = True
    cov_v[yy.ravel() * 4081 + sv.ravel()] = True
    seen = len(np.unique((yy * 4081 + su) * 4081 + sv))
    return (y, u, v), {"u": coverage(cov_u), "v": coverage(cov_v), "uv": seen}


def interleaved_all_triples(yuyv):
    """a UYVY (yuyv False) or YUYV 4:2:2 frame, 4096 x 4096 pixels (2048 texels of 4 bytes per row): texel i carries
    U = i mod 256, V = (i div 256) mod 256 and luma 2 (i div 65536), 2 (i div 65536) + 1, so its two pixels hold two
    triples and the frame every (Y, U, V) once.  -> ((h, w / 2, 4) texels, number of distinct triples)"""
    i = np.arange(N // 2, dtype=np.int64).reshape(SIDE, SIDE // 2)
    U, V, Y0 = i & 255, (i >> 8) & 255, 2 * (i >> 16)
    t = np.empty((SIDE, SIDE // 2, 4), np.uint8)
    if yuyv:
        t[..., 0], t[..., 1], t[..., 2], t[..., 3] = Y0, U, Y0 + 1, V
    else:
        t[..., 0], t[..., 1], t[..., 2], t[..., 3] = U, Y0, V, Y0 + 1
    y, u, v = interleaved_planes(t, yuyv)
    seen = np.zeros(N, bool)
    seen[triple_index(y, u, v).ravel()] = True
    return t, coverage(seen)


def interleaved_planes(t, yuyv):
    """per-pixel (Y, U, V) of an interleaved frame: pixel x reads texel x div 2 and its luma x mod 2"""
    h, tw, _ = t.shape
    y = np.empty((h, 2 * tw), np.uint8)
    if yuyv:
        y[:, 0::2], y[:, 1::2], u, v = t[..., 0], t[..., 2], t[..., 1], t[..., 3]
    else:
        y[:, 0::2], y[:, 1::2], u, v = t[..., 1], t[..., 3], t[..., 0], t[..., 2]
    return y, np.repeat(u, 2, 1), np.repeat(v, 2, 1)


def rgb_all_triples():
    """opaque RGBA8, 4096 x 4096, pixel (x, y) holding one of the 2^24 (r, g, b) colours, each once.
    -> (rgba, number of distinct colours)"""
    r, g, b = _index_planes()
    rgba = np.empty((SIDE, SIDE, 4), np.uint8)
    rgba[..., 0], rgba[..., 1], rgba[..., 2], rgba[..., 3] = r, g, b, 255
    seen = np.zeros(N, bool)
    seen[triple_index(r, g, b).ravel()] = True
    return rgba, coverage(seen)


def rgb_block_triples(part):
    """opaque RGBA8, 4096 x 4096, of constant 2 x 2 blocks: block (bx, by) holds r = bx mod 256, g = by mod 256,
    b = 64 part + bx div 256 + 8 (by div 256), so the four parts hold every colour as a block once.
    -> (rgba, bitmap of the constant-block colours)"""
    nb = SIDE // 2
    by, bx = np.meshgrid(np.arange(nb), np.arange(nb), indexing="ij")
    r, g, b = bx & 255, by & 255, 64 * part + (bx >> 8) + 8 * (by >> 8)
    rgba = np.empty((SIDE, SIDE, 4), np.uint8)
    for c, p in enumerate((r, g, b)):
        rgba[..., c] = np.repeat(np.repeat(p.astype(np.uint8), 2, 0), 2, 1)
    rgba[..., 3] = 255
    return rgba, constant_blocks(rgba)


def constant_blocks(rgba):
    """bitmap of the colours that appear as a constant 2 x 2 block at an even position"""
    q = [rgba[i::2, j::2, :3].astype(np.int64) for i in (0, 1) for j in (0, 1)]
    same = np.all([np.all(q[0] == p, axis=-1) for p in q[1:]], axis=0)
    seen = np.zeros(N, bool)
    seen[triple_index(q[0][..., 0][same], q[0][..., 1][same], q[0][..., 2][same])] = True
    return seen


def all_triples():
    """(a, b, c) byte arrays of every triple, index a | b << 8 | c << 16"""
    i = np.arange(N, dtype=np.int64)
    return i & 255, (i >> 8) & 255, i >> 16


_NEAR_TIE_CACHE = {}


def near_tie_yuv(full_range, delta=TIE_DELTA):
    """the (Y, U, V) triples (a 2^24 bitmap, index Y | U << 8 | V << 16) whose float64 K1 r, g or b lies within delta LSB
    of a rounding tie"""
    key = ("yuv", bool(full_range), delta)
    if key not in _NEAR_TIE_CACHE:
        Y, U, V = all_triples()
        near = np.zeros(N, bool)
        for c in k1_rgb(Y / 255.0, U / 255.0, V / 255.0, full_range):
            near |= tie_distance(c) < delta
        assert near.any(), key
        _NEAR_TIE_CACHE[key] = near
    return _NEAR_TIE_CACHE[key]


def near_tie_rgb(delta=TIE_DELTA):
    """the (r, g, b) colours (a 2^24 bitmap) whose float64 K10 Y' per texel, or whose chroma U' or V' as a constant 2 x 2
    block (the 2 x 2 mean of the colour is the colour), lies within delta LSB of a tie.
    -> (union, Y' per texel only)"""
    key = ("rgb", delta)
    if key not in _NEAR_TIE_CACHE:
        r, g, b = (c / 255.0 for c in all_triples())
        ny = tie_distance(k10_y(r, g, b)) < delta
        near = ny.copy()
        for c in k10_uv(r, g, b):
            near |= tie_distance(c) < delta
        assert ny.any() and near.any()
        _NEAR_TIE_CACHE[key] = (near, ny)
    return _NEAR_TIE_CACHE[key]


# ------------------------------------------------------------------------------------------------
# exact float64 results of whole frames
# ------------------------------------------------------------------------------------------------
def k1_frame_420(planes, full_range, rows):
    """exact (r, g, b) of a 4:2:0 / NV12 frame at `rows` (luma sampled at its texel, chroma interpolated exactly)"""
    y, u, v = planes
    return k1_rgb(y[rows] / 255.0, upsample2_sum16(u, rows) / (16.0 * 255.0), upsample2_sum16(v, rows) / (16.0 * 255.0),
                  full_range)


def k11_frame_420(rgba):
    """exact (Y', U', V') planes of K10/K11 at 4:2:0: Y' per texel, chroma of the 2 x 2 mean"""
    f = rgba[..., :3] / 255.0
    Yp = k10_y(f[..., 0], f[..., 1], f[..., 2])
    m = [mean2x2_sum4(rgba[..., c]) / (4.0 * 255.0) for c in range(3)]
    Up, Vp = k10_uv(*m)
    return Yp, Up, Vp


def report(name, counts):
    print(f"\n{name}: " + ", ".join(f"{k}={v}" for k, v in counts.items()))


# ------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------
def test_near_tie_sets():
    """the near-tie sets are non-empty, nested in delta, and contain every tuple at which the f32 contract leaves rint"""
    sizes = {}
    for fr in (0, 1):
        s = near_tie_yuv(fr)
        sizes[f"K1 {'full' if fr else 'limited'}"] = coverage(s)
        assert coverage(near_tie_yuv(fr, 1e-4)) <= coverage(s)
    union, ny = near_tie_rgb()
    sizes["K10 Y' per texel"], sizes["K10/K11 Y' U' V'"] = coverage(ny), coverage(union)
    report("near-tie set sizes", sizes)
    assert sizes["K1 limited"] == 58256 and sizes["K10/K11 Y' U' V'"] == 100761, sizes


@pytest.mark.parametrize("full_range", [0, 1], ids=["limited", "full"])
def test_k1_planar_444_every_triple(full_range):
    """orc_yuv_planar_to_rgba at 4:4:4 (every plane sampled at its own texel) on every (Y, U, V)"""
    (y, u, v), n = yuv444_all_triples()
    assert n == N
    got = orc.yuv_planar_to_rgba(y, u, v, SIDE, SIDE, SIDE, SIDE, full_range=bool(full_range))
    counts = {}
    for r0 in range(0, SIDE, CHUNK):
        sl = slice(r0, r0 + CHUNK)
        ex = k1_rgb(y[sl] / 255.0, u[sl] / 255.0, v[sl] / 255.0, full_range)
        for c, e in enumerate(ex):
            counts["rgb"[c]] = counts.get("rgb"[c], 0) + tie_rule(got[sl, :, c], e, f"K1 4:4:4 {'rgb'[c]}")
    assert np.all(got[..., 3] == 255)
    report(f"K1 4:4:4 {'full' if full_range else 'limited'}, bytes off rint(float64)", counts)


KINDS_420 = {"limited": ("yuv", "nv12"), "full": ("yuvj",)}


def _check_420(rng, planes):
    """the range's converters (limited: orc_yuv420_to_rgba and orc_nv12_to_rgba, which share one float64 result; full:
    orc_yuv420_to_rgba full range) on one frame -> {kind: bytes off rint(float64)}"""
    y, u, v = planes
    got = {}
    for kind in KINDS_420[rng]:
        if kind == "nv12":
            got[kind] = orc.nv12_to_rgba(y, np.stack([u, v], axis=-1), SIDE, SIDE)
        else:
            got[kind] = orc.yuv420_to_rgba(y, u, v, SIDE, SIDE, full_range=kind == "yuvj")
        assert np.all(got[kind][..., 3] == 255)
    n = dict.fromkeys(got, 0)
    for r0 in range(0, SIDE, CHUNK):
        rows = np.arange(r0, r0 + CHUNK)
        for c, e in enumerate(k1_frame_420(planes, rng == "full", rows)):
            for kind, g in got.items():
                n[kind] += tie_rule(g[rows, :, c], e, f"K1 {kind} {'rgb'[c]}")
    return n


@pytest.mark.parametrize("rng", ["limited", "full"])
def test_k1_420_block_triples(rng):
    """orc_yuv420_to_rgba limited / full and orc_nv12_to_rgba on the four block frames: every (Y, U, V) with the chroma
    delivered exactly, and the interpolated chroma of every block edge"""
    seen = np.zeros(N, bool)
    n = {}
    for part in range(4):
        planes, cov = yuv420_block_triples(part)
        seen |= cov
        for k, v in _check_420(rng, planes).items():
            n[k] = n.get(k, 0) + v
    assert coverage(seen) == N
    report(f"K1 {rng} range block frames, bytes off rint(float64)", n)


@pytest.mark.parametrize("rng", ["limited", "full"])
def test_k1_420_chroma_sums(rng):
    """the same converters on the chroma-sum frame: every interpolated chroma value n / 16 with every Y on both channels"""
    planes, cov = yuv420_chroma_sums()
    assert cov["u"] == cov["v"] == 256 * 4081 and cov["uv"] == 256 * 4081, cov
    report(f"K1 {rng} range chroma sums, bytes off rint(float64)", _check_420(rng, planes))


@pytest.mark.parametrize("yuyv", [0, 1], ids=["uyvy", "yuyv"])
def test_k3_interleaved_every_triple(yuyv):
    """orc_interleaved422_to_rgba on every (Y, U, V): pixel x takes texel x div 2 and its luma x mod 2"""
    t, n = interleaved_all_triples(yuyv)
    assert n == N
    got = orc.interleaved422_to_rgba(t, SIDE, SIDE, yuyv)
    y, u, v = interleaved_planes(t, yuyv)
    counts = {}
    for r0 in range(0, SIDE, CHUNK):
        sl = slice(r0, r0 + CHUNK)
        for c, e in enumerate(k1_rgb(y[sl] / 255.0, u[sl] / 255.0, v[sl] / 255.0, False)):
            counts["rgb"[c]] = counts.get("rgb"[c], 0) + tie_rule(got[sl, :, c], e, f"K3 {'rgb'[c]}")
    report(f"K3 {'yuyv' if yuyv else 'uyvy'}, bytes off rint(float64)", counts)


def test_k10_444_every_colour():
    """orc_rgba_to_yuv_planar_scaled at 4:4:4 (every plane at the source's size) on every (r, g, b)"""
    rgba, n = rgb_all_triples()
    assert n == N
    y, u, v = orc.rgba_to_yuv_planar_scaled(rgba, SIDE, SIDE, SIDE, SIDE)
    counts = {"y": 0, "u": 0, "v": 0}
    for r0 in range(0, SIDE, CHUNK):
        sl = slice(r0, r0 + CHUNK)
        f = rgba[sl, :, :3] / 255.0
        counts["y"] += tie_rule(y[sl], k10_y(f[..., 0], f[..., 1], f[..., 2]), "K10 4:4:4 Y'")
        eu, ev = k10_uv(f[..., 0], f[..., 1], f[..., 2])
        counts["u"] += tie_rule(u[sl], eu, "K10 4:4:4 U'")
        counts["v"] += tie_rule(v[sl], ev, "K10 4:4:4 V'")
    report("K10 4:4:4, bytes off rint(float64)", counts)


def _check_k11(fmt, rgba):
    if fmt == "nv12":
        y, uv = orc.rgba_to_nv12(rgba)
        u, v = uv[..., 0], uv[..., 1]
    else:
        y, u, v = orc.rgba_to_yuv420(rgba)
    ey, eu, ev = k11_frame_420(rgba)
    return {"y": tie_rule(y, ey, f"K11 {fmt} Y'"), "u": tie_rule(u, eu, f"K11 {fmt} U'"), "v": tie_rule(v, ev, f"K11 {fmt} V'")}


@pytest.mark.parametrize("fmt", ["yuv420", "nv12"])
def test_k11_420_block_colours(fmt):
    """orc_rgba_to_yuv420 / orc_rgba_to_nv12 on the four constant-block frames (the chroma of every colour as a 2 x 2
    mean) and on the every-colour frame (2 x 2 means of four different colours)"""
    seen = np.zeros(N, bool)
    counts = {}
    frames = [rgb_block_triples(p) for p in range(4)]
    for rgba, cov in frames:
        seen |= cov
        for k, n in _check_k11(fmt, rgba).items():
            counts[k] = counts.get(k, 0) + n
    del frames
    assert coverage(seen) == N
    rgba, _ = rgb_all_triples()
    for k, n in _check_k11(fmt, rgba).items():
        counts["mixed " + k] = n
    report(f"K11 {fmt}, bytes off rint(float64)", counts)


def test_black_fill_bytes():
    """orc_rgb_to_yuv_bytes (the fill colour, RGBColor::to_yuv) on black, white, the primaries, every near-tie colour
    of its own float64 value and a 52^3 grid"""
    r, g, b = all_triples()
    ey, eu, ev = to_yuv(r, g, b)
    near = (tie_distance(ey) < TIE_DELTA) | (tie_distance(eu) < TIE_DELTA) | (tie_distance(ev) < TIE_DELTA)
    grid = ((r % 5 == 0) & (g % 5 == 0) & (b % 5 == 0))
    idx = np.flatnonzero(near | grid)
    assert near.any() and len(idx) > 140000
    got = np.array([orc.rgb_to_yuv_bytes(int(r[i]), int(g[i]), int(b[i])) for i in idx], np.uint8)
    counts = {k: tie_rule(got[:, c], e[idx], f"to_yuv {k}") for c, (k, e) in enumerate(zip("yuv", (ey, eu, ev)))}
    assert orc.rgb_to_yuv_bytes(0, 0, 0) == (16, 128, 128)
    report(f"to_yuv over {len(idx)} colours ({int(near.sum())} near ties), bytes off rint(float64)", counts)
