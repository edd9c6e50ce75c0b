"""Pins the CPU oracle against every known-answer vector the reference tree physically holds for
the compositor path (SURVEY.md section 8c).  CPU-only (`-m "not gpu"`)."""
import numpy as np
import pytest

from oracle import oracle as orc


# ---- integration-tests/src/render_tests/yuv_tests.rs:32-132 -----------------------------------
GRADIENT_YUV_EXPECTED = [
    89, 0, 0, 255, 100, 5, 3, 255, 160, 0, 0, 255, 165, 2, 0, 255, 204, 0, 0, 255, 207, 1, 0, 255, 239, 0, 0, 255, 241, 1, 0, 255,
    89, 0, 0, 255, 100, 5, 3, 255, 160, 0, 0, 255, 165, 2, 0, 255, 204, 0, 0, 255, 207, 1, 0, 255, 239, 0, 0, 255, 241, 1, 0, 255,
]
GRADIENT_RGBA_EXPECTED = [
    71, 0, 0, 255, 120, 0, 0, 255, 152, 0, 0, 255, 177, 0, 0, 255, 198, 0, 0, 255, 216, 0, 0, 255, 233, 0, 0, 255, 248, 0, 0, 255,
    71, 0, 0, 255, 120, 0, 0, 255, 152, 0, 0, 255, 177, 0, 0, 255, 198, 0, 0, 255, 216, 0, 0, 255, 233, 0, 0, 255, 248, 0, 0, 255,
]
UNIFORM_YUV_EXPECTED = [49, 0, 0, 255] * 16
UNIFORM_RGBA_EXPECTED = [50, 0, 0, 255] * 16


def _gradient_node_texture():
    """What the shader node of yuv_test_gradient leaves in its Rgba8UnormSrgb target: the fragment
    returns vec4(tex_coords.x, 0, 0, 1) with tex_coords.x = (i + .5)/8; the store encodes sRGB."""
    w, h = 8, 2
    img = np.zeros((h, w, 4), np.uint8)
    for i in range(w):
        lin = np.float32((i + 0.5) / 8.0)
        img[:, i] = (orc.lib().orc_srgb_encode_u8(lin), orc.lib().orc_srgb_encode_u8(0.0),
                     orc.lib().orc_srgb_encode_u8(0.0), orc.lib().orc_unorm8(1.0))
    return img


def test_yuv_test_gradient_rgba():
    img = _gradient_node_texture()
    assert img.reshape(-1).tolist() == GRADIENT_RGBA_EXPECTED  # reference tolerance is +-2; we are exact


def test_yuv_test_gradient_yuv_roundtrip():
    img = _gradient_node_texture()
    y, u, v = orc.rgba_to_yuv420(img)
    back = orc.harness_yuv420_to_rgba(y, u, v, 8, 2)
    diff = np.abs(back.reshape(-1).astype(int) - np.array(GRADIENT_YUV_EXPECTED))
    assert diff.max() <= 2, (back.reshape(-1).tolist(), GRADIENT_YUV_EXPECTED)  # yuv_tests.rs:25
    assert diff.max() == 0  # and in fact identical


def _uniform_color_scene(mode):
    # View{background_color: (50,0,0,255)} at 8x2 flattens to one Color layout covering the output
    L = orc.make_layout(orc.LAYOUT_COLOR, 0, 0, 8, 2, color=(50, 0, 0, 255))
    return orc.apply_layouts(8, 2, [L], [None], mode=mode)


@pytest.mark.parametrize("mode", [orc.MODE_GPU_OPTIMIZED, orc.MODE_CPU_OPTIMIZED])
def test_yuv_test_uniform_color(mode):
    img = _uniform_color_scene(mode)
    assert img.reshape(-1).tolist() == UNIFORM_RGBA_EXPECTED
    y, u, v = orc.rgba_to_yuv420(img)
    back = orc.harness_yuv420_to_rgba(y, u, v, 8, 2)
    assert back.reshape(-1).tolist() == UNIFORM_YUV_EXPECTED


# ---- integration-tests/src/render_tests/pixel_input_format_tests.rs:31-152 --------------------
def _through_default_view(node, mode=orc.MODE_GPU_OPTIMIZED):
    """View{children:[InputStream]} at 8x2: transparent Color layout is culled, the child is a
    Texture layout at (0,0) 8x2 with crop = whole texture and the View's overflow-hidden mask
    (dropped by fix_final_render_layout because it contains the layout)."""
    L = orc.make_layout(orc.LAYOUT_TEXTURE, 0, 0, 8, 2, child_index=0, crop=(0, 0, 8, 2))
    return orc.render_layout_node(8, 2, [L], [node], mode=mode)


def test_bgra_pixel_format_input():
    data = np.arange(1, 65, dtype=np.uint8)
    node = orc.bgra_to_rgba(data, 8, 2)
    out = _through_default_view(node)
    exp = []
    for p in range(16):
        b, g, r, a = data[p * 4:p * 4 + 4]
        exp += [r, g, b, a]
    assert out.reshape(-1).tolist() == [int(x) for x in exp]


def test_argb_pixel_format_input():
    data = np.arange(1, 65, dtype=np.uint8)
    node = orc.argb_to_rgba(data, 8, 2)
    out = _through_default_view(node)
    exp = []
    for p in range(16):
        a, r, g, b = data[p * 4:p * 4 + 4]
        exp += [r, g, b, a]
    assert out.reshape(-1).tolist() == [int(x) for x in exp]


# ---- smelter-render/src/transformations/layout/resampler.rs:402-468 ---------------------------
H, V = 0, 1


def test_plans_a_pass_for_every_non_direct_axis():
    assert orc.plan_passes(0.0, 0.0, 640.0, 360.0, 640, 360) == []
    assert orc.plan_passes(100.0, 40.0, 640.0, 360.0, 640, 360) == []
    assert orc.plan_passes(100.0, 0.0, 640.0, 360.0, 640, 300) == [(V, 100)]
    assert orc.plan_passes(0.0, 42.0, 640.0, 360.0, 320, 360) == [(H, 42)]
    frac = orc.plan_passes(100.5, 0.0, 640.0, 360.0, 640, 300)
    assert len(frac) == 2
    sep = orc.plan_passes(0.0, 0.0, 1920.0, 1080.0, 960, 270)
    assert [a for a, _ in sep] == [V, H]


def test_degenerate_scales_do_not_overflow_predecimation():
    assert orc.predecimate_levels(float("inf"), 10) == 16
    assert orc.predecimate_levels(float("nan"), 10) == 0


def test_predecimation_budget():
    # KERNEL_BUDGET = 4 (resampler.rs:19): ratios <= 4 use the kernel alone
    assert orc.predecimate_levels(3840.0, 960) == 0
    assert orc.predecimate_levels(3840.0, 959) == 1
    assert orc.predecimate_levels(7680.0, 480) == 2


# ---- numeric-contract self checks --------------------------------------------------------------
def test_srgb_roundtrip_is_identity():
    L = orc.lib()
    for b in range(256):
        assert L.orc_srgb_encode_u8(L.orc_srgb_decode_u8(b)) == b


def test_f16_matches_numpy():
    L = orc.lib()
    rng = np.random.default_rng(1)
    xs = np.concatenate([rng.standard_normal(2000).astype(np.float32) * 2,
                         (rng.random(2000).astype(np.float32) * 1e-4),
                         np.array([0, -0.0, 1, 65504, 65519.9, 65520, 1e-8, 5.96e-8, 2.98e-8, 6.1e-5], np.float32)])
    for x in xs:
        h = L.orc_f32_to_f16(float(x))
        ref = np.float32(x).astype(np.float16)
        assert h == ref.view(np.uint16), (x, h, ref.view(np.uint16))
        if np.isfinite(ref):
            assert L.orc_f16_to_f32(h) == np.float32(ref)


def test_lanczos_weights_scale4_single_phase():
    # config 3 (3840 -> 960): every output coordinate has the same 25-tap kernel, last tap is 0
    f0, w0, s0 = orc.resample_weights(4.0, 0.0, 0)
    f7, w7, s7 = orc.resample_weights(4.0, 0.0, 7)
    assert len(w0) == 25 and f0 == -10 and f7 == 18
    assert np.array_equal(w0, w7) and s0 == s7
    assert w0[24] == 0.0 and abs(s0 - 4.0) < 0.02
    # symmetric kernel around its centre within float noise of the rotation recurrence
    assert np.allclose(w0[:24], w0[:24][::-1], atol=2e-6)


def test_lanczos_identity_at_unit_scale():
    f, w, s = orc.resample_weights(1.0, 0.0, 5)
    # centre = 5: tap at x=0 has weight 1, the others sit on the zeros of the sinc
    assert f == 2 and len(w) == 7
    assert w[3] == 1.0 and np.abs(np.delete(w, 3)).max() < 1e-6


def test_black_frame_bytes():
    # render_loop.rs:127-139 fills with RGBColor::BLACK.to_yuv()
    assert orc.rgb_to_yuv_bytes(0, 0, 0) == (16, 128, 128)


def test_chroma_upsample_phase_is_quarter():
    """K1 on even sizes: taps .25/.75 exactly (SURVEY appendix A) for every x of every even width
    the renderer can see -- the CUDA kernels hard-code this phase."""
    y = np.full((2, 16), 100, np.uint8)
    u = np.full((1, 8), 128, np.uint8)
    v = np.full((1, 8), 128, np.uint8)
    u[0, 3] = 160
    rgba = orc.yuv420_to_rgba(y, u, v, 16, 2)
    # b channel follows u: pixels 6,7 (chroma texel 3) get .75 weight, 5 and 8 get .25
    b = rgba[0, :, 2].astype(int)
    assert b[6] == b[7] and b[5] == b[8] and b[4] == b[9] and b[6] > b[5] > b[4]


def max_frame_dim():
    """the largest input frame side the renderer accepts: kMaxFrameDim, the bound frame_size_ok checks"""
    import os
    import re
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "smelter_b200", "csrc",
                            "renderer.cpp")).read()
    dim = int(re.search(r"constexpr uint32_t kMaxFrameDim = (\d+);", src).group(1))
    body = re.search(r"static bool frame_size_ok\(const smr_input_frame &f\) \{([^}]*)\}", src).group(1)
    assert body.count("kMaxFrameDim") == 2 and not re.search(r"\d{3,}", body), body
    return dim


def test_even_size_sampler_phases_exhaustive():
    """The CUDA fast paths hard-code the NC-6 taps for even plane sizes; prove the generic formula the
    oracle evaluates gives exactly those taps for EVERY even size the renderer accepts and every coordinate."""
    import ctypes as C
    L = orc.lib()
    L.orc_check_even_size_phases.restype = C.c_long
    assert L.orc_check_even_size_phases(max_frame_dim()) == 0


def test_wide_chroma_restatements_are_consistent():
    """No reference KAT exists for 4:2:2 / 4:4:4 / interleaved frames (parity for them is pinned only through the
    arithmetic they share with the KAT-pinned 4:2:0 path).  Internal consistency of the restatement:
    UYVY == YUYV of the same samples; interleaved (texel-centre chroma) == planar 4:4:4 with the chroma columns
    duplicated; the general planar converter with (w/2, h/2) chroma == the 4:2:0 one; 4:4:4 / 4:2:2 outputs of a
    flat colour == the 4:2:0 bytes."""
    rng = np.random.default_rng(3)
    w, h = 24, 10
    y = rng.integers(16, 236, (h, w), dtype=np.uint8)
    u = rng.integers(16, 241, (h, w // 2), dtype=np.uint8)
    v = rng.integers(16, 241, (h, w // 2), dtype=np.uint8)
    uy = np.empty((h, w // 2, 4), np.uint8)
    uy[..., 0], uy[..., 1], uy[..., 2], uy[..., 3] = u, y[:, 0::2], v, y[:, 1::2]
    yu = np.empty((h, w // 2, 4), np.uint8)
    yu[..., 0], yu[..., 1], yu[..., 2], yu[..., 3] = y[:, 0::2], u, y[:, 1::2], v
    a = orc.interleaved422_to_rgba(uy, w, h, False)
    assert np.array_equal(a, orc.interleaved422_to_rgba(yu, w, h, True))
    assert np.array_equal(a, orc.yuv_planar_to_rgba(y, np.repeat(u, 2, 1), np.repeat(v, 2, 1), w, h, w, h))
    assert np.array_equal(orc.yuv_planar_to_rgba(y, u[::2], v[::2], w, h, w // 2, h // 2),
                          orc.yuv420_to_rgba(y, u[::2], v[::2], w, h))
    # 4:2:2 input: chroma rows are exact, columns interpolate like 4:2:0 -> equals 4:2:0 applied to row-duplicated luma
    flat = np.empty((h, w, 4), np.uint8)
    flat[...] = (200, 40, 90, 255)
    y0, u0, v0 = orc.rgba_to_yuv420_scaled(flat, w, h)
    for cw, ch in ((w // 2, h), (w, h)):
        y1, u1, v1 = orc.rgba_to_yuv_planar_scaled(flat, w, h, cw, ch)
        assert np.array_equal(y0, y1) and u1.shape == (ch, cw)
        assert len(np.unique(u1)) == 1 and u1[0, 0] == u0[0, 0] and v1[0, 0] == v0[0, 0]


def _f32(x):
    return np.float32(x)


def test_interleaved_shader_restated_in_python_floats():
    """interleaved_uyvy_to_rgba.wgsl:24-61 re-derived step by step with numpy float32 scalars (an implementation
    independent of the C restatement) on a small frame, including the column-index round trip of the shader and the
    widths where it degenerates (w = 2: both pixels read the first luma)."""
    rng = np.random.default_rng(12)
    for w, h in ((12, 3), (6, 2), (2, 2)):
        dimx = w // 2
        data = rng.integers(16, 236, (h, dimx, 4), dtype=np.uint8)
        got = orc.interleaved422_to_rgba(data, w, h, False)
        for py in range(h):
            for px in range(w):
                tx = _f32(_f32(px + 0.5) / _f32(w))
                hpw = _f32(_f32(0.5) / _f32(dimx))
                xf = _f32(_f32(_f32(_f32(tx * _f32(dimx)) - hpw) + _f32(0.0001)) * _f32(2.0))
                x_pos = int(xf) if xf > 0 else 0
                tcx = _f32(_f32(_f32(x_pos // 2) / _f32(dimx)) + hpw)
                c = _f32(_f32(tcx * _f32(dimx)) - _f32(0.5))              # texel-space coordinate of the sample
                i0 = int(np.floor(c)); frac = _f32(c - _f32(np.floor(c)))
                wq = int(np.rint(frac * _f32(256.0)))                      # NC-6: 8-bit weight
                assert wq in (0, 256), "the sample must land on a texel centre"
                tex = data[py, min(max(i0 + (wq == 256), 0), dimx - 1)]
                u, y0, v, y1 = [_f32(_f32(t) / _f32(255.0)) for t in tex]
                y = y1 if x_pos % 2 else y0
                k16, rcy, rcc = _f32(_f32(16.0) / _f32(255.0)), _f32(_f32(1.0) / _f32(0.85882352941)), _f32(_f32(1.0) / _f32(0.87843137254))
                cl = lambda t: min(max(t, _f32(0.0)), _f32(1.0))
                y = cl(_f32(_f32(y - k16) * rcy)); u = cl(_f32(_f32(u - k16) * rcc)); v = cl(_f32(_f32(v - k16) * rcc))
                um, vm = _f32(u - _f32(0.5)), _f32(v - _f32(0.5))
                fma = lambda a, b, cc: _f32(np.float64(a) * np.float64(b) + np.float64(cc))   # exact product, one rounding
                r = fma(_f32(1.5748), vm, y)
                g = fma(_f32(-0.4681), vm, fma(_f32(-0.1873), um, y))
                b = fma(_f32(1.8556), um, y)
                exp = [int(np.rint(cl(t) * _f32(255.0))) for t in (r, g, b)] + [255]
                assert got[py, px].tolist() == exp, (w, px, py)


def test_frame_pre_processor_rescale_restated_in_integers():
    """rgba_rescale.wgsl through a plain Rgba8Unorm target (CpuOptimized): every output byte is the correctly rounded
    value of the exact fixed-point bilinear filter (NC-6u) -- re-derived here with Python integers and Fractions."""
    from fractions import Fraction
    rng = np.random.default_rng(4)
    sw, sh, ow, oh = 9, 7, 5, 11
    src = rng.integers(0, 256, (sh, sw, 4), dtype=np.uint8)
    got = orc.rescale_rgba(src, ow, oh, mode=1)

    def tap(o, n_out, n_src):
        c = _f32(_f32(_f32(_f32(o + 0.5) / _f32(n_out)) * _f32(n_src)) - _f32(0.5))
        fl = int(np.floor(c)); w = int(np.rint(_f32(c - _f32(fl)) * _f32(256.0)))
        return min(max(fl, 0), n_src - 1), min(max(fl + 1, 0), n_src - 1), w

    for y in range(oh):
        y0, y1, wy = tap(y, oh, sh)
        for x in range(ow):
            x0, x1, wx = tap(x, ow, sw)
            for c in range(4):
                n = (int(src[y0, x0, c]) * (256 - wx) + int(src[y0, x1, c]) * wx) * (256 - wy) + \
                    (int(src[y1, x0, c]) * (256 - wx) + int(src[y1, x1, c]) * wx) * wy
                v = float(np.float32(Fraction(n, 255 * 65536)))           # one rounding to f32
                assert got[y, x, c] == int(np.rint(np.float32(v) * np.float32(255.0))), (x, y, c)
