"""Parity tests proper: the CUDA path (through the C ABI) against the CPU oracle, BIT-EXACT on every
output byte, on scenes re-typed from the reference's render tests
(integration-tests/src/render_tests/{simple,tiles,view,rescaler,transition}.rs) with the reference's
procedural inputs (harness/input.rs).  Run with `-m gpu` on an H100."""
import numpy as np
import pytest

import smelter_b200 as s
from tests import harness
from tests.parity import OUTPUT_ID, TrackedRenderer, assert_identical, nv12_frame, run_case, wide_chroma_frame, yuv_frame

pytestmark = pytest.mark.gpu

RES = s.Resolution(640, 360)
BG = s.RGBAColor(0x33, 0x33, 0x33, 255)
V = s.ViewComponent
YUV = s.OutputFrameFormat.PlanarYuv420Bytes
NV12 = s.OutputFrameFormat.Nv12WgpuTexture
RGBA = s.OutputFrameFormat.RgbaWgpuTexture


def inputs(n, w=640, h=360):
    return {f"input_{i}": yuv_frame(harness.test_input(i, w, h), w, h) for i in range(1, n + 1)}


def streams(n):
    return [s.InputStreamComponent(input_id=f"input_{i}") for i in range(1, n + 1)]


def check(scene, frames, **kw):
    got, exp, r = run_case(scene, frames, **kw)
    assert_identical(got, exp, type(scene).__name__)
    return r


def test_library_is_the_cuda_path():
    r = s.Renderer()
    assert r.cuda_stream() is not None
    st = r.stats()
    assert st["kernel_launches"] == 0


def test_simple_input_pass_through():
    """simple.rs:18-30"""
    r = check(V(children=streams(1)), inputs(1))
    assert r.stats()["last_render_kernel_launches"] >= 1


@pytest.mark.parametrize("fmt", [YUV, NV12, RGBA])
def test_tiles_02_inputs_all_output_formats(fmt):
    """tiles.rs:85-95 == BASELINE config 1 (2:1 Lanczos3, 13 taps/axis)"""
    check(s.TilesComponent(children=streams(2), background_color=BG), inputs(2), out_format=fmt)


@pytest.mark.parametrize("n", [1, 3, 4, 5, 15])
def test_tiles_n_inputs(n):
    """tiles.rs:73-143"""
    check(s.TilesComponent(children=streams(n), background_color=BG), inputs(n))


def test_tiles_portrait_inputs_with_margin_and_padding():
    """tiles.rs portrait + margin/padding cases: non-integer tile geometry -> fractional Lanczos phases"""
    fr = {f"input_{i}": yuv_frame(harness.test_input(i, 360, 640), 360, 640) for i in range(1, 4)}
    check(s.TilesComponent(children=streams(3), background_color=BG, tile_aspect_ratio=(1, 2), margin=7.0,
                           padding=3.0, horizontal_align=s.HorizontalAlign.Left,
                           vertical_align=s.VerticalAlign.Top), fr)


def test_nv12_input_and_output():
    fr = {f"input_{i}": nv12_frame(harness.smooth_yuv420(i, 640, 360), 640, 360) for i in range(1, 5)}
    check(s.TilesComponent(children=streams(4), background_color=BG), fr, out_format=NV12)


def test_full_range_j420_input():
    y, u, v = harness.random_yuv420(7, 320, 180)
    fr = {"input_1": s.Frame(s.FrameData.PlanarYuvJ420(s.YuvPlanes(y, u, v)), s.Resolution(320, 180))}
    check(V(children=streams(1), background_color=BG), fr, resolution=s.Resolution(320, 180))


def test_random_noise_input_2to1():
    """white-noise planes exercise every rounding boundary of K1 / Lanczos / K10"""
    fr = {f"input_{i}": yuv_frame(harness.random_yuv420(100 + i, 640, 360), 640, 360) for i in range(1, 5)}
    check(s.TilesComponent(children=streams(4), background_color=BG), fr)


def test_root_input_stream_same_size_and_rescaled():
    """pass-through root (BASELINE `single_video_pass_through`): K1 -> K10 only; a root whose size differs
    from the output is stretched by the converter's sampler (render_loop.rs:68-73)"""
    fr = inputs(1)
    check(s.InputStreamComponent(input_id="input_1"), fr)
    check(s.InputStreamComponent(input_id="input_1"), fr, resolution=s.Resolution(320, 200))
    check(s.InputStreamComponent(input_id="input_1"), fr, resolution=s.Resolution(854, 480), out_format=NV12)


def test_missing_frame_gives_black_and_culls_layer():
    """render_loop.rs:24-32,127-139"""
    r = s.Renderer()
    r.register_input("input_1")
    r.update_scene(OUTPUT_ID, RES, YUV, s.InputStreamComponent(input_id="input_1"))
    out = r.render(s.FrameSet(pts=0.0)).frames[OUTPUT_ID]
    y, u, v = out.data.planes
    assert np.all(y == 16) and np.all(u == 128) and np.all(v == 128)
    # missing input inside Tiles: slot reserved, nothing drawn there
    fr = inputs(1)
    r2 = TrackedRenderer()
    for i in (1, 2):
        r2.register_input(f"input_{i}")
    scene = s.TilesComponent(children=streams(2), background_color=BG)
    r2.update_scene(OUTPUT_ID, RES, YUV, scene)
    got, exp, _ = run_case(scene, fr, renderer=r2)
    assert_identical(got, exp, "tiles with a missing input")


def test_stale_frame_is_dropped():
    fr = {"input_1": yuv_frame(harness.test_input(1), 640, 360, pts=1.0)}
    scene = s.TilesComponent(children=streams(1), background_color=BG)
    got, exp, _ = run_case(scene, fr, pts=4.5)  # 4.5 - 3.0 > 1.0 -> stale
    assert_identical(got, exp, "stale")
    assert len(np.unique(got[0])) == 1  # only the background


def test_view_background_borders_radius_shadow():
    """view.rs border_radius / border_width / box_shadow cases"""
    sh = [s.BoxShadow(offset_x=12.0, offset_y=18.0, blur_radius=20.0, color=s.RGBAColor(0, 0, 0, 200)),
          s.BoxShadow(offset_x=-15.0, offset_y=-10.0, blur_radius=6.0, color=s.RGBAColor(0, 255, 0, 255))]
    child = V(position=s.Position.Absolute(width=300.0, height=180.0, left=150.0, top=80.0),
              background_color=s.RGBAColor(255, 0, 0, 255), border_radius=s.BorderRadius(50.0, 10.0, 30.0, 0.0),
              border_width=12.0, border_color=s.RGBAColor(255, 255, 255, 180), box_shadow=sh)
    check(V(children=[child], background_color=BG), {})


def test_view_video_child_with_radius_border_and_overflow_mask():
    """view.rs: rounded video with border inside a rounded, padded parent (nested masks, asymmetric radii)"""
    inner = V(children=streams(1), position=s.Position.Static(width=320.0, height=180.0),
              border_radius=s.BorderRadius(40.0, 8.0, 24.0, 60.0), border_width=6.0,
              border_color=s.RGBAColor(255, 255, 0, 255))
    outer = V(children=[inner], position=s.Position.Absolute(width=400.0, height=260.0, left=120.0, top=50.0),
              border_radius=s.BorderRadius(80.0, 20.0, 50.0, 10.0), padding=s.Padding(10, 10, 10, 120),
              background_color=s.RGBAColor(0, 0, 255, 128))
    check(V(children=[outer], background_color=BG), inputs(1))


def test_semi_transparent_overlay_and_zorder():
    """view.rs:514-574 absolute children over siblings + alpha overlay (BASELINE config 3 ingredients)"""
    kids = [s.RescalerComponent(child=streams(2)[0]), ]
    over = V(position=s.Position.Absolute(width=400.0, height=120.0, left=60.0, bottom=30.0),
             background_color=s.RGBAColor(20, 40, 200, 110), border_radius=s.BorderRadius.new_with_radius(30.0))
    over2 = V(position=s.Position.Absolute(width=200.0, height=200.0, right=20.0, top=20.0),
              children=[s.RescalerComponent(child=streams(2)[1])], border_width=4.0,
              border_color=s.RGBAColor(255, 255, 255, 255))
    check(V(children=kids + [over, over2], background_color=BG), inputs(2))


@pytest.mark.parametrize("mode", [s.RenderingMode.GpuOptimized, s.RenderingMode.CpuOptimized])
def test_stacked_translucent_colour_layers(mode):
    """six overlapping translucent colour views (more than the per-tile blend tables of k_composite) with and
    without radius / border over a video: table path, its overflow to the general path, and both blend modes"""
    kids = [s.RescalerComponent(child=streams(1)[0])]
    for k in range(6):
        kids.append(V(position=s.Position.Absolute(width=360.0 - 30 * k, height=200.0 - 12 * k, left=40.0 + 37 * k,
                                                   top=20.0 + 21 * k),
                      background_color=s.RGBAColor(40 * k, 255 - 35 * k, 90 + 20 * k, 60 + 30 * k),
                      border_radius=s.BorderRadius.new_with_radius(0.0 if k % 2 else 18.0 + k),
                      border_width=3.0 if k == 2 else 0.0, border_color=s.RGBAColor(255, 255, 255, 128)))
    check(V(children=kids, background_color=BG), inputs(1), mode=mode)


@pytest.mark.parametrize("mode_fit", [s.RescaleMode.Fit, s.RescaleMode.Fill])
def test_rescaler_modes_and_alignment(mode_fit):
    """rescaler.rs fit/fill with alignment, border, radius, shadow"""
    resc = s.RescalerComponent(child=streams(1)[0], mode=mode_fit, horizontal_align=s.HorizontalAlign.Right,
                               vertical_align=s.VerticalAlign.Top, border_width=8.0,
                               border_color=s.RGBAColor(255, 0, 255, 255),
                               border_radius=s.BorderRadius.new_with_radius(36.0),
                               box_shadow=[s.BoxShadow(8.0, 8.0, 12.0, s.RGBAColor(0, 0, 0, 255))],
                               position=s.Position.Absolute(width=300.0, height=260.0, left=170.0, top=50.0))
    check(V(children=[resc], background_color=BG), inputs(1))


def test_rescaler_upscale_and_view_subtree():
    """rescaler.rs:76-187: a View subtree rescaled (scale propagates through flatten_child), incl. an
    upscaled video (kernel_scale = 1, 7 taps)"""
    inner = V(position=s.Position.Static(width=320.0, height=180.0), background_color=s.RGBAColor(200, 30, 30, 255),
              border_width=10.0, border_color=s.RGBAColor(250, 250, 250, 255), direction=s.ViewChildrenDirection.Row,
              children=[V(children=streams(1), position=s.Position.Static(width=160.0)),
                        V(background_color=s.RGBAColor(0, 200, 0, 255))])
    fr = {"input_1": yuv_frame(harness.test_input(1, 160, 90), 160, 90)}
    check(s.RescalerComponent(child=inner), fr)


def test_scaling_filter_lanczos3_multiscale_grid():
    """rescaler.rs:838-859 at a reduced size: multiscale grid, 3:1 (19 taps, no box pre-pass)"""
    w, h = 1920, 1080
    fr = {"input_1": yuv_frame(harness.multiscale_grid(w, h), w, h)}
    check(s.RescalerComponent(child=streams(1)[0]), fr, resolution=s.Resolution(640, 360))


def test_box_predecimation_above_4x():
    """resampler.rs:56-58: 1920 -> 300 is 6.4:1 -> one 2x box level, then Lanczos on the reduced source;
    the other axis (1080 -> 270 = 4:1) stays unreduced"""
    w, h = 1920, 1080
    fr = {"input_1": yuv_frame(harness.smooth_yuv420(3, w, h), w, h)}
    resc = s.RescalerComponent(child=V(children=streams(1), position=s.Position.Static(width=1920.0, height=1080.0)),
                               mode=s.RescaleMode.Fill,
                               position=s.Position.Absolute(width=300.0, height=270.0, left=20.0, top=20.0))
    # Fill keeps aspect; use a plain View with explicit stretch instead to get anisotropic ratios
    stretch = V(children=[s.InputStreamComponent(input_id="input_1")], overflow=s.Overflow.Fit,
                position=s.Position.Absolute(width=300.0, height=270.0, left=20.0, top=20.0))
    check(V(children=[resc], background_color=BG), fr)
    check(V(children=[stretch], background_color=BG), fr)


@pytest.mark.parametrize("kind", ["nv12", "yuv420"])
@pytest.mark.parametrize("geom", [(384, 216, 0.0, 0.0), (320, 180, 0.0, 0.0), (240, 135, 0.0, 0.0), (256, 144, 37.0, 21.0), (272, 153, 7.0, 13.0)])
def test_box_reduced_source_in_the_fused_kernel(kind, geom):
    """resampler.rs:56-67 + downsample.wgsl:28-41 with one box level on BOTH axes (ratios in (4, 8]): the any-ratio TMA
    kernel reduces the source 2:1 on the fly (k_resample_tma0<.., BOX>): 5:1, 6:1, 8:1 (the last ratio with one level), 7.5:1
    and the fractional 7.06:1.  Noise input, so that every tap matters; the image edges exercise the clamp of the REDUCED
    texture.  Checked: bytes against the oracle, and that no generic pass ran."""
    dw, dh, left, top = geom
    w, h = 1920, 1080
    mk = nv12_frame if kind == "nv12" else yuv_frame
    fr = {"input_1": mk(harness.random_yuv420(700 + dw, w, h), w, h)}
    layer = s.RescalerComponent(child=s.InputStreamComponent(input_id="input_1"),
                                position=s.Position.Absolute(width=float(dw), height=float(dh), left=left, top=top))
    r = TrackedRenderer()
    r.register_input("input_1")
    r.set_profiling(True)
    scene = V(children=[layer], background_color=BG)
    r.update_scene(OUTPUT_ID, RES, YUV, scene)
    got, exp, _ = run_case(scene, fr, renderer=r)
    assert_identical(got, exp, f"box {kind} {geom}")
    kt = r.kernel_times()
    assert kt["resample_fused"][1] >= 1, kt
    assert kt["resample_box"][1] == 0 and kt["resample_first"][1] == 0 and kt["convert"][1] == 0, kt


@pytest.mark.parametrize("pts", [0.25, 0.5, 0.9])
def test_transition_fractional_geometry(pts):
    """transition.rs: mid-transition layouts have fractional position and size -> non-trivial resample
    phases and K9 bilinear taps"""
    def scene(w, left, tr=None):
        return V(background_color=BG, children=[
            s.RescalerComponent(id="r", child=streams(1)[0], transition=tr,
                                position=s.Position.Absolute(width=w, height=w * 9 / 16, left=left, top=33.0))])
    r = TrackedRenderer()
    r.register_input("input_1")
    r.update_scene(OUTPUT_ID, RES, YUV, scene(200.0, 10.0))
    fr = inputs(1)
    run_case(scene(200.0, 10.0), fr, renderer=r, pts=0.0)
    sc2 = scene(517.0, 101.0, s.Transition(duration=1.0, interpolation_kind=s.InterpolationKind.CubicBezier(0.25, 0.1, 0.25, 1.0)))
    r.update_scene(OUTPUT_ID, RES, YUV, sc2)
    got, exp, _ = run_case(sc2, fr, renderer=r, pts=pts)
    assert_identical(got, exp, f"transition pts={pts}")


def test_rotated_absolute_child():
    """apply_layouts.wgsl:95-157 rotation path (no reference snapshot uses it; oracle = NC-7)"""
    child = V(position=s.Position.Absolute(width=260.0, height=120.0, left=190.0, top=110.0, rotation_degrees=27.0),
              background_color=s.RGBAColor(30, 200, 120, 230), border_radius=s.BorderRadius.new_with_radius(25.0),
              border_width=5.0, border_color=s.RGBAColor(255, 255, 255, 255))
    vid = V(position=s.Position.Absolute(width=160.0, height=90.0, left=40.0, top=40.0, rotation_degrees=-12.5),
            children=streams(1))
    fr = {"input_1": yuv_frame(harness.test_input(4, 160, 90), 160, 90)}
    check(V(children=[child, vid], background_color=BG), fr)


def test_cpu_optimized_mode_bilinear():
    """rescaler.rs:814-836 scaling_filter_bilinear + BASELINE config 2 semantics: gamma-space blend,
    bilinear scaling inside K9, no resampler"""
    fr = {f"input_{i}": nv12_frame(harness.smooth_yuv420(20 + i, 640, 360), 640, 360) for i in range(1, 5)}
    over = V(position=s.Position.Absolute(width=300.0, height=100.0, left=170.0, top=130.0),
             background_color=s.RGBAColor(255, 255, 255, 90), border_radius=s.BorderRadius.new_with_radius(18.0))
    scene = V(background_color=BG, children=[s.TilesComponent(children=streams(4), background_color=BG), over])
    check(scene, fr, mode=s.RenderingMode.CpuOptimized, out_format=NV12)


def test_bgra_argb_inputs_reference_kat():
    """pixel_input_format_tests.rs:31-152 through the real CUDA path (RGBA texture output, exact)"""
    data = np.arange(1, 65, dtype=np.uint8)
    for kind, perm in (("Bgra", (2, 1, 0, 3)), ("Argb", (1, 2, 3, 0))):
        fd = getattr(s.FrameData, kind)(data)
        fr = {"input": s.Frame(fd, s.Resolution(8, 2))}
        r = s.Renderer()
        r.register_input("input")
        r.update_scene(OUTPUT_ID, s.Resolution(8, 2), RGBA, V(children=[s.InputStreamComponent(input_id="input")]))
        out = r.render(s.FrameSet(frames=fr, pts=0.0)).frames[OUTPUT_ID].data.planes[0]
        exp = data.reshape(16, 4)[:, perm]
        assert np.array_equal(out.reshape(16, 4), exp)


def test_yuv_uniform_color_reference_kat():
    """yuv_tests.rs:83-132 through the CUDA path"""
    from oracle import oracle as orc
    scene = V(background_color=s.RGBAColor(50, 0, 0, 255))
    r = s.Renderer()
    r.update_scene(OUTPUT_ID, s.Resolution(8, 2), RGBA, scene)
    rgba = r.render(s.FrameSet(pts=0.0)).frames[OUTPUT_ID].data.planes[0]
    assert rgba.reshape(-1).tolist() == [50, 0, 0, 255] * 16
    r.update_scene(OUTPUT_ID, s.Resolution(8, 2), YUV, scene)
    y, u, v = r.render(s.FrameSet(pts=0.0)).frames[OUTPUT_ID].data.planes
    back = orc.harness_yuv420_to_rgba(y, u, v, 8, 2)
    assert back.reshape(-1).tolist() == [49, 0, 0, 255] * 16


def test_odd_output_size_uses_general_converter():
    fr = inputs(2)
    check(s.TilesComponent(children=streams(2), background_color=BG), fr, resolution=s.Resolution(641, 359))


def test_max_layouts_count_truncates():
    """params.rs:176-182 / shader.rs:152: layouts beyond max_layouts_count are skipped"""
    kids = [V(position=s.Position.Absolute(width=30.0, height=30.0, left=10.0 + 25 * i, top=20.0 + 9 * i),
              background_color=s.RGBAColor(40 * i % 256, 255 - 30 * i % 256, 90, 255)) for i in range(12)]
    check(V(children=kids, background_color=BG), {}, max_layouts=6)


def test_two_outputs_share_an_input():
    """render_loop.rs:232-236: outputs are independent; inputs are shared read-only state"""
    fr = inputs(2)
    r = s.Renderer()
    for i in fr:
        r.register_input(i)
    sc1 = s.TilesComponent(children=streams(2), background_color=BG)
    sc2 = V(children=[s.RescalerComponent(child=streams(2)[1])], background_color=BG)
    r.update_scene("output_1", RES, YUV, sc1)
    r.update_scene("output_2", s.Resolution(320, 180), NV12, sc2)
    out = r.render(s.FrameSet(frames=fr, pts=0.0))
    got1, exp1, _ = run_case(sc1, fr)
    assert_identical([np.asarray(p) for p in out.frames["output_1"].data.planes], exp1, "output_1")
    got2, exp2, _ = run_case(sc2, fr, resolution=s.Resolution(320, 180), out_format=NV12)
    assert_identical([np.asarray(p) for p in out.frames["output_2"].data.planes], exp2, "output_2")


def test_full_size_config3_properties():
    """BASELINE config 3 at full size (16 x 4K -> 4K): size-independent properties instead of the oracle:
    (1) determinism, (2) tile independence: every tile region equals the same input rendered alone into a
    960x540 output, (3) background bytes exact."""
    w, h = 3840, 2160
    base = [harness.smooth_yuv420(40 + i, w, h) for i in range(4)]
    fr = {f"input_{i}": nv12_frame(base[(i - 1) % 4], w, h) for i in range(1, 17)}
    r = s.Renderer()
    for i in fr:
        r.register_input(i)
    r.update_scene(OUTPUT_ID, s.Resolution(w, h), NV12, s.TilesComponent(children=streams(16), background_color=BG))
    a = r.render(s.FrameSet(frames=fr, pts=0.0)).frames[OUTPUT_ID].data.planes
    b = r.render(s.FrameSet(frames=fr, pts=0.0)).frames[OUTPUT_ID].data.planes
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    r1 = s.Renderer()
    r1.register_input("input_1")
    for k in range(4):
        r1.update_scene(OUTPUT_ID, s.Resolution(960, 540), NV12, V(children=[s.RescalerComponent(child=streams(1)[0])]))
        one = r1.render(s.FrameSet(frames={"input_1": fr[f"input_{k + 1}"]}, pts=0.0)).frames[OUTPUT_ID].data.planes
        for slot in (k, k + 4, k + 8, k + 12):
            ty, tx = divmod(slot, 4)
            assert np.array_equal(a[0][ty * 540:(ty + 1) * 540, tx * 960:(tx + 1) * 960], one[0])
            assert np.array_equal(a[1][ty * 270:(ty + 1) * 270, tx * 480:(tx + 1) * 480], one[1])


@pytest.mark.parametrize("kind", ["nv12", "yuv420"])
def test_integer_ratio_4to1_fused_kernel(kind):
    """BASELINE config 3 geometry at 1/3 size: 1280x720 -> 320x180 tiles (exactly 4:1, 25 taps) through the
    register-blocked fused kernel, NV12 and planar, including the clamped border strips"""
    mk = nv12_frame if kind == "nv12" else yuv_frame
    fr = {f"input_{i}": mk(harness.random_yuv420(300 + i, 1280, 720) if i % 2 else harness.smooth_yuv420(300 + i, 1280, 720),
                           1280, 720) for i in range(1, 5)}
    kids = [s.RescalerComponent(child=c, border_radius=s.BorderRadius.new_with_radius(12.0)) for c in streams(4)]
    over = V(position=s.Position.Absolute(width=300.0, height=80.0, left=170.0, bottom=20.0),
             background_color=s.RGBAColor(16, 32, 160, 112), border_radius=s.BorderRadius.new_with_radius(16.0))
    scene = V(background_color=BG, children=[s.TilesComponent(children=kids, background_color=BG), over])
    check(scene, fr, out_format=NV12)


def test_wide_identity_mapping_4k_row():
    """FAST_IDENT / FAST_CONST interior paths at 4K width (largest coordinates the shortcut is allowed for)"""
    w, h = 3840, 64
    fr = {"input_1": nv12_frame(harness.random_yuv420(9, w, h), w, h)}
    scene = V(background_color=BG, children=[
        V(children=streams(1), position=s.Position.Absolute(width=float(w), height=float(h), left=0.0, top=0.0)),
        V(position=s.Position.Absolute(width=900.0, height=40.0, left=1500.0, top=10.0),
          background_color=s.RGBAColor(200, 10, 10, 255), border_width=3.0, border_color=s.RGBAColor(255, 255, 255, 255),
          border_radius=s.BorderRadius.new_with_radius(9.0))])
    check(scene, fr, resolution=s.Resolution(w, h), out_format=NV12)


def test_two_ticks_in_flight_give_the_same_frames():
    """smr_render_begin(k+1) before smr_render_end(k): uploads of the next tick overlap the kernels of the
    current one (double-buffered staging); every tick's output must equal the synchronous result."""
    import ctypes as C
    from smelter_b200 import _ffi as F
    w, h, n = 640, 360, 3
    scene = s.TilesComponent(children=streams(n), background_color=BG)
    ticks = [{f"input_{i}": yuv_frame(harness.random_yuv420(1000 + 10 * k + i, w, h), w, h) for i in range(1, n + 1)}
             for k in range(5)]
    ref = s.Renderer()
    for i in range(1, n + 1):
        ref.register_input(f"input_{i}")
    ref.update_scene(OUTPUT_ID, RES, YUV, scene)
    expected = [[np.array(p) for p in ref.render(s.FrameSet(frames=t, pts=0.0)).frames[OUTPUT_ID].data.planes] for t in ticks]

    r = s.Renderer()
    for i in range(1, n + 1):
        r.register_input(f"input_{i}")
    r.update_scene(OUTPUT_ID, RES, YUV, scene)
    keep, outs = [], []
    def submit(t):
        arr = r._input_frames(s.FrameSet(frames=t, pts=0.0), keep)
        planes = [np.empty(w * h, np.uint8), np.empty(w * h // 4, np.uint8), np.empty(w * h // 4, np.uint8)]
        o = (F.OutputFrame * 1)()
        o[0].output_id = OUTPUT_ID.encode()
        o[0].mem_kind = F.MEM_HOST
        for p in range(3):
            o[0].planes[p] = planes[p].ctypes.data
        keep.append((arr, o))
        outs.append(planes)
        r.render_raw(0, arr, len(t), o, 1, wait=False)
    submit(ticks[0])
    for k in range(1, len(ticks)):
        submit(ticks[k])
        r.wait()  # retires tick k-1
        for got, exp in zip(outs[k - 1], expected[k - 1]):
            assert np.array_equal(got, exp.reshape(-1)), f"tick {k - 1}"
    r.wait()
    for got, exp in zip(outs[-1], expected[-1]):
        assert np.array_equal(got, exp.reshape(-1))


WIDE_KINDS = ["PlanarYuv422", "PlanarYuv444", "InterleavedUyvy422", "InterleavedYuyv422"]


@pytest.mark.parametrize("kind", WIDE_KINDS)
def test_wide_chroma_input_formats(kind):
    """SURVEY 8f-3: FrameData::{PlanarYuv422, PlanarYuv444, InterleavedUyvy422, InterleavedYuyv422} inputs
    (input_texture.rs:86-150, interleaved_{uyvy,yuyv}_to_rgba.wgsl) -- 1:1 pass-through root, a Lanczos-scaled
    tile next to a 4:2:0 one with rounded corners, and the CpuOptimized bilinear path"""
    fr = wide_chroma_frame(kind, 11, 640, 360)
    check(s.InputStreamComponent(input_id="input_1"), {"input_1": fr})
    both = {"input_1": fr, "input_2": inputs(2)["input_2"]}
    kids = [s.RescalerComponent(child=c, border_radius=s.BorderRadius.new_with_radius(20.0)) for c in streams(2)]
    check(s.TilesComponent(children=kids, background_color=BG), both, out_format=NV12)
    check(s.TilesComponent(children=streams(2), background_color=BG), both, mode=s.RenderingMode.CpuOptimized)


@pytest.mark.parametrize("kind", ["InterleavedUyvy422", "PlanarYuv422"])
def test_wide_chroma_input_odd_sizes(kind):
    """odd width / height: the interleaved texture is floor(w/2) texels wide (texture/interleaved_yuv422.rs:18-22)
    and the sampler clamps at its edge; planar 4:2:2 chroma is floor(w/2) wide"""
    w, h = 321, 181
    rng = np.random.default_rng(9)
    if kind == "PlanarYuv422":
        d = s.FrameData.PlanarYuv422(s.YuvPlanes(rng.integers(16, 236, (h, w), dtype=np.uint8),
                                                 rng.integers(16, 241, (h, w // 2), dtype=np.uint8),
                                                 rng.integers(16, 241, (h, w // 2), dtype=np.uint8)))
    else:
        d = s.FrameData.InterleavedUyvy422(rng.integers(16, 236, (h, w // 2, 4), dtype=np.uint8))
    fr = s.Frame(d, s.Resolution(w, h))
    check(V(children=[s.RescalerComponent(child=streams(1)[0])], background_color=BG), {"input_1": fr})
    check(s.InputStreamComponent(input_id="input_1"), {"input_1": fr}, resolution=s.Resolution(w, h), out_format=RGBA)


@pytest.mark.parametrize("fmt", [s.OutputFrameFormat.PlanarYuv422Bytes, s.OutputFrameFormat.PlanarYuv444Bytes])
def test_planar_422_444_outputs(fmt):
    """OutputFrameFormat::{PlanarYuv422Bytes, PlanarYuv444Bytes} (texture/planar_yuv.rs:72-83, rgba_to_yuv.rs:67-116):
    tiles scene, pass-through root (same size and rescaled), missing input (black fill), odd output size"""
    check(s.TilesComponent(children=streams(3), background_color=BG), inputs(3), out_format=fmt)
    check(s.InputStreamComponent(input_id="input_1"), inputs(1), out_format=fmt)
    check(s.InputStreamComponent(input_id="input_1"), inputs(1), out_format=fmt, resolution=s.Resolution(400, 300))
    check(s.InputStreamComponent(input_id="input_1"), {}, out_format=fmt)
    check(s.TilesComponent(children=streams(2), background_color=BG), inputs(2), out_format=fmt,
          resolution=s.Resolution(501, 283))


def test_strided_host_planes_in_and_out():
    """SURVEY 8f-1 (ingest / egress glue): an AVFrame's planes carry a linesize larger than the row
    (copy_plane_from_av, decoder/ffmpeg_utils.rs:67-79; write_plane_to_av_frame, encoder/ffmpeg_utils.rs:77-84).
    The C ABI takes the pitch directly, so the repacking copy on both sides disappears: padded planes in and padded
    planes out must give exactly the bytes of the packed call."""
    from smelter_b200 import _ffi as F
    w, h = 640, 360
    fr = inputs(2)
    scene = s.TilesComponent(children=streams(2), background_color=BG)
    r = s.Renderer()
    for i in fr:
        r.register_input(i)
    r.update_scene(OUTPUT_ID, s.Resolution(w, h), YUV, scene)
    packed = [np.asarray(p) for p in r.render(s.FrameSet(frames=fr, pts=0.0)).frames[OUTPUT_ID].data.planes]

    keep, arr = [], (F.InputFrame * 2)()
    for k, (iid, f) in enumerate(fr.items()):
        arr[k].input_id = iid.encode()
        arr[k].format = F.FRAME_PLANAR_YUV420
        arr[k].width, arr[k].height, arr[k].pts_ns, arr[k].mem_kind = w, h, 0, F.MEM_HOST
        for p, pl in enumerate(f.data.planes):
            pl = np.asarray(pl)
            pitch = pl.shape[1] + 64 + 32 * p                       # linesize > width, different per plane
            buf = np.full((pl.shape[0], pitch), 0xAB, np.uint8)
            buf[:, :pl.shape[1]] = pl
            keep.append(buf)
            arr[k].planes[p], arr[k].pitch[p] = buf.ctypes.data, pitch
    out = (F.OutputFrame * 1)()
    out[0].output_id, out[0].mem_kind = OUTPUT_ID.encode(), F.MEM_HOST
    obufs = []
    for p, (rows, cols) in enumerate(((h, w), (h // 2, w // 2), (h // 2, w // 2))):
        pitch = cols + 48
        b = np.full((rows, pitch), 0xCD, np.uint8)
        obufs.append(b)
        out[0].planes[p], out[0].pitch[p] = b.ctypes.data, pitch
    r.render_raw(0, arr, 2, out, 1, wait=True)
    for p, b in enumerate(obufs):
        cols = packed[p].shape[1]
        assert np.array_equal(b[:, :cols], packed[p]), f"plane {p}"
        assert np.all(b[:, cols:] == 0xCD), "padding bytes must stay untouched"


@pytest.mark.parametrize("kind", ["InterleavedUyvy422", "InterleavedYuyv422"])
def test_interleaved_inputs_through_fused_resampler(kind):
    """capture-card frames (UYVY / YUYV) through the fused convert+Lanczos kernel: exact 4:1 (25 taps), 3:1 and a
    fractional ratio, including the clamped strips at both image edges"""
    big = {f"input_{i}": wide_chroma_frame(kind, 20 + i, 1280, 720) for i in range(1, 5)}
    check(s.TilesComponent(children=streams(4), background_color=BG), big, out_format=NV12)           # 4:1
    one = {"input_1": wide_chroma_frame(kind, 31, 960, 540)}
    check(V(children=[s.RescalerComponent(child=streams(1)[0],
                                          position=s.Position.Absolute(width=320.0, height=180.0, left=40.0, top=30.0))],
            background_color=BG), one)                                                                  # 3:1
    check(V(children=[s.RescalerComponent(child=streams(1)[0],
                                          position=s.Position.Absolute(width=417.0, height=233.0, left=11.0, top=7.0))],
            background_color=BG), one)                                                                  # fractional


@pytest.mark.parametrize("mode", [s.RenderingMode.GpuOptimized, s.RenderingMode.CpuOptimized])
def test_frame_pre_processor(mode):
    """FramePreProcessor::process_to_bytes (state/frame_pre_processor.rs:81-100, rgba_rescale.wgsl): every input
    format to RGBA8 at the source resolution, and rescaled down / up (exact 2:1, fractional, odd target) with the
    linear sampler through the mode's target format; BGRA keeps its alpha"""
    from tests.parity import node_texture
    from oracle import oracle as orc
    r = s.Renderer(s.RendererOptions(rendering_mode=mode))
    pre = s.FramePreProcessor(r)
    w, h = 320, 180
    rng = np.random.default_rng(77)
    frames = [inputs(1, w, h)["input_1"], nv12_frame(harness.smooth_yuv420(5, w, h), w, h),
              wide_chroma_frame("InterleavedUyvy422", 3, w, h), wide_chroma_frame("PlanarYuv444", 4, w, h),
              s.Frame(s.FrameData.Bgra(rng.integers(0, 256, (h, w, 4), dtype=np.uint8)), s.Resolution(w, h))]
    omode = 0 if mode == s.RenderingMode.GpuOptimized else 1
    for fr in frames:
        node = node_texture(fr)
        assert np.array_equal(pre.process_to_bytes(fr), node), fr.data.kind
        for ow, oh in ((160, 90), (211, 97), (480, 271)):
            got = pre.process_to_bytes(fr, s.Resolution(ow, oh))
            exp = orc.rescale_rgba(node, ow, oh, omode)
            assert_identical((got,), (exp,), f"{fr.data.kind} -> {ow}x{oh}")


def test_many_layers_beyond_the_parameter_bank():
    """150 layers (> the 96 that travel in the kernel parameter bank): the composite reads its layer list from
    global / shared memory instead; translucent, opaque, rounded and video layers mixed, more than 40 in one tile"""
    kids = [s.RescalerComponent(child=streams(1)[0])]
    for i in range(148):
        kids.append(V(position=s.Position.Absolute(width=60.0 + (i % 7) * 9, height=40.0 + (i % 5) * 11,
                                                   left=5.0 + (i * 37) % 560, top=4.0 + (i * 53) % 300),
                      background_color=s.RGBAColor((i * 29) % 256, (i * 71) % 256, (i * 13) % 256, 255 if i % 3 else 120),
                      border_radius=s.BorderRadius.new_with_radius(float((i % 4) * 6))))
    # a pile of 45 views on one spot: more than the layers a tile keeps in shared memory
    for i in range(45):
        kids.append(V(position=s.Position.Absolute(width=90.0 - i, height=70.0 - i, left=300.0 + i * 0.5, top=150.0 + i * 0.25),
                      background_color=s.RGBAColor((i * 5) % 256, 200, (i * 17) % 256, 200)))
    check(V(children=kids, background_color=BG), inputs(1), max_layouts=400)


def test_failed_tick_does_not_poison_the_weight_cache():
    """A tick that fails AFTER planning (its second output is not registered) created Lanczos weight-cache entries whose
    k_weights launch never ran; the next good tick must recompute them (ADVICE r1: the cache used to keep the
    uninitialised tables forever).  Two scenes: a grid of two planar inputs, and one UYVY input at exactly 2:1 with a
    zero crop offset, which the LDG-staged kernel resamples at integer ratio 2."""
    fr = inputs(2)
    scene = s.TilesComponent(children=streams(2), background_color=BG)
    r = TrackedRenderer()
    for i in fr:
        r.register_input(i)
    r.update_scene(OUTPUT_ID, RES, YUV, scene)
    r._outputs["ghost"] = (RES, YUV)          # known to the Python mirror only: the library refuses it after output_1
    with pytest.raises(s.RenderSceneError):
        r.render(s.FrameSet(frames=fr, pts=0.0), outputs=[OUTPUT_ID, "ghost"])
    del r._outputs["ghost"]
    got, exp, _ = run_case(scene, fr, renderer=r)
    assert_identical(got, exp, "good tick after a failed one")

    # set_layouts makes the ratio exact: the crop is the whole 640 x 360 frame, the child 320 x 180
    from tests.test_gpu_fused_variants import Job, check as check_fused, make_frame, scene_of
    jobs = [Job("input_1", (0.0, 0.0, 640.0, 360.0), (320, 180))]
    fr = {"input_1": make_frame("uyvy", "extreme", 23, 640, 360)}
    W, H, ids, layouts, _ = scene_of(jobs)
    r = s.Renderer()
    r.register_input("input_1")
    r.set_layouts(OUTPUT_ID, s.Resolution(W, H), RGBA, (W, H), ids, layouts)
    r._outputs["ghost"] = (RES, YUV)
    with pytest.raises(s.RenderSceneError):
        r.render(s.FrameSet(frames=fr, pts=0.0), outputs=[OUTPUT_ID, "ghost"])
    assert [(f["kernel"], f["ratio"]) for f in r.debug_fused_jobs()] == [("ldg", 2)]   # planned by the failed tick
    del r._outputs["ghost"]
    check_fused(jobs, fr, expect=[{"kernel": "ldg", "ratio": 2}], renderer=r, what="UYVY 2:1 good tick after a failed one")


def test_pitch_smaller_than_a_row_is_refused():
    from smelter_b200 import _ffi as F
    import ctypes as C
    r = s.Renderer()
    r.register_input("input_1")
    r.update_scene(OUTPUT_ID, RES, YUV, V(children=streams(1)))
    y, u, v = harness.test_input(1)
    keep = []
    arr = r._input_frames(s.FrameSet(frames={"input_1": yuv_frame((y, u, v), 640, 360)}, pts=0.0), keep)
    arr[0].pitch[0] = 320                      # luma rows are 640 bytes
    out = (F.OutputFrame * 1)()
    bufs = [np.empty(640 * 360, np.uint8), np.empty(320 * 180, np.uint8), np.empty(320 * 180, np.uint8)]
    out[0].output_id = OUTPUT_ID.encode()
    out[0].mem_kind = F.MEM_HOST
    for p in range(3):
        out[0].planes[p] = bufs[p].ctypes.data
    assert r._lib.smr_render(r._h, 0, arr, 1, out, 1) == 1   # SMR_ERR_INVALID_ARGUMENT
    arr[0].pitch[0] = 0
    out[0].pitch[1] = 100                      # chroma rows are 320 bytes
    assert r._lib.smr_render(r._h, 0, arr, 1, out, 1) == 1
    arr[0].pitch[0] = 320                      # the frame pre-processor reads frames by the same rules
    rgba = np.empty(640 * 360 * 4, np.uint8)
    assert r._lib.smr_preprocess_frame(r._h, arr, 0, 0, rgba.ctypes.data, 0, F.MEM_HOST) == 1


def glyph_like_rgba(w, h, seed):
    """premultiplied RGBA8 with soft (anti-aliased) coverage, like a CPU-rasterised text / image layer
    (transformations/text_renderer.rs:282-369 ends in exactly such a texture)"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    cov = np.clip(1.2 * (np.sin(xx / 7.0 + seed) * np.cos(yy / 5.0) + 0.35), 0.0, 1.0)
    cov = np.where(rng.random((h, w)) < 0.05, 0.0, cov)                    # holes: alpha exactly 0
    a = np.rint(cov * 255).astype(np.uint8)
    col = np.stack([np.full((h, w), 230), 40 + (xx * 3) % 200, 200 - (yy * 2) % 180], axis=-1).astype(np.float64)
    rgb = np.rint(col * (a[..., None] / 255.0)).astype(np.uint8)          # premultiplied: rgb <= alpha
    return np.concatenate([rgb, a[..., None]], axis=-1).astype(np.uint8)


@pytest.mark.parametrize("mode", [s.RenderingMode.GpuOptimized, s.RenderingMode.CpuOptimized])
def test_translucent_premultiplied_rgba_layers(mode):
    """SURVEY 8f-2 route (INTEGRATION 3b): a text / image node arrives as a premultiplied RGBA8 input and is an ordinary
    K9 texture layer.  1:1 over video (per-pixel alpha through the blend), scaled by a Rescaler (Lanczos on a
    translucent RGBA source / bilinear in CpuOptimized) and with rounded corners."""
    fr = inputs(1)
    fr["label"] = s.Frame(s.FrameData.Rgba8(glyph_like_rgba(200, 64, 3)), s.Resolution(200, 64), 0.0)
    fr["logo"] = s.Frame(s.FrameData.Rgba8(glyph_like_rgba(96, 96, 5)), s.Resolution(96, 96), 0.0)
    label = V(position=s.Position.Absolute(width=200.0, height=64.0, left=40.0, top=250.0),
              children=[s.InputStreamComponent(input_id="label")])
    logo = s.RescalerComponent(position=s.Position.Absolute(width=171.0, height=150.0, right=20.0, top=15.0),
                               child=s.InputStreamComponent(input_id="logo"),
                               border_radius=s.BorderRadius.new_with_radius(18.0))
    scene = V(background_color=BG, children=[s.RescalerComponent(child=streams(1)[0]), label, logo])
    check(scene, fr, mode=mode)


@pytest.mark.parametrize("mode", [s.RenderingMode.GpuOptimized, s.RenderingMode.CpuOptimized])
def test_add_premultiplied_alpha_pass(mode):
    """wgpu/utils/add_premultiplied_alpha.wgsl:24-35 (PremultiplyAlphaPipeline): straight-alpha RGBA8 asset ->
    premultiplied RGBA8 through the renderer's views, byte-exact against the oracle twin; every alpha value occurs"""
    from oracle import oracle as orc
    rng = np.random.default_rng(11)
    h, w = 64, 256
    rgba = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    rgba[:, :, 3] = np.arange(w, dtype=np.uint8)[None, :]          # alpha 0..255 across the row
    rgba[0, :, :3] = 255
    r = s.Renderer(s.RendererOptions(rendering_mode=mode))
    got = r.premultiply_rgba8(rgba)
    exp = orc.add_premultiplied_alpha(rgba, orc.MODE_GPU_OPTIMIZED if mode == s.RenderingMode.GpuOptimized else orc.MODE_CPU_OPTIMIZED)
    assert np.array_equal(got, exp), f"{np.count_nonzero(got != exp)} bytes differ"
    assert np.all(got[..., :3].astype(int) <= got[..., 3:4].astype(int) + (1 if mode == s.RenderingMode.GpuOptimized else 0) * 255)


def test_set_layouts_renders_like_the_scene():
    """the flattened boundary (smr_set_layouts): feeding the RenderLayout[] of a scene renders the same bytes as the scene"""
    fr = inputs(3)
    kids = [s.RescalerComponent(child=c, border_radius=s.BorderRadius.new_with_radius(12.0)) for c in streams(3)]
    scene = V(background_color=BG, children=[s.TilesComponent(children=kids, background_color=BG, margin=6.0),
                                             V(position=s.Position.Absolute(width=100.0, height=40.0, left=7.0, bottom=9.0),
                                               background_color=s.RGBAColor(10, 20, 30, 99))])
    got, exp, r = run_case(scene, fr)
    assert_identical(got, exp, "scene path")
    ls, root = r.debug_layouts(OUTPUT_ID)
    b = s.Renderer()
    for i in fr:
        b.register_input(i)
    b.set_layouts(OUTPUT_ID, RES, YUV, root, [f"input_{i}" for i in range(1, 4)], ls)
    out = b.render(s.FrameSet(frames=fr, pts=0.0))
    assert_identical([np.asarray(p) for p in out.frames[OUTPUT_ID].data.planes], exp, "flattened path")


def test_codec_shaped_device_surfaces():
    """SURVEY 8f-4 hand-off (INTEGRATION 3d): NV12 frames as a hardware decoder maps them -- device memory, pitch wider than
    the row, the interleaved chroma plane `pitch x aligned_height` bytes below the luma plane -- go in as SMR_MEM_DEVICE
    planes, and the output is written into an encoder-style surface of the same shape.  No host copies (h2d / d2h byte
    counters stay zero); bytes against the oracle on the same frames."""
    import ctypes as C
    import torch
    from smelter_b200 import _ffi as F
    from tests.parity import oracle_output
    w, h, pitch, ah = 1920, 1080, 2048, 1088            # NVDEC: pitch and surface height aligned
    ow, oh, opitch, oah = 1280, 720, 1536, 736
    dev = torch.device("cuda:0")
    fr, surfaces = {}, []
    arr = (F.InputFrame * 2)()
    keep = []
    for i in (1, 2):
        y, u, v = harness.test_input(i, w, h)
        fr[f"input_{i}"] = nv12_frame((y, u, v), w, h)
        surf = torch.zeros((ah * 3 // 2, pitch), dtype=torch.uint8, device=dev)
        surf[:h, :w] = torch.from_numpy(np.ascontiguousarray(y)).to(dev)
        surf[ah:ah + h // 2, :w] = torch.from_numpy(np.stack([u, v], axis=-1).reshape(h // 2, w)).to(dev)
        surfaces.append(surf)
        b = f"input_{i}".encode()
        keep.append(b)
        a = arr[i - 1]
        a.input_id, a.format, a.width, a.height, a.pts_ns, a.mem_kind = b, F.FRAME_NV12, w, h, 0, F.MEM_DEVICE
        a.planes[0], a.planes[1] = surf.data_ptr(), surf.data_ptr() + pitch * ah
        a.pitch[0], a.pitch[1] = pitch, pitch
    scene = s.TilesComponent(children=streams(2), background_color=BG, margin=4.0)
    r = TrackedRenderer()
    for iid in fr:
        r.register_input(iid)
    res = s.Resolution(ow, oh)
    r.update_scene(OUTPUT_ID, res, NV12, scene)
    osurf = torch.zeros((oah * 3 // 2, opitch), dtype=torch.uint8, device=dev)
    out = (F.OutputFrame * 1)()
    ob = OUTPUT_ID.encode()
    out[0].output_id, out[0].mem_kind = ob, F.MEM_DEVICE
    out[0].planes[0], out[0].planes[1] = osurf.data_ptr(), osurf.data_ptr() + opitch * oah
    out[0].pitch[0], out[0].pitch[1] = opitch, opitch
    torch.cuda.synchronize()
    r.render_raw(0, arr, 2, out, 1)
    st = r.stats()
    assert st["h2d_bytes"] == 0 and st["d2h_bytes"] == 0, st
    got_y = osurf[:oh, :ow].cpu().numpy()
    got_uv = osurf[oah:oah + oh // 2, :ow].cpu().numpy().reshape(oh // 2, ow // 2, 2)
    exp = oracle_output(r, scene, fr, res, NV12, 0, 0.0)
    assert_identical((got_y, got_uv), exp, "codec-shaped surfaces")
    assert not osurf[:oh, ow:].any() and not osurf[oh:oah].any(), "bytes outside the visible planes were written"


@pytest.mark.parametrize("fmt", [NV12, YUV])
@pytest.mark.parametrize("ratio", [2, 4])
def test_direct_tiles_match_the_composite_path(fmt, ratio, monkeypatch):
    """Output tiles that lie wholly inside the 1:1 opaque interior of ONE resampled child (nothing painted over them) get
    their Y / chroma bytes straight from the vertical pass of the fused resample kernel (FusedJob.direct_map) and are
    skipped by the composite.  Same scene with SMR_DIRECT_K11=0 (every tile through the composite): identical planes;
    both equal the oracle.  Rounded corners, a translucent overlay and a second, scaled-down showing of an input keep
    plenty of tiles on the composite path next to the direct ones."""
    ow, oh = 1280, 720
    iw, ih = ow // 2 * ratio, oh // 2 * ratio
    fr = {f"input_{i}": (nv12_frame if i % 2 else yuv_frame)(harness.test_input(i, iw, ih), iw, ih) for i in range(1, 5)}
    kids = [s.RescalerComponent(child=c, border_radius=s.BorderRadius.new_with_radius(20.0)) for c in streams(4)]
    overlay = V(position=s.Position.Absolute(width=500.0, height=90.0, left=390.0, bottom=40.0),
                background_color=s.RGBAColor(16, 32, 160, 112), border_radius=s.BorderRadius.new_with_radius(24.0))
    pip = s.RescalerComponent(position=s.Position.Absolute(width=160.0, height=90.0, right=16.0, top=16.0),
                              child=s.InputStreamComponent(input_id="input_2"))
    scene = V(background_color=BG, children=[s.TilesComponent(children=kids, background_color=BG), overlay, pip])
    res = s.Resolution(ow, oh)
    got, exp, r = run_case(scene, fr, resolution=res, out_format=fmt)
    assert_identical(got, exp, "direct tiles")
    n_direct = r.stats()["last_render_direct_tiles"]
    if ratio == 4:
        assert n_direct > 100, n_direct                 # 1280 x 720 = 10 x 45 tiles, most of them inside a child
    else:
        assert n_direct == 0, n_direct                  # 2:1 children stay with the composite (plan_tiles: not worth it there)
    monkeypatch.setenv("SMR_DIRECT_K11", "0")
    got0, _, r0 = run_case(scene, fr, resolution=res, out_format=fmt)
    assert r0.stats()["last_render_direct_tiles"] == 0
    assert_identical(got0, got, "composite path vs direct tiles")


def test_direct_tiles_need_even_positions():
    """a child at an odd frame position cannot share 2 x 2 chroma blocks with the frame: its tiles stay with the composite,
    the child at an even position next to it is written directly; bytes as the oracle's either way"""
    fr = inputs(2, 2560, 1440)
    a = s.RescalerComponent(position=s.Position.Absolute(width=640.0, height=360.0, left=3.0, top=5.0), child=streams(2)[0])
    b = s.RescalerComponent(position=s.Position.Absolute(width=640.0, height=360.0, left=644.0, top=366.0), child=streams(2)[1])
    got, exp, r = run_case(V(background_color=BG, children=[a, b]), fr, resolution=s.Resolution(1286, 730))
    assert_identical(got, exp, "odd and even positions")
    n = r.stats()["last_render_direct_tiles"]
    assert 40 <= n <= 5 * 23, n                         # only b's interior: at most 640 / 128 x 360 / 16 tiles


def test_direct_tiles_not_for_a_child_hanging_over_the_frame_edge():
    """a 4:1 child at an even position whose rectangle leaves the frame (View overflow: visible by position) is composed
    the ordinary way: the resample kernel maps every pixel of a direct job to a tile of the frame, so only children wholly
    inside the frame qualify; the child inside the frame next to it is written directly"""
    fr = inputs(2, 2560, 1440)
    a = s.RescalerComponent(position=s.Position.Absolute(width=640.0, height=360.0, left=960.0, top=-120.0), child=streams(2)[0])
    b = s.RescalerComponent(position=s.Position.Absolute(width=640.0, height=360.0, left=128.0, top=320.0), child=streams(2)[1])
    got, exp, r = run_case(V(background_color=BG, children=[a, b]), fr, resolution=s.Resolution(1280, 720))
    assert_identical(got, exp, "child over the edge")
    n = r.stats()["last_render_direct_tiles"]
    assert 40 <= n <= 5 * 23, n                         # b's interior only
