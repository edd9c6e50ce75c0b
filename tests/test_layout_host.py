"""Host logic (scene -> NestedLayout -> flatten) through the C ABI on a host-only handle
(smr_options.cuda_device = -1).  Expected values are hand-derived from the reference's scene maths
and render-test scenes (integration-tests/src/render_tests/{tiles,view,rescaler,transition}.rs).
CPU-only."""
import math

import pytest

import smelter_b200 as s
from smelter_b200 import _ffi as F

RES = s.Resolution(640, 360)
BG = s.RGBAColor(0x33, 0x33, 0x33, 255)


def host_renderer(mode=s.RenderingMode.GpuOptimized, **kw):
    return s.Renderer(s.RendererOptions(rendering_mode=mode, cuda_device=-1, **kw))


def inputs(n):
    return [s.InputStreamComponent(input_id=f"input_{i}") for i in range(1, n + 1)]


def setup(scene, n_inputs, res=RES, in_res=RES, pts=0.0, r=None):
    r = r or host_renderer()
    for i in range(1, n_inputs + 1):
        r.register_input(f"input_{i}")
    r.update_scene("output_1", res, s.OutputFrameFormat.PlanarYuv420Bytes, scene)
    r.debug_set_inputs(pts, {f"input_{i}": in_res for i in range(1, n_inputs + 1)})
    return r


def rect(l):
    return (l.left, l.top, l.width, l.height)


def test_exports_every_declared_symbol():
    L = F.lib()
    for name in F.EXPORTS:
        assert hasattr(L, name), name


def test_header_and_ffi_agree_on_symbols():
    import os, re
    hdr = open(os.path.join(os.path.dirname(F._HERE), "include", "smelter_b200.h")).read()
    declared = set(re.findall(r"\b(smr_[a-z0-9_]+)\s*\(", hdr)) - {"smr_status"}
    assert declared == set(F.EXPORTS), declared ^ set(F.EXPORTS)


def test_render_without_gpu_fails_loudly():
    r = host_renderer()
    r.update_scene("output_1", RES, s.OutputFrameFormat.PlanarYuv420Bytes, s.ViewComponent())
    with pytest.raises(s.RenderSceneError) as e:
        r.render(s.FrameSet(pts=0.0))
    assert e.value.status == 2  # SMR_ERR_CUDA: no CPU fallback


def test_tiles_02_inputs():
    """tiles.rs:85-95 (BASELINE config 1): two 320x180 tiles at (0,90) and (320,90), grey elsewhere."""
    r = setup(s.TilesComponent(children=inputs(2), background_color=BG), 2)
    ls, root = r.debug_layouts("output_1")
    assert root == (640, 360)
    assert [l.type for l in ls] == [1, 0, 0]
    assert rect(ls[0]) == (0, 0, 640, 360) and (ls[0].color.r, ls[0].color.a) == (0x33, 255)
    assert rect(ls[1]) == (0, 90, 320, 180) and ls[1].child_index == 0
    assert rect(ls[2]) == (320, 90, 320, 180) and ls[2].child_index == 1
    assert (ls[1].crop_left, ls[1].crop_top, ls[1].crop_width, ls[1].crop_height) == (0, 0, 640, 360)
    assert ls[1].masks_len == 0


@pytest.mark.parametrize("n,rows,cols", [(1, 1, 1), (2, 1, 2), (3, 2, 2), (4, 2, 2), (5, 2, 3), (15, 4, 4)])
def test_tiles_grid_shape(n, rows, cols):
    """tiles.rs:73-143: optimal_row_column_count for 16:9 tiles on a 16:9 output."""
    r = setup(s.TilesComponent(children=inputs(n), background_color=BG), n)
    ls, _ = r.debug_layouts("output_1")
    tiles = [l for l in ls if l.type == 0]
    assert len(tiles) == n
    tw = 640 / cols
    assert all(abs(t.width - tw) < 1e-3 and abs(t.height - tw * 9 / 16) < 1e-3 for t in tiles)
    assert len({round(t.top, 2) for t in tiles}) == rows
    # last row is centred (HorizontalAlign::Center default)
    last = [t for t in tiles if abs(t.top - max(x.top for x in tiles)) < 1e-3]
    used = len(last) * tw
    assert abs(min(t.left for t in last) - (640 - used) / 2) < 1e-3


def test_tiles_margin_and_padding():
    """tiles.rs margin_and_padding_with_03_inputs flavour: tile_size / tiles_positions arithmetic."""
    r = setup(s.TilesComponent(children=inputs(3), background_color=BG, margin=10.0, padding=5.0), 3)
    ls, _ = r.debug_layouts("output_1")
    tiles = [l for l in ls if l.type == 0]
    # 2x2 grid: x_scale=(640-20-30)/2/16=18.4375, y_scale=(360-20-30)/2/9=17.2222 -> scale=17.2222
    scale = (360 - 20 - 30) / 2 / 9
    tw, th = 16 * scale, 9 * scale
    assert abs(tiles[0].width - tw) < 1e-3 and abs(tiles[0].height - th) < 1e-3
    add_x = 640 - (tw + 10) * 2 - 30
    assert abs(tiles[0].left - (add_x / 2 + 15)) < 1e-3
    assert abs(tiles[1].left - (add_x / 2 + 15 + tw + 20)) < 1e-3
    assert abs(tiles[0].top - 15) < 1e-3  # additional_y == 0 for the limiting axis
    add_x3 = 640 - (tw + 10) * 1 - 20
    assert abs(tiles[2].left - (add_x3 / 2 + 15)) < 1e-3


def test_tiles_portrait_input_is_fitted_into_tile():
    """tiles_component/layout.rs:107-128 fit_into_tile: 360x640 input in a 640x360 tile."""
    r = setup(s.TilesComponent(children=inputs(1), background_color=BG), 1, in_res=s.Resolution(360, 640))
    ls, _ = r.debug_layouts("output_1")
    t = [l for l in ls if l.type == 0][0]
    assert abs(t.height - 360) < 1e-3 and abs(t.width - 202.5) < 1e-3 and abs(t.left - 218.75) < 1e-3


def test_simple_pass_through_view():
    """simple.rs:18-30: View{children:[InputStream]} -> one texture layout, mask removed as redundant."""
    r = setup(s.ViewComponent(children=inputs(1)), 1)
    ls, _ = r.debug_layouts("output_1")
    assert len(ls) == 1 and ls[0].type == 0
    assert rect(ls[0]) == (0, 0, 640, 360) and ls[0].masks_len == 0 and ls[0].border_width == 0


def test_view_row_with_static_and_dynamic_children():
    """view/layout.rs static_child_size: fixed 100 px + two flexible children share the rest."""
    V = s.ViewComponent
    kids = [V(position=s.Position.Static(width=100.0), background_color=s.RGBAColor(255, 0, 0, 255)),
            V(background_color=s.RGBAColor(0, 255, 0, 255)), V(background_color=s.RGBAColor(0, 0, 255, 255))]
    r = setup(V(children=kids, background_color=BG), 0)
    ls, _ = r.debug_layouts("output_1")
    cols = [l for l in ls if l.type == 1]
    assert [rect(c) for c in cols] == [(0, 0, 640, 360), (0, 0, 100, 360), (100, 0, 270, 360), (370, 0, 270, 360)]


def test_view_column_border_and_padding():
    """view_component.rs:63-69 + layout.rs:129-160: border offsets children, padding adds to position."""
    V = s.ViewComponent
    child = V(position=s.Position.Static(height=50.0), background_color=s.RGBAColor(255, 0, 0, 255))
    root = V(children=[child], direction=s.ViewChildrenDirection.Column, border_width=10.0,
             border_color=s.RGBAColor(255, 255, 255, 255), padding=s.Padding(5, 6, 7, 8), background_color=BG)
    r = setup(root, 0)
    ls, _ = r.debug_layouts("output_1")
    assert rect(ls[0]) == (0, 0, 640, 360) and ls[0].border_width == 10.0
    # content = 620x340; child width = 620 - (6+8); top = border + padding.top; left = border + padding.left
    assert rect(ls[1]) == (18, 15, 606, 50)
    assert ls[1].masks_len == 0  # parent mask (10,10,620,340) contains the child -> dropped


def test_view_absolute_child_and_overflow_mask():
    V = s.ViewComponent
    child = V(position=s.Position.Absolute(width=200.0, height=100.0, right=-50.0, bottom=20.0),
              background_color=s.RGBAColor(255, 0, 0, 255))
    r = setup(V(children=[child], background_color=BG), 0)
    ls, _ = r.debug_layouts("output_1")
    # left = 640 - (-50) - 200 = 490, top = 360 - 20 - 100 = 240; sticks out to the right -> mask kept
    assert rect(ls[1]) == (490, 240, 200, 100)
    assert ls[1].masks_len == 1
    m = ls[1].masks[0]
    assert (m.left, m.top, m.width, m.height) == (0, 0, 640, 360)


def test_view_border_radius_box_shadow_order():
    """flatten.rs:78-81: own shadows first, then [self, children shadows, children]."""
    V = s.ViewComponent
    sh = s.BoxShadow(offset_x=10, offset_y=20, blur_radius=8, color=s.RGBAColor(0, 0, 0, 255))
    child = V(position=s.Position.Absolute(width=100.0, height=100.0, left=50.0, top=60.0),
              background_color=s.RGBAColor(255, 0, 0, 255), border_radius=s.BorderRadius.new_with_radius(20.0),
              box_shadow=[sh])
    r = setup(V(children=[child], background_color=BG), 0)
    ls, _ = r.debug_layouts("output_1")
    assert [l.type for l in ls] == [1, 2, 1]
    assert rect(ls[1]) == (60, 80, 100, 100) and ls[1].blur_radius == 8
    assert list(ls[1].border_radius) == [24.0] * 4  # radius + blur/2, flatten.rs:354
    assert list(ls[2].border_radius) == [20.0] * 4


def test_rescaler_fit_and_fill():
    """rescaler_component/layout.rs:14-57: 640x360 input into a 320x320 rescaler."""
    for mode, exp in [(s.RescaleMode.Fit, (0, 70, 320, 180)), (s.RescaleMode.Fill, (-124.44444, 0, 568.8889, 320))]:
        resc = s.RescalerComponent(child=inputs(1)[0], mode=mode,
                                   position=s.Position.Absolute(width=320.0, height=320.0, left=0.0, top=0.0))
        r = setup(s.ViewComponent(children=[resc], background_color=BG), 1)
        ls, _ = r.debug_layouts("output_1")
        tex = [l for l in ls if l.type == 0][0]
        assert all(abs(a - b) < 1e-2 for a, b in zip(rect(tex), exp)), rect(tex)
        if mode == s.RescaleMode.Fill:
            assert tex.masks_len == 2  # root View mask + rescaler mask both cut the overflow


def test_rescaler_align_and_border():
    resc = s.RescalerComponent(child=inputs(1)[0], horizontal_align=s.HorizontalAlign.Right,
                               vertical_align=s.VerticalAlign.Bottom, border_width=10.0,
                               border_color=s.RGBAColor(255, 255, 255, 255),
                               position=s.Position.Absolute(width=300.0, height=300.0, left=20.0, top=30.0))
    r = setup(s.ViewComponent(children=[resc], background_color=BG), 1)
    ls, _ = r.debug_layouts("output_1")
    # position.with_border: 320x320 at (20,30); content 300x300; scale = 300/640; child 300x168.75 bottom-right
    frame = [l for l in ls if l.type == 1 and l.border_width == 10.0][0]
    assert rect(frame) == (20, 30, 320, 320)
    tex = [l for l in ls if l.type == 0][0]
    assert all(abs(a - b) < 1e-3 for a, b in zip(rect(tex), (30, 40 + 300 - 168.75, 300, 168.75)))


def test_rescaler_scales_view_subtree():
    """rescaler.rs:76-187: rescaling a View with fixed size scales borders/children through flatten_child."""
    V = s.ViewComponent
    inner = V(position=s.Position.Static(width=1280.0, height=720.0), background_color=s.RGBAColor(255, 0, 0, 255),
              border_width=20.0, border_color=s.RGBAColor(255, 255, 255, 255),
              children=[V(position=s.Position.Static(width=640.0), background_color=s.RGBAColor(0, 255, 0, 255))])
    r = setup(s.RescalerComponent(child=inner), 0)
    ls, _ = r.debug_layouts("output_1")
    cols = [l for l in ls if l.type == 1]
    # inner view external size = 1320x760 -> scale = min(640/1320, 360/760) = 0.47368
    sc = min(640 / 1320, 360 / 760)
    outer = [c for c in cols if c.border_width > 0][0]
    assert abs(outer.width - 1320 * sc) < 1e-2 and abs(outer.border_width - 20 * sc) < 1e-3
    green = [c for c in cols if c.color.g == 255][0]
    assert abs(green.width - 640 * sc) < 1e-2


def test_overflow_fit_scales_children():
    V = s.ViewComponent
    kids = [V(position=s.Position.Static(width=400.0, height=100.0), background_color=s.RGBAColor(255, 0, 0, 255)),
            V(position=s.Position.Static(width=400.0, height=100.0), background_color=s.RGBAColor(0, 255, 0, 255))]
    r = setup(V(children=kids, overflow=s.Overflow.Fit, background_color=BG), 0)
    ls, _ = r.debug_layouts("output_1")
    cols = [l for l in ls if l.type == 1]
    assert rect(cols[1]) == (0, 0, 320, 80) and rect(cols[2]) == (320, 0, 320, 80)  # scale = 640/800


def test_missing_input_is_culled_but_keeps_its_tile():
    r = host_renderer()
    for i in (1, 2):
        r.register_input(f"input_{i}")
    r.update_scene("output_1", RES, 0, s.TilesComponent(children=inputs(2), background_color=BG))
    r.debug_set_inputs(0.0, {"input_1": RES})  # input_2 has no frame
    ls, _ = r.debug_layouts("output_1")
    # SURVEY appendix A: the empty child goes through fit_into_tile with 0x0 -> inf scale -> NaN geometry;
    # should_render compares false on NaN so the layout survives flatten but rasterises nothing
    tex = [l for l in ls if l.type == 0]
    assert len(tex) == 2 and rect(tex[0]) == (0, 90, 320, 180)
    assert math.isnan(tex[1].width) and math.isnan(tex[1].left)


def test_stale_input_is_dropped():
    """render_loop.rs:29-32: frame older than stream_fallback_timeout (3 s in the harness) is cleared."""
    r = host_renderer()
    r.register_input("input_1")
    r.update_scene("output_1", RES, 0, s.TilesComponent(children=inputs(1), background_color=BG))
    r.debug_set_inputs(10.0, {"input_1": RES}, frame_pts=6.9)
    live = lambda: [l for l in r.debug_layouts("output_1", 10.0)[0] if l.type == 0 and not math.isnan(l.width)]
    assert len(live()) == 0
    r.debug_set_inputs(10.0, {"input_1": RES}, frame_pts=7.0)
    assert len(live()) == 1


def _transition_scene(width, transition=None):
    return s.ViewComponent(background_color=BG, children=[
        s.ViewComponent(id="box", position=s.Position.Absolute(width=width, height=100.0, left=0.0, top=0.0),
                        background_color=s.RGBAColor(255, 0, 0, 255), transition=transition)])


def test_linear_transition_midpoint_and_end():
    """transition.rs:39-106: a 2 s linear width transition 100 -> 300 starting at the last render pts."""
    r = setup(_transition_scene(100.0), 0)
    r.debug_set_inputs(1.0, {})  # last render at pts = 1 s
    r.update_scene("output_1", RES, 0, _transition_scene(300.0, s.Transition(duration=2.0)))
    w = lambda pts: [l for l in r.debug_layouts("output_1", pts)[0] if l.color.r == 255][0].width
    assert w(1.0) == 100.0 and abs(w(2.0) - 200.0) < 1e-3 and w(3.0) == 300.0 and w(9.0) == 300.0


def test_cubic_bezier_transition_matches_reference_kat():
    """cubic_bezier.rs:140-147: easing(0.294; .25,.1,.25,1) = 0.5014012915764126."""
    r = setup(_transition_scene(100.0), 0)
    r.debug_set_inputs(0.0, {})
    tr = s.Transition(duration=1.0, interpolation_kind=s.InterpolationKind.CubicBezier(0.25, 0.1, 0.25, 1.0))
    r.update_scene("output_1", RES, 0, _transition_scene(200.0, tr))
    w = [l for l in r.debug_layouts("output_1", 0.294)[0] if l.color.r == 255][0].width
    assert abs(w - (100.0 + 100.0 * 0.5014012915764126)) < 1e-4
    tr2 = s.Transition(duration=1.0, interpolation_kind=s.InterpolationKind.CubicBezier(0.85, 0.0, 0.15, 1.0))
    r2 = setup(_transition_scene(100.0), 0)
    r2.debug_set_inputs(0.0, {})
    r2.update_scene("output_1", RES, 0, _transition_scene(200.0, tr2))
    w2 = [l for l in r2.debug_layouts("output_1", 0.5)[0] if l.color.r == 255][0].width
    assert abs(w2 - 150.0) < 1e-4


def test_bounce_transition():
    r = setup(_transition_scene(100.0), 0)
    r.debug_set_inputs(0.0, {})
    r.update_scene("output_1", RES, 0, _transition_scene(200.0, s.Transition(1.0, s.InterpolationKind.Bounce)))
    w = [l for l in r.debug_layouts("output_1", 0.5)[0] if l.color.r == 255][0].width
    assert abs(w - (100 + 100 * (7.5625 * (0.5 - 1.5 / 2.75) ** 2 + 0.75))) < 1e-3


def test_tiles_transition_moves_tiles():
    """tiles_transitions.rs flavour: adding an input re-flows the tiles; ids keep tiles matched."""
    def scene(n, tr=None):
        kids = [s.InputStreamComponent(input_id=f"input_{i}", id=f"c{i}") for i in range(1, n + 1)]
        return s.TilesComponent(id="tiles", children=kids, background_color=BG, transition=tr)
    r = host_renderer()
    for i in (1, 2):
        r.register_input(f"input_{i}")
    r.update_scene("output_1", RES, 0, scene(1))
    r.debug_set_inputs(0.0, {"input_1": RES, "input_2": RES})
    r.update_scene("output_1", RES, 0, scene(2, s.Transition(duration=1.0)))
    mid = [l for l in r.debug_layouts("output_1", 0.5)[0] if l.type == 0]
    # tile c1 travels from (0,0,640,360) to (0,90,320,180); c2 is new and its slot was not occupied -> hidden until the end?
    # (start has a tile at a different position, so the new tile is not shown during the transition)
    c1 = [l for l in mid if l.child_index == 0][0]
    assert rect(c1) == (0, 45, 480, 270)
    assert len(mid) == 1
    end = [l for l in r.debug_layouts("output_1", 1.0)[0] if l.type == 0]
    assert [rect(l) for l in end] == [(0, 90, 320, 180), (320, 90, 320, 180)]


def test_duplicate_component_ids_are_rejected():
    r = host_renderer()
    V = s.ViewComponent
    with pytest.raises(s.UpdateSceneError) as e:
        r.update_scene("output_1", RES, 0, V(id="a", children=[V(id="a")]))
    assert e.value.status == 4 and "More than one component" in str(e.value)


def test_unsupported_component_is_reported():
    class Shader:
        component_type = F.COMPONENT_SHADER
        id = None
    r = host_renderer()
    with pytest.raises(s.UpdateSceneError) as e:
        r.update_scene("output_1", RES, 0, s.ViewComponent(children=[Shader()]))
    assert e.value.status == 5


def test_max_layouts_and_masks_constants():
    assert F.MAX_MASKS == 20
    assert s.RendererOptions().max_layouts_count == 100


def test_fused_resample_row_partition_covers_every_row_once():
    """host logic of the persistent fused-resample launch (renderer.cpp: partition_fused_rows): the output rows of every
    (job, 64-column strip) are cut into equal contiguous shares for the resident blocks.  Every row of every strip must
    belong to exactly one piece, blocks own consecutive pieces, shares are equal up to the 8-row step."""
    import ctypes as C
    from smelter_b200 import _ffi as F
    lib = F.lib()

    def partition(sizes, max_blocks):
        n = len(sizes)
        w = (C.c_int32 * n)(*[s[0] for s in sizes])
        h = (C.c_int32 * n)(*[s[1] for s in sizes])
        cap = 16384
        pieces, begin = (C.c_int32 * (4 * cap))(), (C.c_int32 * cap)()
        npieces, nblocks = C.c_uint32(), C.c_uint32()
        assert lib.smr_debug_partition(w, h, n, max_blocks, pieces, cap, C.byref(npieces), begin, cap, C.byref(nblocks)) == 0
        pc = [tuple(pieces[4 * i:4 * i + 4]) for i in range(npieces.value)]
        return pc, list(begin[:nblocks.value + 1])

    cases = [([(960, 540)] * 16, 444),                       # BASELINE config 3
             ([(1230, 692)] * 32, 444),                      # config 5: ragged last strip
             ([(960, 540)] * 8, 444), ([(320, 180), (417, 233), (1, 1), (64, 8)], 444), ([(64, 8)], 444),
             ([(5, 3)], 12), ([(4096, 4096)], 7), ([(100, 50), (0, 10), (30, 0)], 9)]
    for sizes, max_blocks in cases:
        pc, begin = partition(sizes, max_blocks)
        total = sum(((w + 63) // 64) * h for w, h in sizes if w > 0 and h > 0)
        assert begin[0] == 0 and begin[-1] == len(pc) and all(a < b for a, b in zip(begin, begin[1:]))
        assert len(begin) - 1 <= max_blocks
        covered = {}
        for job, strip, y0, y1 in pc:
            w, h = sizes[job]
            assert 0 <= strip < (w + 63) // 64 and 0 <= y0 < y1 <= h
            for y in range(y0, y1):
                assert (job, strip, y) not in covered
                covered[(job, strip, y)] = True
        assert len(covered) == total
        # pieces are in (job, strip, row) order, so a block's pieces are a contiguous run of that order
        assert pc == sorted(pc)
        shares = [sum(p[3] - p[2] for p in pc[a:b]) for a, b in zip(begin, begin[1:])]
        # every block but the last gets the same share, a multiple of the 8 output rows a block produces per step
        assert len(set(shares[:-1])) <= 1 and all(sh % 8 == 0 for sh in shares[:-1])
        assert len(shares) == 1 or shares[-1] <= shares[0]


def test_output_plane_sizes_for_every_output_format():
    """texture/planar_yuv.rs:64-98 (4:2:0 / 4:2:2 / 4:4:4 chroma plane sizes), nv12.rs:77-88, RGBA; odd sizes floor"""
    import ctypes as C
    lib = F.lib()

    def sizes(w, h, fmt):
        out = (C.c_size_t * 3)()
        st = lib.smr_output_plane_sizes(w, h, fmt, C.byref(out))
        return st, tuple(out)

    assert sizes(640, 360, F.OUT_PLANAR_YUV420) == (0, (640 * 360, 320 * 180, 320 * 180))
    assert sizes(640, 360, F.OUT_PLANAR_YUV422) == (0, (640 * 360, 320 * 360, 320 * 360))
    assert sizes(640, 360, F.OUT_PLANAR_YUV444) == (0, (640 * 360, 640 * 360, 640 * 360))
    assert sizes(640, 360, F.OUT_NV12) == (0, (640 * 360, 320 * 180 * 2, 0))
    assert sizes(640, 360, F.OUT_RGBA8) == (0, (640 * 360 * 4, 0, 0))
    assert sizes(501, 283, F.OUT_PLANAR_YUV422) == (0, (501 * 283, 250 * 283, 250 * 283))
    assert sizes(501, 283, F.OUT_PLANAR_YUV420) == (0, (501 * 283, 250 * 141, 250 * 141))
    assert sizes(640, 360, 5)[0] == 5 and sizes(640, 360, -1)[0] == 5      # SMR_ERR_UNSUPPORTED


def test_unknown_output_format_is_rejected_and_new_formats_accepted():
    r = host_renderer()
    scene = s.ViewComponent(background_color=s.RGBAColor(1, 2, 3, 255))
    for fmt in (s.OutputFrameFormat.PlanarYuv420Bytes, s.OutputFrameFormat.PlanarYuv422Bytes,
                s.OutputFrameFormat.PlanarYuv444Bytes, s.OutputFrameFormat.RgbaWgpuTexture,
                s.OutputFrameFormat.Nv12WgpuTexture):
        r.update_scene("output_1", RES, fmt, scene)
    with pytest.raises(s.UpdateSceneError):
        r.update_scene("output_1", RES, 7, scene)


def test_frame_pre_processor_without_gpu_fails_loudly():
    """no CPU fallback anywhere on the product path: a host-only handle refuses to convert a frame"""
    import numpy as np
    r = host_renderer()
    fr = s.Frame(s.FrameData.InterleavedUyvy422(np.zeros((4, 4, 4), np.uint8)), s.Resolution(8, 4))
    with pytest.raises(s.RendererError) as e:
        s.FramePreProcessor(r).process_to_bytes(fr)
    assert "no CPU fallback" in str(e.value)


def test_set_layouts_flattened_boundary_round_trip():
    """smr_set_layouts (SURVEY 8b, flattened form): the layouts one handle flattened from a scene, handed to another
    handle as RenderLayout[], come back field for field from debug_layouts -- what smr_render then consumes.  They are
    the output's root layout node (debug_node_layouts node 0, the only one), and they replace its scene's image nodes."""
    import numpy as np
    V = s.ViewComponent
    kids = [s.RescalerComponent(child=c, border_radius=s.BorderRadius.new_with_radius(12.0),
                                box_shadow=[s.BoxShadow(3.0, 4.0, 10.0, s.RGBAColor(0, 0, 0, 128))]) for c in inputs(3)]
    scene = V(background_color=BG, children=[s.TilesComponent(children=kids, background_color=BG, margin=6.0),
                                             V(position=s.Position.Absolute(width=100.0, height=40.0, left=7.0, bottom=9.0),
                                               background_color=s.RGBAColor(10, 20, 30, 99), border_width=2.0,
                                               border_color=s.RGBAColor(255, 255, 255, 255))])
    a = setup(scene, 3)
    ls, root = a.debug_layouts("output_1")
    b = host_renderer()
    for i in range(1, 4):
        b.register_input(f"input_{i}")
    b.register_image("image", np.zeros((4, 8, 4), np.uint8))
    b.update_scene("output_1", RES, s.OutputFrameFormat.PlanarYuv420Bytes, V(children=[s.ImageComponent(image_id="image")]))
    assert len(b.debug_image_nodes("output_1")) == 1
    b.set_layouts("output_1", RES, s.OutputFrameFormat.PlanarYuv420Bytes, root, [f"input_{i}" for i in range(1, 4)], ls)
    assert b.debug_image_nodes("output_1") == []
    b.debug_set_inputs(0.0, {f"input_{i}": RES for i in range(1, 4)})
    ls2, root2 = b.debug_layouts("output_1")
    assert root2 == root and len(ls2) == len(ls)
    for x, y in zip(ls, ls2):
        assert bytes(x) == bytes(y)
    ls_node, root_node = b.debug_node_layouts("output_1", 0)
    assert root_node == root2 and [bytes(x) for x in ls_node] == [bytes(y) for y in ls2]
    with pytest.raises(s.RendererError) as e:
        b.debug_node_layouts("output_1", 1)
    assert e.value.status == 1   # SMR_ERR_INVALID_ARGUMENT: no such layout node
    # a later update_scene of the same output replaces the flattened layouts
    b.update_scene("output_1", RES, s.OutputFrameFormat.PlanarYuv420Bytes, V(background_color=BG))
    ls3, _ = b.debug_layouts("output_1")
    assert len(ls3) == 1 and ls3[0].type == 1


def test_tile_plan_of_the_composite():
    """Renderer::plan_tiles' geometric core through smr_debug_tile_plan (device-free), against a restatement in Python:
    a tile is finished by the resample kernel (direct) iff its TOPMOST intersecting layer covers it with one of its
    exact-interior bars and has a fused job (one layer per job); every other tile appears exactly once in the list, most
    expensive first (per intersecting layer 1 inside a bar, 8 otherwise, walking down until an opaque interior)."""
    import ctypes as C
    import numpy as np
    from smelter_b200 import _ffi as F
    lib = F.lib()
    TW, TH = 128, 16

    def plan(boxes, W, H, sort=1):
        b = np.ascontiguousarray(np.array(boxes, np.int32).reshape(-1, 14))
        tx_n, ty_n = (W + TW - 1) // TW, (H + TH - 1) // TH
        owner = (C.c_int32 * (tx_n * ty_n))()
        tiles = (C.c_uint32 * (tx_n * ty_n))()
        n = C.c_uint32()
        st = lib.smr_debug_tile_plan(b.ctypes.data_as(C.POINTER(C.c_int32)), len(b), W, H, sort, owner, tx_n * ty_n, tiles, tx_n * ty_n, C.byref(n))
        assert st == 0
        return list(owner), [(t & 0xffff, t >> 16) for t in tiles[:n.value]]

    def ref(boxes, W, H):
        tx_n, ty_n = (W + TW - 1) // TW, (H + TH - 1) // TH
        owner, cost, job_layer = {}, {}, {}
        for ty in range(ty_n):
            for tx in range(tx_n):
                x0, y0, x1, y1 = tx * TW, ty * TH, min(tx * TW + TW, W), min(ty * TH + TH, H)
                hits = [li for li in range(len(boxes) - 1, -1, -1)
                        if not (boxes[li][0] >= x1 or boxes[li][1] <= x0 or boxes[li][2] >= y1 or boxes[li][3] <= y0)]
                inside = lambda L: (x0 >= L[4] and x1 <= L[5] and y0 >= L[6] and y1 <= L[7]) or (x0 >= L[8] and x1 <= L[9] and y0 >= L[10] and y1 <= L[11])
                own = -1
                if hits:
                    L = boxes[hits[0]]
                    if inside(L) and L[13] >= 0 and job_layer.setdefault(L[13], hits[0]) == hits[0]:
                        own = hits[0]
                owner[(tx, ty)] = own
                c = 0
                for li in hits:
                    c += 1 if inside(boxes[li]) else 8
                    if inside(boxes[li]) and boxes[li][12]:
                        break
                cost[(tx, ty)] = c
        return owner, cost

    def layer(x0, y0, w, h, margin, opaque, job):   # a child rect with interior bars `margin` inside it (corner squares cut out)
        return [x0, x0 + w, y0, y0 + h, x0 + margin, x0 + w - margin, y0 + 2, y0 + h - 2, x0 + 2, x0 + w - 2, y0 + margin, y0 + h - margin, opaque, job]

    W, H = 3840, 2160
    bg = [0, W, 0, H, 0, W, 0, H, 0, W, 0, H, 1, -1]
    grid = [layer(960 * (i % 4), 540 * (i // 4), 960, 540, 34, 1, i) for i in range(16)]
    overlay = [1120, 2720, 1680, 2040, 1170, 2670, 1682, 2038, 1122, 2718, 1730, 1990, 0, -1]
    rng = np.random.default_rng(7)
    random_scene = [bg] + [layer(int(rng.integers(0, W - 700)) & ~1, int(rng.integers(0, H - 400)) & ~1, int(rng.integers(300, 700)), int(rng.integers(100, 400)),
                                 int(rng.integers(2, 40)), int(rng.integers(0, 2)), int(rng.integers(-1, 6))) for _ in range(24)]
    for boxes, w, h in (([bg] + grid + [overlay], W, H), (random_scene, W, H), ([bg] + grid[:4], 1000, 250), ([], 640, 360)):
        owner, tiles = plan(boxes, w, h)
        ro, rc = ref(boxes, w, h)
        tx_n = (w + TW - 1) // TW
        assert {k: v for k, v in ro.items()} == {(i % tx_n, i // tx_n): o for i, o in enumerate(owner)}
        left = [k for k, v in ro.items() if v < 0]
        assert sorted(tiles) == sorted(left) and len(set(tiles)) == len(tiles)           # every tile exactly once
        costs = [rc[t] for t in tiles]
        assert costs == sorted(costs, reverse=True)                                       # most expensive first ...
        for a, b in zip(tiles, tiles[1:]):
            if rc[a] == rc[b]:
                assert (a[1], a[0]) < (b[1], b[0])                                        # ... row-major among equals
        _, unsorted = plan(boxes, w, h, sort=0)
        assert unsorted == sorted(left, key=lambda t: (t[1], t[0]))
    # BASELINE config 3: 70 % of the 4 050 tiles are direct
    owner, tiles = plan([bg] + grid + [overlay], W, H)
    assert 0.65 < sum(o >= 0 for o in owner) / len(owner) < 0.78
