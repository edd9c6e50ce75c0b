"""WebView components (smr_register_web_renderer, smr_web_set_frame, smr_web_set_child_rects, smr_component.web_renderer_id).

The browser stays with the caller, so the pages here are seeded stand-in BGRA planes (premultiplied, some translucent) and
the child rects are typed by hand.  There are no reference snapshots of web scenes: parity with the reference rests on the
shared contract alone (the vertex matrix of transformation_matrices.rs, NC-6 / NC-7, PREMULTIPLIED_ALPHA_BLENDING with an
8-bit store per plane), restated independently in tests/web_oracle.c.

CPU (host-only handle): layouts against the independent engine (tests/layout_ref_web.py), the registry and the refusals.
GPU: every output byte against the oracle, both rendering modes and three output formats.
"""
import ctypes as C
import time

import numpy as np
import pytest

import smelter_b200 as s
from oracle import oracle as orc
from smelter_b200 import _ffi as F
from tests import harness
from tests import layout_ref_web as LW
from tests import oracle_image
from tests import oracle_web
from tests.parity import assert_identical, black, chroma_size, from_ref_layout, layouts_equal, node_texture, nv12_frame, yuv_frame
from tests.test_image_component import pixels
from tests.test_layout_independent import diff, product_layouts, ref_layouts
from tests.test_text_component import label, text_texture

V, R, T, IN, IMG, TXT, WEB = (s.ViewComponent, s.RescalerComponent, s.TilesComponent, s.InputStreamComponent, s.ImageComponent,
                              s.TextComponent, s.WebViewComponent)
YUV, NV12, RGBA = s.OutputFrameFormat.PlanarYuv420Bytes, s.OutputFrameFormat.Nv12WgpuTexture, s.OutputFrameFormat.RgbaWgpuTexture
MODES = [s.RenderingMode.GpuOptimized, s.RenderingMode.CpuOptimized]
FORMATS = [YUV, NV12, RGBA]
OVER, UNDER = F.WEB_NATIVE_OVER_CONTENT, F.WEB_NATIVE_UNDER_CONTENT


def page(w, h, seed, translucent=True):
    """a seeded stand-in for CEF's on_paint: premultiplied BGRA, opaque or with alpha over its whole range"""
    rng = np.random.default_rng(seed)
    p = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    p[..., 1] = (np.arange(w)[None, :] * 255 // max(1, w - 1)) % 256
    if translucent:
        p[::4, :, 3] = 0
        p[1::4, ::3, 3] = 255
    else:
        p[..., 3] = 255
    p[..., :3] = np.minimum(p[..., :3], p[..., 3:4])
    return p


class Pair:
    """a renderer and the independent engine driven together, with the pages, rects and node textures the oracle needs"""

    def __init__(self, out=(640, 360), fmt=YUV, mode=s.RenderingMode.GpuOptimized, device=None, inputs=()):
        opts = s.RendererOptions(rendering_mode=mode) if device is None else s.RendererOptions(rendering_mode=mode, cuda_device=device)
        self.r, self.ref = s.Renderer(opts), LW.StatefulScene(*out)
        self.out, self.fmt, self.mode, self.scene = out, fmt, mode, None
        self.m = orc.MODE_GPU_OPTIMIZED if mode == s.RenderingMode.GpuOptimized else orc.MODE_CPU_OPTIMIZED
        self.inputs = {i: (640, 360) for i in inputs}
        self.pages, self.rects, self.tex, self.px, self.gone = {}, {}, {}, {}, {}
        for i in inputs:
            self.r.register_input(i)

    def register_web(self, instance_id, w, h, embedding=OVER):
        self.r.register_web_renderer(instance_id, w, h, embedding)
        self.ref.register_web(instance_id, w, h, embedding)
        self.rects[instance_id] = []

    def unregister_web(self, instance_id):
        self.r.unregister_web_renderer(instance_id)
        self.ref.unregister_web(instance_id)

    def register_image(self, image_id, frame):
        self.r.register_image(image_id, frame)
        self.ref.register_image(image_id, frame.shape[1], frame.shape[0], [0])
        self.px[image_id] = frame

    def set_frame(self, instance_id, bgra):
        self.r.set_web_frame(instance_id, bgra)
        self.pages[instance_id] = bgra.copy()

    def set_rects(self, instance_id, rects):
        self.r.set_web_child_rects(instance_id, rects)
        self.rects[instance_id] = list(rects)

    def update(self, scene, out=None):
        if out is not None:
            self.out = out
            self.ref.out_w, self.ref.out_h = out
        self.r.update_scene("output_1", s.Resolution(*self.out), self.fmt, scene)
        self.ref.update_scene(scene)
        self.scene = scene
        self.tex = {}   # every web node texture is made anew, transparent

    def check_layouts(self, pts):
        self.r.debug_set_inputs(pts, {k: s.Resolution(*v) for k, v in self.inputs.items()})
        got, root = product_layouts(self.r, pts)
        exp, exp_root = self.ref.layouts(pts, self.inputs)
        assert root == exp_root, f"pts {pts}: root {root} expected {exp_root}"
        d = diff(got, ref_layouts(exp))
        assert d is None, f"pts {pts}: {d}"

    # ---- GPU ----
    def frames(self, pts, stale=()):
        out = {}
        for i, (k, (w, h)) in enumerate(sorted(self.inputs.items())):
            fpts = pts - 5.0 if k in stale else pts     # older than the 3 s stream_fallback_timeout
            if k.startswith("rgba"):        # premultiplied RGBA8, translucent in places
                out[k] = s.Frame(s.FrameData.Rgba8(page(w, h, 40 + i)), s.Resolution(w, h), fpts)
            elif k.startswith("bgra"):
                out[k] = s.Frame(s.FrameData.Bgra(page(w, h, 50 + i, translucent=False)), s.Resolution(w, h), fpts)
            else:
                planes = harness.test_input(i + 1, w, h)
                out[k] = nv12_frame(planes, w, h, fpts) if k.startswith("nv12") else yuv_frame(planes, w, h, fpts)
        return out

    def leaf_texture(self, c, frames, live):
        if isinstance(c, IN):
            return node_texture(frames[c.input_id]) if c.input_id in live else None
        if isinstance(c, IMG):
            px = self.px[c.image_id]
            w, h = LW.LI.resolution(self.ref.images[c.image_id], c.width, c.height)
            return oracle_image.render_image(px, w, h, self.m)
        if isinstance(c, TXT):
            return text_texture(c, self.m)
        return self.web_texture(c, frames, live)

    def web_texture(self, c, frames, live):
        inst = self.ref.webs.get(c.instance_id) or self.gone[c.instance_id]   # an unregistered instance a scene still shows
        prev = self.tex.get(id(c), np.zeros((inst.height, inst.width, 4), np.uint8))
        kids = [self.leaf_texture(k, frames, live) for k in c.children]
        t = oracle_web.render_web(prev, self.pages.get(c.instance_id), kids, self.rects[c.instance_id], inst.embedding, self.m)
        self.tex[id(c)] = t
        return t

    def expected(self, pts, frames, stale=()):
        live = {k for k in frames if k not in stale}
        if isinstance(self.scene, WEB):
            return to_format(self.web_texture(self.scene, frames, live), self.out, self.fmt)
        layouts, (rw, rh) = self.ref.layouts(pts, {k: (f.resolution.width, f.resolution.height) for k, f in frames.items() if k in live})
        got, root = self.r.debug_layouts("output_1", pts)
        assert root == (rw, rh)
        d = layouts_equal(got, layouts)
        assert d is None, d
        nodes = [self.leaf_texture(c, frames, live) for c in leaves(self.scene)]   # every web node is drawn, shown or not
        if rw == 0 or rh == 0:
            return black(s.Resolution(*self.out), self.fmt)
        nodes = [n if n is not None else np.zeros((1, 1, 4), np.uint8) for n in nodes]
        rgba = orc.render_layout_node(rw, rh, [from_ref_layout(l) for l in layouts], nodes, mode=self.m, max_layouts=100)
        return to_format(rgba, self.out, self.fmt)

    def render_check(self, pts, what="", stale=()):
        frames = self.frames(pts, stale)
        got = self.r.render(s.FrameSet(frames=frames, pts=pts)).frames["output_1"]
        assert_identical(tuple(np.asarray(p) for p in got.data.planes), self.expected(pts, frames, stale), f"{what} pts {pts}")


def leaves(comp):
    if isinstance(comp, (IN, IMG, TXT, WEB)):
        return [comp]
    if isinstance(comp, R):
        return leaves(comp.child)
    return [x for c in comp.children for x in leaves(c)]


def to_format(rgba, out, fmt):
    W, H = out
    if fmt == RGBA:
        assert rgba.shape[:2] == (H, W)
        return (rgba,)
    if fmt == NV12:
        return orc.rgba_to_nv12_scaled(rgba, W, H)
    return orc.rgba_to_yuv_planar_scaled(rgba, W, H, *chroma_size(fmt, W, H))


def web(instance_id="page", children=(), id=None):
    return WEB(id=id, instance_id=instance_id, children=list(children))


def cell(x, y, w, h, child, **kw):
    return V(position=s.Position.Absolute(width=float(w), height=float(h), left=float(x), top=float(y)), children=[child], **kw)


# ---- CPU ------------------------------------------------------------------------------------------------------------
def host(**kw):
    return Pair(device=-1, **kw)


LAYOUT_SCENES = {
    "root": lambda: web(children=[IN(id="a", input_id="input_1")]),
    "in_view": lambda: V(children=[IN(input_id="input_1"), web(children=[IN(id="a", input_id="input_1")])]),
    "absolute_in_view": lambda: V(children=[cell(40, 30, 320, 180, web())]),
    "in_tiles": lambda: T(children=[IN(input_id="input_1"), web(), IN(input_id="input_2")]),
    "in_rescaler": lambda: V(children=[R(mode=s.RescaleMode.Fill, child=web(children=[IN(id="a", input_id="input_2")]))]),
}


@pytest.mark.parametrize("name", sorted(LAYOUT_SCENES))
def test_layouts_match_independent_engine(name):
    p = host(inputs=("input_1", "input_2"))
    p.register_web("page", 800, 450)
    p.update(LAYOUT_SCENES[name]())
    for pts in (0.0, 0.5):
        p.check_layouts(pts)


def test_layouts_across_a_transition():
    p = host(inputs=("input_1",))
    p.register_web("page", 1280, 720)
    tr = s.Transition(duration=1.0)
    p.update(V(id="v", children=[IN(input_id="input_1"), web()]))
    p.check_layouts(0.0)
    p.update(V(id="v", direction=s.ViewChildrenDirection.Column, transition=tr, children=[IN(input_id="input_1"), web()]))
    for pts in (0.0, 0.25, 0.5, 0.99, 1.5):
        p.check_layouts(pts)


def _spec_status(r, w, h, emb, instance_id=b"x"):
    return F.lib().smr_register_web_renderer(r._h, instance_id, C.byref(F.WebRendererSpec(w, h, emb)))


def test_registry_and_frame_rules():
    r = s.Renderer(s.RendererOptions(cuda_device=-1))
    for w, h in ((0, 10), (10, 0), (16385, 10), (10, 16385)):
        assert _spec_status(r, w, h, OVER) == 1
    assert _spec_status(r, 64, 32, F.WEB_CHROMIUM_EMBEDDING) == 5
    assert _spec_status(r, 64, 32, 7) == 1
    assert F.lib().smr_register_web_renderer(r._h, None, C.byref(F.WebRendererSpec(64, 32, OVER))) == 1
    assert _spec_status(r, 64, 32, OVER) == 0 and _spec_status(r, 64, 32, UNDER) == 1          # KeyTaken
    f = page(64, 32, 1)
    frame = lambda w, h, pitch=0, kind=F.MEM_HOST, ptr=f.ctypes.data: F.WebFrame(ptr, w, h, pitch, kind)
    assert F.lib().smr_web_set_frame(r._h, b"x", C.byref(frame(64, 32))) == 0
    assert F.lib().smr_web_set_frame(r._h, b"x", C.byref(frame(64, 32, 256))) == 0
    for bad in (frame(63, 32), frame(64, 33), frame(64, 32, 255), frame(64, 32, kind=5), frame(64, 32, ptr=None)):
        assert F.lib().smr_web_set_frame(r._h, b"x", C.byref(bad)) == 1
    assert F.lib().smr_web_set_frame(r._h, b"nope", C.byref(frame(64, 32))) == 1
    rects = (F.WebRect * 2)(F.WebRect(0, 0, 10, 10), F.WebRect(1.5, 2.5, 3, 4))
    assert F.lib().smr_web_set_child_rects(r._h, b"x", rects, 2) == 0
    assert F.lib().smr_web_set_child_rects(r._h, b"x", None, 0) == 0
    assert F.lib().smr_web_set_child_rects(r._h, b"x", None, 1) == 1
    assert F.lib().smr_web_set_child_rects(r._h, b"nope", rects, 2) == 1
    assert F.lib().smr_unregister_web_renderer(r._h, b"nope") == 1
    assert F.lib().smr_unregister_web_renderer(r._h, b"x") == 0 and F.lib().smr_unregister_web_renderer(r._h, b"x") == 1


def _status(r, scene, output_id="output_1"):
    with pytest.raises(s.RendererError) as e:
        r.update_scene(output_id, s.Resolution(640, 360), YUV, scene)
    return e.value.status


def test_scene_refusals_leave_the_scene_as_it_was():
    p = host(inputs=("input_1",))
    p.register_web("page", 800, 450)
    p.register_web("other", 320, 240)
    good = V(children=[IN(input_id="input_1"), web(children=[IN(id="a", input_id="input_1")])])
    p.update(good)
    before = product_layouts(p.r, 0.0)
    c = F.Component()
    F.lib().smr_component_default(F.COMPONENT_WEB_VIEW, C.byref(c))
    assert not c.web_renderer_id
    assert F.lib().smr_update_scene(p.r._h, b"output_1", 640, 360, YUV, C.byref(c)) == 5       # what an older caller sends
    refused = {
        4: [web("missing"),                                                                     # WebRendererNotFound
            V(children=[web(children=[IN(input_id="input_1")])]),                               # WebViewChildWithoutId
            V(children=[web(), web()]),                                                         # one instance, two WebViews
            V(children=[web(children=[IN(id="a", input_id="input_1"), IMG(id="a", image_id="x")])]),   # duplicate ids
            V(id="a", children=[web(children=[IN(id="a", input_id="input_1")])]),
            web(children=[IMG(id="i", image_id="missing")])],                                   # ImageNotFound inside
        5: [web(children=[V(id="v")]), web(children=[R(id="r", child=IN(input_id="input_1"))]), web(children=[T(id="t")]),
            web(children=[web("other", id="w")])],
    }
    for status, scenes in refused.items():
        for scene in scenes:
            assert _status(p.r, scene) == status, scene
            if status == 4:
                with pytest.raises(LW.SceneError):
                    p.ref.update_scene(scene)
            assert product_layouts(p.r, 0.0) == before
    p.check_layouts(0.0)
    # exclusivity across outputs: output_2 may not show "page" while output_1 does, and may once output_1 no longer does
    assert _status(p.r, web("page"), "output_2") == 4
    p.r.update_scene("output_2", s.Resolution(640, 360), YUV, web("other"))
    p.update(V(children=[IN(input_id="input_1")]))
    p.r.update_scene("output_2", s.Resolution(640, 360), YUV, web("page"))
    assert _status(p.r, web("page")) == 4
    # unregistering an instance a scene shows keeps that scene; a new scene cannot name it
    p.r.unregister_web_renderer("other")
    assert _status(p.r, web("other")) == 4


def test_oracle_page_alone_is_the_swapped_page():
    """an opaque page with no child is its own bytes, b and r swapped, in both modes"""
    pg = page(37, 23, 4, translucent=False)
    for m in (orc.MODE_GPU_OPTIMIZED, orc.MODE_CPU_OPTIMIZED):
        got = oracle_web.render_web(np.zeros((23, 37, 4), np.uint8), pg, [], [], OVER, m)
        assert np.array_equal(got, pg[..., [2, 1, 0, 3]])
    assert not oracle_web.render_web(np.zeros((4, 4, 4), np.uint8), None, [], [], OVER).any()


# ---- GPU ------------------------------------------------------------------------------------------------------------
RECTS = {
    "integer": [(40, 30, 320, 180), (400, 200, 200, 112)],
    "fractional": [(40.25, 30.5, 319.75, 180.125), (400.6, 200.3, 201.1, 111.9)],
    "off_page": [(-100, -50, 320, 180), (700, 380, 320, 180)],
    "zero_sized": [(10, 10, 0, 100), (50, 50, 200, 0)],
    "more_rects": [(40, 30, 320, 180), (400, 200, 200, 112), (0, 0, 800, 450)],
    "fewer_rects": [(40, 30, 320, 180)],
    "no_rects": [],
    "mirrored": [(360, 30, -320, 180), (600, 312, -200, -112)],
}


def _two_inputs():
    return [IN(id="a", input_id="input_1"), IN(id="b", input_id="nv12_2")]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("embedding", [OVER, UNDER])
@pytest.mark.parametrize("rects", sorted(RECTS))
def test_rects_and_embeddings_match_oracle(rects, embedding, mode, fmt):
    p = Pair(out=(800, 450) if fmt == RGBA else (640, 360), fmt=fmt, mode=mode, inputs=("input_1", "nv12_2"))
    p.register_web("page", 800, 450, embedding)
    p.update(web(children=_two_inputs()))
    p.render_check(0.0, "no frame yet")                       # transparent
    p.set_frame("page", page(800, 450, 1))
    p.set_rects("page", RECTS[rects])
    p.render_check(0.04, rects)
    p.render_check(0.08, rects + ", again")


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("mode", MODES)
def test_children_of_every_kind_match_oracle(mode, fmt):
    """YUV, NV12, RGBA and BGRA inputs, a stale input, an Image and a Text child; one web view scaled by Lanczos, one
    under a rounded mask beside it"""
    p = Pair(fmt=fmt, mode=mode, inputs=("input_1", "nv12_2", "input_3", "rgba_4", "bgra_5"))
    p.register_image("img", pixels(90, 60, 1, 5)[0])
    p.register_web("page", 800, 450, OVER)
    p.register_web("small", 300, 170, UNDER)
    kids = _two_inputs() + [IN(id="c", input_id="input_3"), IMG(id="i", image_id="img"), label(120, 24, 3, id="t"),
                            IN(id="e", input_id="rgba_4"), IN(id="f", input_id="bgra_5")]
    p.update(V(background_color=s.RGBAColor(10, 20, 30, 255), children=[
        R(child=web("page", kids)),                                                     # 800 x 450 -> Lanczos
        cell(330, 170, 300, 170, web("small", [IN(id="d", input_id="input_1")]),
             border_radius=s.BorderRadius(30.0, 10.0, 40.0, 5.0), overflow=s.Overflow.Hidden)]))
    p.set_frame("page", page(800, 450, 2))
    p.set_frame("small", page(300, 170, 3))
    p.set_rects("page", [(10, 10, 320, 180), (350.5, 20.25, 300, 170), (20, 240, 200, 112), (500, 250, 180, 120), (600, 400, 120, 24),
                         (250.25, 200, 240, 135), (560, 20.5, 200, 150)])
    p.set_rects("small", [(20.5, 10, 250, 140)])
    p.r.set_profiling(True)
    p.render_check(6.0, "children", stale=("input_3",))
    assert p.r.kernel_times()["web"][1] == 1                # both web nodes in one launch
    p.render_check(6.04, "children, input_3 live")


@pytest.mark.gpu
def test_unregistered_instance_keeps_drawing_and_frames_update():
    p = Pair(inputs=("input_1",))
    p.register_web("page", 640, 360, OVER)
    p.update(web(children=[IN(id="a", input_id="input_1")]))
    p.set_frame("page", page(640, 360, 7))
    p.set_rects("page", [(100, 50, 320, 180)])
    p.render_check(0.0)
    p.gone["page"] = p.ref.webs["page"]
    p.unregister_web("page")
    p.render_check(0.04, "unregistered")
    with pytest.raises(s.RendererError):
        p.r.set_web_frame("page", page(640, 360, 8))
    assert _status(p.r, web("page")) == 4


class _Tick:
    """one smr_render_begin with host output planes that stay alive until its smr_render_end.  The planes are page-locked
    (torch pinned memory): a read-back into pageable memory would return only once the tick is complete."""

    def __init__(self, r, pts, frames, out, fmt, torch):
        self.keep = []
        self.in_arr = r._input_frames(s.FrameSet(frames=frames, pts=pts), self.keep)
        sizes = (C.c_size_t * 3)()
        F.lib().smr_output_plane_sizes(out[0], out[1], fmt, C.byref(sizes))
        pinned = [torch.zeros(sizes[p], dtype=torch.uint8).pin_memory() if sizes[p] else None for p in range(3)]
        self.keep.append(pinned)
        self.planes = [t.numpy() if t is not None else None for t in pinned]
        self.out_arr = (F.OutputFrame * 1)()
        self.out_arr[0].output_id = b"output_1"
        self.out_arr[0].mem_kind = F.MEM_HOST
        for p in range(3):
            if self.planes[p] is not None:
                self.out_arr[0].planes[p] = self.planes[p].ctypes.data
        r.render_raw(int(round(pts * 1e9)), self.in_arr, len(frames), self.out_arr, 1, wait=False)


@pytest.mark.gpu
def test_four_ticks_in_flight_across_frames_and_rects():
    """a new frame and rect list every second tick while the earlier ticks are still queued behind a busy render stream:
    each tick shows the frame and rects that were set when it was submitted, and setting a frame does not wait for them"""
    torch = pytest.importorskip("torch")
    p = Pair(inputs=("input_1",))
    p.register_web("page", 640, 360, OVER)
    p.update(V(children=[R(child=IN(input_id="input_1")), cell(100, 60, 400, 225, web(children=[IN(id="a", input_id="input_1")]))]))
    stream = torch.cuda.ExternalStream(p.r.cuda_stream(), device=torch.device("cuda:0"))
    pages = [page(640, 360, 20 + k) for k in range(4)]
    for k in range(4):                       # every kernel loaded, and room in the frame pool for the frames in flight
        p.set_frame("page", pages[k])
        p.r.render(s.FrameSet(frames=p.frames(0.0), pts=0.0))
    done = []
    for batch in range(2):
        ks = range(4 * batch, 4 * batch + 4)
        frames = {k: p.frames(1.0 + k * 0.04) for k in ks}
        with torch.cuda.stream(stream):
            torch.cuda._sleep(1_000_000_000)   # about half a second: the ticks below wait behind it on the render stream
        ticks, t0, steps = [], time.perf_counter(), []
        for k in ks:
            if k % 2 == 0:
                p.set_frame("page", pages[(k // 2) % 4])
                steps.append(("frame", time.perf_counter() - t0))
                p.set_rects("page", [(10 * k, 5 * k, 320 - 8 * k, 180)])
            pts = 1.0 + k * 0.04
            ticks.append((_Tick(p.r, pts, frames[k], p.out, p.fmt, torch), pts, frames[k], p.pages["page"], p.rects["page"]))
            steps.append(("tick", time.perf_counter() - t0))
        took = f"{time.perf_counter() - t0:.3f} s: " + ", ".join(f"{n} {t:.3f}" for n, t in steps)
        # the frames and rects changed while every tick of the batch was in flight
        assert not stream.query(), f"the render stream drained during the batch ({took})"
        for _ in ticks:
            p.r.wait()
        done += ticks
    for t, pts, frames, pg, rects in done:
        p.pages["page"], p.rects["page"] = pg, rects
        assert_identical([pl for pl in t.planes if pl is not None], p.expected(pts, frames), f"tick at {pts}")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_pitched_host_and_device_frames(mode):
    """smr_web_set_frame from a padded device tensor and a padded host plane; both are copied before the call returns"""
    torch = pytest.importorskip("torch")
    p = Pair(out=(320, 180), fmt=RGBA, mode=mode, inputs=("input_1",))
    p.register_web("page", 320, 180, UNDER)
    p.update(web(children=[IN(id="a", input_id="input_1")]))
    p.set_rects("page", [(20.5, 10, 160, 90)])
    pg = page(320, 180, 31)
    big = torch.zeros((180, 344, 4), dtype=torch.uint8, device="cuda:0")
    big[:, :320] = torch.from_numpy(pg).cuda()
    torch.cuda.synchronize()
    assert big[:, :320].stride(0) == 344 * 4
    p.r.set_web_frame("page", big[:, :320], mem_kind=F.MEM_DEVICE)
    p.pages["page"] = pg
    big.fill_(7)
    torch.cuda.synchronize()
    p.render_check(0.0, "device, pitched")
    pg2 = page(320, 180, 32)
    padded = np.full((180, 330, 4), 9, np.uint8)
    padded[:, :320] = pg2
    f = F.WebFrame(padded.ctypes.data, 320, 180, 330 * 4, F.MEM_HOST)
    assert F.lib().smr_web_set_frame(p.r._h, b"page", C.byref(f)) == 0
    p.pages["page"] = pg2
    padded[:] = 9
    p.render_check(0.04, "host, pitched")
