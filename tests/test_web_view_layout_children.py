"""View, Tiles and Rescaler children of WebView components: each is a layout node of its own, below which any component
may appear (Shaders and WebViews included), and each web node is drawn at its depth.

CPU (host-only handle): root layouts and every smr_debug_node_layouts node against the independent engine
(tests/layout_ref_web_layout.py), across scene updates, and the refusals.  GPU: every output byte against the oracle.
"""
import pytest

import smelter_b200 as s
from tests import layout_ref_web_layout as LWL
from tests import oracle_web
from tests import test_shader_component as TS
from tests import test_web_view_component as TW
from tests.test_image_component import pixels
from tests.test_layout_independent import product_layouts
from tests.test_text_component import label

V, R, T, IN, IMG, WEB, SH = (s.ViewComponent, s.RescalerComponent, s.TilesComponent, s.InputStreamComponent, s.ImageComponent,
                             s.WebViewComponent, s.ShaderComponent)
YUV = TW.YUV
web, cell = TW.web, TW.cell


def sized(w, h):
    return s.Position.Static(width=float(w), height=float(h))


class Pair(TS.Pair):
    """the shader test's renderer / independent engine pair, WebViews holding layout nodes; a web node's children are
    drawn at the tick's pts"""

    def __init__(self, **kw):
        super().__init__(**kw)
        self.ref = LWL.StatefulScene(*self.out)

    def leaf_texture(self, c, frames, live, pts=0.0):
        if isinstance(c, WEB):
            return self.web_texture(c, frames, live, pts)
        return super().leaf_texture(c, frames, live, pts)

    def web_texture(self, c, frames, live, pts=0.0):
        inst = self.ref.webs.get(c.instance_id) or self.gone[c.instance_id]
        prev = self.tex.get(id(c), TW.np.zeros((inst.height, inst.width, 4), TW.np.uint8))
        kids = [self.leaf_texture(k, frames, live, pts) for k in c.children]
        t = oracle_web.render_web(prev, self.pages.get(c.instance_id), kids, self.rects[c.instance_id], inst.embedding, self.m)
        self.tex[id(c)] = t
        return t


def host(**kw):
    return Pair(device=-1, **kw)


def _register(p, webs=(("page", 800, 450, TW.OVER), ("other", 320, 180, TW.UNDER))):
    for k in TS.SOURCES:
        p.register_shader(k)
    for w in webs:
        p.register_web(*w)


def _three(prefix="i"):
    return [IN(id=f"{prefix}{k}", input_id=f"input_{k}") for k in (1, 2, 3)]


# ---- CPU ------------------------------------------------------------------------------------------------------------
CASES = {
    "rescaler": (lambda: web(children=[R(id="r", position=sized(320, 180), mode=s.RescaleMode.Fill,
                                         child=IN(input_id="input_1"))]), 1),
    "tiles": (lambda: web(children=[T(id="t", width=600.0, height=300.0, children=_three())]), 1),
    "view_nested": (lambda: web(children=[V(id="v", position=sized(400, 240), background_color=s.RGBAColor(40, 0, 60, 200),
                                            children=[V(children=[IN(input_id="input_1"), IN(input_id="input_2")]),
                                                      label(120, 24, 3), IMG(image_id="img", width=90.0)])]), 1),
    "in_root_view": (lambda: V(children=[IN(input_id="input_1"), web(children=[
        IN(id="a", input_id="input_2"), V(id="v", position=sized(320, 180), children=[IN(input_id="input_3")])])]), 1),
    "shader": (lambda: V(children=[web(children=[V(id="v", position=sized(640, 360), children=[
        SH(shader_id="grade", shader_param=TS.grade(), width=640, height=360, children=[
            V(position=sized(320, 180), children=[IN(input_id="input_1")])])])])]), 2),
    "web_in_web": (lambda: V(children=[IN(input_id="input_1"), web(children=[V(id="v", position=sized(400, 225), children=[
        web("other", id="w", children=[IN(id="a", input_id="input_2")])])])]), 1),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_layouts_and_layout_nodes_match_independent_engine(name):
    p = host(inputs=("input_1", "input_2", "input_3"))
    _register(p)
    p.register_image("img", pixels(90, 60, 1, 5)[0])
    scene, n_nodes = CASES[name]
    p.update(scene())
    assert len(p.nested) == n_nodes
    for pts in (0.0, 0.5):
        p.check_layouts(pts)
        p.check_node_layouts(pts)


def test_layout_children_state_across_scene_updates():
    """a View child of a web under a transition, and a Tiles child reordered with one tile removed: the layout nodes'
    state carries over the scene updates"""
    p = host(inputs=("input_1", "input_2", "input_3"))
    _register(p)
    tr = s.Transition(duration=1.0)

    def scene(direction, ids, t=None):
        return V(children=[IN(input_id="input_1"), web(children=[
            V(id="v", position=sized(400, 240), direction=direction, transition=t,
              children=[IN(id="x", input_id="input_1"), R(child=IN(input_id="input_2"))]),
            T(id="t", width=600.0, height=300.0, transition=t,
              children=[IN(id=i, input_id="input_3" if i == "c" else "input_1") for i in ids])])])
    p.update(scene(s.ViewChildrenDirection.Row, ["a", "b", "c"]))
    assert len(p.nested) == 2
    p.check_layouts(0.0)
    p.check_node_layouts(0.0)
    p.update(scene(s.ViewChildrenDirection.Column, ["c", "a"], tr))
    for pts in (0.0, 0.25, 0.5, 0.99, 1.5):
        p.check_layouts(pts)
        p.check_node_layouts(pts)


def _status(r, scene):
    with pytest.raises(s.RendererError) as e:
        r.update_scene("output_1", s.Resolution(640, 360), YUV, scene)
    return e.value.status


def test_refusals_leave_the_scene_as_it_was():
    p = host(inputs=("input_1",))
    _register(p)
    p.update(V(children=[IN(input_id="input_1"), web(children=[V(id="v", position=sized(320, 180), children=[IN(input_id="input_1")])])]))
    node = TS._Node(p.r, 1)
    before, before_node = product_layouts(p.r, 0.0), product_layouts(node, 0.0)
    grad = lambda *kids, **kw: SH(shader_id="gradient", width=8, height=8, children=list(kids), **kw)
    refused = {
        4: [web(children=[V(position=sized(64, 64), children=[IN(input_id="input_1")])]),        # WebViewChildWithoutId
            web(children=[T(width=64.0, height=64.0)]),
            web(children=[V(id="v", position=sized(64, 64), children=[grad(V())])]),            # a sizeless deeper layout root
            web(children=[V(id="v", position=sized(64, 64), children=[grad(R(child=IN(input_id="input_1")))])]),
            web(children=[V(id="v", position=sized(64, 64), children=[web("page", id="w")])]),  # "page" twice, nested
            web(children=[V(id="v", position=sized(64, 64), children=[grad(web("page", id="w"))])]),
            V(children=[web("other", id="w"), web(children=[T(id="t", width=64.0, height=64.0, children=[web("other", id="x")])])]),
            web(children=[V(id="a", position=sized(64, 64), children=[IN(id="a", input_id="input_1")])]),   # duplicate ids
            web(children=[V(id="v", position=sized(64, 64), children=[web("missing", id="m")])]),     # WebRendererNotFound
            web(children=[V(id="v", position=sized(64, 64), children=[web("other", id="w", children=[IN(input_id="input_1")])])])],
        5: [web(children=[web("other", id="w")]), web(children=[grad(id="x")]),
            web(children=[V(id="v")]), web(children=[V(id="v", position=s.Position.Static(width=64.0))]),
            web(children=[R(id="r", position=s.Position.Static(height=64.0), child=IN(input_id="input_1"))]),
            web(children=[T(id="t", width=64.0)]), web(children=[T(id="t", height=64.0)]),
            web(children=[V(id="v", position=s.Position.Absolute(width=64.0, left=0.0, top=0.0))]),
            web(children=[V(id="v", position=sized(64, 64), children=[web("other", id="w", children=[V(id="x")])])])],
    }
    for status, scenes in refused.items():
        for scene in scenes:
            assert _status(p.r, scene) == status, scene
            if status == 4:
                with pytest.raises(LWL.SceneError):
                    p.ref.update_scene(scene)
            assert product_layouts(p.r, 0.0) == before and product_layouts(node, 0.0) == before_node, scene
    p.check_layouts(0.0)
    p.check_node_layouts(0.0)


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _gpu_pair(fmt, mode, inputs=("input_1", "nv12_2", "input_3"), **kw):
    p = Pair(fmt=fmt, mode=mode, inputs=inputs, **kw)
    for k in TS.SOURCES:
        p.register_shader(k)
    return p


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", TW.FORMATS)
@pytest.mark.parametrize("mode", TW.MODES)
@pytest.mark.parametrize("embedding", [TW.OVER, TW.UNDER])
def test_sized_layout_children_match_oracle(embedding, mode, fmt):
    """a Rescaler the fused kernel Lanczos-scales (640 x 360 -> 320 x 180), a Tiles of three inputs and a View holding a
    View, a Text and an Image, embedded in a page; an input child beside them; a stale input inside the Tiles"""
    p = _gpu_pair(fmt, mode)
    p.register_image("img", pixels(90, 60, 1, 5)[0])
    p.register_web("page", 800, 450, embedding)
    p.update(V(background_color=s.RGBAColor(10, 20, 30, 255), children=[R(child=web(children=[
        R(id="r", position=sized(320, 180), child=IN(input_id="input_1")),
        T(id="t", width=400.0, height=225.0, background_color=s.RGBAColor(0, 60, 0, 255),
          children=[IN(input_id="input_1"), IN(input_id="nv12_2"), IN(input_id="input_3")]),
        V(id="v", position=sized(300, 170), background_color=s.RGBAColor(40, 0, 60, 200), children=[
            V(children=[IN(input_id="nv12_2")]), cell(20, 100, 120, 24, label(120, 24, 3)),
            cell(180, 80, 90, 60, IMG(image_id="img"), border_radius=s.BorderRadius(20.0, 5.0, 30.0, 10.0), overflow=s.Overflow.Hidden)]),
        IN(id="a", input_id="nv12_2")]))]))
    p.set_frame("page", TW.page(800, 450, 2))
    p.set_rects("page", [(10, 10, 320, 180), (350.5, 20.25, 400, 225), (20, 240, 300, 170), (500.25, 280, 240, 135)])
    p.r.set_profiling(True)
    p.render_check(6.0, "layout children", stale=("input_3",))
    assert p.r.kernel_times()["web"][1] == 1                # one web node at depth 2: one launch
    p.render_check(6.04, "layout children, input_3 live")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", TW.MODES)
def test_deep_nestings_match_oracle(mode):
    """web > View > Shader > View > input (web depth 4), and web > View > web > input (depths 3 and 1): one web launch
    per distinct depth"""
    p = _gpu_pair(YUV, mode)
    p.register_web("page", 640, 360, TW.OVER)
    p.register_web("outer", 480, 270, TW.UNDER)
    p.register_web("inner", 320, 180, TW.OVER)
    p.update(V(background_color=s.RGBAColor(10, 20, 30, 255), children=[
        R(child=web("page", children=[V(id="v", position=sized(400, 225), children=[
            SH(shader_id="grade", shader_param=TS.grade(), width=400, height=225, children=[
                V(position=sized(320, 180), children=[R(child=IN(input_id="input_1"))])])])])),
        R(child=web("outer", children=[V(id="w", position=sized(400, 225), children=[
            web("inner", id="x", children=[IN(id="a", input_id="nv12_2")])])]))]))
    for k, (iid, w, h) in enumerate((("page", 640, 360), ("outer", 480, 270), ("inner", 320, 180))):
        p.set_frame(iid, TW.page(w, h, 10 + k))
    p.set_rects("page", [(40.5, 30, 400, 225)])
    p.set_rects("outer", [(20, 10.25, 400, 225)])
    p.set_rects("inner", [(60, 40, 160, 90)])
    p.r.set_profiling(True)
    p.render_check(0.5, "deep")
    assert p.r.kernel_times()["web"][1] == 3                # web depths 1, 3 and 4
    p.render_check(0.54, "deep, again")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", TW.MODES)
def test_web_without_frame_keeps_evaluating_its_layout_child(mode):
    """a web node with no frame is not drawn while its layout child moves through a transition; once it has a frame it
    shows the child where the transition has got to"""
    p = _gpu_pair(YUV, mode)
    p.register_web("page", 640, 360, TW.OVER)
    tr = s.Transition(duration=1.0)
    sc = lambda d, t=None: V(children=[IN(input_id="input_1"), web(children=[
        V(id="v", position=sized(480, 270), direction=d, transition=t, background_color=s.RGBAColor(0, 0, 80, 255),
          children=[IN(id="x", input_id="nv12_2"), T(id="t", children=[IN(input_id="input_1"), IN(input_id="input_3")])])])])
    p.update(sc(s.ViewChildrenDirection.Row))
    p.set_rects("page", [(80, 45, 480, 270)])
    p.render_check(0.0, "no frame")
    p.update(sc(s.ViewChildrenDirection.Column, tr))
    for pts in (0.25, 0.5):
        p.render_check(pts, "no frame, mid-transition")
    p.set_frame("page", TW.page(640, 360, 5))
    for pts in (0.75, 1.5):
        p.render_check(pts, "frame")


@pytest.mark.gpu
def test_four_ticks_in_flight_across_frames_rects_and_a_transition():
    """a new frame and rect list every second tick while the earlier ticks are still queued behind a busy render stream,
    the web's layout child in a transition: each tick shows the frame and rects set when it was submitted, and the layout
    node's composite of its own pts"""
    torch = pytest.importorskip("torch")
    p = _gpu_pair(YUV, s.RenderingMode.GpuOptimized, inputs=("input_1", "nv12_2"))
    p.register_web("page", 640, 360, TW.OVER)
    sc = lambda d, t=None: V(children=[R(child=IN(input_id="input_1")), cell(100, 60, 400, 225, web(children=[
        V(id="v", position=sized(320, 180), direction=d, transition=t,
          children=[R(child=IN(input_id="input_1")), IN(id="b", input_id="nv12_2")])]))])
    p.update(sc(s.ViewChildrenDirection.Row))
    pages = [TW.page(640, 360, 20 + k) for k in range(4)]
    for k in range(4):                       # every kernel loaded, and room in the frame pool for the frames in flight
        p.set_frame("page", pages[k])
        p.r.render(s.FrameSet(frames=p.frames(0.0), pts=0.0))
    p.update(sc(s.ViewChildrenDirection.Column, s.Transition(duration=2.0)))   # from pts 0 to 2: the ticks below are mid-way
    stream = torch.cuda.ExternalStream(p.r.cuda_stream(), device=torch.device("cuda:0"))
    frames = {k: p.frames(1.0 + k * 0.04) for k in range(4)}
    with torch.cuda.stream(stream):
        torch.cuda._sleep(1_000_000_000)   # about half a second: the ticks below wait behind it on the render stream
    ticks = []
    for k in range(4):
        if k % 2 == 0:
            p.set_frame("page", pages[(k // 2 + 1) % 4])
            p.set_rects("page", [(10 * k, 5 * k, 320 - 8 * k, 180)])
        pts = 1.0 + k * 0.04
        ticks.append((TW._Tick(p.r, pts, frames[k], p.out, p.fmt, torch), pts, frames[k], p.pages["page"], p.rects["page"]))
    assert not stream.query(), "the render stream drained before the ticks were checked"
    for _ in ticks:
        p.r.wait()
    for t, pts, fr, pg, rects in ticks:
        p.pages["page"], p.rects["page"] = pg, rects
        TW.assert_identical([pl for pl in t.planes if pl is not None], p.expected(pts, fr), f"tick at {pts}")
