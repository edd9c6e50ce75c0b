"""The independent layout engine (tests/layout_ref.py, with the Text and Image leaves of tests/layout_ref_text.py and
tests/layout_ref_image.py) with WebView components and the web renderer registry.  Test infrastructure.

Restated from the Rust sources, like the engines it extends:

  registry.rs:57-68                  register: KeyTaken when the id exists; unregister: an error when it does not
  scene/validation.rs:35-100         before anything is built: duplicate component ids within an output (a WebView's children
                                     included), then one WebView per instance across every output as it would be after the
                                     update (WebRendererUsageNotExclusive)
  scene/web_view_component.rs:41-71  WebRendererNotFound; then the children are built; then every child needs an id
                                     (WebViewChildWithoutId)
  scene/web_view_component.rs:23-25  the size is the instance's resolution
  scene.rs:101-127, scene/layout.rs:95-158
                                     a WebView is a node child of its layout with a static size and no layout state, like an
                                     Image; its own children are render nodes under it, never laid out
  scene_state.rs:154-196             a WebView root is not a layout node: no layouts

A WebView component here is smelter_b200.WebViewComponent; the product accepts InputStream, Image and Text children only.
"""
import numpy as np

import smelter_b200 as s
from tests import layout_ref as LR
from tests import layout_ref_image as LI
from tests import layout_ref_text as LT

F = LR.F
LEAVES = ("input", "text", "image", "web")
SceneError, RegistryError = LI.SceneError, LI.RegistryError


class Instance:
    """a registered web renderer (compared by identity)"""

    def __init__(self, width, height, embedding):
        self.width, self.height, self.embedding = width, height, embedding


class SNode(LI.SNode):
    """StatefulComponent with the WebView variant"""

    def __init__(self, comp, ctx):
        if not isinstance(comp, s.WebViewComponent):
            if isinstance(comp, (s.TextComponent, s.ImageComponent)):
                LI.SNode.__init__(self, comp, ctx)
            else:
                self._init_component(comp, ctx)
            return
        self.comp, self.kind = comp, "web"
        self.instance = ctx["webs"].get(comp.instance_id)
        if self.instance is None:
            raise SceneError(f"WebRendererNotFound({comp.instance_id})")
        self.children = [SNode(k, ctx) for k in comp.children]
        if any(getattr(k, "id", None) is None for k in comp.children):
            raise SceneError(f"WebViewChildWithoutId({comp.instance_id})")
        self.size = (F(self.instance.width), F(self.instance.height))

    def _init_component(self, comp, ctx):   # LI.SNode._init_component, its children built by this class
        self.comp = comp
        self.kind = ("input" if isinstance(comp, s.InputStreamComponent) else "view" if isinstance(comp, s.ViewComponent)
                     else "rescaler" if isinstance(comp, s.RescalerComponent) else "tiles")
        prev = ctx["prev"].get(comp.id) if getattr(comp, "id", None) is not None else None
        if prev is not None and prev.kind != self.kind:
            prev = None
        last = ctx["last_ns"]
        if self.kind == "input":
            r = ctx["resolutions"].get(comp.input_id)
            self.size = (F(r[0]), F(r[1])) if r is not None else (LR.ZERO, LR.ZERO)
            self.children = []
            return
        kids = [comp.child if comp.child is not None else s.ViewComponent()] if self.kind == "rescaler" else list(comp.children)
        if self.kind in ("view", "rescaler"):
            self.start = prev.params(last) if prev is not None else None
            self.end = LR.params_of(comp)
            changed = prev is not None and LR.comparable(prev.comp) != LR.comparable(comp)
        else:
            self.start = prev.last_layout if prev is not None else None
            self.last_layout = prev.last_layout if prev is not None else None
            changed = False
            if prev is not None:
                ids_a = [getattr(k.comp, "id", None) for k in prev.children]
                ids_b = [getattr(k, "id", None) for k in kids]
                changed = LR.comparable(prev.comp) != LR.comparable(comp) or ids_a != ids_b
        t = comp.transition
        self.transition = LR.TransitionState.new(t, prev.transition if prev is not None else None, changed,
                                                 bool(t.should_interrupt) if t is not None else False, last)
        self.children = [SNode(k, ctx) for k in kids]

    def node_children(self):
        out = []
        for k in self.children:
            out += [k] if k.kind in LEAVES else k.node_children()
        return out


class Engine(LI.Engine):
    def is_layout(self, n):
        return n.kind not in LEAVES

    def width(self, n):
        return n.size[0] if n.kind in LEAVES else self.position(n)[1]

    def height(self, n):
        return n.size[1] if n.kind in LEAVES else self.position(n)[2]

    def update_state(self, n, sizes):      # layout.rs:103-132: Text, Image and WebView have no state
        i = 0
        for k in n.children:
            if k.kind == "input":
                r = sizes[i]
                k.size = (F(r[0]), F(r[1])) if r is not None else (LR.ZERO, LR.ZERO)
                i += 1
            elif k.kind in LEAVES:
                i += 1
            else:
                cnt = len(k.node_children())
                self.update_state(k, sizes[i:i + cnt])
                i += cnt


def web_instance_ids(comp, out):
    if isinstance(comp, s.WebViewComponent):
        out.append(comp.instance_id)
    kids = [comp.child] if isinstance(comp, s.RescalerComponent) and comp.child is not None else getattr(comp, "children", None) or []
    for k in kids:
        web_instance_ids(k, out)
    return out


class StatefulScene(LI.StatefulScene):
    """one output's scene over image and web registries; `others` holds the scenes of the other outputs (for the
    exclusivity of web renderer instances)"""

    def __init__(self, out_w, out_h, images=None, webs=None):
        super().__init__(out_w, out_h, images)
        self.webs = webs if webs is not None else {}
        self.others = []

    def register_web(self, instance_id, width, height, embedding=1):
        if instance_id in self.webs:
            raise RegistryError("KeyTaken")
        self.webs[instance_id] = Instance(width, height, embedding)

    def unregister_web(self, instance_id):
        if instance_id not in self.webs:
            raise RegistryError("NotRegistered")
        del self.webs[instance_id]

    def update_scene(self, scene):
        ids = LI.component_ids(scene, [])
        if len(set(ids)) != len(ids):
            raise SceneError("duplicate component ids")
        used = web_instance_ids(scene, [])
        for other in self.others:
            used += web_instance_ids(other, [])
        if len(set(used)) != len(used):
            raise SceneError("WebRendererUsageNotExclusive")
        if self.scene_tree is not None and self.scene_tree.kind not in LEAVES:   # recalculate_layout at last_pts
            Engine(self.last_ns).layout(self.scene_tree, F(self.out_w), F(self.out_h))
        prev = self.scene_tree.with_id({}) if self.scene_tree is not None else {}
        ctx = {"prev": prev, "last_ns": self.last_ns, "resolutions": dict(self.resolutions), "images": self.images,
               "webs": self.webs}
        tree = SNode(scene, ctx)                     # a SceneError leaves the scene as it was
        self.scene_tree = tree
        self.render_tree = tree.clone()

    def layouts(self, pts, resolutions_by_input_id):
        pts_ns = LR.to_ns(pts)
        self.last_ns, self.resolutions = pts_ns, dict(resolutions_by_input_id)   # register_render_event
        root = self.render_tree
        if root.kind in LEAVES:
            return [], (0, 0)
        eng = Engine(pts_ns)
        leaves = root.node_children()
        in_res = [resolutions_by_input_id.get(k.comp.input_id) if k.kind == "input" else
                  LT.texture_size(k.comp) if k.kind == "text" else
                  (k.instance.width, k.instance.height) if k.kind == "web" else k.resolution for k in leaves]
        eng.update_state(root, in_res)
        p = eng.position(root)
        w = p[1] if p[1] is not None else F(self.out_w)
        h = p[2] if p[2] is not None else F(self.out_h)
        rw, rh = int(np.trunc(w)), int(np.trunc(h))
        nested = eng.layout(root, F(self.out_w), F(self.out_h))
        return LR.flatten(nested, in_res, rw, rh), (rw, rh)
