"""The independent layout engine (tests/layout_ref.py) with Text components.  Test infrastructure.

Restated from the Rust sources, like the engine it extends:

  scene.rs:101-127                 width / height of a Text: Some(resolution), fixed when the scene is built
  scene/text_component.rs:36-53    StatefulTextComponent: the caller's layout resolution, no state
  scene/layout.rs:95-158           a Text is a node child (DFS order); update_state only advances the child index;
                                   layout_content is ChildNode { size: resolution }
  transformations/layout.rs:176-179, text_renderer.rs:77-85
                                   the node texture the flattened layouts see is width x height, or 1 x 1 for 0 x 0
  scene_state.rs:154-196           a Text root is not a layout node: no layouts

A Text component here is smelter_b200.TextComponent; only its id, width and height matter to the layout.
"""
import numpy as np

import smelter_b200 as s
from tests import layout_ref as LR

F = LR.F
LEAVES = ("input", "text")   # StatefulComponent::InputStream / Text


def texture_size(comp):
    """the resolution of a Text component's node texture"""
    return (comp.width, comp.height) if comp.width and comp.height else (1, 1)


class SNode(LR.SNode):
    """StatefulComponent with the Text variant"""

    def __init__(self, comp, ctx):
        if not isinstance(comp, s.TextComponent):
            self._init_component(comp, ctx)
            return
        self.comp, self.kind, self.children = comp, "text", []
        self.size = (F(comp.width), F(comp.height))

    def _init_component(self, comp, ctx):   # LR.SNode.__init__, its children built by this class
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

    def node_children(self):           # layout.rs:93-101
        out = []
        for k in self.children:
            out += [k] if k.kind in LEAVES else k.node_children()
        return out


class Engine(LR.Engine):
    def is_layout(self, n):
        return n.kind not in LEAVES

    def width(self, n):
        return n.size[0] if n.kind in LEAVES else self.position(n)[1]

    def height(self, n):
        return n.size[1] if n.kind in LEAVES else self.position(n)[2]

    def update_state(self, n, sizes):      # layout.rs:103-132: a Text has no state, it only takes its child index
        i = 0
        for k in n.children:
            if k.kind == "input":
                r = sizes[i]
                k.size = (F(r[0]), F(r[1])) if r is not None else (LR.ZERO, LR.ZERO)
                i += 1
            elif k.kind == "text":
                i += 1
            else:
                cnt = len(k.node_children())
                self.update_state(k, sizes[i:i + cnt])
                i += cnt


class StatefulScene(LR.StatefulScene):
    """LR.StatefulScene whose trees may hold Text components"""

    def update_scene(self, scene):
        if self.scene_tree is not None and self.scene_tree.kind not in LEAVES:   # recalculate_layout at last_pts
            Engine(self.last_ns).layout(self.scene_tree, F(self.out_w), F(self.out_h))
        prev = self.scene_tree.with_id({}) if self.scene_tree is not None else {}
        ctx = {"prev": prev, "last_ns": self.last_ns, "resolutions": dict(self.resolutions)}
        self.scene_tree = SNode(scene, ctx)
        self.render_tree = self.scene_tree.clone()

    def layouts(self, pts, resolutions_by_input_id):
        pts_ns = LR.to_ns(pts)
        self.last_ns, self.resolutions = pts_ns, dict(resolutions_by_input_id)   # register_render_event
        root = self.render_tree
        if root.kind in LEAVES:
            return [], (0, 0)
        eng = Engine(pts_ns)
        leaves = root.node_children()
        in_res = [resolutions_by_input_id.get(k.comp.input_id) if k.kind == "input" else texture_size(k.comp) for k in leaves]
        eng.update_state(root, in_res)
        p = eng.position(root)           # SizedLayoutComponent::resolution; Size -> Resolution truncates
        w = p[1] if p[1] is not None else F(self.out_w)
        h = p[2] if p[2] is not None else F(self.out_h)
        rw, rh = int(np.trunc(w)), int(np.trunc(h))
        nested = eng.layout(root, F(self.out_w), F(self.out_h))
        return LR.flatten(nested, in_res, rw, rh), (rw, rh)
