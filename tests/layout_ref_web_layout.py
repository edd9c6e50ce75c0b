"""The independent layout engine with Shaders (tests/layout_ref_shader.py) whose WebViews hold any render node: a View,
Tiles or Rescaler child of a WebView is a layout node of its own, and below it any component may appear, Shaders and
WebViews included.  Test infrastructure.

Restated from the Rust sources, like the engines it extends:

  scene/web_view_component.rs:41-71  WebRendererNotFound; then the children are built (every kind of component); then
                                     every child needs an id (WebViewChildWithoutId)
  scene/validation.rs:35-100         duplicate component ids, then one WebView per instance across every output, at any
                                     depth of nesting (WebRendererUsageNotExclusive)
  scene_state.rs:154-228             a WebView's children are render nodes; a View, Tiles or Rescaler among them is a layout
                                     node whose size is node_size at the last render's pts (UnknownDimensionsForLayoutNodeRoot
                                     without width and height)
"""
import smelter_b200 as s
from tests import layout_ref as LR
from tests import layout_ref_shader as LS
from tests import layout_ref_web as LW

F = LR.F
LEAVES = LS.LEAVES
SceneError, RegistryError = LS.SceneError, LS.RegistryError
Engine, render_nodes, recalculate_layout, component_ids = LS.Engine, LS.render_nodes, LS.recalculate_layout, LS.component_ids


class SNode(LS.SNode):
    """StatefulComponent whose every child, at any depth, is built by this class"""

    def __init__(self, comp, ctx):
        if isinstance(comp, s.WebViewComponent):
            self.comp, self.kind = comp, "web"
            self.instance = ctx["webs"].get(comp.instance_id)
            if self.instance is None:
                raise SceneError(f"WebRendererNotFound({comp.instance_id})")
            self.children = [SNode(k, ctx) for k in comp.children]
            if any(getattr(k, "id", None) is None for k in comp.children):
                raise SceneError(f"WebViewChildWithoutId({comp.instance_id})")
            self.size = (F(self.instance.width), F(self.instance.height))
        elif isinstance(comp, s.ShaderComponent):   # LS.SNode's Shader variant
            self.comp, self.kind = comp, "shader"
            self.shader = ctx["shaders"].get(comp.shader_id)
            if self.shader is None:
                raise SceneError(f"ShaderNotFound({comp.shader_id})")
            if comp.shader_param is not None:
                if self.shader.param_type is None:
                    raise SceneError("ShaderNodeParametersValidationError(NoBindingInShader)")
                LS.validate(comp.shader_param, self.shader.param_type)
            self.children = [SNode(k, ctx) for k in comp.children]
            self.size = (F(comp.width), F(comp.height))
            res = [int(v) if v > 0 else 0 for v in self.size]
            if any(r == 0 or r > 16384 for r in res):
                raise SceneError(f"shader node of {res[0]} x {res[1]}")
        elif isinstance(comp, (s.TextComponent, s.ImageComponent)):
            LS.SNode.__init__(self, comp, ctx)
        else:
            self._init_component(comp, ctx)

    def _init_component(self, comp, ctx):   # LS.SNode._init_component, its children built by this class
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


class StatefulScene(LS.StatefulScene):
    """one output's scene over image, web and shader registries, WebViews holding layout nodes"""

    def update_scene(self, scene):
        ids = component_ids(scene, [])
        if len(set(ids)) != len(ids):
            raise SceneError("duplicate component ids")
        used = LW.web_instance_ids(scene, [])
        for other in self.others:
            used += LW.web_instance_ids(other, [])
        if len(set(used)) != len(used):
            raise SceneError("WebRendererUsageNotExclusive")
        if self.scene_tree is not None:   # recalculate_layout at last_pts
            recalculate_layout(Engine(self.last_ns), self.scene_tree, (F(self.out_w), F(self.out_h)), False)
        prev = self.scene_tree.with_id({}) if self.scene_tree is not None else {}
        ctx = {"prev": prev, "last_ns": self.last_ns, "resolutions": dict(self.resolutions), "images": self.images,
               "webs": self.webs, "shaders": self.shaders}
        tree = SNode(scene, ctx)                     # a SceneError leaves the scene as it was
        for n in render_nodes(tree):                 # build_tree: node_size of every layout node below the root
            p = Engine(self.last_ns).position(n)
            if p[1] is None or p[2] is None:
                raise SceneError("UnknownDimensionsForLayoutNodeRoot")
            n.node_size = (p[1], p[2])
        self.scene_tree = tree
        self.render_tree = tree.clone()
