"""The independent layout engine with WebViews (tests/layout_ref_web.py) extended with Shader components and the shader
registry.  Test infrastructure.

Restated from the Rust sources, like the engines it extends:

  registry.rs:57-68                    register: KeyTaken when the id exists; unregister: an error when it does not
  scene/shader_component.rs:43-72      ShaderNotFound; then the parameter against the shader's type (validation.rs:314-520:
                                       the same kind, a list no longer than the type's, a struct with the same field names
                                       in order; NoBindingInShader without a type); then the children
  scene.rs:101-131, scene/layout.rs:95-158
                                       a Shader is a node child of its layout with its `size` and no layout state; its own
                                       children are render nodes under it, never laid out
  scene_state.rs:154-196               a Shader root is not a layout node: no layouts.  A View, Tiles or Rescaler child of
                                       a Shader is a layout node of its own: its size is node_size at the last render's pts
                                       (UnknownDimensionsForLayoutNodeRoot without width and height, :198-228), its
                                       resolution at pts SizedLayoutComponent::resolution (scene/layout.rs:245-257)
  scene_state.rs:233-262               recalculate_layout: every layout whose parent is not a layout is laid out at its size
                                       when the scene is updated
"""
import smelter_b200 as s
from tests import layout_ref as LR
from tests import layout_ref_web as LW

F = LR.F
LEAVES = LW.LEAVES + ("shader",)
SceneError, RegistryError = LW.SceneError, LW.RegistryError


class Shader:
    """a registered shader: its parameter type (smelter_b200.ShaderParamType or None), compared by identity"""

    def __init__(self, param_type):
        self.param_type = param_type


def validate(v, t):
    if v.kind != t.kind:
        raise SceneError(f"ShaderNodeParametersValidationError(expected {t.kind}, got {v.kind})")
    if t.kind == "list":
        if len(v.value) > t.length:
            raise SceneError("ShaderNodeParametersValidationError(ListTooLong)")
        for x in v.value:
            validate(x, t.item)
    elif t.kind == "struct":
        if len(v.value) != len(t.fields):
            raise SceneError("ShaderNodeParametersValidationError(WrongShaderFieldsAmount)")
        for (n, x), (tn, tt) in zip(v.value, t.fields):
            if n != tn:
                raise SceneError("ShaderNodeParametersValidationError(WrongFieldName)")
            validate(x, tt)


class SNode(LW.SNode):
    """StatefulComponent with the Shader variant"""

    def __init__(self, comp, ctx):
        if not isinstance(comp, s.ShaderComponent):
            if isinstance(comp, (s.TextComponent, s.ImageComponent, s.WebViewComponent)):
                LW.SNode.__init__(self, comp, ctx)
            else:
                self._init_component(comp, ctx)
            return
        self.comp, self.kind = comp, "shader"
        self.shader = ctx["shaders"].get(comp.shader_id)
        if self.shader is None:
            raise SceneError(f"ShaderNotFound({comp.shader_id})")
        if comp.shader_param is not None:
            if self.shader.param_type is None:
                raise SceneError("ShaderNodeParametersValidationError(NoBindingInShader)")
            validate(comp.shader_param, self.shader.param_type)
        self.children = [SNode(k, ctx) for k in comp.children]
        self.size = (F(comp.width), F(comp.height))
        res = [int(v) if v > 0 else 0 for v in self.size]      # Size -> Resolution: `as usize`
        if any(r == 0 or r > 16384 for r in res):              # the reference cannot create such a node texture
            raise SceneError(f"shader node of {res[0]} x {res[1]}")

    def _init_component(self, comp, ctx):   # LW.SNode._init_component, its children built by this class
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


class Engine(LW.Engine):
    def is_layout(self, n):
        return n.kind not in LEAVES

    def width(self, n):
        return n.size[0] if n.kind in LEAVES else self.position(n)[1]

    def height(self, n):
        return n.size[1] if n.kind in LEAVES else self.position(n)[2]

    def update_state(self, n, sizes):      # layout.rs:103-132: a Shader has no state
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


class StatefulScene(LW.StatefulScene):
    """one output's scene over image, web and shader registries"""

    def __init__(self, out_w, out_h):
        super().__init__(out_w, out_h)
        self.shaders = {}

    def register_shader(self, shader_id, param_type=None):
        if shader_id in self.shaders:
            raise RegistryError("KeyTaken")
        self.shaders[shader_id] = Shader(param_type)

    def unregister_shader(self, shader_id):
        if shader_id not in self.shaders:
            raise RegistryError("NotRegistered")
        del self.shaders[shader_id]

    def update_scene(self, scene):
        ids = component_ids(scene, [])
        if len(set(ids)) != len(ids):
            raise SceneError("duplicate component ids")
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

    def layouts(self, pts, resolutions_by_input_id):
        pts_ns = LR.to_ns(pts)
        self.last_ns, self.resolutions = pts_ns, dict(resolutions_by_input_id)   # register_render_event
        root = self.render_tree
        if root.kind in LEAVES:
            return [], (0, 0)
        eng = Engine(pts_ns)
        leaves = root.node_children()
        in_res = self._leaf_resolutions(eng, leaves, resolutions_by_input_id)
        eng.update_state(root, in_res)
        p = eng.position(root)
        w = p[1] if p[1] is not None else F(self.out_w)
        h = p[2] if p[2] is not None else F(self.out_h)
        rw, rh = int(LW.np.trunc(w)), int(LW.np.trunc(h))
        nested = eng.layout(root, F(self.out_w), F(self.out_h))
        return LR.flatten(nested, in_res, rw, rh), (rw, rh)

    def node_layouts(self, k, pts, resolutions_by_input_id):
        """the layouts of layout node k below the root (render graph DFS order, children before parents) at pts, and its
        resolution"""
        pts_ns = LR.to_ns(pts)
        self.last_ns, self.resolutions = pts_ns, dict(resolutions_by_input_id)
        node = render_nodes(self.render_tree)[k]
        eng = Engine(pts_ns)
        in_res = self._leaf_resolutions(eng, node.node_children(), resolutions_by_input_id)
        eng.update_state(node, in_res)
        rw, rh = node_resolution(eng, node)
        nested = eng.layout(node, *node.node_size)
        return LR.flatten(nested, in_res, rw, rh), (rw, rh)

    def _leaf_resolutions(self, eng, leaves, resolutions_by_input_id):
        def layout_res(k):
            r = node_resolution(eng, k)
            return r if 0 < r[0] <= 16384 and 0 < r[1] <= 16384 else None
        return [resolutions_by_input_id.get(k.comp.input_id) if k.kind == "input" else
                  LW.LT.texture_size(k.comp) if k.kind == "text" else
                  (k.instance.width, k.instance.height) if k.kind == "web" else
                (int(k.size[0]), int(k.size[1])) if k.kind == "shader" else
                layout_res(k) if k.kind not in LEAVES else k.resolution for k in leaves]


def render_nodes(n, out=None, top=True):
    """the layout nodes below the root in the render graph's order (build_tree, DFS, a node after its children)"""
    out = [] if out is None else out
    if n.kind in ("shader", "web"):
        for k in n.children:
            render_nodes(k, out, False)
    elif n.kind not in LEAVES:
        for k in n.node_children():
            render_nodes(k, out, False)
        if not top:
            out.append(n)
    return out


def node_resolution(eng, n):
    """SizedLayoutComponent::resolution: the position's width and height at the engine's pts, else node_size, as usize"""
    p = eng.position(n)
    w = p[1] if p[1] is not None else n.node_size[0]
    h = p[2] if p[2] is not None else n.node_size[1]
    return (int(LW.np.trunc(w)) if w > 0 else 0, int(LW.np.trunc(h)) if h > 0 else 0)


def recalculate_layout(eng, n, size, parent_is_layout):
    """scene_state.rs:233-262"""
    if n.kind not in LEAVES:
        if not parent_is_layout:
            if size is None:
                p = eng.position(n)
                size = (p[1], p[2]) if p[1] is not None and p[2] is not None else None
            if size is not None:
                eng.layout(n, *size)
        for k in n.children:
            recalculate_layout(eng, k, None, True)
    else:
        for k in n.children:
            recalculate_layout(eng, k, None, False)


def component_ids(comp, out):
    if getattr(comp, "id", None) is not None:
        out.append(comp.id)
    kids = [comp.child] if isinstance(comp, s.RescalerComponent) and comp.child is not None else getattr(comp, "children", None) or []
    for k in kids:
        component_ids(k, out)
    return out
