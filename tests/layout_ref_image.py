"""The independent layout engine (tests/layout_ref.py, with the Text leaf of tests/layout_ref_text.py) with Image
components and the image registry.  Test infrastructure.

Restated from the Rust sources, like the engines it extends:

  registry.rs:57-68                  register: KeyTaken when the id exists; unregister: an error when it does not
  transformations/image.rs:69-79     one frame is a Bitmap, more are an Animated asset
  animated_image.rs:52-112           frame k's pts is the sum of the delays before it; the duration is the sum of all, 1 ns
                                     when that is zero; more than 1000 frames: TooManyFrames
  animated_image.rs:120-136          animation_pts = (pts - start_pts) % duration; the frame minimising |frame.pts -
                                     animation_pts|, the first one on a tie (min_by_key)
  scene/image_component.rs:57-89     ImageNotFound; the resolution: both sides given -> round(w) x round(h); one side ->
                                     the other through original_aspect_ratio, a usize division width / height; none -> the
                                     asset's size.  `as usize` saturates, NaN -> 0
  scene/image_component.rs:91-120    a component with an id whose previous state is an Image with an equal component and
                                     the same asset (Arc::ptr_eq) keeps start_pts and resolution; anything else starts at
                                     last_render_pts
  scene.rs:101-127, scene/layout.rs:95-158
                                     an Image is a leaf with a static size and a node child without state, like a Text
  scene_state.rs:154-196             an Image root is not a layout node: no layouts

An Image component here is smelter_b200.ImageComponent.  A node texture the reference cannot create (a side of 0 or above
16384, wgpu's limit) is a SceneError here, which is what the product answers.
"""
import math

import numpy as np

import smelter_b200 as s
from tests import layout_ref as LR
from tests import layout_ref_text as LT

F = LR.F
LEAVES = ("input", "text", "image")
USIZE_MAX = 2 ** 64 - 1
MAX_TEXTURE_SIDE = 16384


class SceneError(Exception):
    pass


class RegistryError(Exception):
    pass


class Asset:
    """Image::Bitmap / Image::Animated: compared by identity, as Arc::ptr_eq does"""

    def __init__(self, width, height, delays_ns):
        if len(delays_ns) == 0:
            raise RegistryError("NoFrames")
        if len(delays_ns) > 1000:
            raise RegistryError("TooManyFrames")
        self.width, self.height = width, height
        self.animated = len(delays_ns) > 1
        self.frame_pts, total = [], 0
        for d in delays_ns:
            self.frame_pts.append(total)
            total += d if self.animated else 0
        self.duration = total if total else 1

    def frame_at(self, pts_ns, start_ns):
        if not self.animated:
            return 0
        animation_pts = (pts_ns - start_ns) % self.duration
        return min(range(len(self.frame_pts)), key=lambda i: abs(self.frame_pts[i] - animation_pts))


def as_usize(x):
    """`x as usize` of an f32"""
    x = float(x)
    if math.isnan(x) or x <= 0.0:
        return 0
    return USIZE_MAX if x >= 2.0 ** 64 else int(x)


def round_f32(x):
    """f32::round: half away from zero (exact here: an f32 plus one half is a double)"""
    x = float(x)
    if math.isnan(x) or math.isinf(x):
        return x
    return math.floor(x + 0.5) if x >= 0.0 else -math.floor(-x + 0.5)


def resolution(asset, width, height):
    aspect = F(asset.width // asset.height)          # usize division, then `as f32`
    with np.errstate(divide="ignore", invalid="ignore"):
        if width is not None and height is not None:
            w, h = F(width), F(height)
        elif width is not None:
            w = F(width)
            h = w / aspect
        elif height is not None:
            h = F(height)
            w = h * aspect
        else:
            return asset.width, asset.height
    return as_usize(round_f32(w)), as_usize(round_f32(h))


def component_key(comp):
    """ImageComponent's PartialEq: Option<f32> fields compare as f32 (NaN differs from itself)"""
    f = lambda v: None if v is None else float(F(v))
    return (comp.id, comp.image_id, f(comp.width), f(comp.height))


class SNode(LT.SNode):
    """StatefulComponent with the Image variant"""

    def __init__(self, comp, ctx):
        if isinstance(comp, s.TextComponent):
            LT.SNode.__init__(self, comp, ctx)
            return
        if not isinstance(comp, s.ImageComponent):
            self._init_component(comp, ctx)
            return
        self.comp, self.kind, self.children = comp, "image", []
        asset = ctx["images"].get(comp.image_id)
        if asset is None:
            raise SceneError(f"ImageNotFound({comp.image_id})")
        prev = ctx["prev"].get(comp.id) if comp.id is not None else None
        if (prev is not None and prev.kind == "image" and component_key(prev.comp) == component_key(comp)
                and prev.asset is asset):
            self.asset, self.start_ns, self.resolution = prev.asset, prev.start_ns, prev.resolution
        else:
            self.asset, self.start_ns, self.resolution = asset, ctx["last_ns"], resolution(asset, comp.width, comp.height)
        if not all(1 <= v <= MAX_TEXTURE_SIDE for v in self.resolution):
            raise SceneError(f"node texture of {self.resolution}")
        self.size = (F(self.resolution[0]), F(self.resolution[1]))

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

    def node_children(self):
        out = []
        for k in self.children:
            out += [k] if k.kind in LEAVES else k.node_children()
        return out


class Engine(LT.Engine):
    def is_layout(self, n):
        return n.kind not in LEAVES

    def width(self, n):
        return n.size[0] if n.kind in LEAVES else self.position(n)[1]

    def height(self, n):
        return n.size[1] if n.kind in LEAVES else self.position(n)[2]

    def update_state(self, n, sizes):      # layout.rs:103-132: Text and Image have no state, they only take a child index
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


def component_ids(comp, out):
    if getattr(comp, "id", None) is not None:
        out.append(comp.id)
    kids = [comp.child] if isinstance(comp, s.RescalerComponent) and comp.child is not None else getattr(comp, "children", None) or []
    for k in kids:
        component_ids(k, out)
    return out


class StatefulScene(LT.StatefulScene):
    """one output's scene over an image registry (shared between outputs by passing the same dict)"""

    def __init__(self, out_w, out_h, images=None):
        super().__init__(out_w, out_h)
        self.images = images if images is not None else {}

    def register_image(self, image_id, width, height, delays_ns):
        if image_id in self.images:
            raise RegistryError("KeyTaken")
        self.images[image_id] = Asset(width, height, delays_ns)

    def unregister_image(self, image_id):
        if image_id not in self.images:
            raise RegistryError("NotRegistered")
        del self.images[image_id]

    def update_scene(self, scene):
        ids = component_ids(scene, [])
        if len(set(ids)) != len(ids):                # validation.rs:13,26
            raise SceneError("duplicate component ids")
        if self.scene_tree is not None and self.scene_tree.kind not in LEAVES:   # recalculate_layout at last_pts
            Engine(self.last_ns).layout(self.scene_tree, F(self.out_w), F(self.out_h))
        prev = self.scene_tree.with_id({}) if self.scene_tree is not None else {}
        ctx = {"prev": prev, "last_ns": self.last_ns, "resolutions": dict(self.resolutions), "images": self.images}
        tree = SNode(scene, ctx)                     # a SceneError leaves the scene as it was
        self.scene_tree = tree
        self.render_tree = tree.clone()

    def image_nodes(self):
        """the render tree's image nodes in node-child order (or the Image root): (component, asset, start_ns, (w, h))"""
        root = self.render_tree
        nodes = [root] if root.kind in LEAVES else root.node_children()
        return [(n.comp, n.asset, n.start_ns, n.resolution) for n in nodes if n.kind == "image"]

    def layouts(self, pts, resolutions_by_input_id):
        pts_ns = LR.to_ns(pts)
        self.last_ns, self.resolutions = pts_ns, dict(resolutions_by_input_id)   # register_render_event
        root = self.render_tree
        if root.kind in LEAVES:
            return [], (0, 0)
        eng = Engine(pts_ns)
        leaves = root.node_children()
        in_res = [resolutions_by_input_id.get(k.comp.input_id) if k.kind == "input" else
                  LT.texture_size(k.comp) if k.kind == "text" else k.resolution for k in leaves]
        eng.update_state(root, in_res)
        p = eng.position(root)
        w = p[1] if p[1] is not None else F(self.out_w)
        h = p[2] if p[2] is not None else F(self.out_h)
        rw, rh = int(np.trunc(w)), int(np.trunc(h))
        nested = eng.layout(root, F(self.out_w), F(self.out_h))
        return LR.flatten(nested, in_res, rw, rh), (rw, rh)
