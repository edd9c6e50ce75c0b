"""The product's host layout engine (smelter_b200/csrc/scene.cpp, through the C ABI on a host-only handle) against
the INDEPENDENT restatement tests/layout_ref.py, field for field, on the whole re-typed scene catalogue of the
reference (tests/golden/ref_scenes.py: simple / view / rescaler / tiles / transition / tiles_transitions = 111 in-scope
render tests).  CPU-only."""
import numpy as np
import pytest

import smelter_b200 as s
from tests import layout_ref as LR
from tests import ref_scene_rt as rt
from tests.golden import ref_scenes

CASES = [(m, n) for m, tests in ref_scenes.MODULES.items() for n in tests]
KIND = {0: "child", 1: "color", 2: "shadow"}


def product_layouts(r, pts):
    ls, root = r.debug_layouts("output_1", pts)
    out = []
    for l in ls:
        d = dict(kind=KIND[l.type], top=l.top, left=l.left, width=l.width, height=l.height, rotation=l.rotation_degrees,
                 border_radius=tuple(l.border_radius), masks=[(tuple(m.radius), m.top, m.left, m.width, m.height)
                                                            for m in list(l.masks)[:l.masks_len]])
        if l.type == 2:
            d.update(color=(l.color.r, l.color.g, l.color.b, l.color.a), blur_radius=l.blur_radius)
        else:
            d.update(border_color=(l.border_color.r, l.border_color.g, l.border_color.b, l.border_color.a),
                     border_width=l.border_width)
            if l.type == 1:
                d.update(color=(l.color.r, l.color.g, l.color.b, l.color.a))
            else:
                d.update(index=l.child_index, crop=(l.crop_top, l.crop_left, l.crop_width, l.crop_height))
        out.append(d)
    return out, root


def ref_layouts(ls):
    out = []
    for l in ls:
        d = dict(kind=l.kind, top=l.top, left=l.left, width=l.width, height=l.height, rotation=l.rotation,
                 border_radius=l.border_radius.tup(),
                 masks=[(m.radius.tup(), m.top, m.left, m.width, m.height) for m in l.masks])
        if l.kind == "shadow":
            d.update(color=l.color, blur_radius=l.blur_radius)
        else:
            d.update(border_color=l.border_color, border_width=l.border_width)
            if l.kind == "color":
                d.update(color=l.color)
            else:
                d.update(index=l.index, crop=(l.crop.top, l.crop.left, l.crop.width, l.crop.height))
        out.append(d)
    return out


def same(a, b):
    """bit-for-bit as f32 (NaN == NaN)"""
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, str) or isinstance(b, str):
        return a == b
    fa, fb = np.float32(a), np.float32(b)
    return bool(fa == fb) or bool(np.isnan(fa) and np.isnan(fb))


def diff(got, exp):
    if len(got) != len(exp):
        return f"{len(got)} layouts, expected {len(exp)}: kinds {[g['kind'] for g in got]} vs {[e['kind'] for e in exp]}"
    for i, (g, e) in enumerate(zip(got, exp)):
        if g.keys() != e.keys():
            return f"layout {i}: kind {g['kind']} vs {e['kind']}"
        for k in e:
            if not same(g[k], e[k]):
                return f"layout {i} ({e['kind']}) field {k}: got {g[k]} expected {e[k]}"
    return None


@pytest.mark.parametrize("width", [20000.0, 0.5])
def test_root_outside_the_renderable_range(width):
    """a root too wide to render, or one whose width truncates to 0: smr_render draws only the fallback fill, but
    smr_debug_layouts still reports the root and its layouts as the scene defines them"""
    scene = s.ViewComponent(position=s.Position.Static(width=width, height=300.0), children=[
        s.ViewComponent(position=s.Position.Static(width=100.0, height=100.0), background_color=s.RGBAColor(200, 30, 30, 255)),
        s.InputStreamComponent(input_id="input_1")])
    r = s.Renderer(s.RendererOptions(cuda_device=-1))
    r.register_input("input_1")
    r.update_scene("output_1", s.Resolution(640, 360), s.OutputFrameFormat.PlanarYuv420Bytes, scene)
    r.debug_set_inputs(0.0, {"input_1": s.Resolution(640, 360)})
    got, root = product_layouts(r, 0.0)
    exp_l, exp_root = LR.layouts(scene, 640, 360, {"input_1": (640, 360)})
    assert root == exp_root and not (0 < root[0] <= 16384)
    assert got and diff(got, ref_layouts(exp_l)) is None, diff(got, ref_layouts(exp_l))


@pytest.mark.parametrize("module,name", CASES)
def test_scene_catalogue_layouts(module, name):
    rec = rt.record(ref_scenes.MODULES[module][name])
    if rec is None:
        pytest.skip("text / image / shader components are outside the compositor hot path")
    r = s.Renderer(s.RendererOptions(rendering_mode=rec.mode, cuda_device=-1))
    for i in rec.inputs:
        r.register_input(i.name)
    res = {i.name: (i.resolution.width, i.resolution.height) for i in rec.inputs}
    ref = LR.StatefulScene(rec.resolution.width, rec.resolution.height)
    n_snap = 0
    for kind, arg in rec.steps:
        if kind == "update":
            r.update_scene("output_1", rec.resolution, s.OutputFrameFormat.PlanarYuv420Bytes, arg)
            ref.update_scene(arg)
            continue
        pts = arg
        r.debug_set_inputs(pts, {k: s.Resolution(*v) for k, v in res.items()})
        got, root = product_layouts(r, pts)
        exp_l, exp_root = ref.layouts(pts, res)
        assert root == exp_root, f"{module}/{name} pts {pts}: root {root} expected {exp_root}"
        d = diff(got, ref_layouts(exp_l))
        assert d is None, f"{module}/{name} pts {pts}: {d}"
        n_snap += 1
    assert n_snap > 0
