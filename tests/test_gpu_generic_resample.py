"""The generic resample passes (k_convert, the k_resample box / first / last stages) and the weight kernel against the oracle.

Every resampled child that `Renderer::try_fused_resample` turns down takes the generic passes: vertical-first plans, one-pass
plans, box levels other than (1, 1) (and (1, 1) on odd widths or interleaved sources), and sources the fused kernels do not
read.  Each scene of `REGISTRY` is built with `set_layouts`; a case asks `debug_fused_jobs` that no fused job ran, asks
`debug_resample_stages` for the stages that did and compares them with the plan the oracle's `plan_passes` /
`predecimate_levels` give for the same crop, and compares the RGBA bytes with the oracle.

- `test_registry_covers_the_plan_shapes` (CPU) derives each scene's plan from the oracle and fails when a plan shape, box
  level, source kind or destination shape has no scene.
- Crops the box pass cannot reduce are refused before anything is launched.
- Weight tables of a seeded sweep of mappings, bit for bit against the oracle (GPU) and within a stated tolerance of a
  float64 Lanczos3 (CPU).
- NC-8: the weight kernel's sin / cos equal the oracle's for every float with |x| in [2^-3, 2^4) (GPU).
"""
import math
from dataclasses import dataclass, field
from typing import Dict, List, Tuple

import numpy as np
import pytest

import smelter_b200 as s
from smelter_b200 import _ffi as F
from tests import harness
from tests.parity import OUTPUT_ID, TrackedRenderer, assert_identical, run_case, yuv_frame, nv12_frame
from tests.test_gpu_fused_variants import (RGBA, Job, Placement, extreme_plane, fill_input, make_frame, mismatch_report,
                                           oracle_planes, planes_of, render, scene_of)

# texture kinds (smr_composite_layer_info.tex_kind)
TEX = {"rgba": 1, "yuv": 2, "nv12": 3, "f16": 4, "bgra": 5, "argb": 6, "yuv422": 7, "yuv444": 8, "uyvy": 9, "yuyv": 10}
FOUR_BYTE = ("rgba", "bgra", "argb")


# ------------------------------------------------------------------------------------------------
# frames of every input format, any size
# ------------------------------------------------------------------------------------------------
def any_frame(fmt, content, seed, w, h):
    """a frame of format `fmt` (TEX keys other than f16), w x h; content "extreme" (every byte code, 0 / 255 checkers)
    or "smooth".  Four-byte formats keep their rows as (h, 4 w) so that device placements can pitch them."""
    res = s.Resolution(w, h)
    if fmt in FOUR_BYTE:
        if content == "extreme":
            rng = np.random.default_rng(seed)
            ch = [extreme_plane(rng, w, h) for _ in range(4)]
        else:
            y = harness.smooth_yuv420(seed, w, 4 * h)[0]
            ch = [y[k * h:(k + 1) * h] for k in range(4)]
        t = np.stack(ch, axis=-1).reshape(h, 4 * w)
        kind = {"rgba": "Rgba8", "bgra": "Bgra", "argb": "Argb"}[fmt]
        return s.Frame(s.FrameData(kind, (t,)), res)
    if fmt in ("yuv422", "yuv444"):
        cw = w // 2 if fmt == "yuv422" else w
        if content == "extreme":
            y, u, v = planes_of(content, seed, w, h, cw, h)
        else:
            y, u, v = (harness.smooth_yuv420(seed + k, pw, h)[0] for k, pw in enumerate((w, cw, cw)))
        return s.Frame(s.FrameData("PlanarYuv422" if fmt == "yuv422" else "PlanarYuv444", (y, u, v)), res)
    if fmt in ("uyvy", "yuyv") and w % 2:
        y, u, v = planes_of(content, seed, w, h, w // 2, h)
        ye, yo = y[:, 0:2 * (w // 2):2], y[:, 1:2 * (w // 2):2]
        t = np.empty((h, w // 2, 4), np.uint8)
        if fmt == "uyvy":
            t[..., 0], t[..., 1], t[..., 2], t[..., 3] = u[:h], ye, v[:h], yo
        else:
            t[..., 0], t[..., 1], t[..., 2], t[..., 3] = ye, u[:h], yo, v[:h]
        return s.Frame(s.FrameData("InterleavedUyvy422" if fmt == "uyvy" else "InterleavedYuyv422", (t,)), res)
    if fmt in ("yuv", "nv12") and (w % 2 or h % 2):
        y, u, v = planes_of(content, seed, w, h, w // 2, h // 2)
        if fmt == "nv12":
            return s.Frame(s.FrameData.Nv12(s.NvPlanes(y, np.stack([u, v], axis=-1))), res)
        return s.Frame(s.FrameData("PlanarYuv420", (y, u, v)), res)
    return make_frame(fmt, content, seed, w, h)


# ------------------------------------------------------------------------------------------------
# the plan the oracle gives for one layout
# ------------------------------------------------------------------------------------------------
def cround(x):
    """std::round: half away from zero"""
    return int(math.copysign(math.floor(abs(x) + 0.5), x))


def expected_stages(fmt, src, crop, dst):
    """-> list of stage dicts (debug_resample_stages' fields) of one generic resample; [] when the layout is direct"""
    from oracle import oracle as orc
    f32 = np.float32
    left, top, cw, ch = (float(f32(v)) for v in crop)
    dw, dh = dst
    if orc.plan_passes(left, top, cw, ch, dw, dh) == []:
        return []
    lv = (orc.predecimate_levels(cw, dw), orc.predecimate_levels(ch, dh))
    fx, fy = 1 << lv[0], 1 << lv[1]
    cur, source, kind, out = tuple(src), ("raw" if fmt == "rgba" else "converted"), TEX[fmt], []
    if (fx, fy) != (1, 1):
        red = (-(-src[0] // fx), -(-src[1] // fy))
        out.append(dict(stage="box", axis=-1, box_fx=fx, box_fy=fy, taps=0, perp_offset=0, source=source, src_kind=kind,
                        src=cur, dst=red, dst_f16=1))
        cur, source, kind = red, "f16", TEX["f16"]
    off = (float(f32(left) / f32(fx)), float(f32(top) / f32(fy)))
    ln = (float(f32(cw) / f32(fx)), float(f32(ch) / f32(fy)))
    passes = orc.plan_passes(off[0], off[1], ln[0], ln[1], dw, dh)
    assert passes, "the reduced mapping is direct"
    for i, (axis, perp) in enumerate(passes):
        last = i == len(passes) - 1
        taps = orc.lib().orc_resample_taps(float(f32(ln[axis]) / f32(dst[axis])))
        d = (dw, dh) if last else ((dw, cur[1]) if axis == 0 else (cur[0], dh))
        out.append(dict(stage="last" if last else "first", axis=axis, box_fx=1, box_fy=1, taps=taps, perp_offset=perp,
                        source=source, src_kind=kind, src=cur, dst=d, dst_f16=0 if last else 1))
        cur, source, kind = d, "f16", TEX["f16"]
    return out


# ------------------------------------------------------------------------------------------------
# the registry
# ------------------------------------------------------------------------------------------------
@dataclass
class Case:
    name: str
    inputs: Dict[str, Tuple[str, int, int]]          # input id -> (format, width, height)
    jobs: List[Job]
    placements: Dict[str, Placement] = field(default_factory=dict)   # device planes (default: host)

    def plan(self):
        """expected (stages in launch order, k_convert kinds): one generic resample per distinct (input, crop, size)"""
        per, seen, conv = [], set(), []
        for j in self.jobs:
            key = (j.input_id, tuple(np.float32(c) for c in j.crop), j.dst)
            if key in seen:
                continue
            seen.add(key)
            fmt, w, h = self.inputs[j.input_id]
            st = expected_stages(fmt, (w, h), j.crop, j.dst)
            per.append(st)
            if st and fmt != "rgba" and j.input_id not in [c[0] for c in conv]:
                conv.append((j.input_id, TEX[fmt]))
        order = {"box": 0, "first": 1, "last": 2}
        stages = [x for k in ("box", "first", "last") for st in per for x in st if order[x["stage"]] == order[k]]
        return stages, [c[1] for c in conv]


def one(name, fmt, src, crop, dst, placement=None):
    c = Case(name, {"input_1": (fmt, *src)}, [Job("input_1", crop, dst)])
    if placement is not None:
        c.placements["input_1"] = placement
    return c


def full(w, h):
    return (0.0, 0.0, float(w), float(h))


def _registry():
    R = []
    # plan shapes.  One pass: the other axis is a direct copy at an integer offset (perp_offset), clamped at both edges
    R.append(Case("one-pass-h", {"input_1": ("rgba", 64, 48)},
                  [Job("input_1", (0.0, o, 50.0, 30.0), (37, 30)) for o in (5.0, -3.0, 22.0)]))
    R.append(Case("one-pass-v", {"input_1": ("yuv", 64, 48)},
                  [Job("input_1", (o, 0.0, 40.0, 44.0), (40, 27)) for o in (6.0, -4.0, 30.0)]))
    R.append(one("two-pass-h-first-yuv444", "yuv444", (96, 64), full(96, 64), (40, 30)))
    for fmt in ("yuv", "nv12"):   # the vertical ratio a hair larger: the fused kernels take horizontal-first plans only
        R.append(one(f"two-pass-v-first-{fmt}", fmt, (160, 90), full(160, 90), (80, 44)))
    # as_direct's tolerance of 0.001: offsets 0.0009 / 0.0011, lengths dst +- 0.0009 / +- 0.0011, on each axis
    near = [(0.0009, 40.0), (0.0011, 40.0), (0.0, 40.0009), (0.0, 40.0011), (0.0, 39.9991), (0.0, 39.9989)]
    R.append(Case("as-direct-h", {"input_1": ("rgba", 48, 48)}, [Job("input_1", (o, 2.0, l, 44.0), (40, 30)) for o, l in near]))
    R.append(Case("as-direct-v", {"input_1": ("rgba", 48, 48)}, [Job("input_1", (2.0, o, 44.0, l), (30, 40)) for o, l in near]))
    # ratios
    R.append(one("upscale-both", "rgba", (20, 16), full(20, 16), (50, 37)))
    R.append(one("up-h-down-v", "bgra", (40, 30), full(40, 30), (100, 12)))
    R.append(one("unit-scale-fractional-offset", "argb", (48, 36), (0.25, 0.5, 40.0, 30.0), (40, 30)))
    # box levels; sources that are not a multiple of the factor, so the last block clamps
    R.append(one("box-1-0", "rgba", (203, 40), full(203, 40), (40, 20)))
    R.append(one("box-0-1", "yuv", (40, 202), full(40, 202), (20, 40)))
    R.append(one("box-2-2", "yuv", (402, 302), full(402, 302), (40, 30)))
    R.append(one("box-3-1", "nv12", (530, 90), full(530, 90), (20, 15)))
    R.append(one("box-1-1-odd-width", "yuv", (320, 180), full(320, 180), (53, 30)))
    R.append(one("box-1-1-uyvy", "uyvy", (320, 180), full(320, 180), (60, 30)))
    R.append(one("box-12-from-16384", "rgba", (16384, 2), (0.0, 0.0, 16384.0, 2.0), (1, 2)))
    R.append(one("box-12-12-limit", "rgba", (64, 64), (0.0, 0.0, 16384.0, 16384.0), (1, 1)))
    # sources, host and device (device four-byte rows pitched past 4 w)
    for fmt in FOUR_BYTE:
        R.append(one(f"src-{fmt}-host", fmt, (72, 40), full(72, 40), (30, 17)))
        R.append(one(f"src-{fmt}-device", fmt, (100, 40), full(100, 40), (41, 18), Placement(0, 4)))
    for fmt in ("yuv422", "yuv444"):
        R.append(one(f"src-{fmt}", fmt, (90, 50), full(90, 50), (40, 22)))
    for fmt in ("yuv", "nv12"):
        R.append(one(f"src-{fmt}-odd", fmt, (161, 91), full(161, 91), (60, 40)))
    for fmt in ("uyvy", "yuyv"):
        for w, dst in ((2, (3, 4)), (6, (4, 5)), (7, (3, 9))):
            R.append(one(f"src-{fmt}-w{w}", fmt, (w, 10), full(w, 10), dst))
    R.append(one("src-minimum-2x2", "yuv", (2, 2), full(2, 2), (5, 3)))
    # destinations
    R.append(Case("dst-1x1-1xN-Nx1", {"input_1": ("rgba", 40, 30)},
                  [Job("input_1", full(40, 30), d) for d in ((1, 1), (1, 50), (50, 1))]))
    R.append(one("dst-16384x1", "rgba", (64, 8), full(64, 8), (16384, 1)))
    # crops over every edge, negative offsets included (vertical-first, so the fused kernels leave the 4:2:0 source alone)
    R.append(Case("crops-over-edges", {"input_1": ("yuv", 48, 32)},
                  [Job("input_1", c, (30, 19)) for c in ((-10.0, -7.0, 60.0, 40.0), (20.0, 15.0, 50.0, 40.0),
                                                        (-30.0, 10.0, 40.0, 30.0), (10.0, -25.0, 30.0, 36.0))]))
    # two crops of one input: one k_convert; the same crop twice: resampled once
    R.append(Case("two-crops-one-convert", {"input_1": ("nv12", 96, 54)},
                  [Job("input_1", (0.0, 0.0, 60.0, 54.0), (25, 20)), Job("input_1", (30.0, 10.0, 50.0, 44.0), (20, 17))]))
    R.append(Case("same-crop-twice", {"input_1": ("yuv422", 96, 54), "input_2": ("rgba", 50, 30)},
                  [Job("input_1", full(96, 54), (41, 23)), Job("input_2", full(50, 30), (20, 13)),
                   Job("input_1", full(96, 54), (41, 23))]))
    return R


REGISTRY = _registry()


def plan_shape(stages):
    lanczos = [x for x in stages if x["stage"] != "box"]
    if len(lanczos) == 1:
        return f"one-pass-{'hv'[lanczos[0]['axis']]}"
    return f"two-pass-{'hv'[lanczos[0]['axis']]}-first"


def fused_candidate(fmt, src, st):
    """whether try_fused_resample's format, level and plan checks would let the job through (the scenes must fail them)"""
    w, h = src
    if fmt not in ("yuv", "nv12", "uyvy", "yuyv") or (fmt in ("yuv", "nv12") and (w | h) & 1):
        return False
    if fmt in ("uyvy", "yuyv") and (w & 1 or w < 8):
        return False
    box = [x for x in st if x["stage"] == "box"]
    if box and not (box[0]["box_fx"] == box[0]["box_fy"] == 2 and fmt in ("yuv", "nv12") and st[-1]["dst"][0] % 2 == 0):
        return False
    lan = [x for x in st if x["stage"] != "box"]
    return len(lan) == 2 and lan[0]["axis"] == 0 and all(x["taps"] <= 25 for x in lan)


def test_registry_covers_the_plan_shapes():
    """every plan shape, box level, source kind and destination shape the generic passes take has a scene"""
    assert len({c.name for c in REGISTRY}) == len(REGISTRY)
    shapes, levels, kinds, dsts, perps = set(), set(), set(), set(), set()
    for c in REGISTRY:
        for j in c.jobs:
            fmt, w, h = c.inputs[j.input_id]
            st = expected_stages(fmt, (w, h), j.crop, j.dst)
            assert st, f"{c.name}: {j} is direct"
            assert not fused_candidate(fmt, (w, h), st), f"{c.name}: {j} could take a fused kernel"
            shapes.add(plan_shape(st))
            box = [x for x in st if x["stage"] == "box"]
            lv = (box[0]["box_fx"].bit_length() - 1, box[0]["box_fy"].bit_length() - 1) if box else (0, 0)
            levels.add(lv)
            if lv == (1, 1):
                levels.add(("1-1-odd" if j.dst[0] % 2 else "1-1-even", fmt))
            kinds.add((fmt, "device" if j.input_id in c.placements else "host"))
            dsts.add(j.dst)
            lan = [x for x in st if x["stage"] != "box"]
            if len(lan) == 1:
                perps.add(("neg" if lan[0]["perp_offset"] < 0 else "pos" if lan[0]["perp_offset"] > 0 else "0", lan[0]["axis"]))
    assert {"one-pass-h", "one-pass-v", "two-pass-h-first", "two-pass-v-first"} <= shapes, shapes
    assert {(1, 0), (0, 1), (2, 2), (3, 1), (12, 0), (12, 12)} <= levels and ("1-1-odd", "yuv") in levels and \
        ("1-1-even", "uyvy") in levels, levels
    for fmt in TEX:
        if fmt != "f16":
            assert (fmt, "host") in kinds, fmt
    for fmt in FOUR_BYTE:
        assert (fmt, "device") in kinds, fmt
    assert {(1, 1), (1, 50), (50, 1), (16384, 1)} <= dsts, dsts
    assert {("neg", 0), ("pos", 0), ("neg", 1), ("pos", 1)} <= perps, perps
    assert REGISTRY_BY_NAME["two-pass-v-first-yuv"].plan()[0][0]["axis"] == 1


REGISTRY_BY_NAME = {c.name: c for c in REGISTRY}


def frames_of(case, content, seed):
    return {i: any_frame(fmt, content, seed + k, w, h) for k, (i, (fmt, w, h)) in enumerate(case.inputs.items())}


@pytest.mark.gpu
@pytest.mark.parametrize("case", REGISTRY, ids=lambda c: c.name)
def test_generic_scene(case):
    """no fused job; the stages the oracle plans; the RGBA bytes of the oracle, for extreme and smooth content"""
    stages, conv = case.plan()
    for k, content in enumerate(("extreme", "smooth")):
        fr = frames_of(case, content, 900 + 10 * k)
        r = s.Renderer()
        got = render(r, case.jobs, fr, RGBA, case.placements)
        assert r.debug_fused_jobs() == [], (case.name, r.debug_fused_jobs())
        ran, kinds = r.debug_resample_stages()
        assert ran == stages, f"{case.name}: ran {ran}, the oracle plans {stages}"
        assert kinds == conv, (case.name, kinds, conv)
        rep = mismatch_report(got, oracle_planes(case.jobs, fr, RGBA), case.jobs, [])
        assert rep is None, f"{case.name} {content}: {rep}"


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["yuv", "nv12"])
def test_rescaler_fit_lands_vertical_first(fmt):
    """A Rescaler (Fit) of a 640 x 360 input into 178 x 101: the child is 178 x 100.125, drawn 178 x 100, so the vertical
    ratio (3.6) is a hair above the horizontal one (3.5955) and the plan is vertical-first -- generic passes, not fused"""
    w, h = 640, 360
    mk = nv12_frame if fmt == "nv12" else yuv_frame
    fr = {"input_1": mk(harness.smooth_yuv420(31, w, h), w, h)}
    scene = s.RescalerComponent(child=s.InputStreamComponent(input_id="input_1"), mode=s.RescaleMode.Fit)
    got, exp, r = run_case(scene, fr, resolution=s.Resolution(178, 101), out_format=s.OutputFrameFormat.RgbaWgpuTexture)
    assert_identical(got, exp, f"rescaler fit {fmt}")
    assert r.debug_fused_jobs() == []
    ran, kinds = r.debug_resample_stages()
    assert ran == expected_stages(fmt, (w, h), full(w, h), (178, 100)), ran
    assert [x["axis"] for x in ran] == [1, 0] and kinds == [TEX[fmt]], (ran, kinds)


@pytest.mark.gpu
def test_same_crop_in_two_outputs_is_resampled_once():
    """one (input, crop, size) in two outputs of one tick: one k_convert, one set of stages, both outputs equal the oracle"""
    import torch
    w, h = 96, 54
    fr = {"input_1": any_frame("yuv", "extreme", 77, w, h)}
    jobs = [Job("input_1", (3.5, 1.0, 80.0, 50.0), (34, 20))]   # vertical-first: not a fused job
    W, H, ids, ls, _ = scene_of(jobs)
    r = s.Renderer()
    r.register_input("input_1")
    for oid in ("output_1", "output_2"):
        r.set_layouts(oid, s.Resolution(W, H), RGBA, (W, H), ids, ls)
    keep = []
    arr = (F.InputFrame * 1)()
    fill_input(arr[0], "input_1", fr["input_1"], None, keep)
    outs = [np.zeros((H, W, 4), np.uint8) for _ in range(2)]
    out = (F.OutputFrame * 2)()
    for k, oid in enumerate((b"output_1", b"output_2")):
        out[k].output_id, out[k].mem_kind, out[k].planes[0] = oid, F.MEM_HOST, outs[k].ctypes.data
    torch.cuda.synchronize()
    r.render_raw(0, arr, 1, out, 2)
    assert r.debug_fused_jobs() == []
    ran, kinds = r.debug_resample_stages()
    assert ran == expected_stages("yuv", (w, h), jobs[0].crop, jobs[0].dst) and kinds == [TEX["yuv"]], (ran, kinds)
    exp = oracle_planes(jobs, fr, RGBA)[0]
    for o in outs:
        assert np.array_equal(o, exp)


# ------------------------------------------------------------------------------------------------
# refusals: crops the box pass cannot reduce
# ------------------------------------------------------------------------------------------------
def crop_layout(crop, dst=(4, 4)):
    l = F.RenderLayout()
    l.type, l.width, l.height = 0, float(dst[0]), float(dst[1])
    l.crop_left, l.crop_top, l.crop_width, l.crop_height = crop
    return l


NON_FINITE = [(0.0, 0.0, math.inf, math.inf), (0.0, 0.0, math.inf, 8.0), (0.0, 0.0, math.nan, 8.0), (-math.inf, 0.0, 8.0, 8.0),
              (0.0, math.nan, 8.0, 8.0), (0.0, 0.0, 8.0, -math.inf)]


@pytest.mark.parametrize("crop", NON_FINITE, ids=str)
def test_non_finite_crop_is_refused(crop):
    """smr_set_layouts refuses a texture layout with a non-finite crop field; colour and shadow layouts ignore theirs"""
    r = s.Renderer(s.RendererOptions(cuda_device=-1))
    with pytest.raises(s.renderer.UpdateSceneError) as e:
        r.set_layouts(OUTPUT_ID, s.Resolution(8, 8), RGBA, (8, 8), ["input_1"], [crop_layout(crop)])
    assert e.value.status == 1 and "not finite" in str(e.value)   # SMR_ERR_INVALID_ARGUMENT
    for t in (1, 2):
        l = crop_layout(crop)
        l.type = t
        r.set_layouts(OUTPUT_ID, s.Resolution(8, 8), RGBA, (8, 8), ["input_1"], [l])


def render_status(jobs, frames):
    """one tick through smr_render: (status, error, kernel launches of the handle)"""
    import torch
    W, H, ids, ls, _ = scene_of(jobs)
    r = s.Renderer()
    for i in ids:
        r.register_input(i)
    r.set_layouts(OUTPUT_ID, s.Resolution(W, H), RGBA, (W, H), ids, ls)
    keep = []
    arr = (F.InputFrame * len(ids))()
    for k, i in enumerate(ids):
        fill_input(arr[k], i, frames[i], None, keep)
    o = np.zeros((H, W, 4), np.uint8)
    out = (F.OutputFrame * 1)()
    out[0].output_id, out[0].mem_kind, out[0].planes[0] = OUTPUT_ID.encode(), F.MEM_HOST, o.ctypes.data
    torch.cuda.synchronize()
    st = F.lib().smr_render(r._h, 0, arr, len(ids), out, 1)
    return st, r._err(), r.stats()["kernel_launches"]


@pytest.mark.gpu
@pytest.mark.parametrize("crop,dst", [((0.0, 0.0, 1e9, 1e9), (4, 4)), ((0.0, 0.0, 16384.0, 32768.0), (1, 1)),
                                      ((0.0, 0.0, 3e7, 3e7), (7, 5))], ids=str)
def test_box_factor_above_2_24_is_refused(crop, dst):
    """a finite crop whose box pass would average more than 2^24 texels (levels (16, 16): 2^32; (12, 13): 2^25) is
    SMR_ERR_INVALID_ARGUMENT with no kernel launched; next to it, a good job alone still renders"""
    fr = {"input_1": any_frame("rgba", "extreme", 5, 16, 16), "input_2": any_frame("yuv", "smooth", 6, 32, 32)}
    st, err, launches = render_status([Job("input_2", full(32, 32), (12, 12)), Job("input_1", crop, dst)], fr)
    assert st == 1 and "2^24" in err and launches == 0, (st, err, launches)
    st, err, launches = render_status([Job("input_2", full(32, 32), (12, 12))], fr)
    assert st == 0 and launches > 0, (st, err)


# ------------------------------------------------------------------------------------------------
# weight tables
# ------------------------------------------------------------------------------------------------
def weight_sweep(n=2000, seed=2024):
    """(scale, offset, n_out) of a seeded sweep: the integer ratios, 1 / 64 and 1 at the extremes of offset and n_out; then
    scales log-uniform in [1/64, 4] and, every fourth, the reduced scale of a box level 1..12 (crop / 2^level over dst, as
    AxisMapping::on_reduced_source); offsets 0, integral, fractional, negative, up to 16384; n_out log-uniform in
    [1, 16384]"""
    from oracle import oracle as orc
    rng = np.random.default_rng(seed)
    f32 = np.float32
    out = [(sc, off, no) for sc in (1.0 / 64, 0.5, 1.0, 2.0, 3.0, 4.0)
           for off, no in ((0.0, 1), (0.0, 16384), (16384.0, 16384), (-0.5, 7))]
    while len(out) < n:
        if len(out) % 4 == 3:
            dst = int(rng.integers(1, 4097))
            crop = f32(dst * rng.uniform(4.0001, 4.0 * 2 ** 12))
            lv = orc.predecimate_levels(float(crop), dst)
            scale = (crop / f32(1 << lv)) / f32(dst)
        else:
            scale = f32(2.0 ** rng.uniform(-6.0, 2.0))
        offset = [0.0, float(rng.integers(-64, 16385)), rng.uniform(-64.0, 16384.0), -rng.uniform(0.0, 64.0),
                  float(rng.integers(0, 64)) + float(rng.choice([0.25, 0.5, 0.001, 0.999]))][int(rng.integers(5))]
        n_out = int(np.clip(np.round(2.0 ** rng.uniform(0.0, 14.0)), 1, 16384))
        out.append((float(scale), float(f32(offset)), n_out))
    return out


SWEEP = weight_sweep()


def test_weight_sweep_covers_its_ranges():
    sc = np.array([m[0] for m in SWEEP])
    off = np.array([m[1] for m in SWEEP])
    n = np.array([m[2] for m in SWEEP])
    assert sc.min() <= 1.0 / 60 and sc.max() == 4.0 and {1.0, 2.0, 3.0} <= set(sc.tolist())
    assert off.min() < 0 and off.max() > 16000 and (off == 0).any() and ((off % 1) != 0).any()
    assert n.min() == 1 and n.max() == 16384


def lanczos3_f64(scale, offset, n_out):
    """(first, tap positions x, weights sinc(x) sinc(x / 3)) of every output coordinate, evaluated directly in float64 at
    the positions the f32 centre and first tap give"""
    from oracle import oracle as orc
    f32 = np.float32
    taps = orc.lib().orc_resample_taps(scale)
    ks = max(scale, 1.0)
    o = np.arange(n_out, dtype=np.float32)
    center = (f32(offset) + (o + f32(0.5)) * f32(scale)) - f32(0.5)
    first = np.ceil(center - f32(3.0) * f32(ks))
    x = ((first.astype(np.float64)[:, None] + np.arange(taps)[None, :]) - center.astype(np.float64)[:, None]) / ks
    return first.astype(np.int64), x, np.where(np.abs(x) < 3.0, np.sinc(x) * np.sinc(x / 3.0), 0.0)


# The shader's weights come from sin / cos rotated tap by tap in f32 and divided by (pi x)^2 / 3.  The rotated sines carry
# an absolute error of a few f32 ulps, which that division turns into about 4 ulps / (pi |x|) next to the centre tap.
# Bound on each weight: 2^-19 / min(|x|, 1) (over the sweep the largest |error| * min(|x|, 1) is about 1.1e-6, and
# away from the centre, |x| >= 0.05, the largest error is about 1.9e-5).  A wrong constant, phase or rotation in a
# restatement moves weights by orders of magnitude more.
WEIGHT_ERR = 2.0 ** -19


def test_oracle_weights_are_lanczos3():
    """the oracle's (and so the device's) weights are Lanczos3: each weight within WEIGHT_ERR / min(|x|, 1) of the
    float64 sinc product, and each normalised weight within the bound that error gives after normalisation"""
    from oracle import oracle as orc
    for scale, offset, n_out in SWEEP:
        n = min(n_out, 512)   # the weights depend on the output coordinate only through the centre's phase
        first, w, inv = orc.resample_table(scale, offset, n)
        f64_first, x, w64 = lanczos3_f64(scale, offset, n)
        assert np.array_equal(first, f64_first), (scale, offset)
        ax = np.abs(x)   # below 1e-5 the shader's weight is exactly 1, the sinc product 1 - O(x^2)
        err = np.where(ax < 1e-5, WEIGHT_ERR, WEIGHT_ERR / np.clip(ax, 1e-5, 1.0))
        d = np.abs(w.astype(np.float64) - w64)
        assert (d <= err).all(), (scale, offset, n, float((d / err).max()))
        s64, e_sum = w64.sum(axis=1, keepdims=True), err.sum(axis=1, keepdims=True)
        norm_err = (err + np.abs(w64) * e_sum / s64) / (s64 - e_sum) + 2.0 ** -22
        dn = np.abs(w.astype(np.float64) * inv.astype(np.float64)[:, None] - w64 / s64)
        assert (dn <= norm_err).all(), (scale, offset, n, float((dn / norm_err).max()))


@pytest.mark.gpu
def test_weight_tables_are_the_oracles():
    """every weight, 1 / weight_sum and first tap of every output coordinate of the sweep's mappings, bit for bit"""
    from oracle import oracle as orc
    from tests.test_gpu_int_ratio_ranges import device_weights
    bad = []
    for scale, offset, n_out in SWEEP:
        ef, ew, einv = orc.resample_table(scale, offset, n_out)
        df, dw, dinv = device_weights(scale, offset, n_out)
        for what, a, b in (("first", df, ef), ("weights", dw.view(np.uint32), ew.view(np.uint32)),
                           ("1/wsum", dinv.view(np.uint32), einv.view(np.uint32))):
            if not np.array_equal(a, b):
                o = int(np.argwhere(a != b)[0][0])
                bad.append(f"scale {scale!r} offset {offset!r} n_out {n_out}: {what} differs, first at output {o}")
    assert not bad, f"{len(bad)} of {len(SWEEP)} mappings differ: {bad[:5]}"


# ------------------------------------------------------------------------------------------------
# NC-8 on the device
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_device_sincos_is_correctly_rounded():
    """sin_cr / cos_cr of kernels.cu (fp64 sin / cos rounded to f32) against the oracle's glibc (float)sin((double)x) for all
    117,440,512 floats with |x| in [2^-3, 2^4): every argument k_weights takes once the scale is at most 4"""
    from oracle import oracle as orc
    mant = np.arange(1 << 23, dtype=np.uint32)
    total, n_bad, examples = 0, 0, []
    for e in range(127 - 3, 127 + 4):   # one binade and sign per chunk
        for sign in (0, 1):
            x = ((np.uint32(sign << 31) | np.uint32(e << 23)) | mant).view(np.float32)
            ds, dc = np.empty_like(x), np.empty_like(x)
            assert F.lib().smr_debug_sincos(x.ctypes.data, x.size, ds.ctypes.data, dc.ctypes.data) == 0
            es, ec = orc.sincos_cr(x)
            for name, d, ref in (("sin", ds, es), ("cos", dc, ec)):
                idx = np.flatnonzero(d.view(np.uint32) != ref.view(np.uint32))
                n_bad += idx.size
                examples += [(name, float(x[i]), float(d[i]), float(ref[i])) for i in idx[:4]]
            total += x.size
    assert total == 117440512
    print(f"NC-8 on the device: {total} arguments, {n_bad} sin / cos results differ from the oracle")
    assert n_bad == 0, examples[:10]
