"""Every resample kernel against the float64 restatement of the resampler (tests/resample_ref.py), directly.

The kernels are held byte for byte to the oracle elsewhere; here each case also holds the device's bytes to the
restatement under its acceptance rule, so a mistake the oracle shares with a kernel cannot hide.  Scenes are built with
`set_layouts`: opaque children at integer positions over an RGBA8 output, so each child's output bytes are the
resampled bytes.  Each case checks which kernel ran and that its plan is the restatement's (`debug_fused_jobs`,
`debug_resample_stages`), that the bytes equal the oracle's, and that they meet the rule; it prints the kernel and the
share of bytes off rint(v).

Translucent four-byte children go through the composite's blend, so the GPU cases use opaque sources only; the
resampler's alpha is held to the restatement on the CPU, in tests/test_resample_space.py.
"""
import numpy as np
import pytest

import smelter_b200 as s
from tests import resample_ref as R
from tests.test_gpu_fused_variants import (ALIGNED, REGISTRY as FUSED, RGBA, Job, check, family_job, first_tap,
                                           make_frame, render, scene_of)
from tests.test_gpu_generic_resample import FOUR_BYTE, REGISTRY as GENERIC, any_frame, mismatch_report, oracle_planes

pytestmark = pytest.mark.gpu


def node_of(frame):
    from tests.parity import node_texture
    return node_texture(frame)


def hold_to_restatement(got, jobs, frames, what, fused=None):
    """each job's block of the RGBA output against the restatement; the fused jobs' plans against its plan"""
    _, _, _, _, xs = scene_of(jobs)
    out = got[0]
    for k, (j, x0) in enumerate(zip(jobs, xs)):
        ev = R.evaluate(node_of(frames[j.input_id]), j.crop, j.dst)
        assert ev is not None, (what, j)
        if fused:
            f, pl = fused[k], ev.plan
            assert pl.shape() == "two-pass-h-first" and pl.levels in ((0, 0), (1, 1)), (what, pl)
            assert (f["box"], f["taps_h"], f["taps_v"], f["dst"]) == \
                (int(pl.levels == (1, 1)), pl.passes[0].taps, pl.passes[1].taps, j.dst), (what, f, pl.passes)
        vd = R.assert_rule(out[:j.dst[1], x0:x0 + j.dst[0]], ev, f"{what} job {k}")
        kern = fused[k]["kernel"] if fused else "generic"
        print(f"{what} job {k} [{kern}]: {vd.line()}")


# ------------------------------------------------------------------------------------------------
# the fused kernels: one scene per instantiation, then the geometry edges of each family
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("entry", FUSED, ids=lambda e: e.name)
def test_fused_instantiation(entry):
    """k_resample_tma3 <2|4, planar|NV12> on both ranges, k_resample_tma0 for each window with and without the box,
    k_resample_fused_int <0|2|3|4> on all four sources: extreme content in every plane"""
    fr = {"input_1": make_frame(entry.fmt, "extreme", 17, *entry.src)}
    jobs = [Job("input_1", entry.crop, entry.dst)]
    got, fused, _ = check(jobs, fr, expect=[entry.expect()], what=entry.name)
    hold_to_restatement(got, jobs, fr, entry.name, fused)


def edge_jobs(family):
    """(dw, dh[, crop_left, crop_top, src_w]) of each edge: the last strip 2 columns wide, one strip of 250 rows (the
    row partition cuts it), a source smaller than one TMA box, and the last tile ending at the right image edge"""
    last2 = {"tma3": 58 * 3 + 2, "tma0": 64 * 2 + 2, "ldg": 64 * 2 + 2}[family]
    geoms = [(last2, 40), (40, 250), (24, 6), (12, 4)]
    if family == "tma3":
        x0 = first_tap(4.0, 0.0, 58 * 2)
        geoms.append((58 * 2 + 40, 40, 0.0, 0.0, (x0 & ~15) + 272))
    elif family == "tma0":
        x0 = first_tap(2.0, 0.5, 64 * 2) & ~1
        geoms.append((150, 40, 0.0, 0.0, (x0 & ~15) + 272))
    return geoms


def run_geoms(family, fmt, geoms, what, expect_kernel):
    jobs, frames, places, expect = [], {}, {}, []
    for k, g in enumerate(geoms):
        src, crop, dst, pl, kern = family_job(family, *g)
        iid = f"input_{k}"
        frames[iid] = make_frame(fmt, "extreme", 500 + k, *src)
        places[iid] = pl
        jobs.append(Job(iid, crop, dst))
        expect.append({"kernel": kern} if expect_kernel else None)
    got, fused, _ = check(jobs, frames, placements=places, expect=expect, what=f"{family} {fmt} {what}")
    hold_to_restatement(got, jobs, frames, f"{family} {fmt} {what}", fused)


@pytest.mark.parametrize("fmt", ["yuv", "yuvj", "nv12"])
@pytest.mark.parametrize("family", ["tma3", "tma0", "ldg"])
def test_fused_family_edges(family, fmt):
    run_geoms(family, fmt, edge_jobs(family), "edges", True)


@pytest.mark.parametrize("fmt", ["yuv", "nv12"])
@pytest.mark.parametrize("family", ["tma3", "tma0", "ldg"])
def test_fused_crop_offsets(family, fmt):
    """integral and fractional offsets on each axis, some past 4096 (the offset may move a job to another kernel, so
    only the plan and the bytes are checked)"""
    geoms = [(100, 40, l, t) for l, t in ((8.0, 0.0), (0.37, 0.37), (4100.0, 0.0), (5000.37, 3.5), (0.0, 2050.25))]
    run_geoms(family, fmt, geoms, "crop offsets", False)


def test_cfg3_child_full_size():
    """one child of bench.py's cfg3 scene: a 3840 x 2160 NV12 frame shown 960 x 540 (k_resample_tma3 at 4:1)"""
    fr = {"input_1": make_frame("nv12", "smooth", 7001, 3840, 2160)}
    jobs = [Job("input_1", (0.0, 0.0, 3840.0, 2160.0), (960, 540))]
    got, fused, _ = check(jobs, fr, placements={"input_1": ALIGNED}, expect=[{"kernel": "tma_int", "ratio": 4}],
                          what="cfg3 child")
    hold_to_restatement(got, jobs, fr, "cfg3 child", fused)


# ------------------------------------------------------------------------------------------------
# the generic passes: k_convert + the box / first / last stages
# ------------------------------------------------------------------------------------------------
def opaque_frame(fmt, seed, w, h):
    f = any_frame(fmt, "extreme", seed, w, h)
    if fmt in FOUR_BYTE:
        t = np.array(f.data.planes[0]).reshape(h, w, 4)
        t[..., 0 if fmt == "argb" else 3] = 255
        f = s.Frame(s.FrameData(f.data.kind, (t.reshape(h, 4 * w),)), f.resolution)
    return f


@pytest.mark.parametrize("case", GENERIC, ids=lambda c: c.name)
def test_generic_stages(case):
    """four-byte, 4:2:2 / 4:4:4, interleaved and 4:2:0 sources on every plan shape the generic passes take"""
    fr = {i: opaque_frame(fmt, 1300 + k, w, h) for k, (i, (fmt, w, h)) in enumerate(case.inputs.items())}
    r = s.Renderer()
    got = render(r, case.jobs, fr, RGBA, case.placements)
    assert r.debug_fused_jobs() == [], case.name
    ran, _ = r.debug_resample_stages()
    want, seen = [], set()
    for j in case.jobs:
        key = (j.input_id, j.crop, j.dst)
        if key not in seen:
            seen.add(key)
            fmt, w, h = case.inputs[j.input_id]
            want.append(R.plan((w, h), j.crop, j.dst).stages())
    order = ("box", "first", "last")
    want = [x for st in order for p in want for x in p if x["stage"] == st]
    assert [{k: v for k, v in x.items() if k not in ("source", "src_kind")} for x in ran] == want, case.name
    rep = mismatch_report(got, oracle_planes(case.jobs, fr, RGBA), case.jobs, [])
    assert rep is None, f"{case.name}: {rep}"
    hold_to_restatement(got, case.jobs, fr, case.name)
