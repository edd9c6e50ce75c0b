"""The integer-ratio TMA kernel (k_resample_tma3) with its compiled-in weights and its per-launch luma table.

- The weights of int_weights.h are what the weight kernel computes on the device for the same mapping, bit for bit.
- One tick with full-range and limited-range sources at 2:1 and 4:1 is byte-identical to the oracle.  The luma table
  is built for one range per launch, so planar sources of both ranges take one launch each and NV12 (limited) a third."""
import ctypes as C

import numpy as np
import pytest

import smelter_b200 as s
from smelter_b200 import _ffi
from tests import harness
from tests.parity import OUTPUT_ID, TrackedRenderer, assert_identical, nv12_frame, run_case, yuv_frame
from tests.test_int_weights import header_tables

pytestmark = pytest.mark.gpu

NV12 = s.OutputFrameFormat.Nv12WgpuTexture


def device_weights(scale, offset, out_coord):
    L = _ffi.lib()
    w = (C.c_float * 64)()
    taps, inv = C.c_uint32(), C.c_float()
    st = L.smr_debug_weights(scale, offset, out_coord, w, 64, C.byref(taps), C.byref(inv))
    assert st == 0, st
    return np.array(w[:taps.value], np.float32), np.float32(inv.value)


@pytest.mark.parametrize("S", [2, 3, 4])
def test_header_weights_are_the_device_weights(S):
    w, inv = header_tables()[S]
    for o in (0, 5, 1919):
        dw, dinv = device_weights(float(S), 0.0, o)
        assert np.array_equal(dw.view(np.uint32), w.view(np.uint32)), (S, o)
        assert dinv.view(np.uint32) == inv.view(np.uint32), (S, o)


def full_range_frame(planes, w, h):
    y, u, v = planes
    return s.Frame(s.FrameData.PlanarYuvJ420(s.YuvPlanes(y, u, v)), s.Resolution(w, h), 0.0)


@pytest.mark.parametrize("S", [2, 4])
def test_mixed_range_tick_integer_ratio(S):
    """2 x 2 tiles of 640 x 360 from (640 S) x (360 S) sources: NV12 (limited), planar limited and two planar full range
    inputs in one tick.  Noise on two inputs so that every tap matters; full-range content spans all 256 luma codes."""
    w, h = 640 * S, 360 * S
    fr = {
        "input_1": nv12_frame(harness.random_yuv420(8100 + S, w, h), w, h),
        "input_2": full_range_frame(harness.random_yuv420(8200 + S, w, h), w, h),
        "input_3": yuv_frame(harness.smooth_yuv420(8300 + S, w, h), w, h),
        "input_4": full_range_frame(harness.smooth_yuv420(8400 + S, w, h), w, h),
    }
    y = np.asarray(fr["input_2"].data.planes[0])
    y[:16, :16] = np.arange(256, dtype=np.uint8).reshape(16, 16)
    scene = s.TilesComponent(children=[s.InputStreamComponent(input_id=i) for i in fr],
                             background_color=s.RGBAColor(0x20, 0x30, 0x40, 255))
    r = TrackedRenderer()
    for i in fr:
        r.register_input(i)
    r.set_profiling(True)
    res = s.Resolution(1280, 720)
    r.update_scene(OUTPUT_ID, res, NV12, scene)
    got, exp, _ = run_case(scene, fr, renderer=r, resolution=res, out_format=NV12)
    assert_identical(got, exp, f"mixed ranges {S}:1")
    kt = r.kernel_times()
    # one integer-ratio TMA launch per (source class, range): planar full, planar limited, NV12
    assert kt["resample_fused"][1] == 3, kt
    assert kt["resample_first"][1] == 0 and kt["resample_box"][1] == 0 and kt["convert"][1] == 0, kt
