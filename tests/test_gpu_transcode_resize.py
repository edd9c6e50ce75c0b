"""smr_transcode_resize on an H100: every Y and UV byte of every rendition against the CPU oracle
(tests/transcode_oracle.c), for the three ScalingAlgorithms over downscale ladders, upscales, odd ratios, 1:1 and a
16384-wide strip, with host and device sources and destinations, pitched surfaces and an smr_render output as source."""
import ctypes as C

import numpy as np
import pytest

import smelter_b200 as s
from smelter_b200 import _ffi as F
from tests.oracle_transcode import transcode_resize as oracle

pytestmark = pytest.mark.gpu

ALGOS = (F.SCALE_NEAREST, F.SCALE_BILINEAR, F.SCALE_LANCZOS3)
SHAPES = {
    "4k_ladder": ((3840, 2160), [(1920, 1080), (1280, 720), (854, 480), (640, 360)]),
    "1080_ladder": ((1920, 1080), [(1280, 720), (640, 360), (426, 240)]),
    "upscale_360_1080": ((640, 360), [(1920, 1080)]),
    "upscale_2_16": ((2, 2), [(16, 16)]),
    "odd_ratio": ((1918, 1078), [(1000, 562)]),
    "one_to_one": ((1920, 1080), [(1920, 1080)]),
    "strip": ((16384, 2), [(16384, 2), (1000, 2), (2, 16)]),
}


def random_nv12(w, h, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (h, w), np.uint8), rng.integers(0, 256, (h // 2, w // 2, 2), np.uint8)


def checkerboard_nv12(w, h, cell=8):
    yy, xx = np.mgrid[0:h, 0:w]
    y = np.where(((yy // cell) + (xx // cell)) & 1, 255, 0).astype(np.uint8)
    cy, cx = np.mgrid[0:h // 2, 0:w // 2]
    c = np.where(((cy // (cell // 2)) + (cx // (cell // 2))) & 1, 255, 0).astype(np.uint8)
    return y, np.stack([c, 255 - c], -1)


def nv12(y, uv):
    h, w = y.shape
    return s.Frame(s.FrameData.Nv12(s.NvPlanes(y, uv)), s.Resolution(w, h))


@pytest.fixture(scope="module")
def r():
    rr = s.Renderer()
    yield rr
    rr.close()


def check(got, y, uv, outs, what):
    for (gy, guv), (w, h, algo) in zip(got, outs):
        ey, euv = oracle(y, uv, w, h, algo)
        assert np.array_equal(gy, ey), (what, w, h, algo, int((gy != ey).sum()))
        assert np.array_equal(guv, euv), (what, w, h, algo, int((guv != euv).sum()))


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_random_frames_match_the_oracle(r, shape, algo):
    (w, h), sizes = SHAPES[shape]
    y, uv = random_nv12(w, h, seed=w + h + algo)
    outs = [(ow, oh, algo) for ow, oh in sizes]
    check(r.transcode_resize(nv12(y, uv), outs), y, uv, outs, shape)


@pytest.mark.parametrize("algo", ALGOS)
def test_checkerboard_matches_the_oracle_and_ringing_clamps(r, algo):
    y, uv = checkerboard_nv12(1920, 1080)
    outs = [(1280, 720, algo), (854, 480, algo), (2880, 1620, algo)]
    got = r.transcode_resize(nv12(y, uv), outs)
    check(got, y, uv, outs, "checkerboard")
    if algo == F.SCALE_LANCZOS3:   # overshoot past both ends of the range is stored as 0 and 255
        for gy, guv in got:
            assert (gy == 0).any() and (gy == 255).any() and (guv == 0).any() and (guv == 255).any()


def test_eight_mixed_renditions_in_one_launch(r):
    y, uv = random_nv12(1920, 1080, 7)
    outs = [(1280, 720, 2), (960, 540, 1), (640, 360, 0), (426, 240, 2), (3840, 2160, 1), (2, 2, 2), (1920, 1080, 0),
            (1002, 566, 1)]
    r.set_profiling(True)
    try:
        before = r.kernel_times()["transcode"][1]
        got = r.transcode_resize(nv12(y, uv), outs)
        assert r.kernel_times()["transcode"][1] == before + 1
        r.transcode_resize(nv12(y, uv), outs[:3])
        assert r.kernel_times()["transcode"][1] == before + 2
    finally:
        r.set_profiling(False)
    check(got, y, uv, outs, "eight")


def device_renditions(sizes, pitch_pad=0, sentinel=0xCD):
    """pitched device destinations filled with a sentinel: (Rendition array, surfaces)"""
    import torch
    arr = (F.Rendition * len(sizes))()
    surf = []
    for i, (w, h, algo) in enumerate(sizes):
        py, puv = w + pitch_pad, w + pitch_pad + 2
        ty = torch.full((h + 3, py), sentinel, dtype=torch.uint8, device="cuda:0")
        tuv = torch.full((h // 2 + 3, puv), sentinel, dtype=torch.uint8, device="cuda:0")
        surf.append((ty, tuv))
        arr[i].width, arr[i].height, arr[i].scaling, arr[i].mem_kind = w, h, algo, F.MEM_DEVICE
        arr[i].planes[0], arr[i].planes[1] = ty.data_ptr(), tuv.data_ptr()
        arr[i].pitch[0], arr[i].pitch[1] = py, puv
    return arr, surf


def read_back(surf, sizes, sentinel=0xCD):
    got = []
    for (ty, tuv), (w, h, _) in zip(surf, sizes):
        ay, auv = ty.cpu().numpy(), tuv.cpu().numpy()
        assert (ay[:h, w:] == sentinel).all() and (ay[h:] == sentinel).all(), "bytes past the Y plane were written"
        assert (auv[:h // 2, w:] == sentinel).all() and (auv[h // 2:] == sentinel).all(), "bytes past the UV plane were written"
        got.append((ay[:h, :w].copy(), auv[:h // 2, :w].reshape(h // 2, w // 2, 2).copy()))
    return got


def test_pitched_device_source_crop_and_device_destinations(r):
    """An NVDEC-shaped 1920 x 1088 surface (pitch 2048, chroma below the aligned height) cropped to 1080 rows: the padding
    rows and columns hold garbage and are never read; destinations are pitched device planes whose bytes past each row
    and plane stay at the sentinel."""
    import torch
    w, h, ah, pitch = 1920, 1080, 1088, 2048
    rng = np.random.default_rng(11)
    surf_host = rng.integers(0, 256, (ah * 3 // 2, pitch), np.uint8)   # garbage everywhere, then the crop's bytes
    y, uv = random_nv12(w, h, 12)
    surf_host[:h, :w] = y
    surf_host[ah:ah + h // 2, :w] = uv.reshape(h // 2, w)
    surf = torch.from_numpy(surf_host).to("cuda:0")
    src = F.InputFrame()
    src.input_id, src.format, src.width, src.height, src.mem_kind = b"src", F.FRAME_NV12, w, h, F.MEM_DEVICE
    src.planes[0], src.planes[1] = surf.data_ptr(), surf.data_ptr() + pitch * ah
    src.pitch[0], src.pitch[1] = pitch, pitch
    sizes = [(1280, 720, 2), (854, 480, 1), (640, 360, 0), (1920, 1080, 2)]
    arr, dsurf = device_renditions(sizes, pitch_pad=70)
    torch.cuda.synchronize()
    st0 = r.stats()
    assert r._lib.smr_transcode_resize(r._h, C.byref(src), arr, len(sizes)) == F.SMR_OK, r._err()
    st1 = r.stats()
    assert st1["h2d_bytes"] == st0["h2d_bytes"] and st1["d2h_bytes"] == st0["d2h_bytes"]   # no host copies
    check(read_back(dsurf, sizes), y, uv, sizes, "pitched device")


def test_host_source_device_destinations_and_device_source_host_destinations(r):
    import torch
    y, uv = random_nv12(1280, 720, 21)
    sizes = [(640, 360, 2), (1920, 1080, 1)]
    arr, dsurf = device_renditions(sizes, pitch_pad=6)
    keep = []
    host = r._input_frames(s.FrameSet(frames={"_": nv12(y, uv)}), keep)
    assert r._lib.smr_transcode_resize(r._h, host, arr, len(sizes)) == F.SMR_OK, r._err()
    check(read_back(dsurf, sizes), y, uv, sizes, "host -> device")
    ty, tuv = torch.from_numpy(y).to("cuda:0"), torch.from_numpy(uv).to("cuda:0")
    dev_frame = s.Frame(s.FrameData("Nv12", (ty.data_ptr(), tuv.data_ptr()), device=True), s.Resolution(1280, 720))
    torch.cuda.synchronize()
    check(r.transcode_resize(dev_frame, sizes), y, uv, sizes, "device -> host")


def test_render_output_as_source(r):
    """The library's own NV12 output, left in device memory by smr_render, feeds the transcoder directly."""
    import torch
    from tests import harness
    from tests.parity import yuv_frame
    w, h = 1280, 720
    rr = s.Renderer()
    try:
        rr.register_input("in")
        rr.update_scene("out", s.Resolution(w, h), s.OutputFrameFormat.Nv12WgpuTexture,
                        s.RescalerComponent(child=s.InputStreamComponent(input_id="in")))
        frame = yuv_frame(harness.test_input(1, 1920, 1080), 1920, 1080)
        keep = []
        in_arr = rr._input_frames(s.FrameSet(frames={"in": frame}), keep)
        ty = torch.zeros((h, w), dtype=torch.uint8, device="cuda:0")
        tuv = torch.zeros((h // 2, w), dtype=torch.uint8, device="cuda:0")
        out = (F.OutputFrame * 1)()
        out[0].output_id, out[0].mem_kind = b"out", F.MEM_DEVICE
        out[0].planes[0], out[0].planes[1] = ty.data_ptr(), tuv.data_ptr()
        torch.cuda.synchronize()
        assert rr._lib.smr_render(rr._h, 0, in_arr, 1, out, 1) == F.SMR_OK, rr._err()
        src = s.Frame(s.FrameData("Nv12", (ty.data_ptr(), tuv.data_ptr()), device=True), s.Resolution(w, h))
        sizes = [(640, 360, 2), (854, 480, 1), (426, 240, 0)]
        got = rr.transcode_resize(src, sizes)
        y, uv = ty.cpu().numpy(), tuv.cpu().numpy().reshape(h // 2, w // 2, 2)
        assert y.any()
        check(got, y, uv, sizes, "render output")
    finally:
        rr.close()
