"""gpu-video's frame converters on an H100: every byte of smr_video_nv12_to_rgba against the NC-11 oracle
(tests/video_convert_oracle.c) and of smr_video_rgba_to_nv12 against K11's (orc_rgba_to_nv12_scaled), at the source size and
rescaled, on random bytes and on the joint byte-space frames, from host and pitched device sources into host and pitched
device targets, in both rendering modes."""
import ctypes as C

import numpy as np
import pytest

import smelter_b200 as s
from oracle import oracle as orc
from smelter_b200 import _ffi as F
from tests.c_oracles import nv12_to_rgba as oracle
from tests.test_color_conversion_space import yuv420_block_triples, yuv420_chroma_sums

pytestmark = pytest.mark.gpu

BT709_LIMITED = F.VideoColor(F.COLOR_SPACE_BT709, F.COLOR_RANGE_LIMITED)
UNSPECIFIED_LIMITED = F.VideoColor(F.COLOR_SPACE_UNSPECIFIED, F.COLOR_RANGE_LIMITED)


def random_nv12(w, h, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (h, w), np.uint8), rng.integers(0, 256, (h // 2, w // 2, 2), np.uint8)


def random_rgba(w, h, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 4), np.uint8)


def nv12(y, uv):
    h, w = y.shape
    return s.Frame(s.FrameData.Nv12(s.NvPlanes(y, uv)), s.Resolution(w, h))


def rgba_frame(a):
    h, w, _ = a.shape
    return s.Frame(s.FrameData.Rgba8(a), s.Resolution(w, h))


@pytest.fixture(scope="module")
def r():
    rr = s.Renderer()
    yield rr
    rr.close()


def assert_same(got, want, what):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = got != want
    assert not bad.any(), (what, int(bad.sum()), tuple(np.argwhere(bad)[0]))


# ---------------------------------------------------------------------------------------------------------------------
# NV12 -> RGBA
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", [(3840, 2160), (1920, 1080), (2, 2), (6, 4)])
def test_source_size_random(r, w, h):
    y, uv = random_nv12(w, h, w + h)
    assert_same(r.video_nv12_to_rgba(nv12(y, uv)), oracle(y, uv), (w, h))


@pytest.mark.parametrize("src,dst", [((1920, 1080), (3840, 2160)), ((3840, 2160), (1280, 720)), ((1918, 1078), (1001, 563)),
                                     ((1920, 1080), (1, 1)), ((2, 2), (1, 1)), ((3840, 2160), (1, 1)), ((2, 2), (16, 9)),
                                     ((16384, 2), (16384, 2)), ((16384, 2), (1000, 3)), ((16384, 2), (3, 17)),
                                     ((1920, 1080), (1920, 1081)), ((640, 360), (640, 720))])
def test_scaled_random(r, src, dst):
    y, uv = random_nv12(*src, seed=sum(src) + sum(dst))
    assert_same(r.video_nv12_to_rgba(nv12(y, uv), s.Resolution(*dst)), oracle(y, uv, *dst), (src, dst))


def joint_frames():
    for part in range(4):
        yield f"block{part}", yuv420_block_triples(part)[0]
    yield "chroma_sums", yuv420_chroma_sums()[0]


def test_joint_byte_space_through_the_kernel(r):
    """every exact-chroma (Y, Cb, Cr) and every interpolated chroma value with every luma (the 4096 x 4096 frames of the
    colour-space test), at the source size and at a 2:1 and a 3:2 rescale"""
    for name, (y, u, v) in joint_frames():
        uv = np.ascontiguousarray(np.stack([u, v], -1))
        assert_same(r.video_nv12_to_rgba(nv12(y, uv)), oracle(y, uv), name)
        for dst in ((2048, 2048), (2731, 2731)):
            assert_same(r.video_nv12_to_rgba(nv12(y, uv), s.Resolution(*dst)), oracle(y, uv, *dst), (name, dst))


def test_frame_metadata_and_kernel_class(r):
    y, uv = random_nv12(64, 36, 2)
    want = oracle(y, uv)
    assert_same(r.video_nv12_to_rgba(nv12(y, uv), frame_color=(s.ColorSpace.BT709, s.ColorRange.Limited)), want, "bt709")
    with pytest.raises(s.RendererError) as e:
        r.video_nv12_to_rgba(nv12(y, uv), frame_color=(s.ColorSpace.BT709, s.ColorRange.Full))
    assert e.value.status == 1
    with pytest.raises(s.RendererError) as e:
        r.video_nv12_to_rgba(nv12(y, uv), converter=(s.ColorSpace.BT601Pal, s.ColorRange.Limited))
    assert e.value.status == 5
    r.set_profiling(True)
    try:
        k0 = r.kernel_times()
        r.video_nv12_to_rgba(nv12(y, uv))
        r.video_nv12_to_rgba(nv12(y, uv), s.Resolution(30, 20))
        r.video_rgba_to_nv12(rgba_frame(random_rgba(64, 36, 3)))
        k1 = r.kernel_times()
    finally:
        r.set_profiling(False)
    assert k1["video_convert"][1] == k0["video_convert"][1] + 2 and k1["output"][1] == k0["output"][1] + 1
    assert all(k1[k][1] == k0[k][1] for k in k1 if k not in ("video_convert", "output"))


def device_nv12_surface(y, uv, aligned_h, pitch, seed):
    """an NVDEC-shaped surface: garbage everywhere, the crop's bytes at the top of each plane, chroma below aligned_h rows"""
    import torch
    h, w = y.shape
    host = np.random.default_rng(seed).integers(0, 256, (aligned_h * 3 // 2, pitch), np.uint8)
    host[:h, :w] = y
    host[aligned_h:aligned_h + h // 2, :w] = uv.reshape(h // 2, w)
    surf = torch.from_numpy(host).to("cuda:0")
    f = F.InputFrame()
    f.input_id, f.format, f.width, f.height, f.mem_kind = b"src", F.FRAME_NV12, w, h, F.MEM_DEVICE
    f.planes[0], f.planes[1] = surf.data_ptr(), surf.data_ptr() + pitch * aligned_h
    f.pitch[0], f.pitch[1] = pitch, pitch
    return f, surf


def device_rgba_target(w, h, pitch, sentinel=0xCD):
    import torch
    return torch.full((h + 2, pitch), sentinel, dtype=torch.uint8, device="cuda:0")


def read_rgba_target(t, w, h, sentinel=0xCD):
    a = t.cpu().numpy()
    assert (a[:h, 4 * w:] == sentinel).all() and (a[h:] == sentinel).all(), "bytes past the target were written"
    return a[:h, :4 * w].reshape(h, w, 4).copy()


@pytest.mark.parametrize("dst,pad", [((1920, 1080), 256), ((1920, 1080), 4), ((1280, 720), 68), ((3840, 2160), 12)])
def test_pitched_device_source_crop_into_pitched_device_target(r, dst, pad):
    """a 1920 x 1088 surface (pitch 2048) cropped to 1080 rows, into pitched device targets whose padding keeps its sentinel;
    a pitch that is 4- but not 8-byte aligned takes the 4-byte stores"""
    import torch
    y, uv = random_nv12(1920, 1080, 11)
    src, surf = device_nv12_surface(y, uv, 1088, 2048, 12)
    w, h = dst
    pitch = 4 * w + pad
    t = device_rgba_target(w, h, pitch)
    torch.cuda.synchronize()
    st0 = r.stats()
    assert r._lib.smr_video_nv12_to_rgba(r._h, BT709_LIMITED, C.byref(src), UNSPECIFIED_LIMITED, w, h, t.data_ptr(), pitch,
                                         F.MEM_DEVICE) == F.SMR_OK, r._err()
    st1 = r.stats()
    assert st1["h2d_bytes"] == st0["h2d_bytes"] and st1["d2h_bytes"] == st0["d2h_bytes"]   # no host copies
    assert_same(read_rgba_target(t, w, h), oracle(y, uv, w, h), (dst, pad))


def test_host_and_device_sources_and_targets(r):
    import torch
    y, uv = random_nv12(1280, 720, 21)
    want_same, want_up = oracle(y, uv), oracle(y, uv, 1920, 1080)
    ty, tuv = torch.from_numpy(y).to("cuda:0"), torch.from_numpy(uv).to("cuda:0")
    dev = s.Frame(s.FrameData("Nv12", (ty.data_ptr(), tuv.data_ptr()), device=True), s.Resolution(1280, 720))
    torch.cuda.synchronize()
    for frame, what in ((nv12(y, uv), "host"), (dev, "device")):
        assert_same(r.video_nv12_to_rgba(frame), want_same, (what, "host target"))
        assert_same(r.video_nv12_to_rgba(frame, s.Resolution(1920, 1080)), want_up, (what, "host target, scaled"))
        keep = []
        arr = r._input_frames(s.FrameSet(frames={"_": frame}), keep)
        for (w, h), want in (((1280, 720), want_same), ((1920, 1080), want_up)):
            t = device_rgba_target(w, h, 4 * w)
            torch.cuda.synchronize()
            assert r._lib.smr_video_nv12_to_rgba(r._h, BT709_LIMITED, arr, UNSPECIFIED_LIMITED, w, h, t.data_ptr(), 0,
                                                 F.MEM_DEVICE) == F.SMR_OK, r._err()
            assert_same(read_rgba_target(t, w, h), want, (what, "device target", w, h))


def test_host_target_pitch_keeps_padding(r):
    y, uv = random_nv12(64, 36, 4)
    buf = np.full((36, 64 * 4 + 20), 0xAB, np.uint8)
    keep = []
    arr = r._input_frames(s.FrameSet(frames={"_": nv12(y, uv)}), keep)
    assert r._lib.smr_video_nv12_to_rgba(r._h, BT709_LIMITED, arr, UNSPECIFIED_LIMITED, 0, 0, buf.ctypes.data, buf.shape[1],
                                         F.MEM_HOST) == F.SMR_OK, r._err()
    assert (buf[:, 256:] == 0xAB).all()
    assert_same(buf[:, :256].reshape(36, 64, 4), oracle(y, uv), "host pitch")


def test_rendering_mode_does_not_matter(r):
    y, uv = random_nv12(1918, 1078, 31)
    rc = s.Renderer(s.RendererOptions(rendering_mode=s.RenderingMode.CpuOptimized))
    try:
        for dst in (None, s.Resolution(1001, 563)):
            a, b = r.video_nv12_to_rgba(nv12(y, uv), dst), rc.video_nv12_to_rgba(nv12(y, uv), dst)
            assert_same(a, b, ("modes", dst))
        rgba = random_rgba(640, 360, 32)
        for (ya, uva), (yb, uvb) in ((r.video_rgba_to_nv12(rgba_frame(rgba), d), rc.video_rgba_to_nv12(rgba_frame(rgba), d))
                                     for d in (None, s.Resolution(320, 180))):
            assert_same(ya, yb, "modes y")
            assert_same(uva, uvb, "modes uv")
    finally:
        rc.close()


# ---------------------------------------------------------------------------------------------------------------------
# RGBA -> NV12 (K11 through k_output)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("src,dst", [((1920, 1080), (1920, 1080)), ((1280, 720), (1920, 1080)), ((3840, 2160), (1280, 720)),
                                     ((641, 359), (2, 2)), ((3, 5), (16384, 2)), ((1918, 1078), (1000, 562))])
def test_rgba_to_nv12_random(r, src, dst):
    a = random_rgba(*src, seed=sum(src) + sum(dst))
    gy, guv = r.video_rgba_to_nv12(rgba_frame(a), s.Resolution(*dst))
    wy, wuv = orc.rgba_to_nv12_scaled(a, *dst)
    assert_same(gy, wy, (src, dst, "y"))
    assert_same(guv, wuv, (src, dst, "uv"))


def test_rgba_to_nv12_device_planes_with_sentinels(r):
    """pitched device source and target planes (the y and uv planes at their own pitches, starting at odd addresses);
    bytes past each row and plane keep their sentinel"""
    import torch
    a = random_rgba(1920, 1080, 41)
    sp = 1920 * 4 + 64
    host = np.random.default_rng(42).integers(0, 256, (1090, sp), np.uint8)
    host[:1080, :1920 * 4] = a.reshape(1080, -1)
    surf = torch.from_numpy(host).to("cuda:0")
    src = F.InputFrame()
    src.input_id, src.format, src.width, src.height, src.mem_kind = b"src", F.FRAME_RGBA8, 1920, 1080, F.MEM_DEVICE
    src.planes[0], src.pitch[0] = surf.data_ptr(), sp
    for (w, h) in ((1920, 1080), (1280, 720), (3840, 2160)):
        py, puv = w + 13, w + 6
        ty = torch.full((h + 2, py + 1), 0xCD, dtype=torch.uint8, device="cuda:0")
        tuv = torch.full((h // 2 + 2, puv + 1), 0xCD, dtype=torch.uint8, device="cuda:0")
        planes = (C.c_void_p * 2)(ty.data_ptr() + 1, tuv.data_ptr() + 1)
        torch.cuda.synchronize()
        st0 = r.stats()
        assert r._lib.smr_video_rgba_to_nv12(r._h, BT709_LIMITED, C.byref(src), w, h, planes, (C.c_uint32 * 2)(py, puv),
                                             F.MEM_DEVICE) == F.SMR_OK, r._err()
        st1 = r.stats()
        assert st1["h2d_bytes"] == st0["h2d_bytes"] and st1["d2h_bytes"] == st0["d2h_bytes"]
        ay = ty.cpu().numpy().reshape(-1)[1:1 + (h + 1) * py].reshape(h + 1, py)
        auv = tuv.cpu().numpy().reshape(-1)[1:1 + (h // 2 + 1) * puv].reshape(h // 2 + 1, puv)
        assert (ay[:h, w:] == 0xCD).all() and (ay[h:] == 0xCD).all()
        assert (auv[:h // 2, w:] == 0xCD).all() and (auv[h // 2:] == 0xCD).all()
        wy, wuv = orc.rgba_to_nv12_scaled(a, w, h)
        assert_same(ay[:h, :w], wy, (w, h, "y"))
        assert_same(auv[:h // 2, :w].reshape(h // 2, w // 2, 2), wuv, (w, h, "uv"))


def test_rgba_to_nv12_host_and_device_sources_and_targets(r):
    import torch
    a = random_rgba(1280, 720, 51)
    wy, wuv = orc.rgba_to_nv12_scaled(a, 1280, 720)
    ta = torch.from_numpy(a).to("cuda:0")
    dev = s.Frame(s.FrameData("Rgba8", (ta.data_ptr(),), device=True), s.Resolution(1280, 720))
    torch.cuda.synchronize()
    for frame, what in ((rgba_frame(a), "host"), (dev, "device")):
        gy, guv = r.video_rgba_to_nv12(frame)
        assert_same(gy, wy, (what, "host y"))
        assert_same(guv, wuv, (what, "host uv"))
        keep = []
        arr = r._input_frames(s.FrameSet(frames={"_": frame}), keep)
        t = torch.zeros((720 * 3 // 2, 1280), dtype=torch.uint8, device="cuda:0")
        planes = (C.c_void_p * 2)(t.data_ptr(), t.data_ptr() + 1280 * 720)
        torch.cuda.synchronize()
        assert r._lib.smr_video_rgba_to_nv12(r._h, BT709_LIMITED, arr, 1280, 720, planes, None, F.MEM_DEVICE) == F.SMR_OK, r._err()
        got = t.cpu().numpy()
        assert_same(got[:720], wy, (what, "device y"))
        assert_same(got[720:].reshape(360, 640, 2), wuv, (what, "device uv"))


def test_round_trip_through_both_converters(r):
    """a decoded frame out as RGBA and back as NV12: each step equals its oracle"""
    y, uv = random_nv12(1920, 1080, 61)
    rgba = r.video_nv12_to_rgba(nv12(y, uv))
    assert_same(rgba, oracle(y, uv), "nv12 -> rgba")
    gy, guv = r.video_rgba_to_nv12(rgba_frame(rgba), s.Resolution(1280, 720))
    wy, wuv = orc.rgba_to_nv12_scaled(rgba, 1280, 720)
    assert_same(gy, wy, "rgba -> nv12 y")
    assert_same(guv, wuv, "rgba -> nv12 uv")
