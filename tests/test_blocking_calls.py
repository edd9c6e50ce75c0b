"""The six blocking calls -- smr_preprocess_frame, smr_premultiply_rgba8, smr_render_text, smr_transcode_resize,
smr_video_nv12_to_rgba and smr_video_rgba_to_nv12 -- as a caller counts on them beyond their output bytes (those are held
to the oracle by the tests of each call):

- on a host-only handle, which refusals come before SMR_ERR_CUDA (no device) and which after it;
- the kernel class each call's time is counted under: transcode, video_convert and output; none for preprocess,
  premultiply and text;
- what each call adds to the handle's statistics: one kernel launch, the staged source bytes (rows x row bytes, not the
  caller's pitch) to h2d_bytes and the host target bytes to d2h_bytes; device sources and targets add nothing;
- host target rows are written up to the row's end and no further, and render_text into device memory gives the bytes it
  gives into host memory."""
import ctypes as C

import numpy as np
import pytest

from smelter_b200 import _ffi as F

INVALID, CUDA = 1, 2   # SMR_ERR_INVALID_ARGUMENT, SMR_ERR_CUDA
BT709_LIMITED = F.VideoColor(F.COLOR_SPACE_BT709, F.COLOR_RANGE_LIMITED)
GLYPH = np.dtype(F.GLYPH_DTYPE)
SENTINEL = 0xA5
MASK_GLYPH, COLOR_GLYPH = 1, 0


# ---------------------------------------------------------------------------------------------------------------------
# host-only handle: SMR_ERR_CUDA (2) means every check before the device gate passed
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def host_handle():
    L = F.lib()
    h = C.c_void_p()
    assert L.smr_create(C.byref(F.Options(-1, 0, 100, 3_000_000_000, 30, 1)), C.byref(h)) == F.SMR_OK
    yield L, h
    L.smr_destroy(h)


def fake_frame(fmt=F.FRAME_RGBA8, w=16, h=8, ptr=0x1000):
    """a frame whose planes are never read: every call below stops at or before the device gate"""
    f = F.InputFrame()
    f.input_id, f.format, f.width, f.height, f.mem_kind = b"src", fmt, w, h, F.MEM_HOST
    for p in range(3):
        f.planes[p] = ptr
    return f


def test_preprocess_refuses_a_host_only_handle_before_its_frame_and_target_checks(host_handle):
    L, h = host_handle

    def pre(f, ow=0, oh=0, rgba=0x2000, pitch=0, mem=F.MEM_HOST):
        return L.smr_preprocess_frame(h, C.byref(f) if f is not None else None, ow, oh, rgba, pitch, mem)

    assert pre(None) == INVALID
    assert pre(fake_frame(), rgba=None) == INVALID
    assert pre(fake_frame()) == CUDA
    assert pre(fake_frame(), ow=0, oh=5) == CUDA                     # output resolution out of range
    assert pre(fake_frame(), ow=20000, oh=20) == CUDA
    assert pre(fake_frame(w=0)) == CUDA                              # input resolution out of range
    assert pre(fake_frame(fmt=99)) == CUDA                           # unknown format
    assert pre(fake_frame(ptr=0)) == CUDA                            # null plane
    assert pre(fake_frame(), pitch=60) == CUDA                       # output pitch shorter than a row (64 bytes)
    assert pre(fake_frame(), rgba=0x2002, mem=F.MEM_DEVICE) == CUDA  # device RGBA8 target not 4-byte aligned


def test_premultiply_refuses_a_host_only_handle_after_its_shape_check(host_handle):
    L, h = host_handle

    def pm(f, rgba=0x2000, pitch=0, mem=F.MEM_HOST):
        return L.smr_premultiply_rgba8(h, C.byref(f) if f is not None else None, rgba, pitch, mem)

    assert pm(None) == INVALID
    assert pm(fake_frame(), rgba=None) == INVALID
    assert pm(fake_frame(fmt=F.FRAME_NV12)) == INVALID              # straight-alpha RGBA8 only
    assert pm(fake_frame(fmt=F.FRAME_BGRA)) == INVALID
    assert pm(fake_frame()) == CUDA
    assert pm(fake_frame(w=0)) == CUDA
    assert pm(fake_frame(ptr=0)) == CUDA
    assert pm(fake_frame(), pitch=60) == CUDA
    assert pm(fake_frame(), rgba=0x2002, mem=F.MEM_DEVICE) == CUDA


def test_render_text_refuses_a_host_only_handle_before_its_size_glyph_and_atlas_checks(host_handle):
    L, h = host_handle
    mask = F.Atlas(0x3000, 64, 32, 0)

    def text(w=32, h_=16, glyphs=None, n=0, mask=None, color=None, color_mode=0, rgba=0x2000, pitch=0, mem=F.MEM_HOST):
        return L.smr_render_text(h, w, h_, F.Rgba(0, 0, 0, 0), glyphs, n, C.byref(mask) if mask else None,
                                 C.byref(color) if color else None, color_mode, rgba, pitch, mem)

    g = np.zeros(3, GLYPH)
    g["content"] = MASK_GLYPH
    assert text(rgba=None) == INVALID
    assert text(n=3) == INVALID                                      # glyphs without a glyph list
    assert text(color_mode=2) == INVALID
    assert text() == CUDA
    assert text(w=0) == CUDA                                         # text texture resolution out of range
    assert text(h_=16385) == CUDA
    assert text(glyphs=0x4000, n=(1 << 22) + 1) == CUDA              # too many glyphs
    bad = g.copy()
    bad["content"][1] = 7
    assert text(glyphs=bad.ctypes.data, n=3, mask=mask) == CUDA      # unknown glyph content
    assert text(glyphs=g.ctypes.data, n=3) == CUDA                   # mask glyphs without a mask atlas
    assert text(glyphs=g.ctypes.data, n=3, mask=F.Atlas(0x3000, 64, 32, 63)) == CUDA   # atlas pitch shorter than a row
    assert text(pitch=64) == CUDA                                    # output pitch shorter than a row (128 bytes)
    assert text(rgba=0x2002, mem=F.MEM_DEVICE) == CUDA


# ---------------------------------------------------------------------------------------------------------------------
# GPU: kernel classes and statistics of each call, host -> host and device -> device
# ---------------------------------------------------------------------------------------------------------------------
class Buffers:
    """Pitched planes for one call, in host memory (numpy) or device memory (torch): sources hold random bytes, targets
    a sentinel.  Each plane's pitch is its row plus 16 bytes, so a count of pitch x rows differs from rows x row bytes."""

    def __init__(self, device, seed=5):
        self.device, self.rng, self.keep, self.targets = device, np.random.default_rng(seed), [], []
        self.mem = F.MEM_DEVICE if device else F.MEM_HOST

    def _plane(self, a):
        if not self.device:
            return a, a.ctypes.data, a.shape[1]
        import torch
        t = torch.from_numpy(a).to("cuda:0")
        torch.cuda.synchronize()   # the call runs on the renderer's own stream
        return t, t.data_ptr(), a.shape[1]

    def source(self, rows, row_bytes):
        a, ptr, pitch = self._plane(self.rng.integers(0, 256, (rows, row_bytes + 16), np.uint8))
        self.keep.append(a)
        return ptr, pitch

    def target(self, rows, row_bytes):
        a, ptr, pitch = self._plane(np.full((rows, row_bytes + 16), SENTINEL, np.uint8))
        self.targets.append((a, row_bytes))
        return ptr, pitch

    def frame(self, fmt, w, h, planes):
        """an smr_input_frame of `planes` = [(rows, row bytes)] pitched source planes"""
        f = F.InputFrame()
        f.input_id, f.format, f.width, f.height, f.mem_kind = b"src", fmt, w, h, self.mem
        for p, (rows, row_bytes) in enumerate(planes):
            f.planes[p], f.pitch[p] = self.source(rows, row_bytes)
        return f

    def bytes(self, n):
        """n bytes if these planes are in host memory, else none"""
        return 0 if self.device else n

    def target_rows(self):
        """each target's rows, once the bytes past every row are checked to still hold the sentinel"""
        out = []
        for a, row_bytes in self.targets:
            a = a.cpu().numpy() if self.device else a
            assert (a[:, row_bytes:] == SENTINEL).all(), "bytes past a target row were written"
            out.append(a[:, :row_bytes].copy())
        return out


# Each case makes one call into `b`'s planes and returns (status, h2d bytes, d2h bytes, kernel class or None)
def preprocess(r, b):
    f = b.frame(F.FRAME_NV12, 64, 32, [(32, 64), (16, 64)])
    ptr, pitch = b.target(20, 40 * 4)
    st = r._lib.smr_preprocess_frame(r._h, C.byref(f), 40, 20, ptr, pitch, b.mem)
    return st, b.bytes(64 * 32 + 64 * 16), b.bytes(40 * 4 * 20), None


def premultiply(r, b):
    f = b.frame(F.FRAME_RGBA8, 24, 10, [(10, 24 * 4)])
    ptr, pitch = b.target(10, 24 * 4)
    st = r._lib.smr_premultiply_rgba8(r._h, C.byref(f), ptr, pitch, b.mem)
    return st, b.bytes(24 * 4 * 10), b.bytes(24 * 4 * 10), None


def text(r, b):
    """sources are host memory whatever the target's: the atlases and the glyph list are always staged"""
    rng = np.random.default_rng(3)
    mask = rng.integers(0, 256, (16, 32 + 8), np.uint8)
    color = rng.integers(0, 256, (8, 16 * 4 + 12), np.uint8)
    g = np.zeros(7, GLYPH)
    g["x"], g["y"] = rng.integers(-4, 40, 7), rng.integers(-4, 12, 7)
    g["width"], g["height"] = 10, 6
    g["atlas_x"], g["atlas_y"] = 2, 1
    g["color"] = rng.integers(0, 256, (7, 4))
    g["content"] = [MASK_GLYPH, COLOR_GLYPH] * 3 + [MASK_GLYPH]
    b.keep += [mask, color, g]
    ptr, pitch = b.target(12, 40 * 4)
    st = r._lib.smr_render_text(r._h, 40, 12, F.Rgba(10, 20, 30, 200), g.ctypes.data, len(g),
                                C.byref(F.Atlas(mask.ctypes.data, 32, 16, mask.shape[1])),
                                C.byref(F.Atlas(color.ctypes.data, 16, 8, color.shape[1])), 0, ptr, pitch, b.mem)
    return st, 32 * 16 + 16 * 4 * 8 + GLYPH.itemsize * len(g), b.bytes(40 * 4 * 12), None


def transcode(r, b):
    f = b.frame(F.FRAME_NV12, 64, 32, [(32, 64), (16, 64)])
    outs = (F.Rendition * 2)()
    for i, (w, h) in enumerate([(32, 16), (48, 24)]):
        outs[i].width, outs[i].height, outs[i].scaling, outs[i].mem_kind = w, h, F.SCALE_LANCZOS3, b.mem
        (outs[i].planes[0], outs[i].pitch[0]), (outs[i].planes[1], outs[i].pitch[1]) = b.target(h, w), b.target(h // 2, w)
    st = r._lib.smr_transcode_resize(r._h, C.byref(f), outs, 2)
    return st, b.bytes(64 * 32 + 64 * 16), b.bytes(32 * 16 * 3 // 2 + 48 * 24 * 3 // 2), "transcode"


def nv12_to_rgba(r, b):
    f = b.frame(F.FRAME_NV12, 64, 32, [(32, 64), (16, 64)])
    ptr, pitch = b.target(20, 40 * 4)
    st = r._lib.smr_video_nv12_to_rgba(r._h, BT709_LIMITED, C.byref(f), BT709_LIMITED, 40, 20, ptr, pitch, b.mem)
    return st, b.bytes(64 * 32 + 64 * 16), b.bytes(40 * 4 * 20), "video_convert"


def rgba_to_nv12(r, b):
    f = b.frame(F.FRAME_RGBA8, 24, 10, [(10, 24 * 4)])
    (y, py), (uv, puv) = b.target(16, 32), b.target(8, 32)
    st = r._lib.smr_video_rgba_to_nv12(r._h, BT709_LIMITED, C.byref(f), 32, 16, (C.c_void_p * 2)(y, uv),
                                       (C.c_uint32 * 2)(py, puv), b.mem)
    return st, b.bytes(24 * 4 * 10), b.bytes(32 * 16 * 3 // 2), "output"


CALLS = [preprocess, premultiply, text, transcode, nv12_to_rgba, rgba_to_nv12]


@pytest.fixture(scope="module")
def r():
    import smelter_b200 as s
    rr = s.Renderer()
    rr.set_profiling(True)
    yield rr
    rr.close()


def counted(r, call, b):
    """runs one call; returns its target rows after checking its statistics and kernel class"""
    t0, s0 = r.kernel_times(), r.stats()
    st, h2d, d2h, kclass = call(r, b)
    assert st == F.SMR_OK, r._err()
    t1, s1 = r.kernel_times(), r.stats()
    assert s1["kernel_launches"] - s0["kernel_launches"] == 1
    assert s1["h2d_bytes"] - s0["h2d_bytes"] == h2d
    assert s1["d2h_bytes"] - s0["d2h_bytes"] == d2h
    assert s1["frames_rendered"] == s0["frames_rendered"]
    for name in F.KERNEL_CLASSES:
        assert t1[name][1] - t0[name][1] == (1 if name == kclass else 0), (name, t0[name], t1[name])
    return b.target_rows()


@pytest.mark.gpu
@pytest.mark.parametrize("call", CALLS, ids=[c.__name__ for c in CALLS])
def test_statistics_kernel_class_and_target_bytes(r, call):
    """host -> host, then the same sources (same seed) device -> device: the device targets get the host targets' bytes"""
    host, dev = counted(r, call, Buffers(False)), counted(r, call, Buffers(True))
    assert len(host) == len(dev)
    for i, (a, d) in enumerate(zip(host, dev)):
        assert np.array_equal(a, d), (call.__name__, i, int((a != d).sum()))


@pytest.mark.gpu
def test_transcode_host_and_device_renditions_in_one_call(r):
    """renditions of both memory kinds in one call: the host ones are packed in scratch and copied back, and every
    rendition holds the bytes an all-host call gives"""
    import torch
    sizes = [(32, 16), (48, 24), (16, 8), (64, 32)]
    rng = np.random.default_rng(9)
    y, uv = rng.integers(0, 256, (32, 64), np.uint8), rng.integers(0, 256, (16, 64), np.uint8)
    src = F.InputFrame()
    src.input_id, src.format, src.width, src.height, src.mem_kind = b"src", F.FRAME_NV12, 64, 32, F.MEM_HOST
    src.planes[0], src.planes[1] = y.ctypes.data, uv.ctypes.data

    def run(kinds):
        outs, planes = (F.Rendition * len(sizes))(), []
        for i, ((w, h), mem) in enumerate(zip(sizes, kinds)):
            py, puv = (np.full((h, w + 16), SENTINEL, np.uint8), np.full((h // 2, w + 16), SENTINEL, np.uint8))
            if mem == F.MEM_DEVICE:
                py, puv = torch.from_numpy(py).to("cuda:0"), torch.from_numpy(puv).to("cuda:0")
                outs[i].planes[0], outs[i].planes[1] = py.data_ptr(), puv.data_ptr()
            else:
                outs[i].planes[0], outs[i].planes[1] = py.ctypes.data, puv.ctypes.data
            outs[i].width, outs[i].height, outs[i].scaling, outs[i].mem_kind = w, h, F.SCALE_BILINEAR, mem
            outs[i].pitch[0], outs[i].pitch[1] = w + 16, w + 16
            planes.append((py, puv))
        torch.cuda.synchronize()
        s0 = r.stats()
        assert r._lib.smr_transcode_resize(r._h, C.byref(src), outs, len(sizes)) == F.SMR_OK, r._err()
        s1 = r.stats()
        host_bytes = sum(w * h * 3 // 2 for (w, h), mem in zip(sizes, kinds) if mem == F.MEM_HOST)
        assert s1["d2h_bytes"] - s0["d2h_bytes"] == host_bytes
        assert s1["h2d_bytes"] - s0["h2d_bytes"] == 64 * 32 * 3 // 2
        got = []
        for (py, puv), (w, h) in zip(planes, sizes):
            py, puv = (py.cpu().numpy(), puv.cpu().numpy()) if isinstance(py, torch.Tensor) else (py, puv)
            assert (py[:, w:] == SENTINEL).all() and (puv[:, w:] == SENTINEL).all()
            got.append((py[:, :w].copy(), puv[:, :w].copy()))
        return got

    H, D = F.MEM_HOST, F.MEM_DEVICE
    want = run([H, H, H, H])
    for kinds in ([D, H, D, H], [H, D, H, D], [D, D, D, D]):
        got = run(kinds)
        for i, ((a, b), (c, d)) in enumerate(zip(want, got)):
            assert np.array_equal(a, c) and np.array_equal(b, d), (kinds, i)
