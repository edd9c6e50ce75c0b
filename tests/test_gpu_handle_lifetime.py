"""The device resources a renderer handle owns are released with it, and the caches of device tables it keeps stay valid
for the tick that uses them.

- Lifetime: cycles of create, use every resource kind (streams, events, weight and lane tables, the web-frame pool, a
  shader module, scratch buffers of the blocking calls, peer pools) and destroy leave the device's free memory where it
  was.  The library runs on the runtime's primary context, the one `torch.cuda.mem_get_info` reports on.
- Eviction mid-tick: the weight and lane-table caches are bounded at 4096 entries.  When a tick crosses the bound, the
  entries that tick has already taken stay: the tick's output equals the same tick rendered on a fresh handle.
"""
import numpy as np
import pytest

import smelter_b200 as s
from smelter_b200 import _ffi as F
from tests.parity import OUTPUT_ID
from tests.test_gpu_fused_variants import RGBA, Job, make_frame, render

MiB = 1 << 20
CACHE_BOUND = 4096   # Renderer::bound_cache

GRADIENT = r'''
__device__ float4 smr_fragment(smr_fragment_in in, const smr_base_params &base, const void *params, const smr_textures &tex) {
    return make_float4(in.tex_coords.x, 0.5f, in.tex_coords.y, 1.0f);
}
'''

# one tick of each fused kernel and one generic resample (vertical ratio a hair larger: vertical first, no fused kernel)
LIFETIME_JOBS = [Job("input_1", (0.0, 0.0, 640.0, 360.0), (320, 180)),    # k_resample_tma3, 2:1
                 Job("input_2", (0.0, 0.0, 480.0, 270.0), (320, 180)),    # k_resample_tma0, 1.5:1
                 Job("input_1", (0.0, 0.0, 640.0, 360.0), (321, 181)),    # k_resample_fused_int: odd width
                 Job("input_3", (0.0, 0.0, 160.0, 90.0), (80, 44))]       # generic passes
LIFETIME_FRAMES = {"input_1": ("yuv", 640, 360), "input_2": ("yuv", 480, 270), "input_3": ("yuv", 160, 90)}
# A second output of 1024 children, each 8192 x 2 at its own ratio in (1.05, 1.45) of one 12288 x 16 NV12 input: every
# child takes a horizontal weight table of 8 to 10 taps x 8192 columns (about 290 MiB in all) and a lane table of 4 KiB
# (4 MiB in all).  A cycle that leaked its weight tables would lose about 290 MiB, its lane tables 4 MiB (40 MiB after ten
# cycles), its web-frame pool the 7.9 MiB frame it keeps, its second peer pool 64 MiB.
WIDE_N, WIDE_W, WIDE_H, WIDE_SRC = 1024, 8192, 2, (12288, 16)
WEB_W, WEB_H = 1920, 1080
PEER_POOL_BYTES = 64 * MiB
TOLERANCE = 4 * MiB


def wide_layouts():
    ratios = (1.05 + (np.arange(WIDE_N) + 0.5) / WIDE_N * 0.4).astype(np.float32)
    assert len(np.unique(ratios)) == WIDE_N
    ls = []
    for k, ratio in enumerate(ratios):
        l = F.RenderLayout()
        l.type, l.child_index, l.left, l.top = 0, 0, 0.0, float(k * WIDE_H)
        l.width, l.height = float(WIDE_W), float(WIDE_H)
        l.crop_left, l.crop_top, l.crop_width, l.crop_height = 0.0, 0.0, float(ratio * WIDE_W), float(ratio * WIDE_H)
        ls.append(l)
    return ls


def use_every_resource(frames, nv12, wide, bgra):
    r = s.Renderer(s.RendererOptions(max_layouts_count=WIDE_N))
    r.set_profiling(True)
    r.register_shader("gradient", GRADIENT)
    r.register_web_renderer("web", WEB_W, WEB_H)
    r.set_web_frame("web", bgra)
    for _ in range(3):
        render(r, LIFETIME_JOBS, frames)
    fused = sorted(j["kernel"] for j in r.debug_fused_jobs())
    assert fused == ["ldg", "tma_any", "tma_int"], fused
    stages, _ = r.debug_resample_stages()
    assert stages, "no generic resample pass"
    r.register_input("wide")
    render_tick(r, wide_layouts(), wide, [], output_id="wide", input_id="wide", width=WIDE_W)
    fused = r.debug_fused_jobs()
    assert len(fused) == WIDE_N and all(j["kernel"] == "tma_any" for j in fused)
    r.render_text(40, 12, s.RGBAColor(10, 20, 30, 200), np.zeros(0, F.GLYPH_DTYPE))
    r.transcode_resize(nv12, [(64, 36, s.ScalingAlgorithm.Lanczos3)])
    first, _ = r.peer_pool_alloc(PEER_POOL_BYTES)
    r.peer_pool_free(first)
    r.peer_pool_alloc(PEER_POOL_BYTES)   # left to the handle's destruction
    r.close()


@pytest.mark.gpu
def test_destroyed_handles_release_their_device_memory():
    import torch
    torch.cuda.init()
    frames = {i: make_frame(fmt, "smooth", 40 + k, w, h) for k, (i, (fmt, w, h)) in enumerate(LIFETIME_FRAMES.items())}
    nv12 = make_frame("nv12", "smooth", 50, 128, 72)
    wide = make_frame("nv12", "smooth", 51, *WIDE_SRC)
    bgra = np.random.default_rng(52).integers(0, 256, (WEB_H, WEB_W, 4), dtype=np.uint8)
    use_every_resource(frames, nv12, wide, bgra)   # loads the library's modules, which stay loaded
    free0 = torch.cuda.mem_get_info()[0]
    readings = []
    for _ in range(10):
        use_every_resource(frames, nv12, wide, bgra)
        readings.append(torch.cuda.mem_get_info()[0])
    lost = [(free0 - f) / MiB for f in readings]
    print("MiB of free device memory lost after each cycle:", lost)
    assert free0 - readings[-1] <= TOLERANCE, f"MiB of free device memory lost after each cycle: {lost}"


# ------------------------------------------------------------------------------------------------
# eviction mid-tick
# ------------------------------------------------------------------------------------------------
SRC_W, SRC_H = 128, 72           # one small NV12 input
CHILD_W, CHILD_H = 32, 16        # every child: two weight tables (widths differ) and one lane table
GRID_COLS = 32
TICKS = (512, 1024, 1024, 1024, 1024)   # layouts per tick, each at a ratio no other tick uses


def ratios():
    """distinct f32 ratios in (1, 2.9), none an integer, one per layout of every tick, in tick order"""
    n = sum(TICKS)
    r = (1.0 + (np.arange(n) + 0.5) / n * 1.9).astype(np.float32)
    assert len(np.unique(r)) == n and not np.any(r == np.round(r))
    out, k = [], 0
    for t in TICKS:
        out.append(r[k:k + t])
        k += t
    return out


def tick_layouts(rs):
    ls = []
    for k, ratio in enumerate(rs):
        l = F.RenderLayout()
        l.type, l.child_index = 0, 0
        l.left, l.top = float(k % GRID_COLS * CHILD_W), float(k // GRID_COLS * CHILD_H)
        l.width, l.height = float(CHILD_W), float(CHILD_H)
        # the same ratio on both axes (horizontal pass first); crops stay inside the source
        l.crop_left, l.crop_top = 0.0, 0.0
        l.crop_width, l.crop_height = float(np.float32(ratio) * CHILD_W), float(np.float32(ratio) * CHILD_H)
        ls.append(l)
    return ls


def render_tick(r, layouts, frame, keep, output_id=OUTPUT_ID, input_id="input_1", width=GRID_COLS * CHILD_W):
    """one tick of the layouts (one NV12 input, set_layouts) on r: -> the RGBA output"""
    W, H = width, int(max(l.top + l.height for l in layouts))
    r.set_layouts(output_id, s.Resolution(W, H), RGBA, (W, H), [input_id], layouts)
    arr = (F.InputFrame * 1)()
    y, uv = (np.ascontiguousarray(p).reshape(p.shape[0], -1) for p in frame.data.planes)
    keep += [y, uv]
    arr[0].input_id, arr[0].format = input_id.encode(), F.FRAME_NV12
    arr[0].width, arr[0].height = frame.resolution.width, frame.resolution.height
    arr[0].pts_ns, arr[0].mem_kind = 0, F.MEM_HOST
    arr[0].planes[0], arr[0].planes[1] = y.ctypes.data, uv.ctypes.data
    out = np.zeros(W * H * 4, np.uint8)
    o = (F.OutputFrame * 1)()
    o[0].output_id, o[0].mem_kind, o[0].planes[0] = output_id.encode(), F.MEM_HOST, out.ctypes.data
    r.render_raw(0, arr, 1, o, 1)
    return out.reshape(H, W, 4)


def first_eviction(tables_per_layout):
    """(tick, layout) whose new table finds the cache past its bound, when every layout of every tick takes new tables"""
    n = 0
    for t, count in enumerate(TICKS):
        for i in range(count):
            for _ in range(tables_per_layout):
                if n > CACHE_BOUND:
                    return t, i
                n += 1
    return None


@pytest.mark.gpu
def test_cache_eviction_spares_the_entries_of_the_tick():
    # a lane table (one per layout) finds its cache past the bound at layout 513 of the last tick, a weight table (two
    # per layout) at layout 512 of the third: after hundreds of layouts of the same tick have taken theirs
    assert first_eviction(1) == (4, 513) and first_eviction(2) == (2, 512)
    frame = make_frame("nv12", "smooth", 77, SRC_W, SRC_H)
    per_tick = [tick_layouts(rs) for rs in ratios()]
    keep = []
    r = s.Renderer(s.RendererOptions(max_layouts_count=1024))
    r.register_input("input_1")
    for t, layouts in enumerate(per_tick):
        got = render_tick(r, layouts, frame, keep)
        fused = r.debug_fused_jobs()
        assert len(fused) == len(layouts) and all(j["kernel"] == "tma_any" for j in fused), \
            (t, sorted({j["kernel"] for j in fused}))
        fresh = s.Renderer(s.RendererOptions(max_layouts_count=1024))
        fresh.register_input("input_1")
        exp = render_tick(fresh, layouts, frame, keep)
        fresh.close()
        assert np.array_equal(got, exp), f"tick {t}: {int(np.count_nonzero(got != exp))} bytes differ from a fresh handle's"
    r.close()
