"""Times a cfg3-shaped tick with every input BT.601 against the same tick at BT.709 (smr_set_input_color).

cfg3's scene: 16 x 1920x1080 inputs (planar 4:2:0 and NV12 alternately) in 4 x 4 tiles of a 1920x1080 planar 4:2:0 output,
so every child runs k_resample_tma3 at 4:1 with direct tiles.  The BT.601 tick runs the same kernels with other
immediates, so the expectation is the same time.  Device inputs and outputs, so the tick is on the GPU's clock alone.
Times are the library's own CUDA events around its launches (smr_set_profiling): the sum over kernel classes per tick,
TICKS ticks per round, the two cases alternated for ROUNDS rounds.  The card's name and power limit are printed from the
same run.

    python tools/input_color_probe.py [--ticks 300] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import smelter_b200 as s  # noqa: E402
from smelter_b200 import _ffi as F  # noqa: E402
from smelter_b200.renderer import plane_shapes  # noqa: E402

CASES = [("BT.709 limited", s.YuvMatrix.BT709), ("BT.601 limited", s.YuvMatrix.BT601)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    rng = np.random.default_rng(0)
    n, ow, oh = 16, 1920, 1080
    ids = [f"in{i}" for i in range(n)]
    fmts = [F.FRAME_PLANAR_YUV420 if i % 2 else F.FRAME_NV12 for i in range(n)]
    keep = []
    arr = (F.InputFrame * n)()
    for j, i in enumerate(ids):
        f = arr[j]
        f.input_id, f.format, f.width, f.height, f.mem_kind = i.encode(), fmts[j], 1920, 1080, F.MEM_DEVICE
        for p, (rows, rb) in enumerate(plane_shapes(fmts[j], 1920, 1080)):
            buf = torch.from_numpy(rng.integers(0, 256, (rows, rb), np.uint8)).to("cuda:0")
            keep.append(buf)
            f.planes[p] = buf.data_ptr()
    cases = []
    for name, matrix in CASES:
        r = s.Renderer()
        for i in ids:
            r.register_input(i)
            r.set_input_color(i, matrix, s.YuvRange.Limited)
        r.update_scene("out", s.Resolution(ow, oh), s.OutputFrameFormat.PlanarYuv420Bytes,
                       s.TilesComponent(children=[s.InputStreamComponent(input_id=i) for i in ids]))
        out = (F.OutputFrame * 1)()
        out[0].output_id, out[0].mem_kind = b"out", F.MEM_DEVICE
        dst = torch.empty(ow * oh * 3 // 2, dtype=torch.uint8, device="cuda:0")
        out[0].planes[0], out[0].planes[1], out[0].planes[2] = dst.data_ptr(), dst.data_ptr() + ow * oh, dst.data_ptr() + ow * oh * 5 // 4
        cases.append({"name": name, "r": r, "out": out, "dst": dst, "pts": 0, "tick_ms": [], "fused_ms": []})
    torch.cuda.synchronize()

    def run(c, ticks):
        for _ in range(ticks):
            c["pts"] += 20_000_000
            for j in range(n):
                arr[j].pts_ns = c["pts"]
            c["r"].render_raw(c["pts"], arr, n, c["out"], 1)

    for c in cases:   # warm-up: module load, arenas, weight tables
        run(c, 30)
        c["r"].set_profiling(True)
    for _ in range(args.rounds):
        for c in cases:
            t0 = c["r"].kernel_times()
            run(c, args.ticks)
            t1 = c["r"].kernel_times()
            c["tick_ms"].append((sum(t for t, _ in t1.values()) - sum(t for t, _ in t0.values())) / args.ticks)
            c["fused_ms"].append((t1["resample_fused"][0] - t0["resample_fused"][0]) / args.ticks)
    fused = [j["matrix"] for j in cases[1]["r"].debug_fused_jobs()]
    assert fused and all(m == s.YuvMatrix.BT601 for m in fused), fused
    a, b = cases[0]["dst"].cpu().numpy(), cases[1]["dst"].cpu().numpy()
    print("card (name, power limit, max SM clock):", card())
    for c in cases:
        print(json.dumps({"case": c["name"], "tick_ms_rounds": [round(m, 4) for m in c["tick_ms"]],
                          "resample_fused_ms_rounds": [round(m, 4) for m in c["fused_ms"]],
                          "tick_ms_median": round(float(np.median(c["tick_ms"])), 4)}))
        c["r"].set_profiling(False)
        c["r"].close()
    print(json.dumps({"outputs_differ": bool(not np.array_equal(a, b))}))


if __name__ == "__main__":
    main()
