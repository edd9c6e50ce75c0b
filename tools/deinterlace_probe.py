"""Times k_deinterlace inside smr_render on two interlaced workloads, motion-adaptive, a new frame every tick:

  * 16 x 1920x1080 UYVY inputs in cfg3's scene shape (4 x 4 tiles of a 3840x2160 planar 4:2:0 output);
  * 4 x 1920x1080 planar 4:2:0 inputs in 2 x 2 tiles of a 1920x1080 output.

Device inputs and outputs, so the tick is on the GPU's clock alone.  Times are the library's own CUDA events around the
launch (smr_set_profiling, kernel class "deinterlace"): TICKS ticks per round, three rounds with the cases alternated.
Bytes per tick are what motion-adaptive moves in steady state: the current frame and the history read, the deinterlaced
planes and the next history written (4 x the frame's bytes per input); the rate is set against the H100 SXM data sheet's
3.35 TB/s HBM3 figure (a data-sheet number, not a measured peak).  The card's name and power limit are printed from the
same run.

    python tools/deinterlace_probe.py [--ticks 200] [--rounds 3]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import smelter_b200 as s  # noqa: E402
from smelter_b200 import _ffi as F  # noqa: E402
from smelter_b200.renderer import plane_shapes  # noqa: E402

DATASHEET_HBM_GBS = 3350.0
# (name, inputs, frame format, output size)
CASES = [("16 x 1080i UYVY -> 3840x2160 tiles", 16, F.FRAME_UYVY422, (3840, 2160)),
         ("4 x 1080i YUV420P -> 1920x1080 tiles", 4, F.FRAME_PLANAR_YUV420, (1920, 1080))]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    rng = np.random.default_rng(0)
    cases = []
    for name, n, fmt, (ow, oh) in CASES:
        r = s.Renderer()
        ids = [f"in{i}" for i in range(n)]
        for i in ids:
            r.register_input(i)
            r.set_input_deinterlace(i, s.DeinterlaceMode.MotionAdaptive, s.FieldOrder.TopFirst, 10)
        r.update_scene("out", s.Resolution(ow, oh), s.OutputFrameFormat.PlanarYuv420Bytes,
                       s.TilesComponent(children=[s.InputStreamComponent(input_id=i) for i in ids]))
        shapes = plane_shapes(fmt, 1920, 1080)
        frame_bytes = sum(rows * rb for rows, rb in shapes)
        keep = []
        # two random frame sets alternated: every tick a new pts (the kernel's work does not depend on how much moves)
        sets = []
        for k in range(2):
            arr = (F.InputFrame * n)()
            for j, i in enumerate(ids):
                f = arr[j]
                f.input_id, f.format, f.width, f.height, f.mem_kind = i.encode(), fmt, 1920, 1080, F.MEM_DEVICE
                for p, (rows, rb) in enumerate(shapes):
                    buf = torch.from_numpy(rng.integers(0, 256, (rows, rb), np.uint8)).to("cuda:0")
                    keep.append(buf)
                    f.planes[p] = buf.data_ptr()
            sets.append(arr)
        out = (F.OutputFrame * 1)()
        out[0].output_id, out[0].mem_kind = b"out", F.MEM_DEVICE
        dst = torch.empty(ow * oh * 3 // 2, dtype=torch.uint8, device="cuda:0")
        out[0].planes[0], out[0].planes[1], out[0].planes[2] = dst.data_ptr(), dst.data_ptr() + ow * oh, dst.data_ptr() + ow * oh * 5 // 4
        keep += [out, dst]
        cases.append({"name": name, "r": r, "n": n, "sets": sets, "out": out, "keep": keep, "pts": 0,
                      "bytes": 4 * n * frame_bytes, "ms": [], "tick_ms": []})
    torch.cuda.synchronize()

    def run(c, ticks):
        for _ in range(ticks):
            c["pts"] += 20_000_000
            arr = c["sets"][(c["pts"] // 20_000_000) % 2]
            for j in range(c["n"]):
                arr[j].pts_ns = c["pts"]
            c["r"].render_raw(c["pts"], arr, c["n"], c["out"], 1)

    for c in cases:   # warm-up: module load, arenas, weight tables, the history
        run(c, 20)
        c["r"].set_profiling(True)
    for _ in range(args.rounds):
        for c in cases:
            times0 = c["r"].kernel_times()
            t0, n0 = times0["deinterlace"]
            all0 = sum(t for t, _ in times0.values())
            run(c, args.ticks)
            times1 = c["r"].kernel_times()
            t1, n1 = times1["deinterlace"]
            assert n1 - n0 == args.ticks
            c["ms"].append((t1 - t0) / args.ticks)
            c["tick_ms"].append((sum(t for t, _ in times1.values()) - all0) / args.ticks)
    print("card (name, power limit, max SM clock):", card())
    for c in cases:
        best = min(c["ms"])
        gbs = c["bytes"] / (best * 1e-3) / 1e9
        print(json.dumps({"case": c["name"], "deinterlace_ms_per_tick_rounds": [round(m, 4) for m in c["ms"]],
                          "all_kernels_ms_per_tick_rounds": [round(m, 4) for m in c["tick_ms"]],
                          "bytes_per_tick": c["bytes"], "GB_per_s_best_round": round(gbs, 1),
                          "fraction_of_datasheet_3350_GBs": round(gbs / DATASHEET_HBM_GBS, 3)}))
        c["r"].set_profiling(False)
        c["r"].close()


if __name__ == "__main__":
    main()
