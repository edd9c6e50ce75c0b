"""Times gpu-video's frame converters: smr_video_nv12_to_rgba (k_video_nv12_to_rgba) at 3840x2160 and 1920x1080 at the
source size and 1920x1080 -> 3840x2160, and smr_video_rgba_to_nv12 (k_output) at 3840x2160.  Device source and device
target, so only the kernel is on the GPU's clock.

Times are the library's own CUDA events around the launch (smr_set_profiling, kernel classes "video_convert" and
"output"): CALLS calls per round, three rounds with the cases alternated.  Bytes moved per call are the source read once
plus the target written; the rate is set against the H100 SXM data sheet's 3.35 TB/s HBM3 figure (a data-sheet number,
not a measured peak).  The card's name and power limit are printed from the same run.

    python tools/video_convert_probe.py [--calls 200] [--rounds 3]
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

DATASHEET_HBM_GBS = 3350.0
BT709_LIMITED = F.VideoColor(F.COLOR_SPACE_BT709, F.COLOR_RANGE_LIMITED)
UNSPECIFIED_LIMITED = F.VideoColor(F.COLOR_SPACE_UNSPECIFIED, F.COLOR_RANGE_LIMITED)
# (name, direction, source size, target size)
CASES = [("nv12_to_rgba 3840x2160", "to_rgba", (3840, 2160), (3840, 2160)),
         ("nv12_to_rgba 1920x1080", "to_rgba", (1920, 1080), (1920, 1080)),
         ("nv12_to_rgba 1920x1080 -> 3840x2160", "to_rgba", (1920, 1080), (3840, 2160)),
         ("rgba_to_nv12 3840x2160", "to_nv12", (3840, 2160), (3840, 2160))]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    r = s.Renderer()
    rng = np.random.default_rng(0)
    cases = []
    for name, direction, (w, h), (ow, oh) in CASES:
        src = F.InputFrame()
        src.input_id, src.width, src.height, src.mem_kind = b"src", w, h, F.MEM_DEVICE
        if direction == "to_rgba":
            buf = torch.from_numpy(rng.integers(0, 256, (h * 3 // 2, w), np.uint8)).to("cuda:0")
            src.format = F.FRAME_NV12
            src.planes[0], src.planes[1] = buf.data_ptr(), buf.data_ptr() + w * h
            dst = torch.empty((oh, ow * 4), dtype=torch.uint8, device="cuda:0")
            moved, cls = w * h * 3 // 2 + ow * oh * 4, "video_convert"
        else:
            buf = torch.from_numpy(rng.integers(0, 256, (h, w * 4), np.uint8)).to("cuda:0")
            src.format = F.FRAME_RGBA8
            src.planes[0] = buf.data_ptr()
            dst = torch.empty((oh * 3 // 2, ow), dtype=torch.uint8, device="cuda:0")
            moved, cls = w * h * 4 + ow * oh * 3 // 2, "output"
        planes = (C.c_void_p * 2)(dst.data_ptr(), dst.data_ptr() + ow * oh)
        cases.append({"name": name, "dir": direction, "src": src, "dst": dst, "planes": planes, "ow": ow, "oh": oh,
                      "keep": [buf, dst], "bytes": moved, "cls": cls, "ms": []})
    torch.cuda.synchronize()

    def run(c, calls):
        for _ in range(calls):
            if c["dir"] == "to_rgba":
                st = r._lib.smr_video_nv12_to_rgba(r._h, BT709_LIMITED, C.byref(c["src"]), UNSPECIFIED_LIMITED, c["ow"],
                                                   c["oh"], c["dst"].data_ptr(), 0, F.MEM_DEVICE)
            else:
                st = r._lib.smr_video_rgba_to_nv12(r._h, BT709_LIMITED, C.byref(c["src"]), c["ow"], c["oh"], c["planes"],
                                                   None, F.MEM_DEVICE)
            if st != F.SMR_OK:
                raise RuntimeError(f"{c['name']}: status {st}: {r._err()}")

    for c in cases:   # warm-up: module load
        run(c, 10)
    r.set_profiling(True)
    for _ in range(args.rounds):
        for c in cases:
            t0, n0 = r.kernel_times()[c["cls"]]
            run(c, args.calls)
            t1, n1 = r.kernel_times()[c["cls"]]
            assert n1 - n0 == args.calls
            c["ms"].append((t1 - t0) / args.calls)
    r.set_profiling(False)
    print("card (name, power limit, max SM clock):", card())
    for c in cases:
        best = min(c["ms"])
        gbs = c["bytes"] / (best * 1e-3) / 1e9
        print(json.dumps({"case": c["name"], "ms_per_launch_rounds": [round(m, 4) for m in c["ms"]],
                          "bytes_per_call": c["bytes"], "GB_per_s_best_round": round(gbs, 1),
                          "fraction_of_datasheet_3350_GBs": round(gbs / DATASHEET_HBM_GBS, 3)}))
    r.close()


if __name__ == "__main__":
    main()
