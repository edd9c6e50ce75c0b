"""Times smr_transcode_resize's kernel (k_transcode) on the two transcoder ladders: 3840x2160 -> 1920x1080 / 1280x720 /
854x480 / 640x360 and 1920x1080 -> 1280x720 / 640x360 / 426x240, each with Lanczos3 and with bilinear.  Device source and
device destinations, so only the kernel is on the GPU's clock.

Times are the library's own CUDA events around the launch (smr_set_profiling, kernel class "transcode"): CALLS calls per
round, three rounds with the four cases alternated.  Bytes moved per call are the NV12 crop read once plus every
rendition written; the rate is set against the H100 SXM data sheet's 3.35 TB/s HBM3 figure (a data-sheet number, not a
measured peak).  The card's name and power limit are printed from the same run.

    python tools/transcode_probe.py [--calls 200] [--rounds 3]
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
LADDERS = {"4k": ((3840, 2160), [(1920, 1080), (1280, 720), (854, 480), (640, 360)]),
           "1080p": ((1920, 1080), [(1280, 720), (640, 360), (426, 240)])}
ALGOS = {"lanczos3": F.SCALE_LANCZOS3, "bilinear": F.SCALE_BILINEAR}


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
    for lname, ((w, h), sizes) in LADDERS.items():
        src_y = torch.from_numpy(rng.integers(0, 256, (h, w), np.uint8)).to("cuda:0")
        src_uv = torch.from_numpy(rng.integers(0, 256, (h // 2, w), np.uint8)).to("cuda:0")
        src = F.InputFrame()
        src.input_id, src.format, src.width, src.height, src.mem_kind = b"src", F.FRAME_NV12, w, h, F.MEM_DEVICE
        src.planes[0], src.planes[1] = src_y.data_ptr(), src_uv.data_ptr()
        for aname, algo in ALGOS.items():
            outs = (F.Rendition * len(sizes))()
            keep = [src_y, src_uv]
            for i, (ow, oh) in enumerate(sizes):
                ty = torch.empty((oh * 3 // 2, ow), dtype=torch.uint8, device="cuda:0")
                keep.append(ty)
                outs[i].width, outs[i].height, outs[i].scaling, outs[i].mem_kind = ow, oh, algo, F.MEM_DEVICE
                outs[i].planes[0], outs[i].planes[1] = ty.data_ptr(), ty.data_ptr() + ow * oh
            moved = w * h * 3 // 2 + sum(ow * oh * 3 // 2 for ow, oh in sizes)
            cases.append({"name": f"{lname}/{aname}", "src": src, "outs": outs, "n": len(sizes), "keep": keep,
                          "bytes": moved, "ms": []})
    torch.cuda.synchronize()

    def run(c, calls):
        for _ in range(calls):
            st = r._lib.smr_transcode_resize(r._h, C.byref(c["src"]), c["outs"], c["n"])
            if st != F.SMR_OK:
                raise RuntimeError(f"{c['name']}: status {st}: {r._err()}")

    for c in cases:   # warm-up: module load, tap tables
        run(c, 10)
    r.set_profiling(True)
    for _ in range(args.rounds):
        for c in cases:
            t0, n0 = r.kernel_times()["transcode"]
            run(c, args.calls)
            t1, n1 = r.kernel_times()["transcode"]
            assert n1 - n0 == args.calls
            c["ms"].append((t1 - t0) / args.calls)
    r.set_profiling(False)
    print("card (name, power limit, max SM clock):", card())
    res = []
    for c in cases:
        best = min(c["ms"])
        gbs = c["bytes"] / (best * 1e-3) / 1e9
        row = {"case": c["name"], "ms_per_launch_rounds": [round(m, 4) for m in c["ms"]], "bytes_per_call": c["bytes"],
               "GB_per_s_best_round": round(gbs, 1), "fraction_of_datasheet_3350_GBs": round(gbs / DATASHEET_HBM_GBS, 3)}
        res.append(row)
        print(json.dumps(row))
    r.close()


if __name__ == "__main__":
    main()
