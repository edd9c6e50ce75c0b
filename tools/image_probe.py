#!/usr/bin/env python
"""What animated Image nodes cost per tick on top of bench.py's cfg3 scene (16 x 4K NV12 -> 4K NV12, Tiles 4 x 4).

N in {1, 16} animated 512 x 512 images are shown at 384 x 384 over the tiles; their frame changes at every tick, so every
tick draws every node (the worst case: a tick that keeps its frame launches nothing).  Device-resident inputs and outputs.
Reports ms per tick from CUDA events for the scene without and with the images, alternating between the two handles in
blocks, and the k_image time per launch from smr_set_profiling in a run of its own (profiling serialises the read-back).
Prints the card's name and power limit read in the same run.  GPU only: without a device it fails.

  python tools/image_probe.py [--ticks 200] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import smelter_b200 as s  # noqa: E402
from smelter_b200 import _ffi as F  # noqa: E402

FRAME_NS = 33_333_333
FRAMES = 4


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"name": q[0], "power_limit": q[1], "max_sm_clock": q[2]}


class Handle:
    def __init__(self, torch, dev, wl, n_images):
        W, H, n, iw, ih = wl["W"], wl["H"], wl["n"], wl["iw"], wl["ih"]
        self.r = r = s.Renderer(s.RendererOptions(rendering_mode=wl["mode"]))
        self.ids = [f"input_{i + 1}".encode() for i in range(n)]
        for i in self.ids:
            r.register_input(i.decode())
        rng = np.random.default_rng(7)
        kids = [wl["scene"]]
        for k in range(n_images):
            r.register_image(f"image_{k}", [rng.integers(0, 256, (512, 512, 4), dtype=np.uint8) for _ in range(FRAMES)],
                             [FRAME_NS] * FRAMES)      # one frame per tick
            pos = s.Position.Absolute(width=384.0, height=384.0, left=64.0 + 960.0 * (k % 4), top=48.0 + 540.0 * (k // 4))
            kids.append(s.ViewComponent(position=pos, children=[s.ImageComponent(image_id=f"image_{k}", width=384.0, height=384.0)]))
        scene = s.ViewComponent(children=kids) if n_images else wl["scene"]
        r.update_scene("output_1", s.Resolution(W, H), s.OutputFrameFormat.Nv12WgpuTexture, scene)
        self.planes = [bench.synth_planes_torch(torch, dev, iw, ih, 0x5EED0000 + i) for i in range(n)]
        self.inp = (F.InputFrame * n)()
        for i, (y, uv) in enumerate(self.planes):
            a = self.inp[i]
            a.input_id, a.format, a.width, a.height, a.mem_kind = self.ids[i], F.FRAME_NV12, iw, ih, F.MEM_DEVICE
            a.planes[0], a.planes[1] = y.data_ptr(), uv.data_ptr()
        self.out_y = torch.empty((H, W), dtype=torch.uint8, device=dev)
        self.out_uv = torch.empty((H // 2, W // 2, 2), dtype=torch.uint8, device=dev)
        self.out = (F.OutputFrame * 1)()
        self.out[0].output_id, self.out[0].mem_kind = b"output_1", F.MEM_DEVICE
        self.out[0].planes[0], self.out[0].planes[1] = self.out_y.data_ptr(), self.out_uv.data_ptr()
        self.stream = torch.cuda.ExternalStream(r.cuda_stream(), device=dev)
        self.k, self.n = 0, n

    def ticks(self, count):
        for _ in range(count):
            for a in self.inp:
                a.pts_ns = self.k * FRAME_NS
            self.r.render_raw(self.k * FRAME_NS, self.inp, self.n, self.out, 1, wait=False)
            self.k += 1
            if self.k % 2 == 0:
                self.r.wait()
        while self.k % 2:
            self.ticks(1)

    def timed(self, torch, count):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(self.stream)
        self.ticks(count)
        e1.record(self.stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / count


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("image_probe needs a CUDA device: it measures, and a CPU run measures nothing")
    dev = torch.device("cuda:0")
    wl = bench.workload("cfg3")
    result = {"card": card(), "scene": wl["desc"], "ticks_per_block": args.ticks, "runs": []}
    for n_images in (1, 16):
        plain, images = Handle(torch, dev, wl, 0), Handle(torch, dev, wl, n_images)
        for h in (plain, images):
            h.ticks(40)     # tables, descriptors, arenas, clocks
        ms = {"without": [], "with": []}
        for _ in range(args.rounds):
            ms["without"].append(plain.timed(torch, args.ticks))
            ms["with"].append(images.timed(torch, args.ticks))
        images.r.set_profiling(True)
        images.ticks(args.ticks)
        total, launches = images.r.kernel_times()["image"]
        result["runs"].append({"images": n_images, "ms_per_tick_without": ms["without"], "ms_per_tick_with": ms["with"],
                               "median_delta_ms": float(np.median(ms["with"]) - np.median(ms["without"])),
                               "k_image_launches": launches, "k_image_ms_per_launch": total / max(1, launches)})
        del plain, images
    print(json.dumps(result))


if __name__ == "__main__":
    main()
