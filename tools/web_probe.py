#!/usr/bin/env python
"""What k_web costs: one 1920 x 1080 web view node with four 4K NV12 children, drawn every tick.

The page is a seeded translucent BGRA plane set once; the children are four 3840 x 2160 NV12 inputs in device memory, each
shown at a 960 x 540 rect of the page (the quadrants), so every page pixel samples the page and one child in place.  The
scene root is the WebView (a 1080p NV12 output, so the node texture goes through the stand-alone output kernel only).
Reports the k_web time per launch from smr_set_profiling, and ms per tick from CUDA events for both embedding methods.
Prints the card's name and power limit read in the same run.  GPU only: without a device it fails.

  python tools/web_probe.py [--ticks 200] [--rounds 5]
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
PW, PH, IW, IH = 1920, 1080, 3840, 2160


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"name": q[0], "power_limit": q[1], "max_sm_clock": q[2]}


class Handle:
    def __init__(self, torch, dev, embedding):
        self.r = r = s.Renderer(s.RendererOptions())
        self.ids = [f"input_{i + 1}".encode() for i in range(4)]
        for i in self.ids:
            r.register_input(i.decode())
        r.register_web_renderer("page", PW, PH, embedding)
        rng = np.random.default_rng(11)
        page = rng.integers(0, 256, (PH, PW, 4), dtype=np.uint8)
        page[::2, :, 3] = 128
        page[..., :3] = np.minimum(page[..., :3], page[..., 3:4])
        r.set_web_frame("page", page)
        r.set_web_child_rects("page", [(960.0 * (k % 2), 540.0 * (k // 2), 960.0, 540.0) for k in range(4)])
        kids = [s.InputStreamComponent(id=f"c{k}", input_id=self.ids[k].decode()) for k in range(4)]
        r.update_scene("output_1", s.Resolution(PW, PH), s.OutputFrameFormat.Nv12WgpuTexture,
                       s.WebViewComponent(instance_id="page", children=kids))
        self.planes = [bench.synth_planes_torch(torch, dev, IW, IH, 0x5EED0000 + i) for i in range(4)]
        self.inp = (F.InputFrame * 4)()
        for i, (y, uv) in enumerate(self.planes):
            a = self.inp[i]
            a.input_id, a.format, a.width, a.height, a.mem_kind = self.ids[i], F.FRAME_NV12, IW, IH, F.MEM_DEVICE
            a.planes[0], a.planes[1] = y.data_ptr(), uv.data_ptr()
        self.out_y = torch.empty((PH, PW), dtype=torch.uint8, device=dev)
        self.out_uv = torch.empty((PH // 2, PW // 2, 2), dtype=torch.uint8, device=dev)
        self.out = (F.OutputFrame * 1)()
        self.out[0].output_id, self.out[0].mem_kind = b"output_1", F.MEM_DEVICE
        self.out[0].planes[0], self.out[0].planes[1] = self.out_y.data_ptr(), self.out_uv.data_ptr()
        self.stream = torch.cuda.ExternalStream(r.cuda_stream(), device=dev)
        self.k = 0

    def ticks(self, count):
        for _ in range(count):
            for a in self.inp:
                a.pts_ns = self.k * FRAME_NS
            self.r.render_raw(self.k * FRAME_NS, self.inp, 4, self.out, 1, wait=False)
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
        raise SystemExit("web_probe needs a CUDA device: it measures, and a CPU run measures nothing")
    dev = torch.device("cuda:0")
    result = {"card": card(), "page": [PW, PH], "children": "4 x 3840x2160 NV12 at 960x540 each", "runs": []}
    for name, emb in (("over_content", F.WEB_NATIVE_OVER_CONTENT), ("under_content", F.WEB_NATIVE_UNDER_CONTENT)):
        h = Handle(torch, dev, emb)
        h.ticks(40)     # tables, arenas, clocks
        ms = [h.timed(torch, args.ticks) for _ in range(args.rounds)]
        h.r.set_profiling(True)
        h.ticks(args.ticks)
        total, launches = h.r.kernel_times()["web"]
        result["runs"].append({"embedding": name, "ms_per_tick": ms, "k_web_launches": launches,
                               "k_web_ms_per_launch": total / max(1, launches)})
        del h
    print(json.dumps(result))


if __name__ == "__main__":
    main()
