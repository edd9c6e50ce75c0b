#!/usr/bin/env python
"""What a WGSL shader node costs: the reference's layout_planes.wgsl (four children placed in quarters by its vertex
stage) next to a CUDA shader doing the same work (each plane draws its child into its quarter), at 640 x 360 and
3840 x 2160, over four NV12 inputs of the node's size.

The Shader is the scene root with an NV12 output of the node's size.  Reports the shader kernel's time per launch from
smr_set_profiling (CUDA events), alternating the WGSL and CUDA handles round by round, with the card's name and power
limit read in the same run.  GPU only: without a device it fails.

  python tools/wgsl_probe.py [--ticks 200] [--rounds 3]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import smelter_b200 as s  # noqa: E402
from smelter_b200 import _ffi as F  # noqa: E402
from tools.shader_probe import FRAME_NS, card  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# plane p draws child p into quarter p (0 top-left, 1 top-right, 2 bottom-left, 3 bottom-right), as layout_planes.wgsl
QUARTERS = r'''
__device__ float4 smr_fragment(smr_fragment_in in, const smr_base_params &base, const void *params, const smr_textures &tex) {
    const int p = base.plane_id;
    const float qx = (float)(p & 1) * 0.5f, qy = (float)(p >> 1) * 0.5f;
    const float u = (in.tex_coords.x - qx) * 2.0f, v = (in.tex_coords.y - qy) * 2.0f;
    if (u < 0.0f || u >= 1.0f || v < 0.0f || v >= 1.0f) return make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    return tex.sample((unsigned)p, make_float2(u, v));
}
'''


class Handle:
    def __init__(self, torch, dev, W, H, use_wgsl):
        self.r = r = s.Renderer(s.RendererOptions())
        self.ids = [f"input_{i + 1}".encode() for i in range(4)]
        for i in self.ids:
            r.register_input(i.decode())
        if use_wgsl:
            with open(os.path.join(ROOT, "tests", "golden", "wgsl", "layout_planes.wgsl")) as f:
                r.register_wgsl_shader("probe", f.read())
        else:
            r.register_shader("probe", QUARTERS)
        kids = [s.InputStreamComponent(input_id=i.decode()) for i in self.ids]
        r.update_scene("output_1", s.Resolution(W, H), s.OutputFrameFormat.Nv12WgpuTexture,
                       s.ShaderComponent(shader_id="probe", width=W, height=H, children=kids))
        self.planes = [bench.synth_planes_torch(torch, dev, W, H, 0x5EED0000 + i) for i in range(4)]
        self.inp = (F.InputFrame * 4)()
        for i, (y, uv) in enumerate(self.planes):
            a = self.inp[i]
            a.input_id, a.format, a.width, a.height, a.mem_kind = self.ids[i], F.FRAME_NV12, W, H, F.MEM_DEVICE
            a.planes[0], a.planes[1] = y.data_ptr(), uv.data_ptr()
        self.out_y = torch.empty((H, W), dtype=torch.uint8, device=dev)
        self.out_uv = torch.empty((H // 2, W // 2, 2), dtype=torch.uint8, device=dev)
        self.out = (F.OutputFrame * 1)()
        self.out[0].output_id, self.out[0].mem_kind = b"output_1", F.MEM_DEVICE
        self.out[0].planes[0], self.out[0].planes[1] = self.out_y.data_ptr(), self.out_uv.data_ptr()
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
        self.r.wait()

    def shader_ms(self, count):
        self.r.set_profiling(True)
        self.ticks(count)
        total, launches = self.r.kernel_times()["shader"]
        self.r.set_profiling(False)
        return total / max(1, launches)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("wgsl_probe needs a CUDA device: it measures, and a CPU run measures nothing")
    dev = torch.device("cuda:0")
    result = {"card": card(), "runs": []}
    for W, H in ((640, 360), (3840, 2160)):
        hs = {"wgsl_layout_planes": Handle(torch, dev, W, H, True), "cuda_quarters": Handle(torch, dev, W, H, False)}
        for h in hs.values():
            h.ticks(40)
        ms = {k: [] for k in hs}
        for _ in range(args.rounds):
            for k, h in hs.items():
                ms[k].append(h.shader_ms(args.ticks))
        result["runs"].append({"node": [W, H], "shader_ms_per_launch": ms})
        del hs
    print(json.dumps(result))


if __name__ == "__main__":
    main()
