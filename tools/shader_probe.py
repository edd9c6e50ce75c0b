#!/usr/bin/env python
"""What a shader node costs: a 4K colour grade over one 4K NV12 input, and the same grade over a nested View of sixteen
4K NV12 inputs.

Both scenes have the Shader as their root and a 4K NV12 output, so the shader's node texture goes through the stand-alone
output kernel only.  In the second the shader's child is a 3840 x 2160 View of four rows of four inputs, a layout node of
its own: each input, in a Rescaler, is resampled 4:1 and composited into the node's frame-arena texture, which the shader
then samples.  Reports ms per tick from CUDA events and the time per tick of each kernel class from smr_set_profiling,
with the card's name and power limit read in the same run.  GPU only: without a device it fails.

  python tools/shader_probe.py [--ticks 200] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import smelter_b200 as s  # noqa: E402
from smelter_b200 import _ffi as F  # noqa: E402

FRAME_NS = 33_333_333
OW, OH = 3840, 2160

GRADE = r'''
__device__ float4 smr_fragment(smr_fragment_in in, const smr_base_params &base, const void *params, const smr_textures &tex) {
    const float *g = (const float *)params;
    float4 c = tex.sample(0, in.tex_coords);
    return make_float4(fminf(fmaf(c.x, g[0], g[3] * c.w), c.w), fminf(fmaf(c.y, g[1], g[3] * c.w), c.w),
                       fminf(fmaf(c.z, g[2], g[3] * c.w), c.w), c.w);
}
'''


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"name": q[0], "power_limit": q[1], "max_sm_clock": q[2]}


class Handle:
    def __init__(self, torch, dev, n_inputs, iw, ih, nested, param):
        self.r = r = s.Renderer(s.RendererOptions())
        self.ids = [f"input_{i + 1}".encode() for i in range(n_inputs)]
        for i in self.ids:
            r.register_input(i.decode())
        r.register_shader("probe", GRADE, s.ShaderParamType("list", item=s.ShaderParamType("f32"), length=4))
        kids = [s.InputStreamComponent(input_id=i.decode()) for i in self.ids]
        if nested:   # four rows of four inputs, each fitted into its 960 x 540 cell; the View a layout node of its own
            cells = [s.RescalerComponent(child=k) for k in kids]
            rows = [s.ViewComponent(children=cells[4 * k:4 * k + 4]) for k in range(n_inputs // 4)]
            kids = [s.ViewComponent(position=s.Position.Static(width=float(OW), height=float(OH)),
                                    direction=s.ViewChildrenDirection.Column, children=rows)]
        r.update_scene("output_1", s.Resolution(OW, OH), s.OutputFrameFormat.Nv12WgpuTexture,
                       s.ShaderComponent(shader_id="probe", shader_param=param, width=OW, height=OH, children=kids))
        self.planes = [bench.synth_planes_torch(torch, dev, iw, ih, 0x5EED0000 + i) for i in range(n_inputs)]
        self.inp = (F.InputFrame * n_inputs)()
        for i, (y, uv) in enumerate(self.planes):
            a = self.inp[i]
            a.input_id, a.format, a.width, a.height, a.mem_kind = self.ids[i], F.FRAME_NV12, iw, ih, F.MEM_DEVICE
            a.planes[0], a.planes[1] = y.data_ptr(), uv.data_ptr()
        self.out_y = torch.empty((OH, OW), dtype=torch.uint8, device=dev)
        self.out_uv = torch.empty((OH // 2, OW // 2, 2), dtype=torch.uint8, device=dev)
        self.out = (F.OutputFrame * 1)()
        self.out[0].output_id, self.out[0].mem_kind = b"output_1", F.MEM_DEVICE
        self.out[0].planes[0], self.out[0].planes[1] = self.out_y.data_ptr(), self.out_uv.data_ptr()
        self.stream = torch.cuda.ExternalStream(r.cuda_stream(), device=dev)
        self.n, self.k = n_inputs, 0

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
        raise SystemExit("shader_probe needs a CUDA device: it measures, and a CPU run measures nothing")
    dev = torch.device("cuda:0")
    grade = s.ShaderParam.list([s.ShaderParam.f32(v) for v in (1.25, 0.75, 1.0, 0.0625)])
    result = {"card": card(), "node": [OW, OH], "runs": []}
    for name, n, nested in (("grade_4k_over_one_4k_nv12", 1, False), ("grade_4k_over_a_view_of_16_4k_nv12", 16, True)):
        h = Handle(torch, dev, n, 3840, 2160, nested, grade)
        h.ticks(40)     # tables, arenas, clocks
        ms = [h.timed(torch, args.ticks) for _ in range(args.rounds)]
        h.r.set_profiling(True)
        h.ticks(args.ticks)
        kt = h.r.kernel_times()
        total, launches = kt["shader"]
        result["runs"].append({"scene": name, "ms_per_tick": ms, "shader_launches": launches,
                               "shader_ms_per_launch": total / max(1, launches),
                               "ms_per_tick_by_class": {k: v[0] / args.ticks for k, v in kt.items() if v[1]}})
        del h
    print(json.dumps(result))


if __name__ == "__main__":
    main()
