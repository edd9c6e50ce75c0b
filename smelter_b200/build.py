"""Builds libsmelter_b200.so (C-ABI library: C++ host + sm_90a CUDA kernels) in-tree with nvcc.

No torch, no JIT cache: the .so sits next to this file so that it travels to the GPU box.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libsmelter_b200.so")
SOURCES = ["kernels.cu", "renderer.cpp", "scene.cpp", "wgsl.cpp"]
# the sources a shader module is compiled from at registration (renderer.cpp, NVRTC), embedded as string literals
EMBEDDED = ["kernels.h", "node_sample.cuh", "shader_rt.cuh", "wgsl_rt.cuh"]
EMBEDDED_INC = os.path.join(CSRC, "shader_sources.inc")   # generated, kept out of git
HEADERS = ["node_sample.cuh", "shader_rt.cuh", "wgsl_rt.cuh", "wgsl.h", "kernels.h", "interior.h", "int_weights.h", "scene.h", "ptx_helpers.cuh", "resample_tma.cuh", "resample_tma3.cuh", "resample_tma0.cuh", "transcode.cuh", "video_convert.cuh", "deinterlace.cuh", os.path.join("..", "..", "include", "smelter_b200.h")]

NVCC_FLAGS = [
    "-std=c++17", "-O3",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "-fmad=false",            # numeric contract: only explicit fmaf() is fused
    "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
    "-Xcompiler", "-fPIC,-ffp-contract=off,-Wall",
    "-ccbin", "/usr/bin/g++",
    "-shared",
]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def write_embedded():
    """shader_sources.inc: one raw string literal per EMBEDDED file, named kSrc_<file stem>"""
    out = []
    for name in EMBEDDED:
        with open(os.path.join(CSRC, name)) as f:
            text = f.read()
        assert ')SMRSRC"' not in text
        out.append(f'static const char kSrc_{name.split(".")[0]}[] = R"SMRSRC({text})SMRSRC";\n')
    text = "".join(out)
    if not os.path.exists(EMBEDDED_INC) or open(EMBEDDED_INC).read() != text:
        with open(EMBEDDED_INC, "w") as f:
            f.write(text)


def build(force=False, verbose=False, extra=()):
    if not force and not needs_build():
        return LIB
    write_embedded()
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + list(extra) + ["-o", LIB] + [os.path.join(CSRC, s) for s in SOURCES]
    if verbose:
        print(" ".join(cmd))
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    build(force=True, verbose=True, extra=sys.argv[1:])
    print(LIB)
