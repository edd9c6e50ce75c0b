/*
 * shader_oracle_shim.h -- CPU shim a test shader's CUDA C++ source is compiled against for the shader oracle (TEST
 * INFRASTRUCTURE ONLY, NOT PRODUCT CODE).  tests/c_oracles.py compiles shim + shader + this file's entry point with
 * g++ -ffp-contract=off, so the shader's arithmetic rounds as it does on the GPU (--fmad=false: only fmaf() is fused).
 *
 * Restated from the shader contract in include/smelter_b200.h and the numeric contract in tests/oracle_nc.h:
 *   sample:   textureSample with the linear / ClampToEdge sampler (NC-6) of child i's RGBA8 node texture, through the view:
 *             GpuOptimized decodes the sRGB colour bytes (NC-3), CpuOptimized filters the bytes (NC-6u); an index at or
 *             above texture_count, or a missing texture, is the empty view (0, 0, 0, 0)
 *   planes:   clear to transparent, then max(1, n) full-target planes (plane_id -1 without children), each pixel's
 *             smr_fragment at its centre blended with PREMULTIPLIED_ALPHA_BLENDING and stored as 8 bits (NC-2 / NC-4)
 */
#include <string.h>

#include "oracle_nc.h"

#define __device__

struct float2 { float x, y; };
struct float4 { float x, y, z, w; };
static inline float2 make_float2(float x, float y) { float2 r = {x, y}; return r; }
static inline float4 make_float4(float x, float y, float z, float w) { float4 r = {x, y, z, w}; return r; }

struct smr_fragment_in { float2 tex_coords; float4 position; };
struct smr_base_params { int plane_id; float time; unsigned output_resolution[2]; unsigned texture_count; };
struct smr_textures {
    const uint8_t *const *tex;
    const int *w, *h;
    unsigned count;
    int mode;
    float4 sample(unsigned i, float2 uv) const {
        static const int rgba[4] = {0, 1, 2, 3};
        float out[4];
        if (i >= count) return make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        sample_rgba8(tex[i], w[i], h[i], rgba, mode, uv.x, uv.y, out);
        return make_float4(out[0], out[1], out[2], out[3]);
    }
};

static void blend_fragment(uint8_t *d, float4 c, int mode) {   /* oracle_nc.h's blend of a fragment's colour */
    const float s[4] = {c.x, c.y, c.z, c.w};
    blend(d, s, mode);
}

__device__ float4 smr_fragment(smr_fragment_in in, const smr_base_params &base, const void *params, const smr_textures &tex);

/* out: W x H RGBA8, the node texture after the tick.  tex[k]: child k's RGBA8 node texture of tw[k] x th[k] (NULL: the
 * empty view).  params: the parameter bytes (NULL: none). */
extern "C" void orc_render_shader(int W, int H, int mode, float time, const void *params, const uint8_t *const *tex,
                                  const int *tw, const int *th, int n, uint8_t *out) {
    init_tables();
    memset(out, 0, (size_t)W * H * 4);
    smr_textures t = {tex, tw, th, (unsigned)n, mode};
    smr_base_params base = {0, time, {(unsigned)W, (unsigned)H}, (unsigned)n};
    for (int y = 0; y < H; y++)
        for (int x = 0; x < W; x++) {
            smr_fragment_in in;
            in.position = make_float4((float)x + 0.5f, (float)y + 0.5f, 0.0f, 1.0f);
            in.tex_coords = make_float2(in.position.x / (float)W, in.position.y / (float)H);
            for (int p = 0; p < (n > 0 ? n : 1); p++) {
                base.plane_id = n > 0 ? p : -1;
                blend_fragment(out + ((size_t)y * W + x) * 4, smr_fragment(in, base, params, t), mode);
            }
        }
}
