/*
 * shader_oracle_shim.h -- CPU shim a test shader's CUDA C++ source is compiled against for the shader oracle (TEST
 * INFRASTRUCTURE ONLY, NOT PRODUCT CODE).  tests/oracle_shader.py compiles shim + shader + this file's entry point with
 * g++ -ffp-contract=off, so the shader's arithmetic rounds as it does on the GPU (--fmad=false: only fmaf() is fused).
 *
 * Restated from the shader contract in include/smelter_b200.h and the numeric contract of oracle/smelter_oracle.c:
 *   sample:   textureSample with the linear / ClampToEdge sampler (NC-6) of child i's RGBA8 node texture, through the view:
 *             GpuOptimized decodes the sRGB colour bytes (NC-3), CpuOptimized filters the bytes (NC-6u); an index at or
 *             above texture_count, or a missing texture, is the empty view (0, 0, 0, 0)
 *   planes:   clear to transparent, then max(1, n) full-target planes (plane_id -1 without children), each pixel's
 *             smr_fragment at its centre blended with PREMULTIPLIED_ALPHA_BLENDING and stored as 8 bits (NC-2 / NC-4)
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#define __device__

struct float2 { float x, y; };
struct float4 { float x, y, z, w; };
static inline float2 make_float2(float x, float y) { float2 r = {x, y}; return r; }
static inline float4 make_float4(float x, float y, float z, float w) { float4 r = {x, y, z, w}; return r; }

static float u8n[256], dec[256], thr[255];

static double eotf(double c) { return c <= 0.04045 ? c / 12.92 : pow((c + 0.055) / 1.055, 2.4); }

static void init_tables(void) {
    for (int b = 0; b < 256; b++) {
        u8n[b] = (float)b / 255.0f;                 /* NC-1 */
        dec[b] = (float)eotf((double)b / 255.0);    /* NC-3 */
    }
    for (int k = 0; k < 255; k++) thr[k] = (float)eotf(((double)k + 0.5) / 255.0);   /* NC-4 */
}

static float clamp01(float x) { return fminf(fmaxf(x, 0.0f), 1.0f); }
static uint8_t store_unorm(float x) { return (uint8_t)rintf(clamp01(x) * 255.0f); }
static uint8_t store_srgb(float x) {
    int n = 0;
    x = clamp01(x);
    while (n < 255 && x >= thr[n]) n++;
    return (uint8_t)n;
}

static void tap(float t, int dim, int *i0, int *i1, float *f) {   /* NC-6 */
    float c = t * (float)dim - 0.5f;
    if (c != c) { *i0 = *i1 = 0; *f = 0.0f; return; }
    c = fminf(fmaxf(c, -2.0f), (float)dim + 1.0f);
    float fl = floorf(c);
    *f = rintf((c - fl) * 256.0f) * (1.0f / 256.0f);
    int a = (int)fl, b = a + 1;
    *i0 = a < 0 ? 0 : (a > dim - 1 ? dim - 1 : a);
    *i1 = b < 0 ? 0 : (b > dim - 1 ? dim - 1 : b);
}

static float lerp2(float t00, float t10, float t01, float t11, float fx, float fy) {
    float h0 = fmaf(t10, fx, t00 * (1.0f - fx));
    float h1 = fmaf(t11, fx, t01 * (1.0f - fx));
    return fmaf(h1, fy, h0 * (1.0f - fy));
}

static float lerp2_u8(int t00, int t10, int t01, int t11, float fx, float fy) {   /* NC-6u */
    int wx = (int)(fx * 256.0f), wy = (int)(fy * 256.0f);
    int n = (t00 * (256 - wx) + t10 * wx) * (256 - wy) + (t01 * (256 - wx) + t11 * wx) * wy;
    return (float)n / 16711680.0f;
}

struct smr_fragment_in { float2 tex_coords; float4 position; };
struct smr_base_params { int plane_id; float time; unsigned output_resolution[2]; unsigned texture_count; };
struct smr_textures {
    const uint8_t *const *tex;
    const int *w, *h;
    unsigned count;
    int mode;
    float4 sample(unsigned i, float2 uv) const {
        if (i >= count || !tex[i]) return make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        const uint8_t *t = tex[i];
        int x0, x1, y0, y1;
        float fx, fy, out[4];
        tap(uv.x, w[i], &x0, &x1, &fx);
        tap(uv.y, h[i], &y0, &y1, &fy);
        const uint8_t *p00 = t + ((size_t)y0 * w[i] + x0) * 4, *p10 = t + ((size_t)y0 * w[i] + x1) * 4;
        const uint8_t *p01 = t + ((size_t)y1 * w[i] + x0) * 4, *p11 = t + ((size_t)y1 * w[i] + x1) * 4;
        for (int k = 0; k < 4; k++) {
            if (mode != 0) out[k] = lerp2_u8(p00[k], p10[k], p01[k], p11[k], fx, fy);
            else if (k == 3) out[k] = lerp2(u8n[p00[k]], u8n[p10[k]], u8n[p01[k]], u8n[p11[k]], fx, fy);
            else out[k] = lerp2(dec[p00[k]], dec[p10[k]], dec[p01[k]], dec[p11[k]], fx, fy);
        }
        return make_float4(out[0], out[1], out[2], out[3]);
    }
};

static void blend(uint8_t *d, float4 c, int mode) {   /* PREMULTIPLIED_ALPHA_BLENDING */
    const float s[4] = {clamp01(c.x), clamp01(c.y), clamp01(c.z), clamp01(c.w)};
    const float ia = 1.0f - s[3];
    for (int k = 0; k < 3; k++)
        d[k] = mode == 0 ? store_srgb(fmaf(dec[d[k]], ia, s[k])) : store_unorm(fmaf(u8n[d[k]], ia, s[k]));
    d[3] = store_unorm(fmaf(u8n[d[3]], ia, s[3]));
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
                blend(out + ((size_t)y * W + x) * 4, smr_fragment(in, base, params, t), mode);
            }
        }
}
