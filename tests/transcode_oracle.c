/* transcode_oracle.c -- CPU oracle of smr_transcode_resize: gpu-video's transcoder resize (vulkan_transcoder/shader.wgsl
 * `main` and its samplers) restated per output pixel, for one rendition.  Test infrastructure (tests/c_oracles.py
 * builds it with -ffp-contract=off, so every f32 operation rounds on its own, as DESIGN.md NC-10 requires).
 *
 * Texels are fetched as v / 255 (NC-1) and stored as rint(clamp(x) * 255) (NC-2); sin is evaluated in fp64 and rounded
 * to f32 (NC-8).  Written from the shader, not from the kernel: coordinates and weights are evaluated here per pixel. */
#include "oracle_nc.h"

typedef struct {
    const uint8_t *p;
    int pitch, ch;          /* bytes per row, channels per texel (1: r8unorm, 2: rg8unorm) */
    int w, h;               /* the texture's (cropped) size */
} plane;

static float fetch(const plane *t, int x, int y, int c) { return (float)t->p[(size_t)y * t->pitch + x * t->ch + c] / 255.0f; }

static float sinc(float x) {
    if (fabsf(x) < 1e-6f) return 1.0f;
    const float px = 3.14159265358979323846f * x;
    return (float)sin((double)px) / px;
}

static float lanczos3_weight(float x) {
    if (fabsf(x) >= 3.0f) return 0.0f;
    return sinc(x) * sinc(x / 3.0f);
}

static float mix(float a, float b, float t) { return a * (1.0f - t) + b * t; }

static int clampi(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }

/* the shader's sample_{nearest,bilinear,lanczos3}_{y,uv} at float_coords (fx, fy) of a texture t, channel c */
static float sample(const plane *t, int algo, float fx, float fy, int c) {
    const float in_w = (float)t->w, in_h = (float)t->h;
    if (algo == 0) {
        const float sx = in_w * fx, sy = in_h * fy;
        return fetch(t, (int)(uint32_t)sx, (int)(uint32_t)sy, c);
    }
    const float fcx = in_w * fx - 0.5f, fcy = in_h * fy - 0.5f;
    if (algo == 1) {
        const uint32_t x0 = (uint32_t)fmaxf(floorf(fcx), 0.0f), y0 = (uint32_t)fmaxf(floorf(fcy), 0.0f);
        const uint32_t x1 = x0 + 1 < (uint32_t)t->w - 1 ? x0 + 1 : (uint32_t)t->w - 1;
        const uint32_t y1 = y0 + 1 < (uint32_t)t->h - 1 ? y0 + 1 : (uint32_t)t->h - 1;
        const float ax = fcx - floorf(fcx), ay = fcy - floorf(fcy);
        const float p00 = fetch(t, x0, y0, c), p10 = fetch(t, x1, y0, c), p01 = fetch(t, x0, y1, c), p11 = fetch(t, x1, y1, c);
        return mix(mix(p00, p10, ax), mix(p01, p11, ax), ay);
    }
    const float center_x = floorf(fcx), center_y = floorf(fcy);
    const int max_x = t->w - 1, max_y = t->h - 1;
    float wx[6];   /* the shader evaluates wx inside the dy loop; it does not depend on dy */
    for (int dx = -2; dx <= 3; dx++) wx[dx + 2] = lanczos3_weight(fcx - (center_x + (float)dx));
    float sum = 0.0f, weight_sum = 0.0f;
    for (int dy = -2; dy <= 3; dy++) {
        const int sy = clampi((int)center_y + dy, 0, max_y);
        const float wy = lanczos3_weight(fcy - (center_y + (float)dy));
        for (int dx = -2; dx <= 3; dx++) {
            const int sx = clampi((int)center_x + dx, 0, max_x);
            const float w = wx[dx + 2] * wy;
            sum += fetch(t, sx, sy, c) * w;
            weight_sum += w;
        }
    }
    return sum / weight_sum;
}

/* One rendition of out_w x out_h (even) from the NV12 crop in_w x in_h (even): oy packed out_h x out_w, ouv packed
 * (out_h / 2) x (out_w / 2) {u, v} pairs.  algo: 0 NearestNeighbor, 1 Bilinear, 2 Lanczos3. */
void orc_transcode_resize(const uint8_t *y, int y_pitch, const uint8_t *uv, int uv_pitch, int in_w, int in_h, int out_w,
                          int out_h, int algo, uint8_t *oy, uint8_t *ouv) {
    const plane ty = {y, y_pitch, 1, in_w, in_h}, tuv = {uv, uv_pitch, 2, in_w / 2, in_h / 2};
#pragma omp parallel for schedule(dynamic, 4)
    for (int oyy = 0; oyy < out_h; oyy++) {
        for (int ox = 0; ox < out_w; ox++) {
            const float fx = ((float)ox + 0.5f) / (float)out_w, fy = ((float)oyy + 0.5f) / (float)out_h;
            oy[(size_t)oyy * out_w + ox] = store_unorm(sample(&ty, algo, fx, fy, 0));
            if (ox % 2 == 0 && oyy % 2 == 0) {
                const int ux = ox / 2, uy = oyy / 2, uw = out_w / 2, uh = out_h / 2;
                const float gx = ((float)ux + 0.5f) / (float)uw, gy = ((float)uy + 0.5f) / (float)uh;
                uint8_t *d = ouv + ((size_t)uy * uw + ux) * 2;
                d[0] = store_unorm(sample(&tuv, algo, gx, gy, 0));
                d[1] = store_unorm(sample(&tuv, algo, gx, gy, 1));
            }
        }
    }
}
