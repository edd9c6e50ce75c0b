/*
 * image_oracle.c -- CPU ORACLE for image node textures (TEST INFRASTRUCTURE ONLY, NOT PRODUCT CODE).
 *
 * ImageNode::render (smelter-render/src/transformations/image.rs:178-187) draws an asset frame into a node texture of the
 * node's resolution with wgpu/utils/add_premultiplied_alpha.wgsl.  Written from that shader and from the numeric contract
 * of oracle/smelter_oracle.c (NC-1 .. NC-6u), which it restates for the steps it needs; it lives beside the tests because
 * the committed oracle is the yardstick of every other test and stays as it is.  tests/oracle_image.py compiles it
 * (-ffp-contract=off: only fmaf() is fused) and tests/test_image_component.py pins it to orc_add_premultiplied_alpha at
 * equal sizes.
 *
 *   vs_main:  a full-target quad, tex_coords 0..1: the fragment of target pixel (x, y) has
 *             tex_coords = ((x + .5) / ow, (y + .5) / oh)
 *   fs_main:  color = textureSample(texture, sampler_, tex_coords)      linear / ClampToEdge (common_pipeline.rs:56-65)
 *             a = max(color.a, 0.00001)
 *             (clamp(color.r * a), clamp(color.g * a), clamp(color.b * a), clamp(color.a))
 *   views:    GpuOptimized  source Rgba8UnormSrgb (texels decoded, then filtered: NC-3, NC-6), target stored sRGB (NC-4)
 *             CpuOptimized  source Rgba8Unorm (filtered on the bytes: NC-6u), target stored UNORM8 (NC-2)
 *             alpha is UNORM in both.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

static float u8n[256], dec[256], thr[255];
static int ready = 0;

static double eotf(double c) { return c <= 0.04045 ? c / 12.92 : pow((c + 0.055) / 1.055, 2.4); }

static void init(void) {
    if (ready) return;
    for (int b = 0; b < 256; b++) {
        u8n[b] = (float)b / 255.0f;                 /* NC-1 */
        dec[b] = (float)eotf((double)b / 255.0);    /* NC-3 */
    }
    for (int k = 0; k < 255; k++) thr[k] = (float)eotf(((double)k + 0.5) / 255.0);   /* NC-4 */
    ready = 1;
}

static float clamp01(float x) { return fminf(fmaxf(x, 0.0f), 1.0f); }
static uint8_t store_unorm(float x) { return (uint8_t)rintf(clamp01(x) * 255.0f); }   /* NC-2 */
static uint8_t store_srgb(float x) {                                                  /* NC-4 */
    int n = 0;
    x = clamp01(x);
    while (n < 255 && x >= thr[n]) n++;
    return (uint8_t)n;
}

/* NC-6: texel coordinate t * dim - .5, the fraction quantised to 8 bits, taps clamped to the edge */
static void tap(float t, int dim, int *i0, int *i1, float *f) {
    float c = fminf(fmaxf(t * (float)dim - 0.5f, -2.0f), (float)dim + 1.0f);
    float fl = floorf(c);
    *f = rintf((c - fl) * 256.0f) * (1.0f / 256.0f);
    int a = (int)fl, b = a + 1;
    *i0 = a < 0 ? 0 : (a > dim - 1 ? dim - 1 : a);
    *i1 = b < 0 ? 0 : (b > dim - 1 ? dim - 1 : b);
}

static float lerp2(float t00, float t10, float t01, float t11, float fx, float fy) {   /* NC-6 */
    float h0 = fmaf(t10, fx, t00 * (1.0f - fx));
    float h1 = fmaf(t11, fx, t01 * (1.0f - fx));
    return fmaf(h1, fy, h0 * (1.0f - fy));
}

static float lerp2_u8(int t00, int t10, int t01, int t11, float fx, float fy) {         /* NC-6u */
    int wx = (int)(fx * 256.0f), wy = (int)(fy * 256.0f);
    int n = (t00 * (256 - wx) + t10 * wx) * (256 - wy) + (t01 * (256 - wx) + t11 * wx) * wy;
    return (float)n / 16711680.0f;
}

/* src: sw x sh straight-alpha RGBA8, packed; out: ow x oh premultiplied RGBA8, packed; mode 0 GpuOptimized, 1 CpuOptimized */
void orc_render_image(const uint8_t *src, int sw, int sh, int ow, int oh, int mode, uint8_t *out) {
    init();
    for (int y = 0; y < oh; y++)
        for (int x = 0; x < ow; x++) {
            int x0, x1, y0, y1;
            float fx, fy, c[4];
            tap(((float)x + 0.5f) / (float)ow, sw, &x0, &x1, &fx);
            tap(((float)y + 0.5f) / (float)oh, sh, &y0, &y1, &fy);
            const uint8_t *p00 = src + ((size_t)y0 * sw + x0) * 4, *p10 = src + ((size_t)y0 * sw + x1) * 4;
            const uint8_t *p01 = src + ((size_t)y1 * sw + x0) * 4, *p11 = src + ((size_t)y1 * sw + x1) * 4;
            for (int k = 0; k < 4; k++) {
                if (mode != 0) c[k] = lerp2_u8(p00[k], p10[k], p01[k], p11[k], fx, fy);
                else if (k == 3) c[k] = lerp2(u8n[p00[k]], u8n[p10[k]], u8n[p01[k]], u8n[p11[k]], fx, fy);
                else c[k] = lerp2(dec[p00[k]], dec[p10[k]], dec[p01[k]], dec[p11[k]], fx, fy);
            }
            const float a = fmaxf(c[3], 0.00001f);
            uint8_t *o = out + ((size_t)y * ow + x) * 4;
            for (int k = 0; k < 3; k++) {
                const float v = clamp01(c[k] * a);
                o[k] = mode == 0 ? store_srgb(v) : store_unorm(v);
            }
            o[3] = store_unorm(clamp01(c[3]));
        }
}
