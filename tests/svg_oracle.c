/*
 * svg_oracle.c -- CPU ORACLE for SVG image node textures (TEST INFRASTRUCTURE ONLY, NOT PRODUCT CODE).
 *
 * SvgAsset::render (smelter-render/src/transformations/image/svg_image.rs:59-180) from the caller's raster at the node's
 * size (premultiplied RGBA8, tiny-skia's Pixmap).  CpuOptimized uploads the bytes as they are.  GpuOptimized runs two
 * full-target passes into textures of the same size:
 *   remove_premultiplied_alpha.wgsl through UNORM views: c = textureSample (NC-6u), a = max(c.a, 0.00001),
 *             (clamp(c.r / a), clamp(c.g / a), clamp(c.b / a), clamp(c.a)) stored UNORM8 (NC-2)
 *   add_premultiplied_alpha.wgsl through sRGB views: orc_render_image (tests/image_oracle.c) of that texture at its own
 *             size.
 */
#include "oracle_nc.h"

void orc_render_image(const uint8_t *src, int sw, int sh, int ow, int oh, int mode, uint8_t *out);

/* src: w x h premultiplied RGBA8, packed; mid: w x h scratch; out: the w x h node texture, packed; mode as for
 * orc_render_image */
void orc_render_svg(const uint8_t *src, int w, int h, int mode, uint8_t *mid, uint8_t *out) {
    static const int rgba[4] = {0, 1, 2, 3};
    if (mode != 0) {
        for (size_t i = 0; i < (size_t)w * h * 4; i++) out[i] = src[i];
        return;
    }
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            float c[4];
            sample_rgba8(src, w, h, rgba, 1, ((float)x + 0.5f) / (float)w, ((float)y + 0.5f) / (float)h, c);
            const float a = fmaxf(c[3], 0.00001f);
            uint8_t *o = mid + ((size_t)y * w + x) * 4;
            for (int k = 0; k < 3; k++) o[k] = store_unorm(clamp01(c[k] / a));
            o[3] = store_unorm(clamp01(c[3]));
        }
    orc_render_image(mid, w, h, w, h, 0, out);
}

/* The pixel-centre sample of a texture of the target's own size, for every size 1 .. max_dim and every coordinate: the
 * number of (size, coordinate) pairs whose NC-6 taps are anything but texel x with weight 1 */
long orc_check_same_size_taps(int max_dim) {
    long bad = 0;
    for (int dim = 1; dim <= max_dim; dim++)
        for (int x = 0; x < dim; x++) {
            int i0, i1;
            float f;
            tap(((float)x + 0.5f) / (float)dim, dim, &i0, &i1, &f);
            bad += !((f == 0.0f && i0 == x) || (f == 1.0f && i1 == x));
        }
    return bad;
}
