/*
 * svg_oracle.c -- CPU ORACLE for SVG image node textures (TEST INFRASTRUCTURE ONLY, NOT PRODUCT CODE).
 *
 * SvgAsset::render (smelter-render/src/transformations/image/svg_image.rs:59-180) from the caller's raster at the node's
 * size (premultiplied RGBA8, tiny-skia's Pixmap).  CpuOptimized uploads the bytes as they are.  GpuOptimized runs two
 * full-target passes into textures of the same size:
 *   remove_premultiplied_alpha.wgsl through UNORM views: c = textureSample (NC-6u), a = max(c.a, 0.00001),
 *             (clamp(c.r / a), clamp(c.g / a), clamp(c.b / a), clamp(c.a)) stored UNORM8 (NC-2)
 *   add_premultiplied_alpha.wgsl through sRGB views: orc_render_image of that texture at its own size.
 * It includes tests/image_oracle.c, whose sampler taps, filters, stores and orc_render_image it uses as they are.
 * tests/oracle_svg.py compiles it with the flags tests/oracle_image.py uses.
 */
#include "image_oracle.c"

/* src: w x h premultiplied RGBA8, packed; mid: w x h scratch; out: the w x h node texture, packed; mode as for
 * orc_render_image */
void orc_render_svg(const uint8_t *src, int w, int h, int mode, uint8_t *mid, uint8_t *out) {
    init();
    if (mode != 0) {
        for (size_t i = 0; i < (size_t)w * h * 4; i++) out[i] = src[i];
        return;
    }
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            int x0, x1, y0, y1;
            float fx, fy, c[4];
            tap(((float)x + 0.5f) / (float)w, w, &x0, &x1, &fx);
            tap(((float)y + 0.5f) / (float)h, h, &y0, &y1, &fy);
            const uint8_t *p00 = src + ((size_t)y0 * w + x0) * 4, *p10 = src + ((size_t)y0 * w + x1) * 4;
            const uint8_t *p01 = src + ((size_t)y1 * w + x0) * 4, *p11 = src + ((size_t)y1 * w + x1) * 4;
            for (int k = 0; k < 4; k++) c[k] = lerp2_u8(p00[k], p10[k], p01[k], p11[k], fx, fy);
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
