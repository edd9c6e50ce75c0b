/*
 * image_oracle.c -- CPU ORACLE for image node textures (TEST INFRASTRUCTURE ONLY, NOT PRODUCT CODE).
 *
 * ImageNode::render (smelter-render/src/transformations/image.rs:178-187) draws an asset frame into a node texture of the
 * node's resolution with wgpu/utils/add_premultiplied_alpha.wgsl.  Written from that shader and from the numeric contract
 * as tests/oracle_nc.h states it (NC-1 .. NC-6u).  tests/test_image_component.py pins it to orc_add_premultiplied_alpha at
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
#include "oracle_nc.h"

/* src: sw x sh straight-alpha RGBA8, packed; out: ow x oh premultiplied RGBA8, packed; mode 0 GpuOptimized, 1 CpuOptimized */
void orc_render_image(const uint8_t *src, int sw, int sh, int ow, int oh, int mode, uint8_t *out) {
    static const int rgba[4] = {0, 1, 2, 3};
    init_tables();
    for (int y = 0; y < oh; y++)
        for (int x = 0; x < ow; x++) {
            float c[4];
            sample_rgba8(src, sw, sh, rgba, mode, ((float)x + 0.5f) / (float)ow, ((float)y + 0.5f) / (float)oh, c);
            const float a = fmaxf(c[3], 0.00001f);
            uint8_t *o = out + ((size_t)y * ow + x) * 4;
            for (int k = 0; k < 3; k++) {
                const float v = clamp01(c[k] * a);
                o[k] = mode == 0 ? store_srgb(v) : store_unorm(v);
            }
            o[3] = store_unorm(clamp01(c[3]));
        }
}
