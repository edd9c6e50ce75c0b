/*
 * smelter_oracle.h -- CPU ORACLE (TEST INFRASTRUCTURE ONLY, NOT PRODUCT CODE)
 *
 * A plain-C restatement of the per-output-frame compositor of software-mansion/smelter
 * (`smelter_render::Renderer::render`, smelter-render/src/state.rs:220-252) used ONLY as the
 * checker in tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg.
 * The product (smelter_b200/csrc, libsmelter_b200.so) never includes, links or calls this file.
 *
 * PARITY STATUS: the reference is Rust + wgpu (no rustc, no Vulkan ICD in this image; the golden
 * PNG snapshots live in an un-mounted private submodule).  This oracle is therefore pinned ONLY by
 * the known-answer vectors that are physically present in the reference tree:
 *   - integration-tests/src/render_tests/yuv_tests.rs:32-132          (tests/test_oracle_kat.py)
 *   - integration-tests/src/render_tests/pixel_input_format_tests.rs:31-152
 *   - smelter-render/src/transformations/layout/resampler.rs:402-468  (pass planner truth table)
 *   - smelter-render/src/scene/transition/cubic_bezier.rs tests
 * Beyond those vectors: **parity unpinned** (GPU fixed-function behaviour -- sRGB conversion,
 * UNORM rounding, bilinear weight precision, rasteriser snapping -- is restated from the
 * WebGPU/Vulkan rules, see DESIGN.md "numeric contract").  The planar 4:2:2 / 4:4:4, interleaved
 * UYVY / YUYV and FramePreProcessor-rescale restatements have NO reference vector at all (the reference
 * tests them through snapshots only): parity unpinned for them.
 *
 * Every function cites the reference file:line it follows.
 */
#ifndef SMELTER_ORACLE_H
#define SMELTER_ORACLE_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* RenderingMode (smelter-render/src/types.rs:9-18). WebGl is out of scope. */
enum { ORC_MODE_GPU_OPTIMIZED = 0, ORC_MODE_CPU_OPTIMIZED = 1 };

/* layout_type of apply_layouts.wgsl:66-71 */
enum { ORC_LAYOUT_TEXTURE = 0, ORC_LAYOUT_COLOR = 1, ORC_LAYOUT_BOX_SHADOW = 2 };

#define ORC_MAX_MASKS 20 /* params.rs:15 */

/* ParentMask (apply_layouts.wgsl:58-64, layout.rs:50-57); radius = [tl, tr, br, bl] */
typedef struct {
    float radius[4];
    float top, left, width, height;
} orc_mask;

/* RenderLayout after flatten (layout.rs:59-98) */
typedef struct {
    int32_t type;            /* ORC_LAYOUT_* */
    float top, left, width, height;
    float rotation_degrees;
    float border_radius[4];  /* tl, tr, br, bl */
    uint8_t color[4];        /* Color / BoxShadow: straight (non-premultiplied) sRGB RGBA */
    uint8_t border_color[4];
    float border_width;
    float blur_radius;       /* BoxShadow */
    int32_t child_index;     /* Texture: index into the node-texture array */
    float crop_top, crop_left, crop_width, crop_height;
    int32_t masks_len;
    orc_mask masks[ORC_MAX_MASKS];
} orc_layout;

/* A node texture: premultiplied RGBA8; in GpuOptimized the bytes are sRGB-encoded
 * (node_texture.rs:65-115). data == NULL means "no texture" (cleared input). */
typedef struct {
    int32_t width, height;
    const uint8_t *data; /* width*height*4, tightly packed */
} orc_texture;

/* one-time table init (sRGB LUTs); idempotent, called lazily by everything */
void orc_init(void);

/* --- K1/K2: input conversion (planar_yuv_to_rgba.wgsl:35-58, nv12_to_rgba.wgsl:26-48) ---- */
void orc_yuv420_to_rgba(const uint8_t *y, const uint8_t *u, const uint8_t *v, int w, int h,
                        int full_range, uint8_t *rgba);
void orc_nv12_to_rgba(const uint8_t *y, const uint8_t *uv, int w, int h, uint8_t *rgba);
/* planar 4:2:0 / 4:2:2 / 4:4:4 by chroma plane size (texture/planar_yuv.rs:64-83) */
void orc_yuv_planar_to_rgba(const uint8_t *y, const uint8_t *u, const uint8_t *v, int w, int h, int cw, int ch,
                            int full_range, uint8_t *rgba);
/* K3 interleaved_{uyvy,yuyv}_to_rgba.wgsl; yuyv = 0: U Y0 V Y1, 1: Y0 U Y1 V */
void orc_interleaved422_to_rgba(const uint8_t *data, int w, int h, int yuyv, uint8_t *rgba);
/* K4 (bgra_to_rgba.wgsl / argb_to_rgba.wgsl): pure swizzles */
void orc_bgra_to_rgba(const uint8_t *bgra, int w, int h, uint8_t *rgba);
void orc_argb_to_rgba(const uint8_t *argb, int w, int h, uint8_t *rgba);

/* --- K10/K11: output conversion (rgba_to_yuv.wgsl:26-54, rgba_to_nv12.wgsl:25-52) -------- */
void orc_rgba_to_yuv420(const uint8_t *rgba, int w, int h, uint8_t *y, uint8_t *u, uint8_t *v);
void orc_rgba_to_nv12(const uint8_t *rgba, int w, int h, uint8_t *y, uint8_t *uv);
/* same converters when the root texture (sw x sh) is not the output size (w x h) */
void orc_rgba_to_yuv420_scaled(const uint8_t *rgba, int sw, int sh, int w, int h, uint8_t *y, uint8_t *u,
                               uint8_t *v);
void orc_rgba_to_yuv_planar_scaled(const uint8_t *rgba, int sw, int sh, int w, int h, int cw, int ch, uint8_t *y,
                                   uint8_t *u, uint8_t *v);
void orc_rgba_to_nv12_scaled(const uint8_t *rgba, int sw, int sh, int w, int h, uint8_t *y, uint8_t *uv);
/* RGBColor::to_yuv (scene/types.rs:28-42) stored through an R8Unorm target; black-frame fill
 * of render_loop.rs:127-139 */
void orc_rgb_to_yuv_bytes(uint8_t r, uint8_t g, uint8_t b, uint8_t out_yuv[3]);

/* --- K7/K8: resampler (layout/resampler.rs:285-400, resample.wgsl, downsample.wgsl) ------- */
/* plan: returns 0 = direct (no pass), 1 = single pass, 2 = separable.
 * axis_out[i] (0 = horizontal, 1 = vertical) and perp_out[i] describe each kernel pass;
 * levels_out[2] are the box pre-decimation levels per axis (horizontal, vertical). */
int orc_plan_passes(float crop_left, float crop_top, float crop_w, float crop_h, int dst_w,
                    int dst_h, int axis_out[2], int perp_out[2]);
int orc_predecimate_levels(float crop_len, int dst_len);
/* full resample of one child (GpuOptimized only): src is an sRGB-encoded premultiplied RGBA8 node
 * texture; dst (dst_w*dst_h*4) receives the sRGB-encoded result. Returns 0 if no pass was needed
 * (dst untouched), 1 otherwise. */
int orc_resample(const orc_texture *src, float crop_left, float crop_top, float crop_w,
                 float crop_h, int dst_w, int dst_h, uint8_t *dst);
/* Lanczos3 weights of resample.wgsl:42-86 for one output coordinate. weights must hold
 * orc_resample_taps(scale) floats. Returns `first` (index of the first tap, unclamped). */
int orc_resample_taps(float scale);
int orc_resample_weights(float scale, float offset, int out_coord, float *weights,
                         float *weight_sum);

/* --- K9: apply_layouts (layout/shader.rs:93-167, params.rs:169-333, apply_layouts.wgsl) ---- */
/* Draws `n` layouts (at most max_layouts, shader.rs:152) in order onto a transparent W x H
 * target. textures[i] is the texture bound for layouts[i] when it is a Texture layout
 * (already resampled when needed) and ignored otherwise. */
void orc_apply_layouts(int out_w, int out_h, const orc_layout *layouts,
                       const orc_texture *textures, int n, int max_layouts, int mode,
                       uint8_t *out_rgba);
/* One layout's fragment, per pixel of a W x H target: 1 where the layout covers the pixel and its fragment is the bare
 * colour or sample -- every alpha factor exactly 1 and no border colour mixed in -- else 0. */
void orc_bare_map(int out_w, int out_h, const orc_layout *layout, int mode, uint8_t *out);

/* --- LayoutNode::render (transformations/layout.rs:169-278): resample scaled children, then
 * apply_layouts. nodes[] are the child node textures indexed by orc_layout.child_index. */
void orc_render_layout_node(int out_w, int out_h, const orc_layout *layouts, int n,
                            const orc_texture *nodes, int n_nodes, int max_layouts, int mode,
                            uint8_t *out_rgba);

/* --- test-harness inverse used by every reference snapshot (harness/utils.rs:31-65) ------- */
/* FramePreProcessor's optional rescale (frame_pre_processor.rs:117-132, rgba_rescale.wgsl) */
void orc_rescale_rgba(const uint8_t *rgba, int sw, int sh, int ow, int oh, int mode, uint8_t *out);
/* add_premultiplied_alpha.wgsl:24-35: straight alpha -> premultiplied through the mode's texture views */
void orc_add_premultiplied_alpha(const uint8_t *rgba, int w, int h, int mode, uint8_t *out);
/* glyphon GlyphToRender after clipping (un-vendored dependency glyphon 0.11.0 @ smelter-labs c784922): quad origin in
 * the text texture, size, atlas origin, straight-alpha sRGB colour, content (0 = colour atlas, 1 = mask atlas) */
typedef struct {
    int32_t x, y;
    uint16_t width, height;
    uint16_t atlas_x, atlas_y;
    uint8_t color[4];
    int32_t content;
} orc_glyph;
/* TextRendererNode::render (text_renderer.rs:72-167): clear to background, alpha-blend the glyph quads in order.
 * mask_atlas: R8 (mask_w x mask_h), color_atlas: RGBA8; color_mode 0 = glyphon ColorMode::Accurate, 1 = Web. */
void orc_render_text(int w, int h, const uint8_t background[4], const orc_glyph *glyphs, int n_glyphs, const uint8_t *mask_atlas,
                     int mask_w, int mask_h, const uint8_t *color_atlas, int color_w, int color_h, int color_mode, int mode,
                     uint8_t *out);
void orc_harness_yuv420_to_rgba(const uint8_t *y, const uint8_t *u, const uint8_t *v, int w,
                                int h, uint8_t *rgba);

/* building blocks exposed for unit tests */
float orc_srgb_decode_u8(uint8_t v);    /* sRGB8 -> linear float (texture fetch through srgb view) */
uint8_t orc_srgb_encode_u8(float lin);  /* linear float -> sRGB8 (render-target store) */
uint8_t orc_unorm8(float x);            /* UNORM8 store */
uint16_t orc_f32_to_f16(float x);
float orc_f16_to_f32(uint16_t h);
int orc_num_threads(void);
void orc_set_num_threads(int n);   /* OpenMP team size of the parallel loops (bench: pick the fastest) */

#ifdef __cplusplus
}
#endif
#endif
