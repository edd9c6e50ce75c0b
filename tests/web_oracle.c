/*
 * web_oracle.c -- CPU ORACLE for web view node textures (TEST INFRASTRUCTURE ONLY, NOT PRODUCT CODE).
 *
 * WebRenderer::render (smelter-render/src/transformations/web_renderer/renderer.rs:78-134) with WebRendererShader::render
 * (shader.rs:53-114) and render_website.wgsl.  Written from those sources and from the numeric contract as
 * tests/oracle_nc.h states it (NC-1 .. NC-6u), with NC-7's rasterisation restated here.
 *
 *   no frame:   the node texture is left as it is (transparent from its creation)
 *   planes:     NativeEmbeddingOverContent  the page, then child k at rect k for k < min(children, rects)
 *               NativeEmbeddingUnderContent those children, then the page
 *               the first pass clears to transparent; each pass blends into the texture and stores 8 bits
 *   matrix:     the page: identity.  A child: vertices_transformation_matrix (transformation_matrices.rs:14-68) in f32,
 *               in nalgebra's order, rotation 0: with sx = W/2, sy = H/2
 *                 m00 = (1/sx) * (sx * (w / W))          m03 = (1/sx) * (-(W/2) + (x + w/2))
 *                 m11 = (1/sy) * (sy * (h / H))          m13 = (1/sy) * (H/2 - (y + h/2))
 *   vertex:     the plane's corners (+-1, +-1) -> clip (m03 +- m00, m13 +- m11) -> target pixels by the viewport transform
 *               X = fma(x_clip, sx, sx), Y = fma(-y_clip, sy, sy); tex_coords (0, 0) at clip corner (-1, +1), (1, 1) at (+1, -1)
 *   raster:     NC-7: corners snapped to 1/256 px, pixel (px, py) covered iff its centre lies in [x0, x1) x [y0, y1) of the
 *               snapped box; a quad mirrored on exactly one axis faces back and is culled (cull_mode Back)
 *   fragment:   (u, v) = ((px + .5 - X0) / (X1 - X0), (py + .5 - Y0) / (Y1 - Y0)); the bare textureSample with the
 *               linear / ClampToEdge sampler (NC-6) through the view: GpuOptimized decodes the sRGB colour bytes (NC-3),
 *               CpuOptimized filters the bytes (NC-6u).  The page's sample swaps b and r (its bytes are BGRA).  A missing
 *               child texture is the 1 x 1 transparent default_empty_view.
 *   blend:      PREMULTIPLIED_ALPHA_BLENDING through the target view, per plane (NC-2 / NC-4 stores).
 */
#include <string.h>

#include "oracle_nc.h"

static long long snap256(float v) {
    v = fminf(fmaxf(v, -1e7f), 1e7f);
    return (long long)rintf(v * 256.0f);
}

/* first pixel whose centre 256 * p + 128 is >= the snapped coordinate s */
static long long first_px(long long s) {
    long long a = s - 128, q = a / 256, r = a % 256;
    return q + (r > 0 ? 1 : 0);
}

static void draw_plane(uint8_t *out, int W, int H, int mode, float m00, float m03, float m11, float m13, const uint8_t *tex,
                       int tw, int th, const int order[4]) {
    const float sx = (float)W / 2.0f, sy = (float)H / 2.0f;
    const float X0 = fmaf(m03 - m00, sx, sx), X1 = fmaf(m03 + m00, sx, sx);
    const float Y0 = fmaf(-(m13 + m11), sy, sy), Y1 = fmaf(-(m13 - m11), sy, sy);
    if (!(isfinite(X0) && isfinite(X1) && isfinite(Y0) && isfinite(Y1))) return;
    if ((X1 < X0) != (Y1 < Y0)) return;   /* back-facing */
    long long px0 = first_px(snap256(fminf(X0, X1))), px1 = first_px(snap256(fmaxf(X0, X1)));
    long long py0 = first_px(snap256(fminf(Y0, Y1))), py1 = first_px(snap256(fmaxf(Y0, Y1)));
    if (px0 < 0) px0 = 0;
    if (py0 < 0) py0 = 0;
    if (px1 > W) px1 = W;
    if (py1 > H) py1 = H;
    const float pw = X1 - X0, ph = Y1 - Y0;
    for (long long py = py0; py < py1; py++)
        for (long long px = px0; px < px1; px++) {
            float s[4];
            sample_rgba8(tex, tw, th, order, mode, ((float)px + 0.5f - X0) / pw, ((float)py + 0.5f - Y0) / ph, s);
            blend(out + ((size_t)py * W + px) * 4, s, mode);
        }
}

/* out: W x H RGBA8, the node texture before the render (updated in place when there is a frame).  bgra: the page (NULL: no
 * frame).  children[k]: child k's node texture, RGBA8 of child_w[k] x child_h[k] (NULL: the empty view).  rects: 4 doubles
 * (x, y, width, height) per rect.  embedding: 1 over content, 2 under content.  mode: 0 GpuOptimized, 1 CpuOptimized. */
void orc_render_web(int W, int H, int mode, int embedding, const uint8_t *bgra, const uint8_t *const *children,
                    const int *child_w, const int *child_h, int n_children, const double *rects, int n_rects, uint8_t *out) {
    static const int rgba[4] = {0, 1, 2, 3}, bgra_order[4] = {2, 1, 0, 3};
    init_tables();
    if (!bgra) return;
    memset(out, 0, (size_t)W * H * 4);
    const int n = n_children < n_rects ? n_children : n_rects;
    const float sx = (float)W / 2.0f, sy = (float)H / 2.0f, a = 1.0f / sx, b = 1.0f / sy;
    for (int pass = 0; pass < 2; pass++) {
        const int site_pass = embedding == 1 ? 0 : 1;
        if (pass == site_pass) {
            draw_plane(out, W, H, mode, 1.0f, 0.0f, 1.0f, 0.0f, bgra, W, H, bgra_order);
            continue;
        }
        for (int k = 0; k < n; k++) {
            const float x = (float)rects[4 * k], y = (float)rects[4 * k + 1];
            const float w = (float)rects[4 * k + 2], h = (float)rects[4 * k + 3];
            const float tx = -((float)W / 2.0f) + (x + w / 2.0f), ty = (float)H / 2.0f - (y + h / 2.0f);
            draw_plane(out, W, H, mode, a * (sx * (w / (float)W)), a * tx, b * (sy * (h / (float)H)), b * ty, children[k],
                       child_w[k], child_h[k], rgba);
        }
    }
}
