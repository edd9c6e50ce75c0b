/*
 * web_oracle.c -- CPU ORACLE for web view node textures (TEST INFRASTRUCTURE ONLY, NOT PRODUCT CODE).
 *
 * WebRenderer::render (smelter-render/src/transformations/web_renderer/renderer.rs:78-134) with WebRendererShader::render
 * (shader.rs:53-114) and render_website.wgsl.  Written from those sources and from the numeric contract of
 * oracle/smelter_oracle.c (NC-1 .. NC-7), which it restates for the steps it needs; it lives beside the tests because the
 * committed oracle is the yardstick of every other test and stays as it is.  tests/oracle_web.py compiles it
 * (-ffp-contract=off: only fmaf() is fused).
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
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

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

/* textureSample of a w x h RGBA8 texture (channel order `order`: the byte of output channel k is order[k]) */
static void sample(const uint8_t *t, int w, int h, const int order[4], int mode, float u, float v, float out[4]) {
    static const uint8_t empty[4] = {0, 0, 0, 0};
    if (!t) { t = empty; w = h = 1; }
    int x0, x1, y0, y1;
    float fx, fy;
    tap(u, w, &x0, &x1, &fx);
    tap(v, h, &y0, &y1, &fy);
    const uint8_t *p00 = t + ((size_t)y0 * w + x0) * 4, *p10 = t + ((size_t)y0 * w + x1) * 4;
    const uint8_t *p01 = t + ((size_t)y1 * w + x0) * 4, *p11 = t + ((size_t)y1 * w + x1) * 4;
    for (int k = 0; k < 4; k++) {
        const int b = order[k];
        if (mode != 0) out[k] = lerp2_u8(p00[b], p10[b], p01[b], p11[b], fx, fy);
        else if (k == 3) out[k] = lerp2(u8n[p00[b]], u8n[p10[b]], u8n[p01[b]], u8n[p11[b]], fx, fy);
        else out[k] = lerp2(dec[p00[b]], dec[p10[b]], dec[p01[b]], dec[p11[b]], fx, fy);
    }
}

static void blend(uint8_t *d, const float src[4], int mode) {   /* PREMULTIPLIED_ALPHA_BLENDING */
    float s[4];
    for (int k = 0; k < 4; k++) s[k] = clamp01(src[k]);
    const float ia = 1.0f - s[3];
    for (int k = 0; k < 3; k++)
        d[k] = mode == 0 ? store_srgb(fmaf(dec[d[k]], ia, s[k])) : store_unorm(fmaf(u8n[d[k]], ia, s[k]));
    d[3] = store_unorm(fmaf(u8n[d[3]], ia, s[3]));
}

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
            sample(tex, tw, th, order, mode, ((float)px + 0.5f - X0) / pw, ((float)py + 0.5f - Y0) / ph, s);
            blend(out + ((size_t)py * W + px) * 4, s, mode);
        }
}

/* out: W x H RGBA8, the node texture before the render (updated in place when there is a frame).  bgra: the page (NULL: no
 * frame).  children[k]: child k's node texture, RGBA8 of child_w[k] x child_h[k] (NULL: the empty view).  rects: 4 doubles
 * (x, y, width, height) per rect.  embedding: 1 over content, 2 under content.  mode: 0 GpuOptimized, 1 CpuOptimized. */
void orc_render_web(int W, int H, int mode, int embedding, const uint8_t *bgra, const uint8_t *const *children,
                    const int *child_w, const int *child_h, int n_children, const double *rects, int n_rects, uint8_t *out) {
    static const int rgba[4] = {0, 1, 2, 3}, bgra_order[4] = {2, 1, 0, 3};
    init();
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
