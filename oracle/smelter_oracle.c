/*
 * smelter_oracle.c -- CPU ORACLE (TEST INFRASTRUCTURE ONLY, NOT PRODUCT CODE).  See the header.
 *
 * Literal, multi-pass restatement of the reference compositor: every intermediate texture the
 * reference materialises (RGBA8 node textures, Rgba16Float resampler scratch, the sRGB render
 * target that is read-modified-written once per layout) is materialised here too, so every
 * quantisation point of the reference chain exists at the same place.
 *
 * Numeric contract for behaviour the reference delegates to wgpu / the GPU (DESIGN.md section 3):
 *   NC-1 UNORM8 fetch      v/255.0f (IEEE f32 division)
 *   NC-2 UNORM8 store      rint(clamp(x,0,1)*255.0f), round-half-even, NaN -> 0
 *   NC-3 sRGB8 fetch       f32( eotf_f64(v/255) )  (exact 256-entry table)
 *   NC-4 sRGB8 store       number of k in 0..254 with x >= f32(eotf_f64((k+.5)/255))  (ideal encode + RN)
 *   NC-5 Rgba16Float store round-to-nearest-even f32 -> f16
 *   NC-6u UNORM8 views     linear filter in exact integer arithmetic on the 8-bit texels, rounded once (see filter_u8)
 *   NC-6 linear sampler    texel coord c = t*dim-.5 (f32); weights quantised to 8 fractional bits
 *                          (what llvmpipe's AoS path and NVIDIA's texture units both do); taps clamped;
 *                          h0=fma(t10,fx,t00*(1-fx)) h1=fma(t11,fx,t01*(1-fx)) v=fma(h1,fy,h0*(1-fy))
 *   NC-7 rasteriser        vertices snapped to 1/256 px, pixel centre sampled, top-left rule
 *   NC-8 sin/cos           correctly rounded f32: (float)sin((double)x)
 *   "a*b+c" written as fmaf() below is a single fused op; everything else rounds per operation
 *   (build with -ffp-contract=off).
 */
#include "smelter_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* ------------------------------------------------------------------------------------------ */
/* tables                                                                                      */
/* ------------------------------------------------------------------------------------------ */
static float g_u8n[256];     /* NC-1 */
static float g_dec[256];     /* NC-3 */
static float g_enc_thr[255]; /* NC-4 */
static int g_init_done = 0;

static double eotf_f64(double c) {
    return c <= 0.04045 ? c / 12.92 : pow((c + 0.055) / 1.055, 2.4);
}

__attribute__((constructor)) void orc_init(void) {
    if (g_init_done) return;
    for (int b = 0; b < 256; b++) {
        g_u8n[b] = (float)b / 255.0f;
        g_dec[b] = (float)eotf_f64((double)b / 255.0);
    }
    for (int k = 0; k < 255; k++) g_enc_thr[k] = (float)eotf_f64(((double)k + 0.5) / 255.0);
    g_init_done = 1;
}

void orc_set_num_threads(int n) {
#ifdef _OPENMP
    if (n >= 1) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

int orc_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

static inline float clamp01(float x) { return fminf(fmaxf(x, 0.0f), 1.0f); } /* NaN -> 0 */

uint8_t orc_unorm8(float x) { return (uint8_t)rintf(clamp01(x) * 255.0f); }

float orc_srgb_decode_u8(uint8_t v) { return g_dec[v]; }

uint8_t orc_srgb_encode_u8(float lin) {
    float x = clamp01(lin);
    int lo = 0, hi = 255; /* count of thresholds <= x, thresholds ascending */
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (x >= g_enc_thr[mid]) lo = mid + 1; else hi = mid;
    }
    return (uint8_t)lo;
}

uint16_t orc_f32_to_f16(float x) { /* NC-5, round-to-nearest-even incl. subnormals */
    uint32_t b; memcpy(&b, &x, 4);
    uint32_t sign = (b >> 16) & 0x8000u;
    uint32_t a = b & 0x7fffffffu;
    if (a >= 0x7f800000u) return (uint16_t)(sign | (a > 0x7f800000u ? 0x7e00u : 0x7c00u));
    if (a >= 0x477ff000u) return (uint16_t)(sign | 0x7c00u); /* rounds to >= 65520 -> inf */
    if (a < 0x38800000u) { /* subnormal half or zero */
        if (a < 0x33000000u) return (uint16_t)sign; /* < 2^-25 -> 0 */
        uint32_t e = a >> 23;
        uint32_t m = (a & 0x7fffffu) | 0x800000u;
        uint32_t shift = 126 - e; /* 14..24 */
        uint32_t q = m >> shift, r = m & ((1u << shift) - 1u), half = 1u << (shift - 1);
        if (r > half || (r == half && (q & 1u))) q++;
        return (uint16_t)(sign | q);
    }
    uint32_t h = ((a >> 13) - (112u << 10));
    uint32_t r = a & 0x1fffu;
    if (r > 0x1000u || (r == 0x1000u && (h & 1u))) h++;
    return (uint16_t)(sign | h);
}

float orc_f16_to_f32(uint16_t h) {
    uint32_t sign = ((uint32_t)h & 0x8000u) << 16, e = (h >> 10) & 0x1fu, m = h & 0x3ffu, b;
    if (e == 0) {
        if (m == 0) b = sign;
        else { float f = (float)m * (1.0f / 16777216.0f); memcpy(&b, &f, 4); b |= sign; }
    } else if (e == 31) b = sign | 0x7f800000u | (m << 13);
    else b = sign | ((e + 112u) << 23) | (m << 13);
    float f; memcpy(&f, &b, 4); return f;
}

static inline float sin_cr(float x) { return (float)sin((double)x); } /* NC-8 */
static inline float cos_cr(float x) { return (float)cos((double)x); }

/* ------------------------------------------------------------------------------------------ */
/* NC-6: the one sampler the reference uses everywhere (wgpu/common_pipeline.rs:56-65):        */
/* min/mag Linear, ClampToEdge                                                                 */
/* ------------------------------------------------------------------------------------------ */
typedef struct { int i0, i1; float f; } lin_tap;

static inline lin_tap linear_tap(float t, int dim) {
    lin_tap r;
    float c = t * (float)dim - 0.5f;
    if (!(c == c)) { r.i0 = r.i1 = 0; r.f = 0.0f; return r; }
    c = fminf(fmaxf(c, -2.0f), (float)dim + 1.0f);
    float fl = floorf(c);
    float f = c - fl;
    r.f = rintf(f * 256.0f) * (1.0f / 256.0f);
    int i0 = (int)fl, i1 = i0 + 1;
    r.i0 = i0 < 0 ? 0 : (i0 > dim - 1 ? dim - 1 : i0);
    r.i1 = i1 < 0 ? 0 : (i1 > dim - 1 ? dim - 1 : i1);
    return r;
}

static inline float bilerp(float t00, float t10, float t01, float t11, float fx, float fy) {
    float h0 = fmaf(t10, fx, t00 * (1.0f - fx));
    float h1 = fmaf(t11, fx, t01 * (1.0f - fx));
    return fmaf(h1, fy, h0 * (1.0f - fy));
}

/* NC-6u: linear filtering of a UNORM8 (non-sRGB) view is carried out on the 8-bit texel integers with the
 * 8-bit weights in EXACT arithmetic and rounded once: value = f32( N / (255 * 65536) ),
 * N = (t00*(256-wx) + t10*wx)*(256-wy) + (t01*(256-wx) + t11*wx)*wy.  This is the infinitely precise result
 * of the fixed-point filter of a texture unit, independent of any float operation order; a texel hit gives
 * exactly v/255 (NC-1). */
static inline float filter_u8(int t00, int t10, int t01, int t11, float fx, float fy) {
    int wx = (int)(fx * 256.0f), wy = (int)(fy * 256.0f); /* fx, fy are multiples of 1/256 */
    int n = (t00 * (256 - wx) + t10 * wx) * (256 - wy) + (t01 * (256 - wx) + t11 * wx) * wy;
    return (float)n / 16711680.0f;
}

/* bilinear fetch of one 8-bit channel, UNORM view */
static inline float sample_u8_plane(const uint8_t *p, int w, int h, int pitch_px, int stride,
                                    int ch, float tx, float ty) {
    lin_tap ax = linear_tap(tx, w), ay = linear_tap(ty, h);
    const uint8_t *r0 = p + (size_t)ay.i0 * pitch_px * stride, *r1 = p + (size_t)ay.i1 * pitch_px * stride;
    return filter_u8(r0[ax.i0 * stride + ch], r0[ax.i1 * stride + ch], r1[ax.i0 * stride + ch],
                     r1[ax.i1 * stride + ch], ax.f, ay.f);
}

/* ------------------------------------------------------------------------------------------ */
/* K1 / K2: YUV -> RGBA8 node texture                                                          */
/* planar_yuv_to_rgba.wgsl:35-58, nv12_to_rgba.wgsl:26-48; stored through the Rgba8Unorm view   */
/* ("write to sRGB texture as if it was linear", input_texture/planar_yuv.rs:51)               */
/* ------------------------------------------------------------------------------------------ */
#define K16 (16.0f / 255.0f)
#define RCP_Y (1.0f / 0.85882352941f)  /* x / const is evaluated as x * (1/const) */
#define RCP_C (1.0f / 0.87843137254f)

static inline void yuv_to_rgba_px(float y, float u, float v, int full_range, uint8_t *out) {
    if (!full_range) {
        y = clamp01((y - K16) * RCP_Y);
        u = clamp01((u - K16) * RCP_C);
        v = clamp01((v - K16) * RCP_C);
    }
    float um = u - 0.5f, vm = v - 0.5f;
    float r = fmaf(1.5748f, vm, y);
    float g = fmaf(-0.4681f, vm, fmaf(-0.1873f, um, y));
    float b = fmaf(1.8556f, um, y);
    out[0] = orc_unorm8(r); out[1] = orc_unorm8(g); out[2] = orc_unorm8(b); out[3] = 255;
}

/* any planar variant: the chroma planes are cw x ch (420: w/2 x h/2, 422: w/2 x h, 444: w x h;
 * texture/planar_yuv.rs:64-83) and all three planes are sampled at the SAME normalised coordinate
 * (planar_yuv_to_rgba.wgsl:37-39) */
void orc_yuv_planar_to_rgba(const uint8_t *y, const uint8_t *u, const uint8_t *v, int w, int h, int cw, int ch,
                            int full_range, uint8_t *rgba) {
#pragma omp parallel for schedule(static)
    for (int py = 0; py < h; py++) {
        float ty = ((float)py + 0.5f) / (float)h;
        for (int px = 0; px < w; px++) {
            float tx = ((float)px + 0.5f) / (float)w;
            float yy = sample_u8_plane(y, w, h, w, 1, 0, tx, ty);
            float uu = sample_u8_plane(u, cw, ch, cw, 1, 0, tx, ty);
            float vv = sample_u8_plane(v, cw, ch, cw, 1, 0, tx, ty);
            yuv_to_rgba_px(yy, uu, vv, full_range, rgba + ((size_t)py * w + px) * 4);
        }
    }
}

void orc_yuv420_to_rgba(const uint8_t *y, const uint8_t *u, const uint8_t *v, int w, int h,
                        int full_range, uint8_t *rgba) {
    orc_yuv_planar_to_rgba(y, u, v, w, h, w / 2, h / 2, full_range, rgba); /* texture/planar_yuv.rs:66-71 */
}

/* K3: interleaved 4:2:2 (interleaved_uyvy_to_rgba.wgsl:24-61, interleaved_yuyv_to_rgba.wgsl:24-61).  The frame is
 * uploaded as an Rgba8Unorm texture of (w/2) x h texels, one texel = two pixels (texture/interleaved_yuv422.rs:12-36);
 * the fragment shader turns its interpolated coordinate back into a column index, fetches the texel at its centre
 * (NC-6: the residual bilinear weight rounds to 0) and picks the first or second luma.  Always limited range. */
void orc_interleaved422_to_rgba(const uint8_t *data, int w, int h, int yuyv, uint8_t *rgba) {
    int dimx = w / 2;
    if (dimx < 1) return;
    const float eps = 0.0001f, half_pixel_width = 0.5f / (float)dimx;
#pragma omp parallel for schedule(static)
    for (int py = 0; py < h; py++) {
        float ty = ((float)py + 0.5f) / (float)h;
        for (int px = 0; px < w; px++) {
            float tx = ((float)px + 0.5f) / (float)w;
            float xf = ((tx * (float)dimx - half_pixel_width) + eps) * 2.0f;
            uint32_t x_pos = xf >= 4294967296.0f ? 0xffffffffu : (xf > 0.0f ? (uint32_t)xf : 0u); /* u32(): saturating */
            float tcx = (float)(x_pos / 2u) / (float)dimx + half_pixel_width;
            float t[4];
            for (int c = 0; c < 4; c++) t[c] = sample_u8_plane(data, dimx, h, dimx, 4, c, tcx, ty);
            float uu, vv, yy;
            if (yuyv) { yy = (x_pos & 1u) ? t[2] : t[0]; uu = t[1]; vv = t[3]; }
            else { yy = (x_pos & 1u) ? t[3] : t[1]; uu = t[0]; vv = t[2]; }
            yuv_to_rgba_px(yy, uu, vv, 0, rgba + ((size_t)py * w + px) * 4);
        }
    }
}

void orc_nv12_to_rgba(const uint8_t *y, const uint8_t *uv, int w, int h, uint8_t *rgba) {
    int cw = w / 2, ch = h / 2; /* texture/nv12.rs:77-88 */
#pragma omp parallel for schedule(static)
    for (int py = 0; py < h; py++) {
        float ty = ((float)py + 0.5f) / (float)h;
        for (int px = 0; px < w; px++) {
            float tx = ((float)px + 0.5f) / (float)w;
            float yy = sample_u8_plane(y, w, h, w, 1, 0, tx, ty);
            float uu = sample_u8_plane(uv, cw, ch, cw, 2, 0, tx, ty);
            float vv = sample_u8_plane(uv, cw, ch, cw, 2, 1, tx, ty);
            yuv_to_rgba_px(yy, uu, vv, 0, rgba + ((size_t)py * w + px) * 4);
        }
    }
}

void orc_bgra_to_rgba(const uint8_t *s, int w, int h, uint8_t *d) { /* bgra_to_rgba.wgsl: sample.bgra */
    for (size_t i = 0; i < (size_t)w * h; i++) {
        d[i * 4 + 0] = s[i * 4 + 2]; d[i * 4 + 1] = s[i * 4 + 1];
        d[i * 4 + 2] = s[i * 4 + 0]; d[i * 4 + 3] = s[i * 4 + 3];
    }
}

void orc_argb_to_rgba(const uint8_t *s, int w, int h, uint8_t *d) { /* argb_to_rgba.wgsl: sample.gbar */
    for (size_t i = 0; i < (size_t)w * h; i++) {
        d[i * 4 + 0] = s[i * 4 + 1]; d[i * 4 + 1] = s[i * 4 + 2];
        d[i * 4 + 2] = s[i * 4 + 3]; d[i * 4 + 3] = s[i * 4 + 0];
    }
}

/* ------------------------------------------------------------------------------------------ */
/* K10 / K11: RGBA8 (raw stored bytes, node_texture.rs:104-116) -> YUV                          */
/* rgba_to_yuv.wgsl:26-54 (3 passes), rgba_to_nv12.wgsl:25-52                                   */
/* ------------------------------------------------------------------------------------------ */
static inline void sample_rgb_raw(const uint8_t *rgba, int w, int h, float tx, float ty, float rgb[3]) {
    for (int c = 0; c < 3; c++) rgb[c] = sample_u8_plane(rgba, w, h, w, 4, c, tx, ty);
}
static inline float to_y(const float c[3]) {
    float y = fmaf(c[2], 0.0722f, fmaf(c[1], 0.7152f, c[0] * 0.2126f));
    return fmaf(y, 0.85882352941f, K16);
}
static inline float to_u(const float c[3]) {
    float u = fmaf(c[2], 0.5f, fmaf(c[1], -0.3854f, c[0] * -0.1146f));
    return fmaf(u + 0.5f, 0.87843137254f, K16);
}
static inline float to_v(const float c[3]) {
    float v = fmaf(c[2], -0.0458f, fmaf(c[1], -0.4542f, c[0] * 0.5f));
    return fmaf(v + 0.5f, 0.87843137254f, K16);
}

/* The converters draw a full-screen quad into planes of the OUTPUT size and sample the root texture
 * with the linear sampler, so a root whose size differs from the output is rescaled here
 * (render_loop.rs:68-73, output_texture.rs:49-58). */
static void rgba_to_y_plane(const uint8_t *rgba, int sw, int sh, int w, int h, uint8_t *y) {
#pragma omp parallel for schedule(static)
    for (int py = 0; py < h; py++)
        for (int px = 0; px < w; px++) {
            float c[3];
            sample_rgb_raw(rgba, sw, sh, ((float)px + 0.5f) / (float)w, ((float)py + 0.5f) / (float)h, c);
            y[(size_t)py * w + px] = orc_unorm8(to_y(c));
        }
}

/* planar 420 / 422 / 444 outputs differ only in the chroma plane size cw x ch (texture/planar_yuv.rs:64-83);
 * every plane is a full-target draw sampling the source at its own pixel centres (rgba_to_yuv.rs:67-116) */
void orc_rgba_to_yuv_planar_scaled(const uint8_t *rgba, int sw, int sh, int w, int h, int cw, int ch, uint8_t *y,
                                   uint8_t *u, uint8_t *v) {
    rgba_to_y_plane(rgba, sw, sh, w, h, y);
#pragma omp parallel for schedule(static)
    for (int py = 0; py < ch; py++)
        for (int px = 0; px < cw; px++) {
            float c[3];
            sample_rgb_raw(rgba, sw, sh, ((float)px + 0.5f) / (float)cw, ((float)py + 0.5f) / (float)ch, c);
            u[(size_t)py * cw + px] = orc_unorm8(to_u(c));
            v[(size_t)py * cw + px] = orc_unorm8(to_v(c));
        }
}

void orc_rgba_to_yuv420_scaled(const uint8_t *rgba, int sw, int sh, int w, int h, uint8_t *y, uint8_t *u,
                               uint8_t *v) {
    orc_rgba_to_yuv_planar_scaled(rgba, sw, sh, w, h, w / 2, h / 2, y, u, v);
}

void orc_rgba_to_nv12_scaled(const uint8_t *rgba, int sw, int sh, int w, int h, uint8_t *y, uint8_t *uv) {
    int cw = w / 2, ch = h / 2;
    rgba_to_y_plane(rgba, sw, sh, w, h, y);
#pragma omp parallel for schedule(static)
    for (int py = 0; py < ch; py++)
        for (int px = 0; px < cw; px++) {
            float c[3];
            sample_rgb_raw(rgba, sw, sh, ((float)px + 0.5f) / (float)cw, ((float)py + 0.5f) / (float)ch, c);
            uv[((size_t)py * cw + px) * 2 + 0] = orc_unorm8(to_u(c));
            uv[((size_t)py * cw + px) * 2 + 1] = orc_unorm8(to_v(c));
        }
}

void orc_rgba_to_yuv420(const uint8_t *rgba, int w, int h, uint8_t *y, uint8_t *u, uint8_t *v) {
    orc_rgba_to_yuv420_scaled(rgba, w, h, w, h, y, u, v);
}

void orc_rgba_to_nv12(const uint8_t *rgba, int w, int h, uint8_t *y, uint8_t *uv) {
    orc_rgba_to_nv12_scaled(rgba, w, h, w, h, y, uv);
}

void orc_rgb_to_yuv_bytes(uint8_t r, uint8_t g, uint8_t b, uint8_t out[3]) {
    /* RGBColor::to_yuv, scene/types.rs:28-42: plain (unfused) f32 arithmetic on the CPU */
    float rf = (float)r / 255.0f, gf = (float)g / 255.0f, bf = (float)b / 255.0f;
    float y = rf * 0.2126f + gf * 0.7152f + bf * 0.0722f;
    float u = rf * -0.1146f + gf * -0.3854f + bf * 0.5f;
    float v = rf * 0.5f + gf * -0.4542f + bf * -0.0458f;
    out[0] = orc_unorm8(clamp01((y * 0.85882354f) + (16.0f / 255.0f)));
    out[1] = orc_unorm8(clamp01(((u + 0.5f) * 0.8784314f) + (16.0f / 255.0f)));
    out[2] = orc_unorm8(clamp01(((v + 0.5f) * 0.8784314f) + (16.0f / 255.0f)));
}

/* harness/utils.rs:31-65 -- the CPU inverse every reference snapshot goes through */
void orc_harness_yuv420_to_rgba(const uint8_t *yp, const uint8_t *up, const uint8_t *vp, int w,
                                int h, uint8_t *rgba) {
    int cw_ = w - (w % 2), ch_ = h - (h % 2);
    size_t o = 0;
    for (int i = 0; i < ch_; i++)
        for (int j = 0; j < cw_; j++) {
            float y = (float)yp[(size_t)i * w + j];
            float u = (float)up[(size_t)(i / 2) * (w / 2) + (j / 2)];
            float v = (float)vp[(size_t)(i / 2) * (w / 2) + (j / 2)];
            y = fminf(fmaxf((y - 16.0f) / 0.85882354f, 0.0f), 255.0f);
            u = fminf(fmaxf((u - 16.0f) / 0.8784314f, 0.0f), 255.0f);
            v = fminf(fmaxf((v - 16.0f) / 0.8784314f, 0.0f), 255.0f);
            float r = fminf(fmaxf(y + 1.5748f * (v - 128.0f), 0.0f), 255.0f);
            float g = fminf(fmaxf(y - 0.1873f * (u - 128.0f) - 0.4681f * (v - 128.0f), 0.0f), 255.0f);
            float b = fminf(fmaxf(y + 1.8556f * (u - 128.0f), 0.0f), 255.0f);
            rgba[o++] = (uint8_t)r; rgba[o++] = (uint8_t)g; rgba[o++] = (uint8_t)b; rgba[o++] = 255;
        }
}

/* ------------------------------------------------------------------------------------------ */
/* K7 / K8: Lanczos3 resampler                                                                 */
/* ------------------------------------------------------------------------------------------ */
#define KERNEL_BUDGET 4.0f           /* resampler.rs:19 */
#define MAX_PREDECIMATE_LEVELS 16    /* resampler.rs:23 */
#define PI_F 3.14159265359f          /* resample.wgsl:29 */

static int is_same_px(float a, float b) { return fabsf(a - b) < 0.001f; } /* resampler.rs:398-400 */

/* AxisMapping::as_direct, resampler.rs:72-76 ; returns 1 and *off when direct */
static int as_direct(float crop_offset, float crop_len, int dst_len, int *off) {
    float rounded = roundf(crop_offset); /* f32::round: half away from zero */
    if (is_same_px(crop_len, (float)dst_len) && is_same_px(crop_offset, rounded)) {
        *off = (int)rounded;
        return 1;
    }
    return 0;
}

int orc_predecimate_levels(float crop_len, int dst_len) { /* resampler.rs:56-58 */
    float scale = crop_len / (float)dst_len;
    float l = ceilf(log2f(scale / KERNEL_BUDGET));
    l = (l > 0.0f) ? l : 0.0f; /* f32::max(NaN,0)=0 */
    uint32_t lv = (l >= 4294967296.0f) ? 0xffffffffu : (uint32_t)l; /* saturating `as u32` */
    return (int)(lv < MAX_PREDECIMATE_LEVELS ? lv : MAX_PREDECIMATE_LEVELS);
}

int orc_plan_passes(float crop_left, float crop_top, float crop_w, float crop_h, int dst_w,
                    int dst_h, int axis_out[2], int perp_out[2]) { /* resampler.rs:122-145 */
    int hoff = 0, voff = 0;
    int hd = as_direct(crop_left, crop_w, dst_w, &hoff);
    int vd = as_direct(crop_top, crop_h, dst_h, &voff);
    if (hd && vd) return 0;
    if (!hd && vd) { axis_out[0] = 0; perp_out[0] = voff; return 1; }
    if (hd && !vd) { axis_out[0] = 1; perp_out[0] = hoff; return 1; }
    float hs = crop_w / (float)dst_w, vs = crop_h / (float)dst_h;
    if (vs > hs) { axis_out[0] = 1; axis_out[1] = 0; } else { axis_out[0] = 0; axis_out[1] = 1; }
    perp_out[0] = perp_out[1] = 0;
    return 2;
}

int orc_resample_taps(float scale) { /* resample.wgsl:43-48 */
    float kernel_scale = fmaxf(scale, 1.0f);
    float support = 3.0f * kernel_scale;
    return (int)ceilf(2.0f * support) + 1;
}

int orc_resample_weights(float scale, float offset, int out_coord, float *weights,
                         float *weight_sum) { /* resample.wgsl:42-86 */
    float kernel_scale = fmaxf(scale, 1.0f);
    float inv_k = 1.0f / kernel_scale;
    float support = 3.0f * kernel_scale;
    float center = (offset + ((float)out_coord + 0.5f) * scale) - 0.5f;
    float first = ceilf(center - support);
    int taps = (int)ceilf(2.0f * support) + 1;
    float x0 = (first - center) * inv_k;
    float s1 = sin_cr(PI_F * x0), c1 = cos_cr(PI_F * x0);
    float s3 = sin_cr(PI_F * x0 / 3.0f), c3 = cos_cr(PI_F * x0 / 3.0f);
    float sd1 = sin_cr(PI_F * inv_k), cd1 = cos_cr(PI_F * inv_k);
    float sd3 = sin_cr(PI_F * inv_k / 3.0f), cd3 = cos_cr(PI_F * inv_k / 3.0f);
    const float pi2 = PI_F * PI_F;
    float wsum = 0.0f;
    for (int t = 0; t < taps; t++) {
        float x = x0 + (float)t * inv_k;
        float w = 0.0f;
        if (fabsf(x) < 1e-5f) w = 1.0f;
        else if (fabsf(x) < 3.0f) w = ((3.0f * s1) * s3) / ((pi2 * x) * x);
        weights[t] = w;
        wsum += w;
        float ns1 = s1 * cd1 + c1 * sd1;
        c1 = c1 * cd1 - s1 * sd1;
        s1 = ns1;
        float ns3 = s3 * cd3 + c3 * sd3;
        c3 = c3 * cd3 - s3 * sd3;
        s3 = ns3;
    }
    *weight_sum = wsum;
    return (int)first;
}

/* a linear-light float texture view used inside the resampler */
typedef struct {
    int w, h;
    const uint8_t *srgb8; /* sRGB-encoded RGBA8 (fetched through the srgb view: decode) or */
    const uint16_t *f16;  /* Rgba16Float */
} rs_src;

static inline void rs_load(const rs_src *s, int x, int y, float out[4]) {
    if (s->srgb8) {
        const uint8_t *p = s->srgb8 + ((size_t)y * s->w + x) * 4;
        out[0] = g_dec[p[0]]; out[1] = g_dec[p[1]]; out[2] = g_dec[p[2]]; out[3] = g_u8n[p[3]];
    } else {
        const uint16_t *p = s->f16 + ((size_t)y * s->w + x) * 4;
        for (int c = 0; c < 4; c++) out[c] = orc_f16_to_f32(p[c]);
    }
}

/* one resample.wgsl pass: target (tw x th) f16 or srgb8 */
static void rs_kernel_pass(const rs_src *s, int axis, float scale, float offset, int perp_offset,
                           int tw, int th, uint16_t *dst_f16, uint8_t *dst_srgb8) {
    int taps = orc_resample_taps(scale);
    int n_out = axis == 1 ? th : tw;
    float *wtab = (float *)malloc(sizeof(float) * (size_t)taps * n_out);
    float *inv = (float *)malloc(sizeof(float) * n_out);
    int *first = (int *)malloc(sizeof(int) * n_out);
    for (int o = 0; o < n_out; o++) {
        float ws;
        first[o] = orc_resample_weights(scale, offset, o, wtab + (size_t)o * taps, &ws);
        inv[o] = 1.0f / ws; /* `sum / weight_sum` evaluated as sum * (1/weight_sum) */
    }
    int max_src = (axis == 1 ? s->h : s->w) - 1;
    int max_perp = (axis == 1 ? s->w : s->h) - 1;
#pragma omp parallel for schedule(static)
    for (int py = 0; py < th; py++)
        for (int px = 0; px < tw; px++) {
            int o = axis == 1 ? py : px;
            int perp = (axis == 1 ? px : py) + perp_offset;
            perp = perp < 0 ? 0 : (perp > max_perp ? max_perp : perp);
            const float *w = wtab + (size_t)o * taps;
            float sum[4] = {0, 0, 0, 0};
            for (int t = 0; t < taps; t++) {
                int src = first[o] + t;
                src = src < 0 ? 0 : (src > max_src ? max_src : src);
                float tx[4];
                if (axis == 1) rs_load(s, perp, src, tx); else rs_load(s, src, perp, tx);
                for (int c = 0; c < 4; c++) sum[c] = fmaf(tx[c], w[t], sum[c]);
            }
            size_t di = ((size_t)py * tw + px) * 4;
            for (int c = 0; c < 4; c++) {
                float r = sum[c] * inv[o];
                if (dst_f16) dst_f16[di + c] = orc_f32_to_f16(r);
                else dst_srgb8[di + c] = c < 3 ? orc_srgb_encode_u8(r) : orc_unorm8(r);
            }
        }
    free(wtab); free(inv); free(first);
}

/* downsample.wgsl:28-41 */
static void rs_box_pass(const rs_src *s, int fx, int fy, int tw, int th, uint16_t *dst) {
    float denom = (float)((uint32_t)fx * (uint32_t)fy);
#pragma omp parallel for schedule(static)
    for (int py = 0; py < th; py++)
        for (int px = 0; px < tw; px++) {
            float sum[4] = {0, 0, 0, 0};
            for (int dy = 0; dy < fy; dy++)
                for (int dx = 0; dx < fx; dx++) {
                    int sx = px * fx + dx, sy = py * fy + dy;
                    sx = sx > s->w - 1 ? s->w - 1 : sx;
                    sy = sy > s->h - 1 ? s->h - 1 : sy;
                    float t[4];
                    rs_load(s, sx, sy, t);
                    for (int c = 0; c < 4; c++) sum[c] += t[c];
                }
            for (int c = 0; c < 4; c++) dst[((size_t)py * tw + px) * 4 + c] = orc_f32_to_f16(sum[c] / denom);
        }
}

int orc_resample(const orc_texture *src, float crop_left, float crop_top, float crop_w,
                 float crop_h, int dst_w, int dst_h, uint8_t *dst) { /* resampler.rs:305-378 */
    int axis[2], perp[2];
    if (orc_plan_passes(crop_left, crop_top, crop_w, crop_h, dst_w, dst_h, axis, perp) == 0) return 0;
    int lv[2] = {orc_predecimate_levels(crop_w, dst_w), orc_predecimate_levels(crop_h, dst_h)};
    int fac[2] = {1 << lv[0], 1 << lv[1]};
    rs_src cur = {src->width, src->height, src->data, NULL};
    uint16_t *reduced = NULL, *mid = NULL;
    if (fac[0] != 1 || fac[1] != 1) {
        int rw = (src->width + fac[0] - 1) / fac[0], rh = (src->height + fac[1] - 1) / fac[1];
        reduced = (uint16_t *)malloc((size_t)rw * rh * 8);
        rs_box_pass(&cur, fac[0], fac[1], rw, rh, reduced);
        cur.w = rw; cur.h = rh; cur.srgb8 = NULL; cur.f16 = reduced;
    }
    /* AxisMapping::on_reduced_source, resampler.rs:60-67 */
    float off[2] = {crop_left / (float)fac[0], crop_top / (float)fac[1]};
    float len[2] = {crop_w / (float)fac[0], crop_h / (float)fac[1]};
    int dlen[2] = {dst_w, dst_h};
    int n = orc_plan_passes(off[0], off[1], len[0], len[1], dst_w, dst_h, axis, perp);
    if (n == 0) { free(reduced); return 0; } /* reference: expect() panics; unreachable */
    if (n == 2) {
        int a = axis[0];
        int mw = a == 0 ? dlen[0] : cur.w, mh = a == 1 ? dlen[1] : cur.h; /* output_size */
        mid = (uint16_t *)malloc((size_t)mw * mh * 8);
        rs_kernel_pass(&cur, a, len[a] / (float)dlen[a], off[a], perp[0], mw, mh, mid, NULL);
        cur.w = mw; cur.h = mh; cur.srgb8 = NULL; cur.f16 = mid;
        axis[0] = axis[1]; perp[0] = perp[1];
    }
    int a = axis[0];
    rs_kernel_pass(&cur, a, len[a] / (float)dlen[a], off[a], perp[0], dst_w, dst_h, NULL, dst);
    free(reduced); free(mid);
    return 1;
}

/* ------------------------------------------------------------------------------------------ */
/* K9: apply_layouts.wgsl                                                                       */
/* ------------------------------------------------------------------------------------------ */
static double srgb_to_linear_host(uint8_t c) { /* wgpu/utils.rs:74-81 (note: `<`, f64) */
    double x = (double)c / 255.0;
    return x < 0.04045 ? x / 12.92 : pow((x + 0.055) / 1.055, 2.4);
}

static void shader_color(const uint8_t c[4], int mode, float out[4]) { /* wgpu/utils.rs:51-71 */
    double a = (double)c[3] / 255.0;
    if (mode == ORC_MODE_GPU_OPTIMIZED) {
        out[0] = (float)(a * srgb_to_linear_host(c[0]));
        out[1] = (float)(a * srgb_to_linear_host(c[1]));
        out[2] = (float)(a * srgb_to_linear_host(c[2]));
    } else {
        out[0] = (float)(a * (double)c[0] / 255.0);
        out[1] = (float)(a * (double)c[1] / 255.0);
        out[2] = (float)(a * (double)c[2] / 255.0);
    }
    out[3] = (float)a;
}

static inline float smoothstep_f(float e0, float e1, float x) {
    float t = clamp01((x - e0) / (e1 - e0));
    return (t * t) * (3.0f - 2.0f * t);
}

/* apply_layouts.wgsl:246-256; radius = [tl, tr, br, bl] */
static inline float rounded_rect_sdf(float dx, float dy, float sx, float sy, const float radius[4]) {
    float hx = sx / 2.0f, hy = sy / 2.0f;
    float rx, ry;
    if (dx < 0.0f) { rx = radius[0]; ry = radius[3]; } else { rx = radius[1]; ry = radius[2]; }
    if (dy < 0.0f) rx = ry;
    float qx = (fabsf(dx) - hx) + rx, qy = (fabsf(dy) - hy) + rx;
    float mx = fmaxf(qx, 0.0f), my = fmaxf(qy, 0.0f);
    return (fminf(fmaxf(qx, qy), 0.0f) + sqrtf(mx * mx + my * my)) - rx;
}

/* NC-7: quad of vertices_transformation_matrix (apply_layouts.wgsl:127-157) rasterised with
 * 8 sub-pixel bits and the top-left rule. */
typedef struct {
    int rotated;
    int64_t x0, x1, y0, y1;     /* unrotated: covered iff x0 <= 256*px+128 < x1 (same in y) */
    int64_t vx[4], vy[4];       /* rotated: snapped vertices, clockwise on screen */
    int bx0, bx1, by0, by1;     /* conservative pixel bbox [bx0,bx1) x [by0,by1) */
    float cx, cy, cs, sn;       /* centre (fb coords), cos/sin */
} quad;

static inline int64_t snap256(float v) { return (int64_t)rintf(v * 256.0f); }

static int quad_setup(quad *q, float left, float top, float w, float h, float rot_deg, int W, int H) {
    if (!(left == left) || !(top == top) || !(w == w) || !(h == h) || !(rot_deg == rot_deg)) return 0;
    if (fabsf(left) > 1e7f || fabsf(top) > 1e7f || fabsf(w) > 1e7f || fabsf(h) > 1e7f) return 0;
    float hw = w / 2.0f, hh = h / 2.0f;
    q->cx = left + hw; q->cy = top + hh;
    q->rotated = rot_deg != 0.0f;
    float minx, maxx, miny, maxy;
    if (!q->rotated) {
        q->cs = 1.0f; q->sn = 0.0f;
        q->x0 = snap256(q->cx - hw); q->x1 = snap256(q->cx + hw);
        q->y0 = snap256(q->cy - hh); q->y1 = snap256(q->cy + hh);
        minx = q->cx - hw; maxx = q->cx + hw; miny = q->cy - hh; maxy = q->cy + hh;
    } else {
        float ang = rot_deg * (PI_F / 180.0f); /* radians() */
        q->cs = cos_cr(ang); q->sn = sin_cr(ang);
        /* local y-up corners, clockwise on screen: TL, TR, BR, BL */
        const float lx[4] = {-hw, hw, hw, -hw}, ly[4] = {hh, hh, -hh, -hh};
        minx = miny = 1e30f; maxx = maxy = -1e30f;
        for (int i = 0; i < 4; i++) {
            float xr = lx[i] * q->cs - ly[i] * q->sn, yr = lx[i] * q->sn + ly[i] * q->cs;
            float X = q->cx + xr, Y = q->cy - yr;
            q->vx[i] = snap256(X); q->vy[i] = snap256(Y);
            minx = fminf(minx, X); maxx = fmaxf(maxx, X); miny = fminf(miny, Y); maxy = fmaxf(maxy, Y);
        }
    }
    float fx0 = floorf(minx) - 1.0f, fx1 = ceilf(maxx) + 1.0f, fy0 = floorf(miny) - 1.0f, fy1 = ceilf(maxy) + 1.0f;
    q->bx0 = (int)fmaxf(fx0, 0.0f); q->by0 = (int)fmaxf(fy0, 0.0f);
    q->bx1 = (int)fminf(fx1, (float)W); q->by1 = (int)fminf(fy1, (float)H);
    return q->bx0 < q->bx1 && q->by0 < q->by1;
}

static inline int quad_covers(const quad *q, int px, int py) {
    int64_t X = (int64_t)px * 256 + 128, Y = (int64_t)py * 256 + 128;
    if (!q->rotated) return X >= q->x0 && X < q->x1 && Y >= q->y0 && Y < q->y1;
    for (int i = 0; i < 4; i++) {
        int j = (i + 1) & 3;
        int64_t dx = q->vx[j] - q->vx[i], dy = q->vy[j] - q->vy[i];
        int64_t e = dx * (Y - q->vy[i]) - dy * (X - q->vx[i]);
        int top_left = (dy < 0) || (dy == 0 && dx > 0);
        if (e < 0 || (e == 0 && !top_left)) return 0;
    }
    return 1;
}

/* textureSample of the child through NodeTextureState::view() (srgb view in GpuOptimized) */
static inline void sample_node(const orc_texture *t, int mode, float tx, float ty, float out[4]) {
    static const uint8_t empty[4] = {0, 0, 0, 0}; /* default_empty_view: 1x1 transparent */
    const uint8_t *d = t && t->data ? t->data : empty;
    int w = t && t->data ? t->width : 1, h = t && t->data ? t->height : 1;
    lin_tap ax = linear_tap(tx, w), ay = linear_tap(ty, h);
    const uint8_t *p00 = d + ((size_t)ay.i0 * w + ax.i0) * 4, *p10 = d + ((size_t)ay.i0 * w + ax.i1) * 4;
    const uint8_t *p01 = d + ((size_t)ay.i1 * w + ax.i0) * 4, *p11 = d + ((size_t)ay.i1 * w + ax.i1) * 4;
    if (mode == ORC_MODE_GPU_OPTIMIZED) { /* srgb view: texels are decoded to float, then filtered (NC-6) */
        for (int c = 0; c < 3; c++) out[c] = bilerp(g_dec[p00[c]], g_dec[p10[c]], g_dec[p01[c]], g_dec[p11[c]], ax.f, ay.f);
        out[3] = bilerp(g_u8n[p00[3]], g_u8n[p10[3]], g_u8n[p01[3]], g_u8n[p11[3]], ax.f, ay.f);
    } else { /* plain Rgba8Unorm node texture: NC-6u on all four channels */
        for (int c = 0; c < 4; c++) out[c] = filter_u8(p00[c], p10[c], p01[c], p11[c], ax.f, ay.f);
    }
}

/* FramePreProcessor::rescale_node_texture (state/frame_pre_processor.rs:117-132) with rgba_rescale.wgsl:24-27:
 * one full-target draw, `blend: None` (rgba_rescale.rs:38-42): each target pixel is the linear-filtered sample of
 * the node texture at its centre, stored through the target format (sRGB encode in GpuOptimized, plain UNORM8 in
 * CpuOptimized; RescaleTexture::new :199-206). */
/* wgpu/utils/add_premultiplied_alpha.wgsl:24-35 (PremultiplyAlphaPipeline): the full-screen quad samples the
 * straight-alpha source at texel centres (one texel, weight 1) through its view, multiplies the colour by
 * max(alpha, 1e-5), clamps and stores through the target view. */
void orc_add_premultiplied_alpha(const uint8_t *rgba, int w, int h, int mode, uint8_t *out) {
    orc_init();
#pragma omp parallel for schedule(static)
    for (int i = 0; i < w * h; i++) {
        const uint8_t *t = rgba + (size_t)i * 4;
        uint8_t *o = out + (size_t)i * 4;
        const float a = g_u8n[t[3]], am = fmaxf(a, 0.00001f);
        for (int c = 0; c < 3; c++) {
            const float v = clamp01((mode == ORC_MODE_GPU_OPTIMIZED ? g_dec[t[c]] : g_u8n[t[c]]) * am);
            o[c] = mode == ORC_MODE_GPU_OPTIMIZED ? orc_srgb_encode_u8(v) : orc_unorm8(v);
        }
        o[3] = orc_unorm8(clamp01(a));
    }
}

/* TextRendererNode::render (transformations/text_renderer.rs:72-167): the node texture is cleared to the component's
 * background colour (`LoadOp::Clear(convert_to_shader_color(..))`, :141-150, stored through the target view) and
 * glyphon's TextRenderer draws one quad per prepared glyph over it.  glyphon is an un-vendored git dependency
 * (0.11.0 @ smelter-labs rev c784922, Cargo.lock:2298); what is restated here is its published shader + pipeline:
 *   vertex:   quad = pos + {0, dim}, uv = atlas origin + {0, dim} in integer texels (so every covered pixel centre hits
 *             the centre of exactly one atlas texel: a plain texel fetch, whatever the sampler's filter);
 *             glyph colour -> linear (srgb_to_linear per channel, alpha untouched) in ColorMode::Accurate -- the mode
 *             TextAtlas::new selects (:95-100) -- or left as it is in ColorMode::Web;
 *   fragment: mask glyph:  (colour.rgb, colour.a * mask)      mask atlas = R8Unorm
 *             colour glyph: the colour-atlas texel             colour atlas = Rgba8UnormSrgb (Accurate) / Rgba8Unorm (Web)
 *   blend:    wgpu::BlendState::ALPHA_BLENDING -- rgb: src * src.a + dst * (1 - src.a); a: src.a + dst.a * (1 - src.a),
 *             on the clamped source, destination read and result stored through the node texture's view
 *             (sRGB in GpuOptimized, plain UNORM8 in CpuOptimized).
 * The glyph list is glyphon's `GlyphToRender` after its CPU-side clipping to TextBounds; shaping and rasterisation
 * (cosmic-text / swash) stay on the CPU side of the boundary.  PARITY UNPINNED: render_tests/text.rs holds snapshots only. */
void orc_render_text(int w, int h, const uint8_t background[4], const orc_glyph *glyphs, int n_glyphs, const uint8_t *mask_atlas,
                     int mask_w, int mask_h, const uint8_t *color_atlas, int color_w, int color_h, int color_mode, int mode,
                     uint8_t *out) {
    orc_init();
    float bg[4];
    shader_color(background, mode, bg);
    for (int i = 0; i < w * h; i++) {
        uint8_t *o = out + (size_t)i * 4;
        for (int c = 0; c < 3; c++) o[c] = mode == ORC_MODE_GPU_OPTIMIZED ? orc_srgb_encode_u8(bg[c]) : orc_unorm8(bg[c]);
        o[3] = orc_unorm8(bg[3]);
    }
    const int accurate = color_mode == 0;
    for (int gi = 0; gi < n_glyphs; gi++) {
        const orc_glyph *G = &glyphs[gi];
        float col[4];
        for (int c = 0; c < 3; c++) col[c] = accurate ? g_dec[G->color[c]] : g_u8n[G->color[c]];
        col[3] = g_u8n[G->color[3]];
        for (int dy = 0; dy < (int)G->height; dy++) {
            const int py = G->y + dy;
            if (py < 0 || py >= h) continue;
            for (int dx = 0; dx < (int)G->width; dx++) {
                const int px = G->x + dx;
                if (px < 0 || px >= w) continue;
                const int ax = (int)G->atlas_x + dx, ay = (int)G->atlas_y + dy;
                float s[4];
                if (G->content == 1) {   /* ContentType::Mask */
                    /* texel outside the atlas: ClampToEdge of glyphon's sampler */
                    const int cx = ax < mask_w ? ax : mask_w - 1, cy = ay < mask_h ? ay : mask_h - 1;
                    const float cov = mask_atlas ? g_u8n[mask_atlas[(size_t)cy * mask_w + cx]] : 0.0f;
                    s[0] = col[0]; s[1] = col[1]; s[2] = col[2]; s[3] = col[3] * cov;
                } else {                 /* ContentType::Color */
                    const int cx = ax < color_w ? ax : color_w - 1, cy = ay < color_h ? ay : color_h - 1;
                    const uint8_t *t = color_atlas ? color_atlas + ((size_t)cy * color_w + cx) * 4 : NULL;
                    for (int c = 0; c < 3; c++) s[c] = t ? (accurate ? g_dec[t[c]] : g_u8n[t[c]]) : 0.0f;
                    s[3] = t ? g_u8n[t[3]] : 0.0f;
                }
                for (int c = 0; c < 4; c++) s[c] = clamp01(s[c]);
                const float a = s[3], ia = 1.0f - a;
                uint8_t *d = out + ((size_t)py * w + px) * 4;
                for (int c = 0; c < 3; c++) {
                    if (mode == ORC_MODE_GPU_OPTIMIZED) d[c] = orc_srgb_encode_u8(fmaf(g_dec[d[c]], ia, s[c] * a));
                    else d[c] = orc_unorm8(fmaf(g_u8n[d[c]], ia, s[c] * a));
                }
                d[3] = orc_unorm8(fmaf(g_u8n[d[3]], ia, a));
            }
        }
    }
}

void orc_rescale_rgba(const uint8_t *rgba, int sw, int sh, int ow, int oh, int mode, uint8_t *out) {
    orc_texture t = {sw, sh, rgba};
#pragma omp parallel for schedule(static)
    for (int py = 0; py < oh; py++)
        for (int px = 0; px < ow; px++) {
            float sm[4];
            sample_node(&t, mode, ((float)px + 0.5f) / (float)ow, ((float)py + 0.5f) / (float)oh, sm);
            uint8_t *o = out + ((size_t)py * ow + px) * 4;
            for (int c = 0; c < 3; c++) o[c] = mode == ORC_MODE_GPU_OPTIMIZED ? orc_srgb_encode_u8(sm[c]) : orc_unorm8(sm[c]);
            o[3] = orc_unorm8(sm[3]);
        }
}

/* PREMULTIPLIED_ALPHA_BLENDING through the node texture's view (common_pipeline.rs:125) */
static inline void blend_store(uint8_t *dst, const float src_in[4], int mode) {
    float s[4];
    for (int c = 0; c < 4; c++) s[c] = clamp01(src_in[c]);
    float ia = 1.0f - s[3];
    if (mode == ORC_MODE_GPU_OPTIMIZED) {
        for (int c = 0; c < 3; c++) dst[c] = orc_srgb_encode_u8(fmaf(g_dec[dst[c]], ia, s[c]));
    } else {
        for (int c = 0; c < 3; c++) dst[c] = orc_unorm8(fmaf(g_u8n[dst[c]], ia, s[c]));
    }
    dst[3] = orc_unorm8(fmaf(g_u8n[dst[3]], ia, s[3]));
}

/* One layout as draw_layout sees it: the quad, the shader colours, the texture */
typedef struct {
    const orc_layout *L;
    const orc_texture *tex;
    quad q;
    float left, top, w, h;      /* the quad (box shadow: grown by blur_radius) */
    float color[4], border_color[4];
    int tw, th, nmask, mode;
} layer_ctx;

static int layer_setup(layer_ctx *c, int W, int H, const orc_layout *L, const orc_texture *tex, int mode) {
    c->L = L; c->tex = tex; c->mode = mode;
    c->left = L->left; c->top = L->top; c->w = L->width; c->h = L->height;
    if (L->type == ORC_LAYOUT_BOX_SHADOW) { /* apply_layouts.wgsl:215-229 */
        float bw = L->width + 2.0f * L->blur_radius, bh = L->height + 2.0f * L->blur_radius;
        c->left = L->left - L->blur_radius; c->top = L->top - L->blur_radius; c->w = bw; c->h = bh;
    }
    if (!quad_setup(&c->q, c->left, c->top, c->w, c->h, L->rotation_degrees, W, H)) return 0;
    shader_color(L->color, mode, c->color);
    shader_color(L->border_color, mode, c->border_color);
    c->tw = tex && tex->data ? tex->width : 1; c->th = tex && tex->data ? tex->height : 1;
    c->nmask = L->masks_len < ORC_MAX_MASKS ? L->masks_len : ORC_MAX_MASKS;
    return 1;
}

/* vs_main's interpolated attributes + fs_main (apply_layouts.wgsl:258-377) at a covered pixel: the premultiplied source.
 * *bare = 1 when every alpha factor is exactly 1 and the branch taken does not mix in the border colour, so the source
 * is the layer's bare colour or sample. */
static void fragment(const layer_ctx *c, int px, int py, float src[4], int *bare) {
    const orc_layout *L = c->L;
    const quad *q = &c->q;
    float pcx = (float)px + 0.5f, pcy = (float)py + 0.5f;
    /* interpolated vertex attributes */
    float lx, ly, u, v;
    if (!q->rotated) {
        lx = (pcx - c->left) - c->w * 0.5f;
        ly = c->h * 0.5f - (pcy - c->top);
        u = (pcx - c->left) / c->w;
        v = (pcy - c->top) / c->h;
    } else {
        float dx = pcx - q->cx, dyu = q->cy - pcy;
        lx = dx * q->cs + dyu * q->sn;
        ly = dyu * q->cs - dx * q->sn;
        u = lx / c->w + 0.5f;
        v = 0.5f - ly / c->h;
    }
    float mask_alpha = 1.0f;
    for (int i = 0; i < c->nmask; i++) {
        const orc_mask *m = &L->masks[i];
        float d = rounded_rect_sdf((m->left + m->width / 2.0f) - pcx, (m->top + m->height / 2.0f) - pcy,
                                   m->width, m->height, m->radius);
        mask_alpha = mask_alpha * smoothstep_f(-0.5f, 0.5f, -d);
    }
    for (int ch = 0; ch < 4; ch++) src[ch] = 0.0f;
    *bare = 0;
    if (L->type == ORC_LAYOUT_TEXTURE) {
        float tx = u * (L->crop_width / (float)c->tw) + (L->crop_left / (float)c->tw);
        float ty = v * (L->crop_height / (float)c->th) + (L->crop_top / (float)c->th);
        float sample[4];
        sample_node(c->tex, c->mode, tx, ty, sample);
        float edge = -rounded_rect_sdf(lx, ly, L->width, L->height, L->border_radius);
        float bw = L->border_width;
        if (bw < 1.0f) {
            float ca = smoothstep_f(-0.5f, 0.5f, edge);
            for (int ch = 0; ch < 4; ch++) src[ch] = (sample[ch] * ca) * mask_alpha;
            *bare = ca == 1.0f && mask_alpha == 1.0f;
        } else if (mask_alpha < 0.01f) {
            /* transparent */
        } else if (edge > bw / 2.0f) {
            float ba = smoothstep_f(bw - 0.5f, bw + 0.5f, edge);
            for (int ch = 0; ch < 4; ch++)
                src[ch] = (c->border_color[ch] * (1.0f - ba) + sample[ch] * ba) * mask_alpha;
            *bare = ba == 1.0f && mask_alpha == 1.0f;
        } else {
            float ca = smoothstep_f(-0.5f, 0.5f, edge);
            for (int ch = 0; ch < 4; ch++) src[ch] = (c->border_color[ch] * ca) * mask_alpha;
        }
    } else if (L->type == ORC_LAYOUT_COLOR) {
        float edge = -rounded_rect_sdf(lx, ly, L->width, L->height, L->border_radius);
        float bw = L->border_width;
        if (bw < 1.0f) {
            float ca = smoothstep_f(-0.5f, 0.5f, edge);
            for (int ch = 0; ch < 4; ch++) src[ch] = (c->color[ch] * ca) * mask_alpha;
            *bare = ca == 1.0f && mask_alpha == 1.0f;
        } else if (edge > bw / 2.0f) {
            float ba = smoothstep_f(bw, bw + 1.0f, edge);
            for (int ch = 0; ch < 4; ch++)
                src[ch] = (c->border_color[ch] * (1.0f - ba) + c->color[ch] * ba) * mask_alpha;
            *bare = ba == 1.0f && mask_alpha == 1.0f;
        } else {
            float ca = smoothstep_f(-0.5f, 0.5f, edge);
            for (int ch = 0; ch < 4; ch++) src[ch] = (c->border_color[ch] * ca) * mask_alpha;
        }
    } else {
        float edge = -rounded_rect_sdf(lx, ly, L->width, L->height, L->border_radius);
        float br = L->blur_radius;
        float ba = smoothstep_f(-br / 2.0f, br / 2.0f, edge) * mask_alpha;
        for (int ch = 0; ch < 4; ch++) src[ch] = c->color[ch] * ba;
    }
}

static void draw_layout(int W, int H, const orc_layout *L, const orc_texture *tex, int mode, uint8_t *out) {
    layer_ctx c;
    if (!layer_setup(&c, W, H, L, tex, mode)) return;
#pragma omp parallel for schedule(static)
    for (int py = c.q.by0; py < c.q.by1; py++)
        for (int px = c.q.bx0; px < c.q.bx1; px++) {
            if (!quad_covers(&c.q, px, py)) continue;
            float src[4];
            int bare;
            fragment(&c, px, py, src, &bare);
            blend_store(out + ((size_t)py * W + px) * 4, src, mode);
        }
}

/* Per pixel of a W x H target: 1 where the layout covers the pixel and its fragment is the bare colour or sample (every
 * alpha factor exactly 1, no border colour mixed in), else 0.  The layer interiors the compositor proves must lie inside. */
void orc_bare_map(int W, int H, const orc_layout *L, int mode, uint8_t *out) {
    orc_init();
    memset(out, 0, (size_t)W * H);
    layer_ctx c;
    if (!layer_setup(&c, W, H, L, NULL, mode)) return;
#pragma omp parallel for schedule(static)
    for (int py = c.q.by0; py < c.q.by1; py++)
        for (int px = c.q.bx0; px < c.q.bx1; px++) {
            if (!quad_covers(&c.q, px, py)) continue;
            float src[4];
            int bare;
            fragment(&c, px, py, src, &bare);
            out[(size_t)py * W + px] = (uint8_t)bare;
        }
}

void orc_apply_layouts(int W, int H, const orc_layout *layouts, const orc_texture *textures, int n,
                       int max_layouts, int mode, uint8_t *out) {
    memset(out, 0, (size_t)W * H * 4); /* LoadOp::Clear(TRANSPARENT), shader.rs:135 */
    int m = n < max_layouts ? n : max_layouts;
    for (int i = 0; i < m; i++) draw_layout(W, H, &layouts[i], textures ? &textures[i] : NULL, mode, out);
}

void orc_render_layout_node(int W, int H, const orc_layout *layouts_in, int n, const orc_texture *nodes,
                            int n_nodes, int max_layouts, int mode, uint8_t *out) {
    orc_layout *layouts = (orc_layout *)malloc(sizeof(orc_layout) * (size_t)(n ? n : 1));
    orc_texture *tex = (orc_texture *)calloc((size_t)(n ? n : 1), sizeof(orc_texture));
    uint8_t **owned = (uint8_t **)calloc((size_t)(n ? n : 1), sizeof(uint8_t *));
    memcpy(layouts, layouts_in, sizeof(orc_layout) * (size_t)n);
    for (int i = 0; i < n; i++) {
        orc_layout *L = &layouts[i];
        if (L->type != ORC_LAYOUT_TEXTURE) continue;
        const orc_texture *node = (L->child_index >= 0 && L->child_index < n_nodes) ? &nodes[L->child_index] : NULL;
        if (!node || !node->data) continue; /* default_empty_view */
        tex[i] = *node;
        if (mode != ORC_MODE_GPU_OPTIMIZED) continue; /* layout_renderer.rs:22-28: no resampler */
        /* resample_scaled_children, layout.rs:238-278 */
        float rw = roundf(L->width), rh = roundf(L->height);
        int dw = (rw >= 1.0f) ? (rw > 16384.0f ? 16384 : (int)rw) : 1;
        int dh = (rh >= 1.0f) ? (rh > 16384.0f ? 16384 : (int)rh) : 1;
        int ax[2], pp[2];
        if (orc_plan_passes(L->crop_left, L->crop_top, L->crop_width, L->crop_height, dw, dh, ax, pp) == 0) continue;
        owned[i] = (uint8_t *)malloc((size_t)dw * dh * 4);
        orc_resample(node, L->crop_left, L->crop_top, L->crop_width, L->crop_height, dw, dh, owned[i]);
        tex[i].width = dw; tex[i].height = dh; tex[i].data = owned[i];
        L->crop_top = 0.0f; L->crop_left = 0.0f; L->crop_width = (float)dw; L->crop_height = (float)dh;
    }
    orc_apply_layouts(W, H, layouts, tex, n, max_layouts, mode, out);
    for (int i = 0; i < n; i++) free(owned[i]);
    free(owned); free(tex); free(layouts);
}

/* ------------------------------------------------------------------------------------------ */
/* self-check used by tests: for even plane sizes the K1/K2 chroma taps of NC-6 are exactly     */
/* (x/2-1, x/2; f=.75) for even x and ((x-1)/2, (x+1)/2; f=.25) for odd x (clamped), the luma   */
/* tap and the K10 chroma tap (f=.5 between 2c and 2c+1) likewise.  Returns the mismatch count. */
/* ------------------------------------------------------------------------------------------ */
long orc_check_even_size_phases(int max_dim) {
    long bad = 0;
    for (int w = 2; w <= max_dim; w += 2) {
        int cw = w / 2;
        for (int x = 0; x < w; x++) {
            float t = ((float)x + 0.5f) / (float)w;
            lin_tap c = linear_tap(t, cw);
            int e0 = (x & 1) ? (x - 1) / 2 : x / 2 - 1, e1 = e0 + 1;
            float ef = (x & 1) ? 0.25f : 0.75f;
            if (e0 < 0) e0 = 0;
            if (e1 > cw - 1) e1 = cw - 1;
            if (c.i0 != e0 || c.i1 != e1 || c.f != ef) bad++;
            lin_tap l = linear_tap(t, w); /* luma: must select texel x with weight exactly 1 */
            if (!((l.f == 0.0f && l.i0 == x) || (l.f == 1.0f && l.i1 == x))) bad++;
        }
        for (int c = 0; c < cw; c++) { /* K10: chroma target texel c samples the full-res texture */
            lin_tap k = linear_tap(((float)c + 0.5f) / (float)cw, w);
            if (k.i0 != 2 * c || k.i1 != 2 * c + 1 || k.f != 0.5f) bad++;
        }
    }
    return bad;
}
