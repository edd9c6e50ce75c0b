/*
 * input_color_oracle.c -- the YUV -> RGBA8 node texture of an input with a colour setting (smr_set_input_color, DESIGN.md
 * NC-13), for the tests of that setting (TEST INFRASTRUCTURE ONLY, NOT PRODUCT CODE).  K1 / K2 / K3 restated from
 * oracle/smelter_oracle.c, the committed oracle, with the matrix's chroma coefficients and the range as arguments:
 * matrix 0 BT.709, 1 BT.601; full_range 0 limited, 1 full, for every YUV format.  At BT.709 and a format's own range the
 * bytes are the committed oracle's (tests/test_input_color.py checks it over the joint byte space).
 */
#include "oracle_nc.h"

#define K16 (16.0f / 255.0f)
#define RCP_Y (1.0f / 0.85882352941f)  /* x / const is evaluated as x * (1/const) */
#define RCP_C (1.0f / 0.87843137254f)

/* one channel of a w x h plane of `stride`-byte texels (pitch w texels), NC-6u at the normalised coordinate (tx, ty) */
static inline float sample_plane(const uint8_t *p, int w, int h, int stride, int ch, float tx, float ty) {
    int x0, x1, y0, y1;
    float fx, fy;
    tap(tx, w, &x0, &x1, &fx);
    tap(ty, h, &y0, &y1, &fy);
    const uint8_t *r0 = p + (size_t)y0 * w * stride, *r1 = p + (size_t)y1 * w * stride;
    return lerp2_u8(r0[x0 * stride + ch], r0[x1 * stride + ch], r1[x0 * stride + ch], r1[x1 * stride + ch], fx, fy);
}

static inline void to_rgba(float y, float u, float v, int full_range, int matrix, uint8_t *out) {
    const float rv = matrix ? 1.402f : 1.5748f, gu = matrix ? -0.3441f : -0.1873f;
    const float gv = matrix ? -0.7141f : -0.4681f, bu = matrix ? 1.772f : 1.8556f;
    if (!full_range) {
        y = clamp01((y - K16) * RCP_Y);
        u = clamp01((u - K16) * RCP_C);
        v = clamp01((v - K16) * RCP_C);
    }
    const float um = u - 0.5f, vm = v - 0.5f;
    out[0] = store_unorm(fmaf(rv, vm, y));
    out[1] = store_unorm(fmaf(gv, vm, fmaf(gu, um, y)));
    out[2] = store_unorm(fmaf(bu, um, y));
    out[3] = 255;
}

/* planar 4:2:0 / 4:2:2 / 4:4:4 by chroma plane size: the three planes are sampled at the same normalised coordinate */
void ico_yuv_planar_to_rgba(const uint8_t *y, const uint8_t *u, const uint8_t *v, int w, int h, int cw, int ch,
                            int full_range, int matrix, uint8_t *rgba) {
#pragma omp parallel for schedule(static)
    for (int py = 0; py < h; py++) {
        const float ty = ((float)py + 0.5f) / (float)h;
        for (int px = 0; px < w; px++) {
            const float tx = ((float)px + 0.5f) / (float)w;
            to_rgba(sample_plane(y, w, h, 1, 0, tx, ty), sample_plane(u, cw, ch, 1, 0, tx, ty),
                    sample_plane(v, cw, ch, 1, 0, tx, ty), full_range, matrix, rgba + ((size_t)py * w + px) * 4);
        }
    }
}

void ico_nv12_to_rgba(const uint8_t *y, const uint8_t *uv, int w, int h, int full_range, int matrix, uint8_t *rgba) {
    const int cw = w / 2, ch = h / 2;
#pragma omp parallel for schedule(static)
    for (int py = 0; py < h; py++) {
        const float ty = ((float)py + 0.5f) / (float)h;
        for (int px = 0; px < w; px++) {
            const float tx = ((float)px + 0.5f) / (float)w;
            to_rgba(sample_plane(y, w, h, 1, 0, tx, ty), sample_plane(uv, cw, ch, 2, 0, tx, ty),
                    sample_plane(uv, cw, ch, 2, 1, tx, ty), full_range, matrix, rgba + ((size_t)py * w + px) * 4);
        }
    }
}

/* K3: the (w / 2) x h texels of UYVY (yuyv = 0) or YUYV; the column index comes back from the interpolated coordinate and
 * the texel is fetched at its centre */
void ico_interleaved422_to_rgba(const uint8_t *data, int w, int h, int yuyv, int full_range, int matrix, uint8_t *rgba) {
    const int dimx = w / 2;
    if (dimx < 1) return;
    const float eps = 0.0001f, half_pixel_width = 0.5f / (float)dimx;
#pragma omp parallel for schedule(static)
    for (int py = 0; py < h; py++) {
        const float ty = ((float)py + 0.5f) / (float)h;
        for (int px = 0; px < w; px++) {
            const float tx = ((float)px + 0.5f) / (float)w;
            const float xf = ((tx * (float)dimx - half_pixel_width) + eps) * 2.0f;
            const uint32_t x_pos = xf >= 4294967296.0f ? 0xffffffffu : (xf > 0.0f ? (uint32_t)xf : 0u);   /* u32(): saturating */
            const float tcx = (float)(x_pos / 2u) / (float)dimx + half_pixel_width;
            float t[4];
            for (int c = 0; c < 4; c++) t[c] = sample_plane(data, dimx, h, 4, c, tcx, ty);
            float yy, uu, vv;
            if (yuyv) { yy = (x_pos & 1u) ? t[2] : t[0]; uu = t[1]; vv = t[3]; }
            else { yy = (x_pos & 1u) ? t[3] : t[1]; uu = t[0]; vv = t[2]; }
            to_rgba(yy, uu, vv, full_range, matrix, rgba + ((size_t)py * w + px) * 4);
        }
    }
}
