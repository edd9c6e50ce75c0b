/*
 * oracle_nc.h -- the numeric contract of DESIGN.md §3 as the C oracles under tests/ use it (TEST INFRASTRUCTURE ONLY, NOT
 * PRODUCT CODE).  Restated from oracle/smelter_oracle.c, the committed oracle, which stays as it is because it is the
 * yardstick of every other test.  Plain C that also compiles as C++ (the shader shim is built with g++); every file that
 * includes it is compiled with -ffp-contract=off, so only the fmaf() calls are fused.
 */
#ifndef ORACLE_NC_H
#define ORACLE_NC_H

#include <math.h>
#include <stddef.h>
#include <stdint.h>

static float u8n[256], dec[256], thr[255];
static int tables_ready = 0;

/* NC-3 / NC-4: the sRGB EOTF in double */
static inline double eotf(double c) { return c <= 0.04045 ? c / 12.92 : pow((c + 0.055) / 1.055, 2.4); }

/* the NC-1, NC-3 and NC-4 tables, built on the first call */
static inline void init_tables(void) {
    if (tables_ready) return;
    for (int b = 0; b < 256; b++) {
        u8n[b] = (float)b / 255.0f;                 /* NC-1 */
        dec[b] = (float)eotf((double)b / 255.0);    /* NC-3 */
    }
    for (int k = 0; k < 255; k++) thr[k] = (float)eotf(((double)k + 0.5) / 255.0);   /* NC-4 */
    tables_ready = 1;
}

/* NC-2's clamp: NaN -> 0 */
static inline float clamp01(float x) { return fminf(fmaxf(x, 0.0f), 1.0f); }

/* NC-2: UNORM8 store */
static inline uint8_t store_unorm(float x) { return (uint8_t)rintf(clamp01(x) * 255.0f); }

/* NC-4: sRGB8 store, the number of thresholds at or below x */
static inline uint8_t store_srgb(float x) {
    int n = 0;
    x = clamp01(x);
    while (n < 255 && x >= thr[n]) n++;
    return (uint8_t)n;
}

/* NC-6: texel coordinate t * dim - .5, the fraction quantised to 8 bits, taps clamped to the edge.  A NaN coordinate
 * needs no case of its own: fmaxf(NaN, -2) is -2, so it gives taps 0, 0 and fraction 0. */
static inline void tap(float t, int dim, int *i0, int *i1, float *f) {
    float c = fminf(fmaxf(t * (float)dim - 0.5f, -2.0f), (float)dim + 1.0f);
    float fl = floorf(c);
    *f = rintf((c - fl) * 256.0f) * (1.0f / 256.0f);
    int a = (int)fl, b = a + 1;
    *i0 = a < 0 ? 0 : (a > dim - 1 ? dim - 1 : a);
    *i1 = b < 0 ? 0 : (b > dim - 1 ? dim - 1 : b);
}

/* NC-6: the bilinear filter of four decoded texels */
static inline float lerp2(float t00, float t10, float t01, float t11, float fx, float fy) {
    float h0 = fmaf(t10, fx, t00 * (1.0f - fx));
    float h1 = fmaf(t11, fx, t01 * (1.0f - fx));
    return fmaf(h1, fy, h0 * (1.0f - fy));
}

/* NC-6u: the bilinear filter of four bytes in integers, rounded once */
static inline float lerp2_u8(int t00, int t10, int t01, int t11, float fx, float fy) {
    int wx = (int)(fx * 256.0f), wy = (int)(fy * 256.0f);
    int n = (t00 * (256 - wx) + t10 * wx) * (256 - wy) + (t01 * (256 - wx) + t11 * wx) * wy;
    return (float)n / 16711680.0f;
}

/* NC-6 / NC-6u: textureSample with the linear / ClampToEdge sampler of a w x h RGBA8 texture (NULL: the 1 x 1 transparent
 * empty view) through the view: mode 0 (GpuOptimized) decodes the sRGB colour bytes (NC-3), mode 1 (CpuOptimized)
 * filters the bytes.  The byte of output channel k is order[k]. */
static inline void sample_rgba8(const uint8_t *t, int w, int h, const int order[4], int mode, float u, float v, float out[4]) {
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

/* PREMULTIPLIED_ALPHA_BLENDING of src over the RGBA8 pixel d through the target view, stored as 8 bits (NC-2 / NC-4) */
static inline void blend(uint8_t *d, const float src[4], int mode) {
    float s[4];
    for (int k = 0; k < 4; k++) s[k] = clamp01(src[k]);
    const float ia = 1.0f - s[3];
    for (int k = 0; k < 3; k++)
        d[k] = mode == 0 ? store_srgb(fmaf(dec[d[k]], ia, s[k])) : store_unorm(fmaf(u8n[d[k]], ia, s[k]));
    d[3] = store_unorm(fmaf(u8n[d[3]], ia, s[3]));
}

#endif
