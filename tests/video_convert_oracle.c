/* video_convert_oracle.c -- CPU oracle of smr_video_nv12_to_rgba: gpu-video's NV12 -> RGBA converter restated per target
 * pixel from DESIGN.md NC-11.  Test infrastructure (tests/c_oracles.py builds it with -ffp-contract=off, so every f32
 * operation rounds on its own).  The reverse converter is K11, whose oracle is orc_rgba_to_nv12_scaled.
 *
 * Written from the contract, not from the kernel: every pixel takes the general sampler (four taps per plane, integer
 * filter, one rounding), the matrix keeps all nine products, and the constants are rounded from double here. */
#include "oracle_nc.h"

/* NC-6u: channel ch of a plane of `stride`-byte texels at columns x[0], x[1] and rows y[0], y[1] with fractions fx, fy */
static float sample_plane(const uint8_t *p, int pitch, int stride, int ch, const int x[2], const int y[2], float fx,
                          float fy) {
#define T(i, j) p[(size_t)y[j] * pitch + (size_t)x[i] * stride + ch]
    return lerp2_u8(T(0, 0), T(1, 0), T(0, 1), T(1, 1), fx, fy);
#undef T
}

/* One RGBA8 target of ow x oh (packed) from the NV12 crop w x h (even sides; y and uv read at their pitches). */
void orc_video_nv12_to_rgba(const uint8_t *y, int y_pitch, const uint8_t *uv, int uv_pitch, int w, int h, int ow, int oh,
                            uint8_t *rgba) {
    const float bias = (float)(16.0 / 255.0), scale_y = (float)(255.0 / 219.0), scale_c = (float)(255.0 / 224.0);
    /* mat3x3 columns as the constructor lists them; rgb[j] = dot(s, m[j]) in the order s0, s1, s2 */
    const float m[3][3] = {{(float)1.0, (float)0.0, (float)1.5748},
                           {(float)1.0, (float)-0.1873, (float)-0.4681},
                           {(float)1.0, (float)1.8556, (float)0.0}};
#pragma omp parallel for schedule(static)
    for (int py = 0; py < oh; py++) {
        const float v = ((float)py + 0.5f) / (float)oh;
        int ly[2], cy[2];
        float fly, fcy;
        tap(v, h, &ly[0], &ly[1], &fly);
        tap(v, h / 2, &cy[0], &cy[1], &fcy);
        for (int px = 0; px < ow; px++) {
            const float u = ((float)px + 0.5f) / (float)ow;
            int lx[2], cx[2];
            float flx, fcx;
            tap(u, w, &lx[0], &lx[1], &flx);
            tap(u, w / 2, &cx[0], &cx[1], &fcx);
            const float yuv[3] = {sample_plane(y, y_pitch, 1, 0, lx, ly, flx, fly),
                                  sample_plane(uv, uv_pitch, 2, 0, cx, cy, fcx, fcy),
                                  sample_plane(uv, uv_pitch, 2, 1, cx, cy, fcx, fcy)};
            const float d[3] = {yuv[0] - bias, yuv[1] - 0.5f, yuv[2] - 0.5f};
            const float s[3] = {d[0] * scale_y, d[1] * scale_c, d[2] * scale_c};
            uint8_t *o = rgba + ((size_t)py * ow + px) * 4;
            for (int j = 0; j < 3; j++) {
                const float a = s[0] * m[j][0], b = s[1] * m[j][1], c = s[2] * m[j][2];
                o[j] = store_unorm((a + b) + c);
            }
            o[3] = 255;
        }
    }
}
