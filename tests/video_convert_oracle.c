/* video_convert_oracle.c -- CPU oracle of smr_video_nv12_to_rgba: gpu-video's NV12 -> RGBA converter restated per target
 * pixel from DESIGN.md NC-11.  Test infrastructure (tests/oracle_video_convert.py builds it with -ffp-contract=off, so
 * every f32 operation rounds on its own).  The reverse converter is K11, whose oracle is orc_rgba_to_nv12_scaled.
 *
 * Written from the contract, not from the kernel: every pixel takes the general sampler (four taps per plane, integer
 * filter, one rounding), the matrix keeps all nine products, and the constants are rounded from double here. */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

typedef struct {
    int i0, i1;   /* the two texels of one axis, clamped to the edge */
    int w1;       /* the second texel's weight in 1/256 (the first has 256 - w1) */
} axis_tap;

static int clampi(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }

/* NC-6: c = t * n - 0.5, weight quantised to 8 fractional bits, clamp-to-edge */
static axis_tap tap_at(float t, int n) {
    const float c = t * (float)n - 0.5f;
    const float fl = floorf(c);
    axis_tap a;
    a.w1 = (int)rintf((c - fl) * 256.0f);
    a.i0 = clampi((int)fl, 0, n - 1);
    a.i1 = clampi((int)fl + 1, 0, n - 1);
    return a;
}

/* NC-6u: channel ch of a plane of `stride`-byte texels, filtered in integers and rounded once to f32 */
static float sample_unorm(const uint8_t *p, int pitch, int stride, int ch, axis_tap ax, axis_tap ay) {
#define T(x, y) ((int64_t)p[(size_t)(y) * pitch + (size_t)(x) * stride + ch])
    const int64_t top = T(ax.i0, ay.i0) * (256 - ax.w1) + T(ax.i1, ay.i0) * ax.w1;
    const int64_t bot = T(ax.i0, ay.i1) * (256 - ax.w1) + T(ax.i1, ay.i1) * ax.w1;
#undef T
    const int64_t n = top * (256 - ay.w1) + bot * ay.w1;
    /* the double quotient is within 2^-53 of n / (255 * 65536), which is never that close to an f32 rounding tie */
    return (float)((double)n / (255.0 * 65536.0));
}

/* NC-2 */
static uint8_t store(float x) {
    if (!(x > 0.0f)) return 0;
    if (x > 1.0f) x = 1.0f;
    return (uint8_t)rintf(x * 255.0f);
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
        const axis_tap ly = tap_at(v, h), cy = tap_at(v, h / 2);
        for (int px = 0; px < ow; px++) {
            const float u = ((float)px + 0.5f) / (float)ow;
            const axis_tap lx = tap_at(u, w), cx = tap_at(u, w / 2);
            const float yuv[3] = {sample_unorm(y, y_pitch, 1, 0, lx, ly), sample_unorm(uv, uv_pitch, 2, 0, cx, cy),
                                  sample_unorm(uv, uv_pitch, 2, 1, cx, cy)};
            const float d[3] = {yuv[0] - bias, yuv[1] - 0.5f, yuv[2] - 0.5f};
            const float s[3] = {d[0] * scale_y, d[1] * scale_c, d[2] * scale_c};
            uint8_t *o = rgba + ((size_t)py * ow + px) * 4;
            for (int j = 0; j < 3; j++) {
                const float a = s[0] * m[j][0], b = s[1] * m[j][1], c = s[2] * m[j][2];
                o[j] = store((a + b) + c);
            }
            o[3] = 255;
        }
    }
}
