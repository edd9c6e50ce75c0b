// node_sample.cuh -- the device tables, the NC-6 sampler of node textures (every texture kind) and the
// PREMULTIPLIED_ALPHA_BLENDING store, shared by kernels.cu and the shader modules NVRTC compiles at registration
// (renderer.cpp embeds this file as a string), so that a shader plane and a web plane sample, blend and round alike.
// Included inside namespace smr::dev, after kernels.h.  Each module has its own copy of the c_* tables; the host copies
// the values kernels.cu holds into a shader module when it loads it.

__device__ float c_u8n[256];
__device__ float c_dec[256];
__device__ float c_thr[256];  // 255 used
__device__ float c_yl[256];   // limited-range luma, already expanded: clamp01((n/255 - 16/255) * RCP_Y)
// finer buckets (exponent + top 8 mantissa bits): every bucket holds AT MOST ONE threshold, so the encode is the
// bucket's count plus one comparison -- no search loop (checked on the host when the table is built)
#define ENC1_KEY0 ((127 - 13) << 8)
#define ENC1_KEYS ((13 << 8) + 1)
__device__ unsigned char c_enc1[ENC1_KEYS + 3];

struct Tables {  // per-block shared-memory copies (divergent indices would serialise in constant memory)
    float u8n[256];
    float dec[256];
    float thr[256];
    float yl[256];
};

__device__ __forceinline__ void load_tables(Tables &t) {
    for (int i = threadIdx.y * blockDim.x + threadIdx.x; i < 256; i += blockDim.x * blockDim.y) {
        t.u8n[i] = c_u8n[i];
        t.dec[i] = c_dec[i];
        t.thr[i] = c_thr[i];
        t.yl[i] = c_yl[i];
    }
    __syncthreads();
}

__device__ __forceinline__ float clamp01(float x) { return __saturatef(x); }  // [0,1], NaN -> 0 (== fmin(fmax(x,0),1))

__device__ __forceinline__ int unorm8(float x) { return __float2int_rn(clamp01(x) * 255.0f); }  // NC-2

// NC-4: the encoded byte is the number of decision thresholds <= x (thr[] ascending, thr[255] is a sentinel).
// c_enc1[] holds that count at the lower edge of each bucket of the float's (exponent, top 8 mantissa bits); a bucket
// contains at most one threshold (checked when the table is built), so one comparison finishes the count -- no
// pow(), no search loop, no divergence.  The table is read through L1 (3.3 KB, read-only).
__device__ __forceinline__ int srgb_encode(const Tables &t, float lin) {
    const float x = clamp01(lin);                                  // NaN -> 0
    const int k = max((__float_as_int(x) >> 15) - ENC1_KEY0, 0);   // below 2^-13 < thr[0]: bucket 0, count 0
    const int e = __ldg(c_enc1 + k);
    return e + (x >= t.thr[e] ? 1 : 0);
}

// ------------------------------------------------------------------------------------------------
// NC-6 sampler
// ------------------------------------------------------------------------------------------------
struct LinTap {
    int i0, i1;
    float f;
};

__device__ __forceinline__ LinTap linear_tap(float t, int dim) {
    LinTap r;
    float c = t * (float)dim - 0.5f;
    if (!(c == c)) { r.i0 = r.i1 = 0; r.f = 0.0f; return r; }
    c = fminf(fmaxf(c, -2.0f), (float)dim + 1.0f);
    float fl = floorf(c);
    float f = c - fl;
    r.f = rintf(f * 256.0f) * (1.0f / 256.0f);
    int i0 = (int)fl, i1 = i0 + 1;
    r.i0 = min(max(i0, 0), dim - 1);
    r.i1 = min(max(i1, 0), dim - 1);
    return r;
}

__device__ __forceinline__ float bilerp(float t00, float t10, float t01, float t11, float fx, float fy) {
    float h0 = fmaf(t10, fx, t00 * (1.0f - fx));
    float h1 = fmaf(t11, fx, t01 * (1.0f - fx));
    return fmaf(h1, fy, h0 * (1.0f - fy));
}

// NC-6u: UNORM8 (non-sRGB) views are filtered in exact integer arithmetic on the 8-bit texels and rounded once:
// value = f32(N / (255*65536)).  f32(n/255) is evaluated division-free and EXACTLY as fma(n, c, n*lo) with
// c = f32(1/255), lo = f32(1/255 - c) (checked for every n <= 255*65536); powers of two scale exactly.
__device__ __forceinline__ float div255(float nf, float pow2) {
    const float c = __uint_as_float(0x3b808081u) * pow2, lo = __uint_as_float(0xaf7efeffu) * pow2;  // folded at compile time
    return fmaf(nf, c, nf * lo);
}
__device__ __forceinline__ float filter_u8(int t00, int t10, int t01, int t11, float fx, float fy) {
    const int wx = (int)(fx * 256.0f), wy = (int)(fy * 256.0f);
    const int n = (t00 * (256 - wx) + t10 * wx) * (256 - wy) + (t01 * (256 - wx) + t11 * wx) * wy;
    return div255((float)n, 1.0f / 65536.0f);
}

// channel ch of a UNORM8 plane of `stride`-byte texels, NC-6u at the taps (ax, ay)
__device__ __forceinline__ float sample_u8(const uint8_t *p, int pitch, int stride, int ch, const LinTap &ax, const LinTap &ay) {
    const uint8_t *r0 = p + (size_t)ay.i0 * pitch, *r1 = p + (size_t)ay.i1 * pitch;
    const int t00 = __ldg(r0 + ax.i0 * stride + ch), t10 = __ldg(r0 + ax.i1 * stride + ch);
    const int t01 = __ldg(r1 + ax.i0 * stride + ch), t11 = __ldg(r1 + ax.i1 * stride + ch);
    return filter_u8(t00, t10, t01, t11, ax.f, ay.f);
}
__device__ __forceinline__ float sample_plane(const Tables &T, const uint8_t *p, int pitch, int stride, int ch,
                                              const LinTap &ax, const LinTap &ay) {
    return sample_u8(p, pitch, stride, ch, ax, ay);
}

// ------------------------------------------------------------------------------------------------
// K1/K2/K4: one texel of the (possibly virtual) RGBA8 node texture of an input
// planar_yuv_to_rgba.wgsl:35-58, nv12_to_rgba.wgsl:26-48, bgra_to_rgba.wgsl, argb_to_rgba.wgsl
// ------------------------------------------------------------------------------------------------
#define K16 (16.0f / 255.0f)
#define RCP_Y (1.0f / 0.85882352941f)
#define RCP_C (1.0f / 0.87843137254f)

// The chroma coefficients of the YUV -> RGB matrix rows, by Tex::matrix: 0 BT.709 (K1-K3), 1 BT.601 (NC-13, from Kr = 0.299
// and Kb = 0.114).  The only place they appear: every reader takes them from here, as immediates where the matrix is a
// template parameter.
struct YuvCoef {
    float rv, gu, gv, bu;   // r = y + rv (v - .5); g = y + gu (u - .5) + gv (v - .5); b = y + bu (u - .5)
};
__host__ __device__ constexpr YuvCoef yuv_coef(int matrix) {
    return matrix == 1 ? YuvCoef{1.402f, -0.3441f, -0.7141f, 1.772f} : YuvCoef{1.5748f, -0.1873f, -0.4681f, 1.8556f};
}

__device__ __forceinline__ uchar4 yuv_to_rgba8(float y, float u, float v, int full_range, int matrix) {
    const YuvCoef k = yuv_coef(matrix);
    if (!full_range) {
        y = clamp01((y - K16) * RCP_Y);
        u = clamp01((u - K16) * RCP_C);
        v = clamp01((v - K16) * RCP_C);
    }
    float um = u - 0.5f, vm = v - 0.5f;
    float r = fmaf(k.rv, vm, y);
    float g = fmaf(k.gv, vm, fmaf(k.gu, um, y));
    float b = fmaf(k.bu, um, y);
    return make_uchar4((unsigned char)unorm8(r), (unsigned char)unorm8(g), (unsigned char)unorm8(b), 255);
}

// luma already expanded (Tables::yl or Tables::u8n), chroma still raw; results as integers for callers that index a table next
__device__ __forceinline__ void yuv_to_rgb8n(float yn, float u, float v, int full_range, const YuvCoef &k, int &r8, int &g8, int &b8) {
    if (!full_range) {
        u = clamp01((u - K16) * RCP_C);
        v = clamp01((v - K16) * RCP_C);
    }
    float um = u - 0.5f, vm = v - 0.5f;
    r8 = unorm8(fmaf(k.rv, vm, yn));
    g8 = unorm8(fmaf(k.gv, vm, fmaf(k.gu, um, yn)));
    b8 = unorm8(fmaf(k.bu, um, yn));
}

// MAT: the matrix, or -1 for the texture's (s.matrix).  RANGE422: the range of the 4:2:2, 4:4:4 and interleaved kinds, or -1
// for the texture's (s.full_range); the 4:2:0 kinds always read s.full_range.  Callers that are specialised for one
// matrix and range pass them, so that the coefficients are immediates.
template <int MAT = -1, int RANGE422 = -1>
__device__ __forceinline__ uchar4 node_texel(const Tables &T, const Tex &s, int x, int y) {
    const int mat = MAT < 0 ? s.matrix : MAT;
    const int fr422 = RANGE422 < 0 ? s.full_range : RANGE422;
    switch (s.kind) {
        case TEX_RGBA8:
            return __ldg(reinterpret_cast<const uchar4 *>(s.p0 + (size_t)y * s.pitch0) + x);
        case TEX_BGRA: {
            uchar4 v = __ldg(reinterpret_cast<const uchar4 *>(s.p0 + (size_t)y * s.pitch0) + x);
            return make_uchar4(v.z, v.y, v.x, v.w);
        }
        case TEX_ARGB: {
            uchar4 v = __ldg(reinterpret_cast<const uchar4 *>(s.p0 + (size_t)y * s.pitch0) + x);
            return make_uchar4(v.y, v.z, v.w, v.x);
        }
        case TEX_YUV420:
        case TEX_NV12: {
            int cw = s.width / 2, ch = s.height / 2;
            if (((s.width | s.height) & 1) == 0) {
                // Even sizes: the NC-6 taps are exactly texel (x,y) for luma and the .25/.75 pair for chroma
                // (proved for every even size <= 16384 by oracle test test_even_size_sampler_phases_exhaustive).
                int x0 = (x & 1) ? (x >> 1) : max((x >> 1) - 1, 0), x1 = (x & 1) ? min((x >> 1) + 1, cw - 1) : (x >> 1);
                int y0 = (y & 1) ? (y >> 1) : max((y >> 1) - 1, 0), y1 = (y & 1) ? min((y >> 1) + 1, ch - 1) : (y >> 1);
                const int kx = (x & 1) ? 1 : 3, ky = (y & 1) ? 1 : 3;   // weight of the second tap, in quarters
                float yy = T.u8n[__ldg(s.p0 + (size_t)y * s.pitch0 + x)];
                int nu, nv;   // 16 x the interpolated chroma byte value (NC-6u with the .25/.75 taps)
                if (s.kind == TEX_YUV420) {
                    const uint8_t *u0 = s.p1 + (size_t)y0 * s.pitch1, *u1 = s.p1 + (size_t)y1 * s.pitch1;
                    const uint8_t *v0 = s.p2 + (size_t)y0 * s.pitch2, *v1 = s.p2 + (size_t)y1 * s.pitch2;
                    nu = ((int)__ldg(u0 + x0) * (4 - kx) + (int)__ldg(u0 + x1) * kx) * (4 - ky) +
                         ((int)__ldg(u1 + x0) * (4 - kx) + (int)__ldg(u1 + x1) * kx) * ky;
                    nv = ((int)__ldg(v0 + x0) * (4 - kx) + (int)__ldg(v0 + x1) * kx) * (4 - ky) +
                         ((int)__ldg(v1 + x0) * (4 - kx) + (int)__ldg(v1 + x1) * kx) * ky;
                } else {
                    const uchar2 *r0 = reinterpret_cast<const uchar2 *>(s.p1 + (size_t)y0 * s.pitch1);
                    const uchar2 *r1 = reinterpret_cast<const uchar2 *>(s.p1 + (size_t)y1 * s.pitch1);
                    uchar2 a = __ldg(r0 + x0), b = __ldg(r0 + x1), c = __ldg(r1 + x0), d = __ldg(r1 + x1);
                    nu = ((int)a.x * (4 - kx) + (int)b.x * kx) * (4 - ky) + ((int)c.x * (4 - kx) + (int)d.x * kx) * ky;
                    nv = ((int)a.y * (4 - kx) + (int)b.y * kx) * (4 - ky) + ((int)c.y * (4 - kx) + (int)d.y * kx) * ky;
                }
                const float uu = div255((float)nu, 0.0625f), vv = div255((float)nv, 0.0625f);
                return yuv_to_rgba8(yy, uu, vv, s.full_range, mat);
            }
            float tx = ((float)x + 0.5f) / (float)s.width, ty = ((float)y + 0.5f) / (float)s.height;
            LinTap ax = linear_tap(tx, s.width), ay = linear_tap(ty, s.height);
            LinTap cx = linear_tap(tx, cw), cy = linear_tap(ty, ch);
            float yy = sample_plane(T, s.p0, s.pitch0, 1, 0, ax, ay);
            float uu, vv;
            if (s.kind == TEX_YUV420) {
                uu = sample_plane(T, s.p1, s.pitch1, 1, 0, cx, cy);
                vv = sample_plane(T, s.p2, s.pitch2, 1, 0, cx, cy);
            } else {
                uu = sample_plane(T, s.p1, s.pitch1, 2, 0, cx, cy);
                vv = sample_plane(T, s.p1, s.pitch1, 2, 1, cx, cy);
            }
            return yuv_to_rgba8(yy, uu, vv, s.full_range, mat);
        }
        case TEX_YUV422:
        case TEX_YUV444: {   // the three planes are sampled at the same normalised coordinate (NC-6)
            const int cw = s.kind == TEX_YUV444 ? s.width : s.width / 2, ch = s.height;
            float tx = ((float)x + 0.5f) / (float)s.width, ty = ((float)y + 0.5f) / (float)s.height;
            LinTap ax = linear_tap(tx, s.width), ay = linear_tap(ty, s.height);
            LinTap cx = linear_tap(tx, cw), cy = linear_tap(ty, ch);
            float yy = sample_plane(T, s.p0, s.pitch0, 1, 0, ax, ay);
            float uu = sample_plane(T, s.p1, s.pitch1, 1, 0, cx, cy);
            float vv = sample_plane(T, s.p2, s.pitch2, 1, 0, cx, cy);
            return yuv_to_rgba8(yy, uu, vv, fr422, mat);
        }
        case TEX_UYVY:
        case TEX_YUYV: {   // K3 (interleaved_{uyvy,yuyv}_to_rgba.wgsl:24-61): column index back from the coordinate
            const int dimx = s.width / 2;
            const float eps = 0.0001f, hpw = 0.5f / (float)dimx;
            float tx = ((float)x + 0.5f) / (float)s.width, ty = ((float)y + 0.5f) / (float)s.height;
            float xf = ((tx * (float)dimx - hpw) + eps) * 2.0f;
            unsigned x_pos = xf >= 4294967296.0f ? 0xffffffffu : (xf > 0.0f ? (unsigned)xf : 0u);
            float tcx = (float)(x_pos / 2u) / (float)dimx + hpw;
            LinTap ax = linear_tap(tcx, dimx), ay = linear_tap(ty, s.height);
            float t[4];
#pragma unroll
            for (int c = 0; c < 4; c++) t[c] = sample_plane(T, s.p0, s.pitch0, 4, c, ax, ay);
            const bool second = x_pos & 1u;
            if (s.kind == TEX_YUYV) return yuv_to_rgba8(second ? t[2] : t[0], t[1], t[3], fr422, mat);
            return yuv_to_rgba8(second ? t[3] : t[1], t[0], t[2], fr422, mat);
        }
        default:
            return make_uchar4(0, 0, 0, 0);
    }
}

// K1/K2 for the aligned 2x2 pixel quad (x, y), x and y even, of an even-sized YUV texture.  The four pixels
// share one 3x3 chroma neighbourhood: texels and horizontal interpolants are computed once (bilerp of NC-6 is
// horizontal-then-vertical, so sharing the horizontal terms is bit-exact).  Requires 2 <= x <= W-4, 2 <= y <= H-4.
__device__ __forceinline__ bool yuv_quad_ok(const Tex &s, int x, int y) {
    return (s.kind == TEX_NV12 || s.kind == TEX_YUV420) && (((s.width | s.height | x | y) & 1) == 0) && x >= 2 &&
           x + 3 <= s.width - 1 && y >= 2 && y + 3 <= s.height - 1;
}
// The chroma of the aligned 2x2 pixel quad over chroma texel (cx, cy) of an even-sized 4:2:0 texture at the pixel centres:
// NC-6's .25 / .75 taps, in exact integers, with texels packed u in bits 0..15 and v in bits 16..31 so that both channels
// share every integer multiply-add (max 4080 < 65536).  quad_chroma_row: texels a, b, d of columns cx - 1, cx, cx + 1 of
// one chroma row -> its horizontal terms for the quad's even and odd pixel; quad_chroma16: the terms of rows cy - 1 .. cy + 1
// -> 16 x the interpolated chroma of pixels (0,0), (1,0), (0,1), (1,1).
__device__ __forceinline__ void quad_chroma_row(unsigned a, unsigned b, unsigned d, unsigned &he, unsigned &ho) {
    he = a + 3u * b;   // even pixel: taps (cx-1, cx), weights (1/4, 3/4)
    ho = 3u * b + d;   // odd pixel:  taps (cx, cx+1), weights (3/4, 1/4)
}
__device__ __forceinline__ void quad_chroma16(const unsigned he[3], const unsigned ho[3], unsigned &n00, unsigned &n10,
                                              unsigned &n01, unsigned &n11) {
    // even row: chroma rows (cy-1, cy) weights (1/4, 3/4) ; odd row: (cy, cy+1) weights (3/4, 1/4)
    n00 = he[0] + 3u * he[1]; n10 = ho[0] + 3u * ho[1]; n01 = 3u * he[1] + he[2]; n11 = 3u * ho[1] + ho[2];
}
__device__ __forceinline__ void yuv_quad(const Tables &T, const Tex &s, int x, int y, uchar4 &p00, uchar4 &p10,
                                         uchar4 &p01, uchar4 &p11) {
    const int cx = x >> 1, cy = y >> 1;
    unsigned he[3], ho[3];
#pragma unroll
    for (int i = 0; i < 3; i++) {
        unsigned a, b, d;
        if (s.kind == TEX_NV12) {
            const uchar2 *rp = reinterpret_cast<const uchar2 *>(s.p1 + (size_t)(cy - 1 + i) * s.pitch1) + cx;
            const uchar2 ta = __ldg(rp - 1), tb = __ldg(rp), td = __ldg(rp + 1);
            a = ta.x | (ta.y << 16); b = tb.x | (tb.y << 16); d = td.x | (td.y << 16);
        } else {
            const uint8_t *ru = s.p1 + (size_t)(cy - 1 + i) * s.pitch1 + cx, *rv = s.p2 + (size_t)(cy - 1 + i) * s.pitch2 + cx;
            a = __ldg(ru - 1) | (__ldg(rv - 1) << 16); b = __ldg(ru) | (__ldg(rv) << 16); d = __ldg(ru + 1) | (__ldg(rv + 1) << 16);
        }
        quad_chroma_row(a, b, d, he[i], ho[i]);
    }
    const uchar2 y0 = __ldg(reinterpret_cast<const uchar2 *>(s.p0 + (size_t)y * s.pitch0 + x));
    const uchar2 y1 = __ldg(reinterpret_cast<const uchar2 *>(s.p0 + (size_t)(y + 1) * s.pitch0 + x));
    unsigned n00, n10, n01, n11;
    quad_chroma16(he, ho, n00, n10, n01, n11);
    p00 = yuv_to_rgba8(T.u8n[y0.x], div255((float)(n00 & 0xffffu), 0.0625f), div255((float)(n00 >> 16), 0.0625f), s.full_range, s.matrix);
    p10 = yuv_to_rgba8(T.u8n[y0.y], div255((float)(n10 & 0xffffu), 0.0625f), div255((float)(n10 >> 16), 0.0625f), s.full_range, s.matrix);
    p01 = yuv_to_rgba8(T.u8n[y1.x], div255((float)(n01 & 0xffffu), 0.0625f), div255((float)(n01 >> 16), 0.0625f), s.full_range, s.matrix);
    p11 = yuv_to_rgba8(T.u8n[y1.y], div255((float)(n11 & 0xffffu), 0.0625f), div255((float)(n11 >> 16), 0.0625f), s.full_range, s.matrix);
}

// textureSample of a child through NodeTextureState::view()
__device__ __forceinline__ float4 sample_node(const Tables &T, const Tex *tex, int mode, float tx, float ty,
                                              bool &exact, uchar4 &texel) {
    exact = false;
    if (tex == nullptr || tex->kind == TEX_NONE) return make_float4(0.f, 0.f, 0.f, 0.f);  // default_empty_view
    const Tex &S = *tex;
    LinTap ax = linear_tap(tx, S.width), ay = linear_tap(ty, S.height);
    const float *lut = mode == 0 ? T.dec : T.u8n;
    // a weight of exactly 1 on the second tap is the same single-texel hit as a weight of 0
    if (ax.f == 1.0f) { ax.i0 = ax.i1; ax.f = 0.0f; }
    if (ay.f == 1.0f) { ay.i0 = ay.i1; ay.f = 0.0f; }
    uchar4 p00 = node_texel(T, S, ax.i0, ay.i0);
    if (ax.f == 0.0f && ay.f == 0.0f) {  // exact texel hit: the other three weights are zero
        exact = true;
        texel = p00;
        return make_float4(lut[p00.x], lut[p00.y], lut[p00.z], T.u8n[p00.w]);
    }
    uchar4 p10, p01, p11;
    if (ax.i1 == ax.i0 + 1 && ay.i1 == ay.i0 + 1 && yuv_quad_ok(S, ax.i0, ay.i0)) {
        yuv_quad(T, S, ax.i0, ay.i0, p00, p10, p01, p11);  // the 4 taps are one chroma-aligned quad (e.g. exact 2:1)
    } else {
        p10 = ax.f != 0.0f ? node_texel(T, S, ax.i1, ay.i0) : p00;
        p01 = ay.f != 0.0f ? node_texel(T, S, ax.i0, ay.i1) : p00;
        p11 = (ax.f != 0.0f && ay.f != 0.0f) ? node_texel(T, S, ax.i1, ay.i1) : (ax.f != 0.0f ? p10 : p01);
    }
    float4 r;
    if (mode != 0) {   // CpuOptimized: plain Rgba8Unorm node textures -> NC-6u on all four channels
        r.x = filter_u8(p00.x, p10.x, p01.x, p11.x, ax.f, ay.f);
        r.y = filter_u8(p00.y, p10.y, p01.y, p11.y, ax.f, ay.f);
        r.z = filter_u8(p00.z, p10.z, p01.z, p11.z, ax.f, ay.f);
        r.w = filter_u8(p00.w, p10.w, p01.w, p11.w, ax.f, ay.f);
        return r;
    }
    r.x = bilerp(lut[p00.x], lut[p10.x], lut[p01.x], lut[p11.x], ax.f, ay.f);
    r.y = bilerp(lut[p00.y], lut[p10.y], lut[p01.y], lut[p11.y], ax.f, ay.f);
    r.z = bilerp(lut[p00.z], lut[p10.z], lut[p01.z], lut[p11.z], ax.f, ay.f);
    r.w = bilerp(T.u8n[p00.w], T.u8n[p10.w], T.u8n[p01.w], T.u8n[p11.w], ax.f, ay.f);
    return r;
}

// textureGather(c, ...) of a child through the same view: component c of the four texels of sample_node's bilinear
// footprint (NC-6's taps, clamped to the edge), in the order (i0, i1), (i1, i1), (i1, i0), (i0, i0) of (x, y).  Each texel
// is decoded as a sample's taps are (NC-3 colour in GpuOptimized, NC-1 otherwise and for alpha); a YUV texture goes
// through node_texel, the per-texel fetch of sample_node's bilinear path.
__device__ __forceinline__ float4 gather_node(const Tables &T, const Tex *tex, int mode, float tx, float ty, int c) {
    if (tex == nullptr || tex->kind == TEX_NONE) return make_float4(0.f, 0.f, 0.f, 0.f);  // default_empty_view
    const LinTap ax = linear_tap(tx, tex->width), ay = linear_tap(ty, tex->height);
    const float *lut = mode == 0 && c < 3 ? T.dec : T.u8n;
    float r[4];
#pragma unroll 1
    for (int k = 0; k < 4; k++) {   // one node_texel in the code: a YUV fetch is long
        const uchar4 p = node_texel(T, *tex, k == 1 || k == 2 ? ax.i1 : ax.i0, k < 2 ? ay.i1 : ay.i0);
        r[k] = lut[c == 0 ? p.x : c == 1 ? p.y : c == 2 ? p.z : p.w];
    }
    return make_float4(r[0], r[1], r[2], r[3]);
}

// PREMULTIPLIED_ALPHA_BLENDING through the target's view: decode dst -> blend -> encode (per layer)
__device__ __forceinline__ uchar4 blend(const Tables &T, int mode, uchar4 dst, float4 s) {
    s.x = clamp01(s.x); s.y = clamp01(s.y); s.z = clamp01(s.z); s.w = clamp01(s.w);
    if (s.x == 0.0f && s.y == 0.0f && s.z == 0.0f && s.w == 0.0f) return dst;  // encode(decode(b)) == b
    float ia = 1.0f - s.w;
    uchar4 o;
    if (ia == 0.0f) {  // opaque source: fma(dst, 0, s) == s, the destination is never read
        if (mode == 0) {
            o.x = (unsigned char)srgb_encode(T, s.x);
            o.y = (unsigned char)srgb_encode(T, s.y);
            o.z = (unsigned char)srgb_encode(T, s.z);
        } else {
            o.x = (unsigned char)unorm8(s.x);
            o.y = (unsigned char)unorm8(s.y);
            o.z = (unsigned char)unorm8(s.z);
        }
        o.w = 255;
        return o;
    }
    if (mode == 0) {
        o.x = (unsigned char)srgb_encode(T, fmaf(T.dec[dst.x], ia, s.x));
        o.y = (unsigned char)srgb_encode(T, fmaf(T.dec[dst.y], ia, s.y));
        o.z = (unsigned char)srgb_encode(T, fmaf(T.dec[dst.z], ia, s.z));
    } else {
        o.x = (unsigned char)unorm8(fmaf(T.u8n[dst.x], ia, s.x));
        o.y = (unsigned char)unorm8(fmaf(T.u8n[dst.y], ia, s.y));
        o.z = (unsigned char)unorm8(fmaf(T.u8n[dst.z], ia, s.z));
    }
    o.w = (unsigned char)unorm8(fmaf(T.u8n[dst.w], ia, s.w));
    return o;
}

// The job of block b in a launch that draws several node textures: the last i with tile_begin[i] <= b
__device__ __forceinline__ int tile_job(const int32_t *__restrict__ tile_begin, int n_jobs, int b) {
    int lo = 0, hi = n_jobs - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (tile_begin[mid] <= b) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// Thread (0, 0) of such a launch: the block's job copied to the caller's shared `J`, and its 32 x 8 tile's origin
template <class Job>
__device__ __forceinline__ void load_block_job(const Job *__restrict__ jobs, const int32_t *__restrict__ tile_begin, int n_jobs,
                                               Job &J, int *origin) {
    const int b = (int)blockIdx.x, lo = tile_job(tile_begin, n_jobs, b);
    J = jobs[lo];
    const int t = b - tile_begin[lo], tiles_x = (J.dst.width + 31) / 32;
    origin[0] = (t % tiles_x) * 32;
    origin[1] = (t / tiles_x) * 8;
}
