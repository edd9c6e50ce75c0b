// wgsl_rt.cuh -- what a WGSL shader translated by wgsl.cpp is compiled against, by NVRTC at smr_register_wgsl_shader.
// Never compiled by nvcc: renderer.cpp embeds it as a string and puts it in front of the translated source, which is then
// compiled as shader_rt.cuh describes.  It defines SMR_WGSL, which selects the rasterising main section of shader_rt.cuh.
//
// Every WGSL operation the translator emits is one of the functions below, so that the WGSL rules C++ does not give hold
// without undefined behaviour: i32 arithmetic wraps (it runs in u32), integer division by 0 gives the dividend and % by 0
// gives 0, INT_MIN / -1 gives INT_MIN and INT_MIN % -1 gives 0, shift counts are masked to the bit width, f32 -> i32 / u32
// conversions saturate (NaN gives 0), and an index into an array, vector or matrix is clamped to its last element (naga's
// Restrict policy).  Float arithmetic is plain IEEE f32 (--fmad=false: nothing is contracted).
#define SMR_WGSL 1

template <class T, int N> struct wv { T v[N]; };
template <int C, int R> struct wm { wv<float, R> c[C]; };
template <class T, int N> struct wa { T a[N]; };

template <class I> __device__ inline unsigned wg_idx(I i, unsigned n) { unsigned u = (unsigned)i; return u < n ? u : n - 1; }

// ---- scalars ----
__device__ inline int w_add(int a, int b) { return (int)((unsigned)a + (unsigned)b); }
__device__ inline int w_sub(int a, int b) { return (int)((unsigned)a - (unsigned)b); }
__device__ inline int w_mul(int a, int b) { return (int)((unsigned)a * (unsigned)b); }
__device__ inline int w_div(int a, int b) { return b == 0 ? a : (b == -1 && a == (-2147483647 - 1)) ? a : a / b; }
__device__ inline int w_mod(int a, int b) { return b == 0 || (b == -1 && a == (-2147483647 - 1)) ? 0 : a % b; }
__device__ inline unsigned w_add(unsigned a, unsigned b) { return a + b; }
__device__ inline unsigned w_sub(unsigned a, unsigned b) { return a - b; }
__device__ inline unsigned w_mul(unsigned a, unsigned b) { return a * b; }
__device__ inline unsigned w_div(unsigned a, unsigned b) { return b == 0 ? a : a / b; }
__device__ inline unsigned w_mod(unsigned a, unsigned b) { return b == 0 ? 0u : a % b; }
__device__ inline float w_add(float a, float b) { return a + b; }
__device__ inline float w_sub(float a, float b) { return a - b; }
__device__ inline float w_mul(float a, float b) { return a * b; }
__device__ inline float w_div(float a, float b) { return a / b; }
__device__ inline float w_mod(float a, float b) { return a - b * truncf(a / b); }   // WGSL: e1 - e2 * trunc(e1 / e2)
__device__ inline int w_neg(int a) { return (int)(0u - (unsigned)a); }
__device__ inline float w_neg(float a) { return -a; }
__device__ inline int w_shl(int a, unsigned b) { return (int)((unsigned)a << (b & 31u)); }
__device__ inline unsigned w_shl(unsigned a, unsigned b) { return a << (b & 31u); }
__device__ inline int w_shr(int a, unsigned b) { return a >> (b & 31u); }   // arithmetic, as WGSL's i32 >>
__device__ inline unsigned w_shr(unsigned a, unsigned b) { return a >> (b & 31u); }
template <class T> __device__ inline T w_and(T a, T b) { return a & b; }
template <class T> __device__ inline T w_or(T a, T b) { return a | b; }
template <class T> __device__ inline T w_xor(T a, T b) { return a ^ b; }
__device__ inline bool w_and(bool a, bool b) { return a && b; }
__device__ inline bool w_or(bool a, bool b) { return a || b; }
template <class T> __device__ inline T w_bnot(T a) { return ~a; }
__device__ inline bool w_lnot(bool a) { return !a; }
template <class T> __device__ inline bool w_eq(T a, T b) { return a == b; }
template <class T> __device__ inline bool w_ne(T a, T b) { return a != b; }
template <class T> __device__ inline bool w_lt(T a, T b) { return a < b; }
template <class T> __device__ inline bool w_le(T a, T b) { return a <= b; }
template <class T> __device__ inline bool w_gt(T a, T b) { return a > b; }
template <class T> __device__ inline bool w_ge(T a, T b) { return a >= b; }

// conversions (value constructors): wc<To>(from)
template <class To> __device__ inline To wc(float x);
template <> __device__ inline float wc<float>(float x) { return x; }
template <> __device__ inline int wc<int>(float x) {
    return x != x ? 0 : x >= 2147483648.0f ? 2147483647 : x < -2147483648.0f ? (-2147483647 - 1) : (int)x;
}
template <> __device__ inline unsigned wc<unsigned>(float x) {
    return x != x ? 0u : x >= 4294967296.0f ? 4294967295u : x <= -1.0f ? 0u : (unsigned)x;
}
template <> __device__ inline bool wc<bool>(float x) { return x != 0.0f; }
template <class To> __device__ inline To wc(int x) { return (To)x; }
template <class To> __device__ inline To wc(unsigned x) { return (To)x; }
template <class To> __device__ inline To wc(bool x) { return x ? (To)1 : (To)0; }
template <> __device__ inline bool wc<bool>(int x) { return x != 0; }
template <> __device__ inline bool wc<bool>(unsigned x) { return x != 0u; }
template <> __device__ inline bool wc<bool>(bool x) { return x; }
template <class To, class T, int N> __device__ inline wv<To, N> wc(const wv<T, N> &a) {
    wv<To, N> r;
    for (int i = 0; i < N; i++) r.v[i] = wc<To>(a.v[i]);
    return r;
}
template <class To> __device__ inline To wbits(float x) { return (To)__float_as_uint(x); }
template <> __device__ inline float wbits<float>(float x) { return x; }
template <class To> __device__ inline To wbits(unsigned x);
template <> __device__ inline float wbits<float>(unsigned x) { return __uint_as_float(x); }
template <> __device__ inline unsigned wbits<unsigned>(unsigned x) { return x; }
template <> __device__ inline int wbits<int>(unsigned x) { return (int)x; }
template <class To> __device__ inline To wbits(int x) { return wbits<To>((unsigned)x); }

// ---- vectors and matrices: componentwise ----
#define WG_VBIN(f)                                                                                                       \
    template <class T, int N> __device__ inline auto f(const wv<T, N> &a, const wv<T, N> &b) {                           \
        wv<decltype(f(a.v[0], b.v[0])), N> r;                                                                            \
        for (int i = 0; i < N; i++) r.v[i] = f(a.v[i], b.v[i]);                                                          \
        return r;                                                                                                        \
    }
#define WG_VUN(f)                                                                                                        \
    template <class T, int N> __device__ inline auto f(const wv<T, N> &a) {                                              \
        wv<decltype(f(a.v[0])), N> r;                                                                                    \
        for (int i = 0; i < N; i++) r.v[i] = f(a.v[i]);                                                                  \
        return r;                                                                                                        \
    }
#define WG_VTRI(f)                                                                                                       \
    template <class T, int N> __device__ inline wv<T, N> f(const wv<T, N> &a, const wv<T, N> &b, const wv<T, N> &c) {    \
        wv<T, N> r;                                                                                                      \
        for (int i = 0; i < N; i++) r.v[i] = f(a.v[i], b.v[i], c.v[i]);                                                  \
        return r;                                                                                                        \
    }
WG_VBIN(w_add) WG_VBIN(w_sub) WG_VBIN(w_div) WG_VBIN(w_mod) WG_VBIN(w_shl) WG_VBIN(w_shr)
WG_VBIN(w_and) WG_VBIN(w_or) WG_VBIN(w_xor) WG_VBIN(w_eq) WG_VBIN(w_ne) WG_VBIN(w_lt) WG_VBIN(w_le) WG_VBIN(w_gt) WG_VBIN(w_ge)
WG_VUN(w_neg) WG_VUN(w_bnot) WG_VUN(w_lnot)
template <class T, int N> __device__ inline wv<T, N> w_mul(const wv<T, N> &a, const wv<T, N> &b) {
    wv<T, N> r;
    for (int i = 0; i < N; i++) r.v[i] = w_mul(a.v[i], b.v[i]);
    return r;
}
template <int N, class T> __device__ inline wv<T, N> wsplat(T s) {
    wv<T, N> r;
    for (int i = 0; i < N; i++) r.v[i] = s;
    return r;
}
template <int... I, class T, int N> __device__ inline wv<T, (int)sizeof...(I)> wsw(const wv<T, N> &a) { return {{a.v[I]...}}; }

// vecN / matCxR constructors from a list of scalars and vectors, in order
template <class T, int N> struct wcat {
    wv<T, N> r;
    int k = 0;
    __device__ void put(T s) { r.v[k++] = s; }
    template <int M> __device__ void put(const wv<T, M> &a) { for (int i = 0; i < M; i++) r.v[k++] = a.v[i]; }
};
template <class T, int N, class... A> __device__ inline wv<T, N> wvec(const A &...a) {
    wcat<T, N> b;
    (b.put(a), ...);
    return b.r;
}
template <int C, int R, class... A> __device__ inline wm<C, R> wmat(const A &...a) {
    wv<float, C * R> f = wvec<float, C * R>(a...);
    wm<C, R> m;
    for (int c = 0; c < C; c++)
        for (int r = 0; r < R; r++) m.c[c].v[r] = f.v[c * R + r];
    return m;
}
template <int C, int R> __device__ inline wm<C, R> w_add(const wm<C, R> &a, const wm<C, R> &b) {
    wm<C, R> m;
    for (int c = 0; c < C; c++) m.c[c] = w_add(a.c[c], b.c[c]);
    return m;
}
template <int C, int R> __device__ inline wm<C, R> w_sub(const wm<C, R> &a, const wm<C, R> &b) {
    wm<C, R> m;
    for (int c = 0; c < C; c++) m.c[c] = w_sub(a.c[c], b.c[c]);
    return m;
}
template <int C, int R> __device__ inline wm<C, R> w_mul(const wm<C, R> &a, float s) {
    wm<C, R> m;
    for (int c = 0; c < C; c++) m.c[c] = w_mul(a.c[c], wsplat<R>(s));
    return m;
}
template <int C, int R> __device__ inline wm<C, R> w_mul(float s, const wm<C, R> &a) { return w_mul(a, s); }
// matrix products: each result component a sum in index order, from 0
template <int C, int R> __device__ inline wv<float, R> w_mul(const wm<C, R> &a, const wv<float, C> &v) {
    wv<float, R> r;
    for (int i = 0; i < R; i++) {
        float s = a.c[0].v[i] * v.v[0];
        for (int c = 1; c < C; c++) s = s + a.c[c].v[i] * v.v[c];
        r.v[i] = s;
    }
    return r;
}
template <int C, int R> __device__ inline wv<float, C> w_mul(const wv<float, R> &v, const wm<C, R> &a) {
    wv<float, C> r;
    for (int c = 0; c < C; c++) {
        float s = v.v[0] * a.c[c].v[0];
        for (int i = 1; i < R; i++) s = s + v.v[i] * a.c[c].v[i];
        r.v[c] = s;
    }
    return r;
}
template <int K, int R, int C> __device__ inline wm<C, R> w_mul(const wm<K, R> &a, const wm<C, K> &b) {
    wm<C, R> m;
    for (int c = 0; c < C; c++) m.c[c] = w_mul(a, b.c[c]);
    return m;
}
template <int C, int R> __device__ inline wm<R, C> wb_transpose(const wm<C, R> &a) {
    wm<R, C> m;
    for (int c = 0; c < C; c++)
        for (int r = 0; r < R; r++) m.c[r].v[c] = a.c[c].v[r];
    return m;
}

// ---- builtins ----
__device__ inline float wb_abs(float x) { return fabsf(x); }
__device__ inline int wb_abs(int x) { return x < 0 ? w_neg(x) : x; }
__device__ inline unsigned wb_abs(unsigned x) { return x; }
__device__ inline float wb_min(float a, float b) { return fminf(a, b); }
__device__ inline float wb_max(float a, float b) { return fmaxf(a, b); }
__device__ inline int wb_min(int a, int b) { return a < b ? a : b; }
__device__ inline int wb_max(int a, int b) { return a > b ? a : b; }
__device__ inline unsigned wb_min(unsigned a, unsigned b) { return a < b ? a : b; }
__device__ inline unsigned wb_max(unsigned a, unsigned b) { return a > b ? a : b; }
template <class T> __device__ inline T wb_clamp(T e, T lo, T hi) { return wb_min(wb_max(e, lo), hi); }
__device__ inline float wb_mix(float a, float b, float t) { return a * (1.0f - t) + b * t; }
__device__ inline float wb_step(float edge, float x) { return x >= edge ? 1.0f : 0.0f; }
__device__ inline float wb_smoothstep(float lo, float hi, float x) {
    float t = wb_clamp((x - lo) / (hi - lo), 0.0f, 1.0f);
    return t * t * (3.0f - 2.0f * t);
}
__device__ inline float wb_floor(float x) { return floorf(x); }
__device__ inline float wb_ceil(float x) { return ceilf(x); }
__device__ inline float wb_fract(float x) { return x - floorf(x); }
__device__ inline float wb_round(float x) { return rintf(x); }
__device__ inline float wb_trunc(float x) { return truncf(x); }
__device__ inline float wb_sqrt(float x) { return sqrtf(x); }
__device__ inline float wb_inverseSqrt(float x) { return 1.0f / sqrtf(x); }
__device__ inline float wb_pow(float a, float b) { return powf(a, b); }
__device__ inline float wb_exp(float x) { return expf(x); }
__device__ inline float wb_exp2(float x) { return exp2f(x); }
__device__ inline float wb_log(float x) { return logf(x); }
__device__ inline float wb_log2(float x) { return log2f(x); }
__device__ inline float wb_sin(float x) { return sinf(x); }
__device__ inline float wb_cos(float x) { return cosf(x); }
__device__ inline float wb_tan(float x) { return tanf(x); }
__device__ inline float wb_asin(float x) { return asinf(x); }
__device__ inline float wb_acos(float x) { return acosf(x); }
__device__ inline float wb_atan(float x) { return atanf(x); }
__device__ inline float wb_atan2(float y, float x) { return atan2f(y, x); }
__device__ inline float wb_sign(float x) { return x > 0.0f ? 1.0f : x < 0.0f ? -1.0f : 0.0f; }
__device__ inline int wb_sign(int x) { return x > 0 ? 1 : x < 0 ? -1 : 0; }
template <class T> __device__ inline T wb_select(T f, T t, bool c) { return c ? t : f; }
WG_VUN(wb_abs) WG_VBIN(wb_min) WG_VBIN(wb_max) WG_VTRI(wb_clamp) WG_VTRI(wb_mix) WG_VBIN(wb_step) WG_VTRI(wb_smoothstep)
WG_VUN(wb_floor) WG_VUN(wb_ceil) WG_VUN(wb_fract) WG_VUN(wb_round) WG_VUN(wb_trunc) WG_VUN(wb_sqrt) WG_VUN(wb_inverseSqrt)
WG_VBIN(wb_pow) WG_VUN(wb_exp) WG_VUN(wb_exp2) WG_VUN(wb_log) WG_VUN(wb_log2) WG_VUN(wb_sin) WG_VUN(wb_cos) WG_VUN(wb_tan)
WG_VUN(wb_asin) WG_VUN(wb_acos) WG_VUN(wb_atan) WG_VBIN(wb_atan2) WG_VUN(wb_sign)
template <class T, int N> __device__ inline wv<T, N> wb_select(const wv<T, N> &f, const wv<T, N> &t, const wv<bool, N> &c) {
    wv<T, N> r;
    for (int i = 0; i < N; i++) r.v[i] = c.v[i] ? t.v[i] : f.v[i];
    return r;
}
template <class T, int N> __device__ inline wv<T, N> wb_select(const wv<T, N> &f, const wv<T, N> &t, bool c) { return c ? t : f; }
// dot, length, distance, normalize: sums in component order
template <class T, int N> __device__ inline T wb_dot(const wv<T, N> &a, const wv<T, N> &b) {
    T s = w_mul(a.v[0], b.v[0]);
    for (int i = 1; i < N; i++) s = w_add(s, w_mul(a.v[i], b.v[i]));
    return s;
}
__device__ inline float wb_length(float x) { return fabsf(x); }
template <int N> __device__ inline float wb_length(const wv<float, N> &a) { return sqrtf(wb_dot(a, a)); }
template <class V> __device__ inline float wb_distance(const V &a, const V &b) { return wb_length(w_sub(a, b)); }
template <int N> __device__ inline wv<float, N> wb_normalize(const wv<float, N> &a) { return w_div(a, wsplat<N>(wb_length(a))); }
__device__ inline wv<float, 3> wb_cross(const wv<float, 3> &a, const wv<float, 3> &b) {
    return {{a.v[1] * b.v[2] - a.v[2] * b.v[1], a.v[2] * b.v[0] - a.v[0] * b.v[2], a.v[0] * b.v[1] - a.v[1] * b.v[0]}};
}
template <int N> __device__ inline bool wb_any(const wv<bool, N> &a) { bool r = false; for (int i = 0; i < N; i++) r = r || a.v[i]; return r; }
template <int N> __device__ inline bool wb_all(const wv<bool, N> &a) { bool r = true; for (int i = 0; i < N; i++) r = r && a.v[i]; return r; }
__device__ inline bool wb_any(bool a) { return a; }
__device__ inline bool wb_all(bool a) { return a; }

// numeric builtins (DESIGN.md, "WGSL builtins"): each rule is written out there and restated in numpy by
// tests/test_wgsl_builtins.py
__device__ inline float wb_saturate(float x) { return wb_clamp(x, 0.0f, 1.0f); }
__device__ inline float wb_degrees(float x) { return x * __uint_as_float(0x42652ee1u); }   // f32(180 / pi)
__device__ inline float wb_radians(float x) { return x * __uint_as_float(0x3c8efa35u); }   // f32(pi / 180)
__device__ inline float wb_fma(float a, float b, float c) { return fmaf(a, b, c); }
__device__ inline float wb_sinh(float x) { return sinhf(x); }
__device__ inline float wb_cosh(float x) { return coshf(x); }
__device__ inline float wb_tanh(float x) { return tanhf(x); }
__device__ inline float wb_asinh(float x) { return asinhf(x); }
__device__ inline float wb_acosh(float x) { return acoshf(x); }
__device__ inline float wb_atanh(float x) { return atanhf(x); }
// f32 -> f16 (round to nearest even, no flush) and back, in PTX: NVRTC compiles this without cuda_fp16.h
__device__ inline unsigned short wg_f16(float x) { unsigned short h; asm("cvt.rn.f16.f32 %0, %1;" : "=h"(h) : "f"(x)); return h; }
__device__ inline float wg_f32(unsigned short h) { float x; asm("cvt.f32.f16 %0, %1;" : "=f"(x) : "h"(h)); return x; }
__device__ inline float wb_quantizeToF16(float x) { return wg_f32(wg_f16(x)); }
WG_VUN(wb_saturate) WG_VUN(wb_degrees) WG_VUN(wb_radians) WG_VTRI(wb_fma) WG_VUN(wb_sinh) WG_VUN(wb_cosh) WG_VUN(wb_tanh)
WG_VUN(wb_asinh) WG_VUN(wb_acosh) WG_VUN(wb_atanh) WG_VUN(wb_quantizeToF16)
__device__ inline float wb_ldexp(float x, int e) { return ldexpf(x, e); }
template <int N> __device__ inline wv<float, N> wb_ldexp(const wv<float, N> &x, const wv<int, N> &e) {
    wv<float, N> r;
    for (int i = 0; i < N; i++) r.v[i] = ldexpf(x.v[i], e.v[i]);
    return r;
}
// the predeclared result structs: __frexp_result_f32 / _vecN_f32 { fract, exp } and __modf_result* { fract, whole }
template <class F, class E> struct wfrexp { F m_fract; E m_exp; };
template <class F> struct wmodf { F m_fract; F m_whole; };
__device__ inline wfrexp<float, int> wb_frexp(float x) {   // the fraction's magnitude in [0.5, 1); 0 gives (0, 0)
    wfrexp<float, int> r;
    r.m_fract = frexpf(x, &r.m_exp);
    return r;
}
template <int N> __device__ inline wfrexp<wv<float, N>, wv<int, N>> wb_frexp(const wv<float, N> &x) {
    wfrexp<wv<float, N>, wv<int, N>> r;
    for (int i = 0; i < N; i++) r.m_fract.v[i] = frexpf(x.v[i], &r.m_exp.v[i]);
    return r;
}
__device__ inline wmodf<float> wb_modf(float x) { const float w = truncf(x); return {x - w, w}; }
template <int N> __device__ inline wmodf<wv<float, N>> wb_modf(const wv<float, N> &x) {
    wmodf<wv<float, N>> r;
    for (int i = 0; i < N; i++) { r.m_whole.v[i] = truncf(x.v[i]); r.m_fract.v[i] = x.v[i] - r.m_whole.v[i]; }
    return r;
}
// cofactor expansion along the first column, terms added left to right; a[r][c] is row r, column c
template <int N> __device__ inline float wg_det(const float (&a)[N][N]) {
    float s = 0.0f;
    for (int i = 0; i < N; i++) {
        float m[N - 1][N - 1];
        for (int r = 0, k = 0; r < N; r++) {
            if (r == i) continue;
            for (int c = 1; c < N; c++) m[k][c - 1] = a[r][c];
            k++;
        }
        const float t = a[i][0] * wg_det<N - 1>(m);
        s = i == 0 ? t : (i & 1) ? s - t : s + t;
    }
    return s;
}
template <> __device__ inline float wg_det<1>(const float (&a)[1][1]) { return a[0][0]; }
template <int N> __device__ inline float wb_determinant(const wm<N, N> &m) {
    float a[N][N];
    for (int r = 0; r < N; r++)
        for (int c = 0; c < N; c++) a[r][c] = m.c[c].v[r];
    return wg_det<N>(a);
}
template <int N> __device__ inline wv<float, N> wb_faceForward(const wv<float, N> &e1, const wv<float, N> &e2, const wv<float, N> &e3) {
    return wb_dot(e2, e3) < 0.0f ? e1 : w_neg(e1);
}
template <int N> __device__ inline wv<float, N> wb_reflect(const wv<float, N> &e1, const wv<float, N> &e2) {
    const float k = 2.0f * wb_dot(e2, e1);
    wv<float, N> r;
    for (int i = 0; i < N; i++) r.v[i] = e1.v[i] - k * e2.v[i];
    return r;
}
template <int N> __device__ inline wv<float, N> wb_refract(const wv<float, N> &e1, const wv<float, N> &e2, float e3) {
    const float d = wb_dot(e2, e1), k = 1.0f - e3 * e3 * (1.0f - d * d);
    wv<float, N> r;
    if (k < 0.0f) return wsplat<N>(0.0f);
    const float s = e3 * d + sqrtf(k);
    for (int i = 0; i < N; i++) r.v[i] = e3 * e1.v[i] - s * e2.v[i];
    return r;
}

// bit builtins, i32 and u32
__device__ inline unsigned wb_countOneBits(unsigned x) { return (unsigned)__popc(x); }
__device__ inline int wb_countOneBits(int x) { return __popc((unsigned)x); }
__device__ inline unsigned wb_countLeadingZeros(unsigned x) { return (unsigned)__clz((int)x); }   // 32 for 0
__device__ inline int wb_countLeadingZeros(int x) { return __clz(x); }
__device__ inline unsigned wb_countTrailingZeros(unsigned x) { return x ? (unsigned)(__ffs((int)x) - 1) : 32u; }
__device__ inline int wb_countTrailingZeros(int x) { return (int)wb_countTrailingZeros((unsigned)x); }
__device__ inline unsigned wb_reverseBits(unsigned x) { return __brev(x); }
__device__ inline int wb_reverseBits(int x) { return (int)__brev((unsigned)x); }
__device__ inline unsigned wb_firstTrailingBit(unsigned x) { return x ? (unsigned)(__ffs((int)x) - 1) : 0xffffffffu; }
__device__ inline int wb_firstTrailingBit(int x) { return (int)wb_firstTrailingBit((unsigned)x); }
__device__ inline unsigned wb_firstLeadingBit(unsigned x) { return x ? 31u - (unsigned)__clz((int)x) : 0xffffffffu; }
__device__ inline int wb_firstLeadingBit(int x) {   // the highest bit that differs from the sign bit; -1 for 0 and -1
    const unsigned u = x < 0 ? ~(unsigned)x : (unsigned)x;
    return u ? 31 - __clz((int)u) : -1;
}
__device__ inline unsigned wg_bitmask(unsigned c) { return c >= 32u ? 0xffffffffu : (1u << c) - 1u; }   // bits [0, c)
__device__ inline unsigned wb_extractBits(unsigned e, unsigned offset, unsigned count) {
    const unsigned o = min(offset, 32u), c = min(count, 32u - o);
    return c == 0u ? 0u : (e >> o) & wg_bitmask(c);
}
__device__ inline int wb_extractBits(int e, unsigned offset, unsigned count) {   // sign-extended from bit c - 1
    const unsigned o = min(offset, 32u), c = min(count, 32u - o);
    return c == 0u ? 0 : (int)(wb_extractBits((unsigned)e, o, c) << (32u - c)) >> (32u - c);
}
__device__ inline unsigned wb_insertBits(unsigned e, unsigned newbits, unsigned offset, unsigned count) {
    const unsigned o = min(offset, 32u), c = min(count, 32u - o);
    if (c == 0u) return e;
    const unsigned mask = wg_bitmask(c) << o;
    return (e & ~mask) | ((newbits << o) & mask);
}
__device__ inline int wb_insertBits(int e, int newbits, unsigned offset, unsigned count) {
    return (int)wb_insertBits((unsigned)e, (unsigned)newbits, offset, count);
}
WG_VUN(wb_countOneBits) WG_VUN(wb_countLeadingZeros) WG_VUN(wb_countTrailingZeros) WG_VUN(wb_reverseBits)
WG_VUN(wb_firstTrailingBit) WG_VUN(wb_firstLeadingBit)
template <class T, int N> __device__ inline wv<T, N> wb_extractBits(const wv<T, N> &e, unsigned offset, unsigned count) {
    wv<T, N> r;
    for (int i = 0; i < N; i++) r.v[i] = wb_extractBits(e.v[i], offset, count);
    return r;
}
template <class T, int N> __device__ inline wv<T, N> wb_insertBits(const wv<T, N> &e, const wv<T, N> &b, unsigned offset, unsigned count) {
    wv<T, N> r;
    for (int i = 0; i < N; i++) r.v[i] = wb_insertBits(e.v[i], b.v[i], offset, count);
    return r;
}
__device__ inline unsigned wb_dot4U8Packed(unsigned a, unsigned b) {
    unsigned s = 0u;
    for (int i = 0; i < 32; i += 8) s += ((a >> i) & 255u) * ((b >> i) & 255u);
    return s;
}
__device__ inline int wb_dot4I8Packed(unsigned a, unsigned b) {
    int s = 0;
    for (int i = 0; i < 32; i += 8) s += (int)(signed char)(a >> i) * (int)(signed char)(b >> i);
    return s;
}

// packing: component i goes to byte / half-word i, from the least significant
template <int N> __device__ inline unsigned wg_pack(const wv<float, N> &e, float lo, float scale) {
    unsigned r = 0u;
    for (int i = 0; i < N; i++) {
        const int q = (int)floorf(0.5f + scale * wb_min(1.0f, wb_max(lo, e.v[i])));
        r |= ((unsigned)q & (N == 4 ? 0xffu : 0xffffu)) << (i * (32 / N));
    }
    return r;
}
__device__ inline unsigned wb_pack4x8snorm(const wv<float, 4> &e) { return wg_pack(e, -1.0f, 127.0f); }
__device__ inline unsigned wb_pack4x8unorm(const wv<float, 4> &e) { return wg_pack(e, 0.0f, 255.0f); }
__device__ inline unsigned wb_pack2x16snorm(const wv<float, 2> &e) { return wg_pack(e, -1.0f, 32767.0f); }
__device__ inline unsigned wb_pack2x16unorm(const wv<float, 2> &e) { return wg_pack(e, 0.0f, 65535.0f); }
__device__ inline unsigned wb_pack2x16float(const wv<float, 2> &e) { return (unsigned)wg_f16(e.v[0]) | ((unsigned)wg_f16(e.v[1]) << 16); }
__device__ inline wv<float, 4> wb_unpack4x8snorm(unsigned x) {
    wv<float, 4> r;
    for (int i = 0; i < 4; i++) r.v[i] = wb_max((float)(signed char)(x >> (8 * i)) / 127.0f, -1.0f);
    return r;
}
__device__ inline wv<float, 4> wb_unpack4x8unorm(unsigned x) {
    wv<float, 4> r;
    for (int i = 0; i < 4; i++) r.v[i] = (float)((x >> (8 * i)) & 255u) / 255.0f;
    return r;
}
__device__ inline wv<float, 2> wb_unpack2x16snorm(unsigned x) {
    return {{wb_max((float)(short)x / 32767.0f, -1.0f), wb_max((float)(short)(x >> 16) / 32767.0f, -1.0f)}};
}
__device__ inline wv<float, 2> wb_unpack2x16unorm(unsigned x) { return {{(float)(x & 0xffffu) / 65535.0f, (float)(x >> 16) / 65535.0f}}; }
__device__ inline wv<float, 2> wb_unpack2x16float(unsigned x) { return {{wg_f32((unsigned short)x), wg_f32((unsigned short)(x >> 16))}}; }

// the uniform: read at WGSL uniform-address-space offsets from the node's parameter bytes (zero-padded to its size)
template <class T> __device__ inline T wld(const unsigned char *p) { return *(const T *)p; }
template <class T, int N> __device__ inline wv<T, N> wldv(const unsigned char *p) {
    wv<T, N> r;
    for (int i = 0; i < N; i++) r.v[i] = *(const T *)(p + 4 * i);
    return r;
}

// A texture value is its index into the header's textures (an unsigned); the header has one sampler, so a sampler value
// carries nothing
struct wg_sampler {};

// the header's bindings: textures (group 0) through sampler_ (group 2), as smr_textures samples them
struct wg_textures {
    const smr::dev::Tables *T;
    const smr::dev::Tex *tex;
    unsigned count;
    int mode;
    __device__ wv<float, 4> sample(unsigned i, const wv<float, 2> &uv) const {
        bool exact;
        uchar4 texel;
        float4 c = smr::dev::sample_node(*T, i < count ? tex + i : nullptr, mode, uv.v[0], uv.v[1], exact, texel);
        return {{c.x, c.y, c.z, c.w}};
    }
    // the empty view is 1 x 1
    __device__ wv<unsigned, 2> dims(unsigned i) const {
        if (i >= count || tex[i].kind == smr::dev::TEX_NONE) return {{1u, 1u}};
        return {{(unsigned)tex[i].width, (unsigned)tex[i].height}};
    }
    // A node texture has one mip level and naga's Restrict policy clamps levels: a level, bias or gradient selects
    // level 0, so these are textureSample itself (the arguments are still evaluated, as WGSL evaluates them).
    __device__ wv<float, 4> sample_level(unsigned i, const wv<float, 2> &uv, float) const { return sample(i, uv); }
    __device__ wv<float, 4> sample_bias(unsigned i, const wv<float, 2> &uv, float) const { return sample(i, uv); }
    __device__ wv<float, 4> sample_grad(unsigned i, const wv<float, 2> &uv, const wv<float, 2> &, const wv<float, 2> &) const {
        return sample(i, uv);
    }
    template <class L> __device__ wv<unsigned, 2> dims(unsigned i, L) const { return dims(i); }
    __device__ unsigned levels(unsigned) const { return 1u; }
    // textureSampleBaseClampToEdge: each coordinate clamped to [0.5 / dim, 1 - 0.5 / dim], then the level-0 sample
    __device__ wv<float, 4> sample_clamped(unsigned i, const wv<float, 2> &uv) const {
        const wv<unsigned, 2> d = dims(i);
        wv<float, 2> c;
        for (int k = 0; k < 2; k++) {
            const float lo = 0.5f / (float)d.v[k];
            c.v[k] = wb_min(wb_max(uv.v[k], lo), 1.0f - lo);
        }
        return sample(i, c);
    }
    __device__ wv<float, 4> gather(int c, unsigned i, const wv<float, 2> &uv) const {
        float4 r = smr::dev::gather_node(*T, i < count ? tex + i : nullptr, mode, uv.v[0], uv.v[1], c);
        return {{r.x, r.y, r.z, r.w}};
    }
};
