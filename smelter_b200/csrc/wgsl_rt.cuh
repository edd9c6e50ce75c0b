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

// the uniform: read at WGSL uniform-address-space offsets from the node's parameter bytes (zero-padded to its size)
template <class T> __device__ inline T wld(const unsigned char *p) { return *(const T *)p; }
template <class T, int N> __device__ inline wv<T, N> wldv(const unsigned char *p) {
    wv<T, N> r;
    for (int i = 0; i < N; i++) r.v[i] = *(const T *)(p + 4 * i);
    return r;
}

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
};
