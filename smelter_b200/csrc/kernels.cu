// kernels.cu -- hand-written sm_90a kernels of the per-output-frame compositor.
//
// Replaces the reference's WGSL shader set (SURVEY 2.2 K1..K11):
//   k_convert     planar_yuv_to_rgba.wgsl / nv12_to_rgba.wgsl / bgra / argb           (K1,K2,K4)
//   k_weights     the per-output-coordinate part of resample.wgsl:42-86               (K8 setup)
//   k_resample    resample.wgsl (Lanczos3 pass) and downsample.wgsl (box pass)         (K7,K8)
//   k_composite_p / k_composite_multi
//                 apply_layouts.wgsl: every layout of every output in ONE launch, painter's order kept per
//                 pixel in registers, fixed-function sRGB blend emulated per layer, fused with
//                 rgba_to_yuv.wgsl / rgba_to_nv12.wgsl on the way out                   (K9,K10,K11)
//   k_output      rgba_to_yuv / rgba_to_nv12 stand-alone (root size != output size, odd sizes)
//   k_fill        r8/rg8_fill_value.wgsl (black frame)                                  (K6)
//   k_transcode   gpu-video's vulkan_transcoder/shader.wgsl: NV12 -> up to eight NV12 renditions (transcode.cuh)
//   k_video_nv12_to_rgba  gpu-video's nv12_to_rgba.wgsl: NV12 -> RGBA8 at any size (video_convert.cuh)
//   k_deinterlace field / motion-adaptive deinterlacing of interlaced input planes (deinterlace.cuh; the reference has none)
//
// Numeric contract: identical to oracle/smelter_oracle.c (DESIGN.md section 3).  Compiled with
// -fmad=false: only explicit fmaf() is fused, every other operation rounds separately, division and
// sqrt are IEEE.  No tensor cores: there is no dense contraction on this path (HBM / FP32-ALU bound).
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <atomic>
#include <type_traits>
#include <cstring>
#include <utility>
#include <vector>

#include "kernels.h"
#include "interior.h"
#include "int_weights.h"

namespace smr {
namespace dev {

#include "ptx_helpers.cuh"

// ------------------------------------------------------------------------------------------------
// tables (NC-1, NC-3, NC-4) -- pushed from the host so host and device agree bit-for-bit.  Plain global
// memory: every block copies them to shared memory with one coalesced load per warp (a per-thread index into
// the constant bank would serialise 32 ways).
// ------------------------------------------------------------------------------------------------
#define ENC_KEY0 ((127 - 13) << 5)   // srgb_encode buckets: from x = 2^-13 (< thr[0]) ...
#define ENC_KEYS ((13 << 5) + 1)     // ... up to x = 1.0
__device__ unsigned char c_enc0[420];

#include "node_sample.cuh"

static thread_local char g_err[256] = {0};   // a launch and the read of its error happen on the same thread
const char *last_launch_error() { return g_err; }
static bool check_launch(const char *what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        snprintf(g_err, sizeof(g_err), "%s: %s", what, cudaGetErrorString(e));
        return false;
    }
    return true;
}

void upload_tables(const float *u8n, const float *dec, const float *thr) {
    float t[256];
    for (int i = 0; i < 255; i++) t[i] = thr[i];
    t[255] = 3.0e38f;
    cudaMemcpyToSymbol(c_u8n, u8n, sizeof(float) * 256);
    cudaMemcpyToSymbol(c_dec, dec, sizeof(float) * 256);
    cudaMemcpyToSymbol(c_thr, t, sizeof(float) * 256);
    float yl[256];  // same two f32 operations as yuv_to_rgba8's limited-range branch (no contraction possible)
    for (int i = 0; i < 256; i++) {
        volatile float d = u8n[i] - (16.0f / 255.0f);
        volatile float m = d * (1.0f / 0.85882352941f);
        yl[i] = m < 0.0f ? 0.0f : (m > 1.0f ? 1.0f : m);
    }
    cudaMemcpyToSymbol(c_yl, yl, sizeof(float) * 256);
    unsigned char enc0[420] = {0};
    for (int k = 0; k < ENC_KEYS; k++) {
        const uint32_t bits = (uint32_t)(k + ENC_KEY0) << 18;   // lower edge of the bucket
        float lo;
        memcpy(&lo, &bits, 4);
        int e = 0;
        while (e < 255 && lo >= t[e]) e++;
        enc0[k] = (unsigned char)e;
    }
    cudaMemcpyToSymbol(c_enc0, enc0, sizeof(enc0));
    static unsigned char enc1[ENC1_KEYS + 3];
    for (int k = 0; k < ENC1_KEYS; k++) {
        const uint32_t bits = (uint32_t)(k + ENC1_KEY0) << 15;
        float lo;
        memcpy(&lo, &bits, 4);
        int e = 0;
        while (e < 255 && lo >= t[e]) e++;
        enc1[k] = (unsigned char)e;
        if (k > 0 && enc1[k] - enc1[k - 1] > 1) {   // two thresholds inside one bucket: the one-compare encode would be wrong
            fprintf(stderr, "smelter_b200: sRGB encode bucket table is too coarse at key %d\n", k);
            abort();
        }
    }
    cudaMemcpyToSymbol(c_enc1, enc1, sizeof(enc1));
}

__global__ void __launch_bounds__(256) k_convert(Tex src, uint8_t *dst, int dst_pitch) {
    __shared__ Tables T;
    load_tables(T);
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= src.width || y >= src.height) return;
    reinterpret_cast<uchar4 *>(dst + (size_t)y * dst_pitch)[x] = node_texel(T, src, x, y);
}

int launch_convert_to_rgba(const Tex &src, uint8_t *dst, int dst_pitch, Stream s) {
    dim3 b(32, 8), g((src.width + 31) / 32, (src.height + 7) / 8);
    k_convert<<<g, b, 0, (cudaStream_t)s>>>(src, dst, dst_pitch);
    return check_launch("k_convert") ? 1 : -1;
}

// ------------------------------------------------------------------------------------------------
// K8 setup: Lanczos3 weights, resample.wgsl:42-86.  sin/cos are NC-8 (correctly rounded f32, through
// the fp64 unit); the rotation recurrence is the shader's.
// ------------------------------------------------------------------------------------------------
#define PI_F 3.14159265359f

__device__ __forceinline__ float sin_cr(float x) { return (float)sin((double)x); }
__device__ __forceinline__ float cos_cr(float x) { return (float)cos((double)x); }

__global__ void k_weights(const WeightJob *jobs) {
    const WeightJob J = jobs[blockIdx.y];
    int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= J.n_out) return;
    float kernel_scale = fmaxf(J.scale, 1.0f);
    float inv_k = 1.0f / kernel_scale;
    float support = 3.0f * kernel_scale;
    float center = (J.offset + ((float)o + 0.5f) * J.scale) - 0.5f;
    float first = ceilf(center - support);
    float x0 = (first - center) * inv_k;
    float s1 = sin_cr(PI_F * x0), c1 = cos_cr(PI_F * x0);
    float s3 = sin_cr(PI_F * x0 / 3.0f), c3 = cos_cr(PI_F * x0 / 3.0f);
    float sd1 = sin_cr(PI_F * inv_k), cd1 = cos_cr(PI_F * inv_k);
    float sd3 = sin_cr(PI_F * inv_k / 3.0f), cd3 = cos_cr(PI_F * inv_k / 3.0f);
    const float pi2 = PI_F * PI_F;
    float wsum = 0.0f;
    float *w = J.weights + (size_t)o * J.taps;
    for (int t = 0; t < J.taps; t++) {
        float x = x0 + (float)t * inv_k;
        float wt = 0.0f;
        if (fabsf(x) < 1e-5f) wt = 1.0f;
        else if (fabsf(x) < 3.0f) wt = ((3.0f * s1) * s3) / ((pi2 * x) * x);
        w[t] = wt;
        wsum += wt;
        float ns1 = s1 * cd1 + c1 * sd1;
        c1 = c1 * cd1 - s1 * sd1;
        s1 = ns1;
        float ns3 = s3 * cd3 + c3 * sd3;
        c3 = c3 * cd3 - s3 * sd3;
        s3 = ns3;
    }
    J.inv_wsum[o] = 1.0f / wsum;
    float fc = fminf(fmaxf(first, -1.0e9f), 1.0e9f);
    J.first[o] = (int)fc;
}

// k_weights of one mapping read back: the whole table, n_out x taps weights, and per output coordinate its 1 / weight_sum
// and first tap
int debug_weights(float scale, float offset, int n_out, float *w_host, size_t cap, int *taps_out, float *inv_host,
                  int32_t *first_host) {
    const float ks = fmaxf(scale, 1.0f);
    const int taps = (int)ceilf(2.0f * (3.0f * ks)) + 1;
    *taps_out = taps;
    const size_t nw = (size_t)n_out * taps;
    if (nw > cap) return 0;
    unsigned char *d = nullptr;
    if (cudaMalloc(&d, sizeof(WeightJob) + sizeof(float) * (nw + n_out) + sizeof(int32_t) * n_out) != cudaSuccess) return -1;
    WeightJob j{};
    j.scale = scale; j.offset = offset; j.n_out = n_out; j.taps = taps;
    j.weights = reinterpret_cast<float *>(d + sizeof(WeightJob));
    j.inv_wsum = j.weights + nw;
    j.first = reinterpret_cast<int32_t *>(j.inv_wsum + n_out);
    bool ok = cudaMemcpy(d, &j, sizeof(j), cudaMemcpyHostToDevice) == cudaSuccess &&
              launch_weights(reinterpret_cast<const WeightJob *>(d), &j, 1, nullptr) == 1 &&
              cudaMemcpy(w_host, j.weights, sizeof(float) * nw, cudaMemcpyDeviceToHost) == cudaSuccess &&
              cudaMemcpy(inv_host, j.inv_wsum, sizeof(float) * n_out, cudaMemcpyDeviceToHost) == cudaSuccess &&
              cudaMemcpy(first_host, j.first, sizeof(int32_t) * n_out, cudaMemcpyDeviceToHost) == cudaSuccess;
    cudaFree(d);
    return ok ? 1 : -1;
}

__global__ void k_debug_sincos(const float *x, int n, float *s, float *c) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    s[i] = sin_cr(x[i]);
    c[i] = cos_cr(x[i]);
}

// sin_cr / cos_cr, the NC-8 functions k_weights calls, on n host values
int debug_sincos(const float *x_host, int n, float *s_host, float *c_host) {
    float *d = nullptr;
    if (cudaMalloc(&d, sizeof(float) * 3 * (size_t)n) != cudaSuccess) return -1;
    bool ok = cudaMemcpy(d, x_host, sizeof(float) * n, cudaMemcpyHostToDevice) == cudaSuccess;
    if (ok) {
        k_debug_sincos<<<(n + 255) / 256, 256>>>(d, n, d + n, d + 2 * (size_t)n);
        ok = check_launch("k_debug_sincos") &&
             cudaMemcpy(s_host, d + n, sizeof(float) * n, cudaMemcpyDeviceToHost) == cudaSuccess &&
             cudaMemcpy(c_host, d + 2 * (size_t)n, sizeof(float) * n, cudaMemcpyDeviceToHost) == cudaSuccess;
    }
    cudaFree(d);
    return ok ? 1 : -1;
}

int launch_weights(const WeightJob *jobs_dev, const WeightJob *jobs_host, int n, Stream s) {
    if (n <= 0) return 0;
    int max_out = 1;
    for (int i = 0; i < n; i++) max_out = jobs_host[i].n_out > max_out ? jobs_host[i].n_out : max_out;
    dim3 b(128), g((max_out + 127) / 128, n);
    k_weights<<<g, b, 0, (cudaStream_t)s>>>(jobs_dev);
    return check_launch("k_weights") ? 1 : -1;
}

// ------------------------------------------------------------------------------------------------
// K7/K8: resampler passes.  One launch runs the same pass stage of every resampled child of the
// frame (blockIdx.z = job).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float4 rs_load(const Tables &T, const Tex &s, int x, int y) {
    if (s.kind == TEX_F16) {
        const uint2 raw = __ldg(reinterpret_cast<const uint2 *>(s.p0 + (size_t)y * s.pitch0) + x);
        __half2 a = *reinterpret_cast<const __half2 *>(&raw.x), b = *reinterpret_cast<const __half2 *>(&raw.y);
        float2 fa = __half22float2(a), fb = __half22float2(b);
        return make_float4(fa.x, fa.y, fb.x, fb.y);
    }
    uchar4 p = node_texel(T, s, x, y);  // fetched through the srgb view: decode rgb, alpha linear
    return make_float4(T.dec[p.x], T.dec[p.y], T.dec[p.z], T.u8n[p.w]);
}

__device__ __forceinline__ void rs_store(const Tables &T, const ResampleJob &J, int x, int y, float4 r) {
    if (J.dst_f16) {
        __half2 a = __floats2half2_rn(r.x, r.y), b = __floats2half2_rn(r.z, r.w);  // NC-5
        uint2 raw;
        raw.x = *reinterpret_cast<unsigned int *>(&a);
        raw.y = *reinterpret_cast<unsigned int *>(&b);
        reinterpret_cast<uint2 *>(J.dst + (size_t)y * J.dst_pitch)[x] = raw;
    } else {
        uchar4 o = make_uchar4((unsigned char)srgb_encode(T, r.x), (unsigned char)srgb_encode(T, r.y),
                               (unsigned char)srgb_encode(T, r.z), (unsigned char)unorm8(r.w));
        reinterpret_cast<uchar4 *>(J.dst + (size_t)y * J.dst_pitch)[x] = o;
    }
}

__global__ void __launch_bounds__(256) k_resample(const ResampleJob *jobs) {
    __shared__ Tables T;
    load_tables(T);
    const ResampleJob &J = jobs[blockIdx.z];
    int px = blockIdx.x * blockDim.x + threadIdx.x, py = blockIdx.y * blockDim.y + threadIdx.y;
    if (px >= J.dst_w || py >= J.dst_h) return;
    const Tex &S = J.src;
    if ((unsigned)J.box_fx * (unsigned)J.box_fy > 1u) {  // downsample.wgsl:28-41
        float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int dy = 0; dy < J.box_fy; dy++)
            for (int dx = 0; dx < J.box_fx; dx++) {
                int sx = min(px * J.box_fx + dx, S.width - 1), sy = min(py * J.box_fy + dy, S.height - 1);
                float4 t = rs_load(T, S, sx, sy);
                sum.x += t.x; sum.y += t.y; sum.z += t.z; sum.w += t.w;
            }
        float d = (float)((unsigned)J.box_fx * (unsigned)J.box_fy);
        rs_store(T, J, px, py, make_float4(sum.x / d, sum.y / d, sum.z / d, sum.w / d));
        return;
    }
    int o = J.axis == 1 ? py : px;
    int max_src = (J.axis == 1 ? S.height : S.width) - 1;
    int max_perp = (J.axis == 1 ? S.width : S.height) - 1;
    int perp = min(max((J.axis == 1 ? px : py) + J.perp_offset, 0), max_perp);
    const float *w = J.weights + (size_t)o * J.taps;
    int first = __ldg(J.first + o);
    float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int t = 0; t < J.taps; t++) {
        float wt = __ldg(w + t);
        if (wt == 0.0f) continue;  // exact: adds +-0 to a sum that is never -0
        int src = min(max(first + t, 0), max_src);
        float4 tx = J.axis == 1 ? rs_load(T, S, perp, src) : rs_load(T, S, src, perp);
        sum.x = fmaf(tx.x, wt, sum.x);
        sum.y = fmaf(tx.y, wt, sum.y);
        sum.z = fmaf(tx.z, wt, sum.z);
        sum.w = fmaf(tx.w, wt, sum.w);
    }
    float inv = __ldg(J.inv_wsum + o);
    rs_store(T, J, px, py, make_float4(sum.x * inv, sum.y * inv, sum.z * inv, sum.w * inv));
}

int launch_resample(const ResampleJob *jobs_dev, const ResampleJob *jobs_host, int n, Stream s) {
    if (n <= 0) return 0;
    int mw = 1, mh = 1;
    for (int i = 0; i < n; i++) {
        mw = jobs_host[i].dst_w > mw ? jobs_host[i].dst_w : mw;
        mh = jobs_host[i].dst_h > mh ? jobs_host[i].dst_h : mh;
    }
    dim3 b(32, 8), g((mw + 31) / 32, (mh + 7) / 8, n);
    k_resample<<<g, b, 0, (cudaStream_t)s>>>(jobs_dev);
    return check_launch("k_resample") ? 1 : -1;
}

// ------------------------------------------------------------------------------------------------
// K1/K2 + K8 + K8 fused: the common resample (YUV input, horizontal pass first, then vertical).
//
// One block owns a strip of 64 output columns and a run of output rows and streams DOWN the source:
//   phase A  each warp takes whole source rows: converts the strip's source pixels ONCE (K1/K2 -> RGBA8
//            quantisation -> sRGB decode), runs the horizontal Lanczos pass out of a per-warp shared-memory
//            row and stores the f16-quantised result into a ring of intermediate rows in shared memory;
//   phase B  each warp produces one output row: vertical Lanczos pass out of the ring, sRGB8 encode,
//            coalesced stores.
// Neither the RGBA8 node texture (4 B/px of the INPUT resolution) nor the Rgba16Float intermediate ever
// reaches HBM; a source row is converted once per strip.  Bit-identical to running K1, resample.wgsl pass 1
// (-> f16) and pass 2 (-> sRGB8) separately: every quantisation point is reproduced.
//
// Template parameter S: 0 = any ratio <= 4 (per-column weights and first-tap indices from shared memory);
// 2, 3, 4 = INTEGER horizontal ratio with a zero crop offset -- every grid / mosaic of the BASELINE configs.  Then first(o) = S*o + const and every output column
// has the same TAPS = 6S+1 weights (exact small-integer arithmetic in resample.wgsl:45-50), which allows:
//   * weights as immediates: every FFMA takes int_weight<S>(j) from int_weights.h, as k_resample_tma3 does;
//   * register blocking: a lane produces 2 adjacent output columns from one (S+TAPS)-long window;
//   * 64-column strips (less horizontal halo), one source row per warp step, so only ~4 KB of shared memory
//     per warp and 3 blocks (24 warps) per SM;
//   * K1/K2 on chroma-aligned pixel PAIRS (the .25/.75 taps of the two pixels share 3 chroma texels per row),
//     raw bytes of the next pair prefetched into registers while the current one is converted;
//   * conflict-free shared memory: value i of a row sits at i + i/(2S)  (lane stride 2S+1, odd);
//   * the f16 intermediate is kept AS f16 (half2 per lane) in the ring.
// Accumulation order per output is tap 0..TAPS-1 exactly as in the shader, so results are bit-identical.
// ------------------------------------------------------------------------------------------------
#define W64_TW 64
#define W64_WARPS 8
#define W64_RING 64

template <int S>   // S = 0: any ratio <= 4 (weights per column from shared memory)
struct W64 {
    static constexpr int SS = S == 0 ? 4 : S;                           // sizing ratio
    static constexpr int TAPS = 6 * SS + 1;
    static constexpr int SPAN = (W64_TW - 1) * SS + TAPS + 3;          // + chroma alignment / ceil slack
    static constexpr int ROWLEN = S == 0 ? ((SPAN + 2 + 7) & ~7) : (((SPAN + SPAN / (2 * SS) + 2) + 7) & ~7);
    struct Smem {
        Tables T;
        __half2 ring[W64_RING][3][W64_TW / 2];
        float4 srow[W64_WARPS][ROWLEN];                                // decoded source row, (r, g, b, -) per pixel
        float hw[S == 0 ? TAPS * W64_TW : 1];                          // any-ratio: the strip's weights, [tap][column]
    };
    // slot of pixel i in a source row: integer ratios pad one slot per 2*S so that the lanes' windows (stride 2*S
    // pixels) start 2*S+1 float4 apart -- conflict-free LDS.128; any-ratio rows are stored densely
    static __device__ __forceinline__ int pos(int i) { return S == 0 ? i : i + i / (2 * SS); }
};
// The host sends a job here at any ratio <= 4 with at most kFusedMaxTaps taps per axis and checks no span or ring bound:
// at those limits a strip's source span, ceil(63 * ratio) + taps + 2 pixels, fits a row, and the source rows of eight
// output rows, ceil(7 * ratio) + taps + 2, fit the ring.
static_assert((W64_TW - 1) * 4 + kFusedMaxTaps + 2 <= W64<0>::SPAN, "a strip's source span must fit a row");
static_assert((W64_WARPS - 1) * 4 + kFusedMaxTaps + 2 <= W64_RING, "eight output rows' source rows must fit the ring");

// Pull [p, p + bytes) towards L2, clipped to the plane [lo, hi): one bulk prefetch of exactly the span (16-byte
// granules) instead of whole 128-byte lines -- neighbouring strips' lines are not dragged in a second time.
__device__ __forceinline__ void prefetch_l2_span(const uint8_t *p, int bytes, const uint8_t *lo, const uint8_t *hi) {
    unsigned long long a = (unsigned long long)(p < lo ? lo : p), e = (unsigned long long)(p + bytes < hi ? p + bytes : hi);
    a = (a + 15ull) & ~15ull;
    if (e <= a + 16ull) return;
    const unsigned size = (unsigned)((e - a) & ~15ull);
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(a), "r"(size) : "memory");
}

// SRC: 0 planar 4:2:0 (K1), 1 NV12 (K2), 2 UYVY, 3 YUYV (K3: texel-centre chroma, no interpolation -- for even
// widths >= 8 the shader's coordinate round trip lands on pixel x's own texel (x >> 1) with weight exactly 1)
// MAT: the matrix (Tex::matrix) of every source of the launch.  FULL: the range of every source of the launch for the
// interleaved sources (the host keys their launches by it); 4:2:0 sources read the range per job, with FULL false.
template <int S, int SRC, int MAT, bool FULL>
__global__ void __launch_bounds__(32 * W64_WARPS, 3) k_resample_fused_int(const FusedJob *jobs, const FusedPiece *pieces,
                                                                            const int *piece_begin) {
    constexpr bool NV12 = SRC == 1, IL = SRC >= 2;
    using K = W64<S>;
    constexpr int TAPS = K::TAPS;  // S > 0: exact tap count; S == 0: upper bound (the job's taps_h is used)
    constexpr int WIN = S + TAPS;  // S > 0: window feeding 2 adjacent output columns
    extern __shared__ __align__(16) unsigned char fs_raw[];
    typename K::Smem &M = *reinterpret_cast<typename K::Smem *>(fs_raw);
    load_tables(M.T);
    const int lane = threadIdx.x, warp = threadIdx.y;
    // Persistent grid: exactly (SMs x resident blocks) blocks, each owning an EQUAL share of the launch's output
    // rows as a short list of pieces (job, strip, row range) cut by the host -- no partial last wave.
    for (int pi = __ldg(piece_begin + blockIdx.x); pi < __ldg(piece_begin + blockIdx.x + 1); pi++) {
    const FusedPiece P = pieces[pi];
    const FusedJob &J = jobs[P.job];
    const int th = S == 0 ? J.taps_h : TAPS;
    const int ox0 = P.strip * W64_TW;
    const int oy_begin = P.oy_begin, oy_end = P.oy_end;
    const Tex &src = J.src;
    const int W = src.width, H = src.height, chei = H >> 1;
    const int tv = J.taps_v;
    const int xa = __ldg(J.first_h + ox0);      // S > 0: first(o) = S*o + const
    const int xa_e = xa & ~1;                   // chroma-aligned start
    const int d0 = xa - xa_e;
    // generic ratio: per-column first tap, 1/weight_sum and weights (columns 2*lane and 2*lane+1)
    const int oc0 = min(ox0 + 2 * lane, J.dst_w - 1), oc1 = min(ox0 + 2 * lane + 1, J.dst_w - 1);
    int gi0 = 0, gD = 0, npairs_g = 0;
    float inv0, inv1;
    if constexpr (S == 0) {
        const int f0 = __ldg(J.first_h + oc0), f1 = __ldg(J.first_h + oc1);
        gi0 = f0 - xa_e; gD = f1 - f0;
        inv0 = __ldg(J.inv_h + oc0); inv1 = __ldg(J.inv_h + oc1);
        const int o_last = min(ox0 + W64_TW - 1, J.dst_w - 1);
        npairs_g = (min(__ldg(J.first_h + o_last) + th - xa_e, K::SPAN) + 1) >> 1;
        for (int t = warp; t < th; t += W64_WARPS) {   // [tap][column]: conflict-free reads in A2
            M.hw[t * W64_TW + 2 * lane] = __ldg(J.w_h + (size_t)oc0 * th + t);
            M.hw[t * W64_TW + 2 * lane + 1] = __ldg(J.w_h + (size_t)oc1 * th + t);
        }
        __syncthreads();
    } else {
        inv0 = inv1 = int_inv<S>();
    }
    // S > 0: the strip's pair count is a constant (d0 = 1 needs one pair less for S = 3; the extra one is harmless)
    constexpr int NP = ((W64_TW - 1) * K::SS + TAPS + 2) >> 1, NIT = (NP + 31) / 32;
    const int npairs = S == 0 ? npairs_g : NP;
    const int full_range = src.full_range;
    constexpr YuvCoef kc = yuv_coef(MAT);
    // pairs whose pixels and chroma taps need no clamping: x = xa_e + 2p >= 2 and x + 3 <= W - 1
    // (interleaved sources have no chroma neighbours: x >= 0 and x + 1 <= W - 1)
    const int p_in_lo = IL ? (xa_e >= 0 ? 0 : (1 - xa_e) >> 1) : (xa_e >= 2 ? 0 : (2 - xa_e + 1) >> 1);
    const int p_in_hi = IL ? (W - 2 - xa_e) >> 1 : (W - 4 - xa_e) >> 1;
    const int p_hi = min(p_in_hi, npairs - 1);   // last pair of the strip on the unclamped path
    // S > 0: pixel x is stored at slot x - xa so that lane l's window starts at slot 2*S*l (compile-time offsets)
    const int dsh = S == 0 ? 0 : d0;

    int produced_hi = -0x40000000;
    for (int o0 = oy_begin; o0 < oy_end; o0 += W64_WARPS) {
        const int o_l = min(o0 + W64_WARPS - 1, oy_end - 1);
        const int need_lo = min(max(__ldg(J.first_v + o0), 0), H - 1);
        const int need_hi = min(max(__ldg(J.first_v + o_l) + tv - 1, 0), H - 1);
        const int start = max(produced_hi + 1, need_lo);
        {   // pull the NEXT group's source rows towards L2 while this group computes: 32 rows x (luma, chroma) spans
            const int tid = warp * 32 + lane;
            const int nr = need_hi + 1 + (tid >> 2), part = tid & 3;
            if (tid < 128 && nr < H) {
                const int xb = max(xa_e - 2, 0), span = K::SPAN + 4;   // the strip's pixels plus the chroma neighbours
                if (IL) {
                    if (part == 0) prefetch_l2_span(src.p0 + (size_t)nr * src.pitch0 + 2 * xb, 2 * span, src.p0, src.p0 + (size_t)H * src.pitch0);
                } else if (part == 0) {
                    prefetch_l2_span(src.p0 + (size_t)nr * src.pitch0 + xb, span, src.p0, src.p0 + (size_t)H * src.pitch0);
                } else if ((nr & 1) == 0) {
                    const int cyn = min(nr >> 1, chei - 1);
                    if (NV12) {
                        if (part == 1) prefetch_l2_span(src.p1 + (size_t)cyn * src.pitch1 + xb, span, src.p1, src.p1 + (size_t)chei * src.pitch1);
                    } else if (part == 1) {
                        prefetch_l2_span(src.p1 + (size_t)cyn * src.pitch1 + (xb >> 1), span >> 1, src.p1, src.p1 + (size_t)chei * src.pitch1);
                    } else if (part == 2) {
                        prefetch_l2_span(src.p2 + (size_t)cyn * src.pitch2 + (xb >> 1), span >> 1, src.p2, src.p2 + (size_t)chei * src.pitch2);
                    }
                }
            }
        }
        // ---- phase A: one source row per warp step -----------------------------------------------------
        for (int r = start + warp; r <= need_hi; r += W64_WARPS) {
            float4 *row = M.srow[warp];
            // A1: K1/K2 -> u8 -> sRGB decode of the strip's pixels of row r
            {
                const uint8_t *yrow = src.p0 + (size_t)r * src.pitch0;
                const int cy0 = (r & 1) ? (r >> 1) : max((r >> 1) - 1, 0), cy1 = (r & 1) ? min((r >> 1) + 1, chei - 1) : (r >> 1);
                const uint8_t *c0a = IL ? nullptr : src.p1 + (size_t)cy0 * src.pitch1, *c1a = IL ? nullptr : src.p1 + (size_t)cy1 * src.pitch1;
                const uint8_t *c0b = (NV12 || IL) ? nullptr : src.p2 + (size_t)cy0 * src.pitch2;
                const uint8_t *c1b = (NV12 || IL) ? nullptr : src.p2 + (size_t)cy1 * src.pitch2;
                const bool odd = r & 1;
                // raw bytes of one pixel pair, each in a full register: luma pair (y0 | y1 << 8) and the three chroma
                // taps of both chroma rows (NV12: u | v << 8 as loaded; planar: u | v << 16)
                struct Raw { unsigned y, a0, b0, d0, a1, b1, d1; };
                auto load_raw = [&](int pp, Raw &R) {
                    const int x = xa_e + 2 * pp, cx = x >> 1;
                    if (IL) {   // one texel = the pixel pair: {U,Y0,V,Y1} or {Y0,U,Y1,V}
                        R.y = __ldg(reinterpret_cast<const unsigned int *>(yrow) + cx);
                        return;
                    }
                    if (NV12) {
                        const unsigned short *r0 = reinterpret_cast<const unsigned short *>(c0a) + cx;
                        const unsigned short *r1 = reinterpret_cast<const unsigned short *>(c1a) + cx;
                        R.a0 = __ldg(r0 - 1); R.b0 = __ldg(r0); R.d0 = __ldg(r0 + 1);
                        R.a1 = __ldg(r1 - 1); R.b1 = __ldg(r1); R.d1 = __ldg(r1 + 1);
                    } else {
                        R.a0 = __ldg(c0a + cx - 1) | ((unsigned)__ldg(c0b + cx - 1) << 16);
                        R.b0 = __ldg(c0a + cx) | ((unsigned)__ldg(c0b + cx) << 16);
                        R.d0 = __ldg(c0a + cx + 1) | ((unsigned)__ldg(c0b + cx + 1) << 16);
                        R.a1 = __ldg(c1a + cx - 1) | ((unsigned)__ldg(c1b + cx - 1) << 16);
                        R.b1 = __ldg(c1a + cx) | ((unsigned)__ldg(c1b + cx) << 16);
                        R.d1 = __ldg(c1a + cx + 1) | ((unsigned)__ldg(c1b + cx + 1) << 16);
                    }
                    R.y = __ldg(reinterpret_cast<const unsigned short *>(yrow + x));
                };
                auto spread = [&](unsigned c) { return NV12 ? __byte_perm(c, 0, 0x4140) : c; };  // -> u | v << 16
                auto put = [&](int i, int r8, int g8, int b8) {
                    row[K::pos(i)] = make_float4(M.T.dec[r8], M.T.dec[g8], M.T.dec[b8], 0.0f);
                };
                auto convert_store = [&](const Raw &R, int p) {
                    if constexpr (IL) {
                        const unsigned t = R.y;
                        const unsigned ub = SRC == 2 ? (t & 0xffu) : ((t >> 8) & 0xffu), vb = SRC == 2 ? ((t >> 16) & 0xffu) : (t >> 24);
                        const unsigned y0 = SRC == 2 ? ((t >> 8) & 0xffu) : (t & 0xffu), y1 = SRC == 2 ? (t >> 24) : ((t >> 16) & 0xffu);
                        const float u = M.T.u8n[ub], v = M.T.u8n[vb];   // texel hit: exactly b / 255 (NC-1)
                        const int i = 2 * p - dsh;
                        int r8, g8, b8;
                        yuv_to_rgb8n(FULL ? M.T.u8n[y0] : M.T.yl[y0], u, v, FULL, kc, r8, g8, b8);
                        if (i >= 0) put(i, r8, g8, b8);
                        yuv_to_rgb8n(FULL ? M.T.u8n[y1] : M.T.yl[y1], u, v, FULL, kc, r8, g8, b8);
                        put(i + 1, r8, g8, b8);
                        return;
                    }
                    // NC-6u chroma: u in bits 0..15, v in bits 16..31 of one register (max 4080 < 65536)
                    const unsigned a0 = spread(R.a0), b0 = 3u * spread(R.b0), e0 = spread(R.d0);
                    const unsigned a1 = spread(R.a1), b1 = 3u * spread(R.b1), e1 = spread(R.d1);
                    // even pixel: taps (cx-1, cx) weights (1/4, 3/4); odd pixel: taps (cx, cx+1) weights (3/4, 1/4)
                    const unsigned he0 = a0 + b0, ho0 = b0 + e0, he1 = a1 + b1, ho1 = b1 + e1;
                    // row weights: even row (1/4, 3/4) on chroma rows (cy0, cy1); odd row (3/4, 1/4)
                    const unsigned ne = odd ? 3u * he0 + he1 : he0 + 3u * he1;
                    const unsigned no = odd ? 3u * ho0 + ho1 : ho0 + 3u * ho1;
                    const float ue = div255((float)(ne & 0xffffu), 0.0625f), ve = div255((float)(ne >> 16), 0.0625f);
                    const float uo = div255((float)(no & 0xffffu), 0.0625f), vo = div255((float)(no >> 16), 0.0625f);
                    const int i = 2 * p - dsh;
                    int r8, g8, b8;
                    // luma by arithmetic, not by table: f32(y/255) exactly (div255), then the same two f32 operations as the
                    // table entry -- trades one conflict-prone LDS per pixel for three FP32 instructions
                    auto luma = [&](unsigned yb) {
                        const float yn = div255((float)yb, 1.0f);
                        return full_range ? yn : clamp01((yn - K16) * RCP_Y);
                    };
                    yuv_to_rgb8n(luma(R.y & 0xffu), ue, ve, full_range, kc, r8, g8, b8);
                    if (i >= 0) put(i, r8, g8, b8);
                    yuv_to_rgb8n(luma(R.y >> 8), uo, vo, full_range, kc, r8, g8, b8);
                    put(i + 1, r8, g8, b8);
                };
                auto inside = [&](int pp) { return pp >= p_in_lo && pp <= p_hi; };
                auto border = [&](int p) {   // image border: resample.wgsl clamps the tap index
                    const int x = xa_e + 2 * p, i = 2 * p - dsh;
                    const uchar4 pe = node_texel<MAT, FULL>(M.T, src, min(max(x, 0), W - 1), r);
                    const uchar4 po = node_texel<MAT, FULL>(M.T, src, min(max(x + 1, 0), W - 1), r);
                    if (i >= 0) put(i, pe.x, pe.y, pe.z);
                    put(i + 1, po.x, po.y, po.z);
                };
                // unclamped pairs: the next pair's bytes are in flight while this one converts
                Raw cur, nxt;
                bool ok = inside(lane);
                if (ok) load_raw(lane, cur);
                if constexpr (S != 0) {
#pragma unroll
                    for (int it = 0; it < NIT; it++) {
                        const int p = lane + 32 * it;
                        const bool ok_n = it + 1 < NIT && inside(p + 32);
                        if (ok_n) load_raw(p + 32, nxt);
                        if (ok) convert_store(cur, p);
                        cur = nxt; ok = ok_n;
                    }
                } else {
                    for (int p = lane; p < npairs; p += 32) {
                        const bool ok_n = inside(p + 32);
                        if (ok_n) load_raw(p + 32, nxt);
                        if (ok) convert_store(cur, p);
                        cur = nxt; ok = ok_n;
                    }
                }
                if (p_in_lo > 0 || p_hi < npairs - 1)   // strips touching the left / right image edge only
                    for (int p = lane; p < npairs; p += 32)
                        if (!inside(p)) border(p);
            }
            __syncwarp();
            // A2: horizontal Lanczos, each lane 2 adjacent output columns; one LDS.128 feeds six FMAs
            {
                __half2 *ringrow = &M.ring[r & (W64_RING - 1)][0][0];
                float r0 = 0.f, g0 = 0.f, b0 = 0.f, r1 = 0.f, g1 = 0.f, b1 = 0.f;
                if constexpr (S == 0) {
                    const float *w0 = M.hw + 2 * lane, *w1 = M.hw + 2 * lane + 1 - gD * W64_TW;
                    const int win = th + gD;  // union of the two columns' windows (first is non-decreasing)
                    const float4 *sp = row + gi0;
#pragma unroll 4
                    for (int j = 0; j < win; j++) {
                        const float4 v = sp[j];
                        if (j < th) { const float w = w0[j * W64_TW]; r0 = fmaf(v.x, w, r0); g0 = fmaf(v.y, w, g0); b0 = fmaf(v.z, w, b0); }
                        if (j >= gD) { const float w = w1[j * W64_TW]; r1 = fmaf(v.x, w, r1); g1 = fmaf(v.y, w, g1); b1 = fmaf(v.z, w, b1); }
                    }
                } else {
                    const float4 *sp = row + (2 * S + 1) * lane;   // pos(2*S*lane + j) = (2*S+1)*lane + pos(j)
#pragma unroll
                    for (int j = 0; j < WIN; j++) {
                        const float4 v = sp[K::pos(j)];
                        if (j < TAPS) { const float w = int_weight<S>(j); r0 = fmaf(v.x, w, r0); g0 = fmaf(v.y, w, g0); b0 = fmaf(v.z, w, b0); }
                        if (j >= S) { const float w = int_weight<S>(j - S); r1 = fmaf(v.x, w, r1); g1 = fmaf(v.y, w, g1); b1 = fmaf(v.z, w, b1); }
                    }
                }
                ringrow[lane] = __floats2half2_rn(r0 * inv0, r1 * inv1);  // NC-5
                ringrow[W64_TW / 2 + lane] = __floats2half2_rn(g0 * inv0, g1 * inv1);
                ringrow[W64_TW + lane] = __floats2half2_rn(b0 * inv0, b1 * inv1);
            }
            __syncwarp();
        }
        produced_hi = max(produced_hi, need_hi);
        __syncthreads();
        // ---- phase B: vertical pass, one output row per warp, 2 columns per lane (any ratio) ----------------
        const int oy = o0 + warp;
        if (oy < oy_end) {
            const int fv = __ldg(J.first_v + oy);
            const float *wv = J.w_v + (size_t)oy * tv;
            float r0 = 0.f, g0 = 0.f, b0 = 0.f, r1 = 0.f, g1 = 0.f, b1 = 0.f;
            const bool inside = fv >= 0 && fv + tv - 1 <= H - 1;
            for (int t = 0; t < tv; t++) {
                const float wt = __ldg(wv + t);
                const int row = inside ? fv + t : min(max(fv + t, 0), H - 1);
                const __half2 *p = &M.ring[row & (W64_RING - 1)][0][0];
                const float2 vr = __half22float2(p[lane]), vg = __half22float2(p[W64_TW / 2 + lane]), vb = __half22float2(p[W64_TW + lane]);
                r0 = fmaf(vr.x, wt, r0); r1 = fmaf(vr.y, wt, r1);
                g0 = fmaf(vg.x, wt, g0); g1 = fmaf(vg.y, wt, g1);
                b0 = fmaf(vb.x, wt, b0); b1 = fmaf(vb.y, wt, b1);
            }
            const float inv_v = __ldg(J.inv_v + oy);
            const int ox = ox0 + 2 * lane;
            uchar4 oa = make_uchar4((unsigned char)srgb_encode(M.T, r0 * inv_v), (unsigned char)srgb_encode(M.T, g0 * inv_v),
                                    (unsigned char)srgb_encode(M.T, b0 * inv_v), 255);
            uchar4 ob = make_uchar4((unsigned char)srgb_encode(M.T, r1 * inv_v), (unsigned char)srgb_encode(M.T, g1 * inv_v),
                                    (unsigned char)srgb_encode(M.T, b1 * inv_v), 255);
            uchar4 *drow = reinterpret_cast<uchar4 *>(J.dst + (size_t)oy * J.dst_pitch);
            if (ox + 1 < J.dst_w && (J.dst_pitch & 7) == 0) {
                uint2 pk;
                pk.x = *reinterpret_cast<unsigned int *>(&oa);
                pk.y = *reinterpret_cast<unsigned int *>(&ob);
                *reinterpret_cast<uint2 *>(drow + ox) = pk;
            } else {
                if (ox < J.dst_w) drow[ox] = oa;
                if (ox + 1 < J.dst_w) drow[ox + 1] = ob;
            }
        }
        __syncthreads();
    }
    }  // pieces
}

}  // namespace dev
}  // namespace smr
namespace smr {
namespace dev {
// rgba_to_yuv.wgsl:26-54 on raw stored bytes
__device__ __forceinline__ float to_y(float r, float g, float b) {
    float y = fmaf(b, 0.0722f, fmaf(g, 0.7152f, r * 0.2126f));
    return fmaf(y, 0.85882352941f, K16);
}
__device__ __forceinline__ float to_u(float r, float g, float b) {
    float u = fmaf(b, 0.5f, fmaf(g, -0.3854f, r * -0.1146f));
    return fmaf(u + 0.5f, 0.87843137254f, K16);
}
__device__ __forceinline__ float to_v(float r, float g, float b) {
    float v = fmaf(b, -0.0458f, fmaf(g, -0.4542f, r * 0.5f));
    return fmaf(v + 0.5f, 0.87843137254f, K16);
}

// K10 / K11 of one 2 x 2 block of final target bytes (little-endian RGBA8 words; rgba_to_yuv.wgsl / rgba_to_nv12.wgsl), the
// very operations of the composite's fused output stage: Y per pixel from the raw bytes, chroma from the exact mean of
// the four bytes (NC-6u at the .5 / .5 taps of an even-sized target).  (X, Y) even: frame position of the block.
__device__ __forceinline__ void emit_yuv_2x2(const FusedJob &J, int X, int Y, uint32_t p00, uint32_t p10, uint32_t p01, uint32_t p11) {
    using namespace tma;
    // The arithmetic of the composite's output stage, operation for operation, two values per instruction (packed FP32) and
    // without the conversion unit (I2F / F2I run at a fraction of the FP32 rate): a byte or 16-bit field goes under the
    // exponent of 2^23 by PRMT and 2^23 is subtracted (exact); the UNORM8 store rounds by the magic add (== __float2int_rn
    // below 2^22); clamp01 is the .SAT of the producing fma.
    const float2 m23 = splat(-8388608.0f);
    const float2 c = splat(__uint_as_float(0x3b808081u)), lo = splat(__uint_as_float(0xaf7efeffu));   // div255(n, 1): fma(n, c, n * lo)
    auto pairf = [&](uint32_t a, uint32_t b, uint32_t sel) {   // exact floats of one byte of a and of b
        return add2(make_float2(__uint_as_float(__byte_perm(a, 0x4B000000u, sel)), __uint_as_float(__byte_perm(b, 0x4B000000u, sel))), m23);
    };
    auto unit = [&](float2 n) { return fma2(n, c, mul2(n, lo)); };                                      // T.u8n[] of two bytes
    auto store2 = [&](float2 x01) -> uint32_t {   // two unorm8(): x01 already clamped to [0, 1]; bytes in bits 0..7 and 8..15
        const float2 q = add2_after_mul(mul2(x01, splat(255.0f)), splat(12582912.0f));
        return (__float_as_uint(q.x) & 0xffu) | ((__float_as_uint(q.y) & 0xffu) << 8);
    };
    auto lum2 = [&](uint32_t a, uint32_t b) -> uint32_t {   // to_y() of two pixels
        const float2 r = unit(pairf(a, b, 0x7540u)), g = unit(pairf(a, b, 0x7541u)), bl = unit(pairf(a, b, 0x7542u));
        const float2 y = fma2(bl, splat(0.0722f), fma2(g, splat(0.7152f), mul2(r, splat(0.2126f))));
        return store2(make_float2(__saturatef(fmaf(y.x, 0.85882352941f, K16)), __saturatef(fmaf(y.y, 0.85882352941f, K16))));
    };
    *reinterpret_cast<unsigned short *>(J.out0 + (size_t)Y * J.out_pitch0 + X) = (unsigned short)lum2(p00, p10);
    *reinterpret_cast<unsigned short *>(J.out0 + (size_t)(Y + 1) * J.out_pitch0 + X) = (unsigned short)lum2(p01, p11);
    // sums of the four bytes per channel, two channels per word: (r, b) in the 16-bit halves of one, (g, a) of the other
    const uint32_t m = 0x00ff00ffu;
    const uint32_t srb = (p00 & m) + (p10 & m) + (p01 & m) + (p11 & m);
    const uint32_t sga = ((p00 >> 8) & m) + ((p10 >> 8) & m) + ((p01 >> 8) & m) + ((p11 >> 8) & m);
    const float2 c4 = splat(__uint_as_float(0x3b808081u) * 0.25f), lo4 = splat(__uint_as_float(0xaf7efeffu) * 0.25f);   // div255(n, 0.25)
    const float2 nrg = add2(make_float2(__uint_as_float(__byte_perm(srb, 0x4B000000u, 0x7610u)), __uint_as_float(__byte_perm(sga, 0x4B000000u, 0x7610u))), m23);
    const float nb = __uint_as_float(__byte_perm(srb, 0x4B000000u, 0x7632u)) - 8388608.0f;
    const float2 rg = fma2(nrg, c4, mul2(nrg, lo4));
    const float b = fmaf(nb, c4.x, nb * lo4.x);
    // (to_u, to_v) as one packed chain: the two matrix rows side by side
    float2 uv = mul2(splat(rg.x), make_float2(-0.1146f, 0.5f));
    uv = fma2(splat(rg.y), make_float2(-0.3854f, -0.4542f), uv);
    uv = fma2(splat(b), make_float2(0.5f, -0.0458f), uv);
    uv = add2(uv, splat(0.5f));
    const uint32_t cuv = store2(make_float2(__saturatef(fmaf(uv.x, 0.87843137254f, K16)), __saturatef(fmaf(uv.y, 0.87843137254f, K16))));
    if (J.out_format == 4) {   // NV12: texel (X / 2, Y / 2) of the interleaved plane sits at byte X
        *reinterpret_cast<unsigned short *>(J.out1 + (size_t)(Y >> 1) * J.out_pitch1 + X) = (unsigned short)cuv;
    } else {
        J.out1[(size_t)(Y >> 1) * J.out_pitch1 + (X >> 1)] = (unsigned char)(cuv & 0xffu);
        J.out2[(size_t)(Y >> 1) * J.out_pitch2 + (X >> 1)] = (unsigned char)(cuv >> 8);
    }
}

#include "resample_tma.cuh"
#include "resample_tma3.cuh"
#include "resample_tma0.cuh"

// ------------------------------------------------------------------------------------------------
// The compiled instantiations of the three fused kernel families, one table built once from each family's template
// parameter lists: launch_resample_fused looks a launch's variant up here and launches the entry's kernel
// ------------------------------------------------------------------------------------------------
struct FusedEntry {
    FusedVariant key;
    const void *fn;     // the __global__ function
    int smem;           // dynamic shared memory, bytes
    dim3 block;
    int groups;         // eight-warp groups per block: the host cuts a launch's work for nblocks groups
    const char *name;   // in a launch error
};

template <int... V> using ints = std::integer_sequence<int, V...>;
// f(a, b, ...) for every combination of a in the first list, b in the second, ..., each a std::integral_constant
template <class F> static void each(F &&f) { f(); }
template <class F, int... V, class... Lists> static void each(F &&f, ints<V...>, Lists... rest);
template <class F, class C, class... Lists> static void each_with(F &f, C c, Lists... rest) {   // f(c, ...) over the rest
    each([&](auto... tail) { f(c, tail...); }, rest...);
}
template <class F, int... V, class... Lists> static void each(F &&f, ints<V...>, Lists... rest) {
    (each_with(f, std::integral_constant<int, V>{}, rest...), ...);
}

static const std::vector<FusedEntry> &fused_table() {
    static const std::vector<FusedEntry> table = [] {
        std::vector<FusedEntry> t;
        using two = ints<0, 1>;
        // k_resample_fused_int: any ratio (0) or 2 / 3 / 4, every source class; the range is a parameter of the interleaved
        // sources only
        each([&](auto S, auto SRC, auto MAT, auto FULL) {
            if constexpr (!FULL || SRC >= 2)
                t.push_back({{FusedVariant::LDG, S, 0, 0, SRC, FULL, MAT}, (const void *)k_resample_fused_int<S, SRC, MAT, FULL != 0>,
                             (int)sizeof(typename W64<S>::Smem), dim3(32, W64_WARPS), 1, "k_resample_fused_int"});
        }, ints<0, 2, 3, 4>{}, ints<0, 1, 2, 3>{}, two{}, two{});
        // k_resample_tma3: ratio 2 / 4 on planar 4:2:0 and NV12
        each([&](auto S, auto SRC, auto FULL, auto MAT) {
            t.push_back({{FusedVariant::TMA_INT, S, 0, 0, SRC, FULL, MAT}, (const void *)tma_int::k_resample_tma3<S, SRC, FULL != 0, MAT>,
                         tma_int::Cfg<S>::SMEM, dim3(32, tma::kWarps * tma_int::kGroups), tma_int::kGroups, "k_resample_tma3"});
        }, ints<2, 4>{}, two{}, two{}, two{});
        // k_resample_tma0: planar 4:2:0 and NV12, every window of kTma0Window, with and without the box reduction
        each([&](auto SRC, auto W, auto BOX, auto MAT) {
            t.push_back({{FusedVariant::TMA_ANY, 0, W, BOX, SRC, 0, MAT}, (const void *)tma_any::k_resample_tma0<SRC, kTma0Window[W], BOX, MAT>,
                         tma_any::Cfg::SMEM, dim3(32, tma::kWarps * tma_any::kGroups), tma_any::kGroups, "k_resample_tma0"});
        }, two{}, ints<0, 1, 2, 3>{}, two{}, two{});
        return t;
    }();
    return table;
}

int fused_variants(FusedVariant *out, int cap) {
    const std::vector<FusedEntry> &table = fused_table();
    for (int i = 0; i < cap && i < (int)table.size(); i++) out[i] = table[i].key;
    return (int)table.size();
}

int launch_resample_fused(const FusedVariant &v, const FusedJob *jobs_dev, const FusedPiece *pieces_dev, const int *piece_begin_dev,
                          int nblocks, Stream s) {
    static_assert(tma_int::Cfg<4>::NOUT == kTmaStripCols4 && tma_int::Cfg<2>::NOUT == kTmaStripCols2 &&
                  tma_int::Cfg<4>::RROWS == kTmaRing4 && tma_int::Cfg<2>::RROWS == kTmaRing2, "integer-ratio kernel");
    static_assert(tma_any::kGroups == kTma0Groups && tma_any::Cfg::MAXT == kTma0MaxTaps && tma_any::Cfg::WINP_MAX == kTma0Window[3] &&
                  tma_any::Cfg::RROWS == kTmaRing4, "any-ratio kernel");
    static_assert(tma::kLumaBox == 2 * kTmaLumaBoxW && tma::kChunkRows == kTmaLumaBoxH && tma::kNv12Box == 2 * kTmaNv12BoxW &&
                  tma::kPlanarBox == kTmaPlanarBoxW && tma::kChromaRows == kTmaChromaBoxH, "TMA boxes");
    if (nblocks <= 0) return 0;
    const std::vector<FusedEntry> &table = fused_table();
    const auto e = std::find_if(table.begin(), table.end(), [&](const FusedEntry &x) { return x.key == v; });
    if (e == table.end()) {
        snprintf(g_err, sizeof(g_err), "no fused resample kernel for kind %d, ratio %d, window %d, box %d, source class %d, range %d, matrix %d",
                 (int)v.kind, v.ratio, v.window, v.box, v.src, v.range, v.matrix);
        return -1;
    }
    // the attribute is per device: several handles of one process may drive different GPUs from different threads
    static std::vector<std::atomic<unsigned long long>> attr_set(table.size());
    std::atomic<unsigned long long> &done = attr_set[e - table.begin()];
    int dev = 0;
    cudaGetDevice(&dev);
    const unsigned long long bit = 1ull << (dev & 63);
    if (!(done.load(std::memory_order_acquire) & bit)) {
        cudaFuncSetAttribute(e->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, e->smem);
        done.fetch_or(bit, std::memory_order_release);
    }
    void *args[] = {(void *)&jobs_dev, (void *)&pieces_dev, (void *)&piece_begin_dev, (void *)&nblocks};   // k_resample_fused_int takes the first three
    cudaLaunchKernel(e->fn, dim3((nblocks + e->groups - 1) / e->groups), e->block, args, (size_t)e->smem, (cudaStream_t)s);
    return check_launch(e->name) ? 1 : -1;
}

// ------------------------------------------------------------------------------------------------
// FAST_HALF: K1/K2 of one source row of an aligned 8-pixel run (x0 even, interior: 2 <= x0, x0 + 9 <= W - 1, chroma rows
// inside), the conversion of the TMA-staged kernels (tma::convert_pair); the bytes of pixels (2i, 2i + 1) are ADDED to
// sums[i][c].  The result of yuv_to_rgba8() bit for bit (same operations, two pixels per instruction).
// ------------------------------------------------------------------------------------------------
// one source row: yw = its 8 luma bytes, v[k] = 3 * heavy + light chroma texel cx - 1 + k (u in bits 0..15, v in 16..31)
__device__ __forceinline__ void half_row_convert(const uint32_t (&yw)[2], const uint32_t (&v)[6], float nk16, float rcp_y, float rcp_c,
                                                 const YuvCoef &kc, int (&sums)[4][3]) {
#pragma unroll
    for (int p = 0; p < 4; p++) {
        float2 qr, qg, qb;
        tma::convert_pair(yw, v, p, nk16, rcp_y, rcp_c, kc, qr, qg, qb);
        sums[p][0] += (int)(__float_as_uint(qr.x) & 0xffu) + (int)(__float_as_uint(qr.y) & 0xffu);
        sums[p][1] += (int)(__float_as_uint(qg.x) & 0xffu) + (int)(__float_as_uint(qg.y) & 0xffu);
        sums[p][2] += (int)(__float_as_uint(qb.x) & 0xffu) + (int)(__float_as_uint(qb.y) & 0xffu);
    }
}

template <bool NV12>
__device__ __forceinline__ void half_row_sums(const Tex &S, int x0, int r, float nk16, float rcp_y, float rcp_c, const YuvCoef &kc,
                                              int (&sums)[4][3]) {
    const uint8_t *yrow = S.p0 + (size_t)r * S.pitch0 + x0;
    const uint32_t yw[2] = {__ldg(reinterpret_cast<const uint32_t *>(yrow)), __ldg(reinterpret_cast<const uint32_t *>(yrow) + 1)};
    const int ch = r >> 1, cl = (r & 1) ? ch + 1 : ch - 1, cx = x0 >> 1;
    uint32_t v[6];
#pragma unroll
    for (int k = 0; k < 6; k++) {
        uint32_t h, l;
        if (NV12) {
            const uint32_t th = __ldg(reinterpret_cast<const unsigned short *>(S.p1 + (size_t)ch * S.pitch1) + (cx - 1 + k));
            const uint32_t tl = __ldg(reinterpret_cast<const unsigned short *>(S.p1 + (size_t)cl * S.pitch1) + (cx - 1 + k));
            h = __byte_perm(th, 0, 0x4140); l = __byte_perm(tl, 0, 0x4140);
        } else {
            h = __ldg(S.p1 + (size_t)ch * S.pitch1 + cx - 1 + k) | ((uint32_t)__ldg(S.p2 + (size_t)ch * S.pitch2 + cx - 1 + k) << 16);
            l = __ldg(S.p1 + (size_t)cl * S.pitch1 + cx - 1 + k) | ((uint32_t)__ldg(S.p2 + (size_t)cl * S.pitch2 + cx - 1 + k) << 16);
        }
        v[k] = 3u * h + l;
    }
    half_row_convert(yw, v, nk16, rcp_y, rcp_c, kc, sums);
}

// NV12, x0 % 4 == 0, chroma plane 4-byte aligned: both source rows (r even, r + 1) of one output row.  The three chroma rows
// they touch are loaded once as 16-byte windows [x0 - 4, x0 + 12) and spread once; the heavy row (r / 2) is shared.
__device__ __forceinline__ void half_pair_sums_nv12(const Tex &S, int x0, int r, float nk16, float rcp_y, float rcp_c, const YuvCoef &kc,
                                                    int (&sums)[4][3]) {
    const int ch = r >> 1;
    auto spread_row = [&](int crow, uint32_t (&t)[6]) {
        const uint32_t *w = reinterpret_cast<const uint32_t *>(S.p1 + (size_t)crow * S.pitch1 + x0 - 4);
        const uint32_t w0 = __ldg(w), w1 = __ldg(w + 1), w2 = __ldg(w + 2), w3 = __ldg(w + 3);
        t[0] = __byte_perm(w0, 0, 0x4342); t[1] = __byte_perm(w1, 0, 0x4140); t[2] = __byte_perm(w1, 0, 0x4342);
        t[3] = __byte_perm(w2, 0, 0x4140); t[4] = __byte_perm(w2, 0, 0x4342); t[5] = __byte_perm(w3, 0, 0x4140);
    };
    uint32_t th[6], tl[6], v[6];
    spread_row(ch, th);
#pragma unroll
    for (int k = 0; k < 6; k++) th[k] *= 3u;
#pragma unroll
    for (int half = 0; half < 2; half++) {
        spread_row(half ? ch + 1 : ch - 1, tl);
#pragma unroll
        for (int k = 0; k < 6; k++) v[k] = th[k] + tl[k];
        const uint32_t *yrow = reinterpret_cast<const uint32_t *>(S.p0 + (size_t)(r + half) * S.pitch0 + x0);
        const uint32_t yw[2] = {__ldg(yrow), __ldg(yrow + 1)};
        half_row_convert(yw, v, nk16, rcp_y, rcp_c, kc, sums);
    }
}

// ------------------------------------------------------------------------------------------------
// K9 (+K10/K11): composite
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float smoothstep_f(float e0, float e1, float x) {
    float t = clamp01((x - e0) / (e1 - e0));
    return (t * t) * (3.0f - 2.0f * t);
}

// apply_layouts.wgsl:246-256; radius = [tl, tr, br, bl]
__device__ __forceinline__ float rounded_rect_sdf(float dx, float dy, float sx, float sy, const float *radius) {
    float hx = sx / 2.0f, hy = sy / 2.0f;
    float rx, ry;
    if (dx < 0.0f) { rx = radius[0]; ry = radius[3]; } else { rx = radius[1]; ry = radius[2]; }
    if (dy < 0.0f) rx = ry;
    float qx = (fabsf(dx) - hx) + rx, qy = (fabsf(dy) - hy) + rx;
    float mx = fmaxf(qx, 0.0f), my = fmaxf(qy, 0.0f);
    return (fminf(fmaxf(qx, qy), 0.0f) + sqrtf(mx * mx + my * my)) - rx;
}

__device__ __forceinline__ bool quad_covers(const LayerDev &L, int px, int py) {  // NC-7
    if (px < L.px0 || px >= L.px1 || py < L.py0 || py >= L.py1) return false;
    if (!L.rotated) return true;
    long long X = (long long)px * 256 + 128, Y = (long long)py * 256 + 128;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        int j = (i + 1) & 3;
        long long dx = L.vx[j] - L.vx[i], dy = L.vy[j] - L.vy[i];
        long long e = dx * (Y - L.vy[i]) - dy * (X - L.vx[i]);
        bool top_left = (dy < 0) || (dy == 0 && dx > 0);
        if (e < 0 || (e == 0 && !top_left)) return false;
    }
    return true;
}

// vs_main + fs_main of apply_layouts.wgsl for one covered pixel
// `pass` is set when the fragment is an unmodified opaque texel: blending it through the sRGB target
// reproduces the texel's bytes exactly (encode(decode(b)) == b), so the caller copies `texel`.
__device__ __forceinline__ float4 shade(const Tables &T, const CompositeJob &J, const LayerDev &L, int px, int py,
                                        bool &pass, uchar4 &texel) {
    pass = false;
    float pcx = (float)px + 0.5f, pcy = (float)py + 0.5f;
    float lx, ly, u, v;
    if (!L.rotated) {
        lx = (pcx - L.left) - L.width * 0.5f;
        ly = L.height * 0.5f - (pcy - L.top);
        u = (pcx - L.left) / L.width;
        v = (pcy - L.top) / L.height;
    } else {
        float dx = pcx - L.cx, dyu = L.cy - pcy;
        lx = dx * L.cs + dyu * L.sn;
        ly = dyu * L.cs - dx * L.sn;
        u = lx / L.width + 0.5f;
        v = 0.5f - ly / L.height;
    }
    float mask_alpha = 1.0f;
    for (int i = 0; i < L.mask_count; i++) {
        const MaskDev &m = J.masks[L.mask_begin + i];
        float d = rounded_rect_sdf((m.left + m.width / 2.0f) - pcx, (m.top + m.height / 2.0f) - pcy, m.width,
                                   m.height, m.radius);
        mask_alpha = mask_alpha * smoothstep_f(-0.5f, 0.5f, -d);
    }
    float edge = -rounded_rect_sdf(lx, ly, L.content_w, L.content_h, L.border_radius);
    float4 src = make_float4(0.f, 0.f, 0.f, 0.f);
    if (L.type == 0) {
        float tx = u * L.crop_sx + L.crop_ox;
        float ty = v * L.crop_sy + L.crop_oy;
        bool exact;
        float4 sample = sample_node(T, L.tex >= 0 ? &J.textures[L.tex] : nullptr, J.mode, tx, ty, exact, texel);
        float bw = L.border_width;
        if (bw < 1.0f) {
            float ca = smoothstep_f(-0.5f, 0.5f, edge);
            pass = exact && ca == 1.0f && mask_alpha == 1.0f && texel.w == 255;
            src = make_float4((sample.x * ca) * mask_alpha, (sample.y * ca) * mask_alpha,
                              (sample.z * ca) * mask_alpha, (sample.w * ca) * mask_alpha);
        } else if (mask_alpha < 0.01f) {
            // transparent
        } else if (edge > bw / 2.0f) {
            float ba = smoothstep_f(bw - 0.5f, bw + 0.5f, edge);
            float ib = 1.0f - ba;
            src = make_float4((L.border_color[0] * ib + sample.x * ba) * mask_alpha,
                              (L.border_color[1] * ib + sample.y * ba) * mask_alpha,
                              (L.border_color[2] * ib + sample.z * ba) * mask_alpha,
                              (L.border_color[3] * ib + sample.w * ba) * mask_alpha);
        } else {
            float ca = smoothstep_f(-0.5f, 0.5f, edge);
            src = make_float4((L.border_color[0] * ca) * mask_alpha, (L.border_color[1] * ca) * mask_alpha,
                              (L.border_color[2] * ca) * mask_alpha, (L.border_color[3] * ca) * mask_alpha);
        }
    } else if (L.type == 1) {
        float bw = L.border_width;
        if (bw < 1.0f) {
            float ca = smoothstep_f(-0.5f, 0.5f, edge);
            src = make_float4((L.color[0] * ca) * mask_alpha, (L.color[1] * ca) * mask_alpha,
                              (L.color[2] * ca) * mask_alpha, (L.color[3] * ca) * mask_alpha);
        } else if (edge > bw / 2.0f) {
            float ba = smoothstep_f(bw, bw + 1.0f, edge);
            float ib = 1.0f - ba;
            src = make_float4((L.border_color[0] * ib + L.color[0] * ba) * mask_alpha,
                              (L.border_color[1] * ib + L.color[1] * ba) * mask_alpha,
                              (L.border_color[2] * ib + L.color[2] * ba) * mask_alpha,
                              (L.border_color[3] * ib + L.color[3] * ba) * mask_alpha);
        } else {
            float ca = smoothstep_f(-0.5f, 0.5f, edge);
            src = make_float4((L.border_color[0] * ca) * mask_alpha, (L.border_color[1] * ca) * mask_alpha,
                              (L.border_color[2] * ca) * mask_alpha, (L.border_color[3] * ca) * mask_alpha);
        }
    } else {
        float br = L.blur_radius;
        float ba = smoothstep_f(-br / 2.0f, br / 2.0f, edge) * mask_alpha;
        src = make_float4(L.color[0] * ba, L.color[1] * ba, L.color[2] * ba, L.color[3] * ba);
    }
    return src;
}

// general per-pixel path: full fragment shader + fixed-function blend.  Kept out of line: the fast paths of
// k_composite cover almost every pixel and the instruction cache matters more than the call.
__device__ __noinline__ uchar4 shade_blend(const Tables &T, const CompositeJob &J, const LayerDev &L, int X, int Y,
                                           uchar4 dst) {
    // per-pixel version of the host's interior bars (LayerDev::ix0..): straight edges of rounded layers and masks need
    // no SDF -- only the corner squares do
    if (interior_shortcut(L, J.masks + L.mask_begin, X, Y)) {
        if (L.type == 1) {  // bare colour
            if (L.fast & FAST_CONST) return *reinterpret_cast<const uchar4 *>(&L.const_bytes);
            return blend(T, J.mode, dst, make_float4(L.color[0], L.color[1], L.color[2], L.color[3]));
        }
        bool exact;
        uchar4 texel;
        float4 sample;
        if (L.fast & FAST_IDENT) {
            texel = node_texel(T, J.textures[L.tex], X + L.tx_off, Y + L.ty_off);
            exact = true;
            const float *lut = J.mode == 0 ? T.dec : T.u8n;
            sample = make_float4(lut[texel.x], lut[texel.y], lut[texel.z], T.u8n[texel.w]);
        } else {
            const float u = (((float)X + 0.5f) - L.left) / L.width, v = (((float)Y + 0.5f) - L.top) / L.height;
            sample = sample_node(T, L.tex >= 0 ? &J.textures[L.tex] : nullptr, J.mode, u * L.crop_sx + L.crop_ox,
                                 v * L.crop_sy + L.crop_oy, exact, texel);
        }
        if (exact && texel.w == 255) return texel;  // encode(decode(b)) == b
        return blend(T, J.mode, dst, sample);
    }
    bool pass;
    uchar4 texel;
    float4 src = shade(T, J, L, X, Y, pass, texel);
    return pass ? texel : blend(T, J.mode, dst, src);
}

#ifndef SMR_COMPOSITE_BLOCKS
#define SMR_COMPOSITE_BLOCKS 3   // resident blocks per SM the composite kernels are compiled for
#endif
#define CT_W 4           // pixels per thread, x
#define CT_H 2           // pixels per thread, y
#define CB_X 32          // threads per block, x
#define CB_Y 8
#define CT_ITERS 1       // vertical steps per thread (1: a block covers 128 x 16 pixels; more starves 1080p frames of blocks)
#define MAX_TILE_LAYERS 1024
#define SM_LAYERS 40     // layers of a tile kept in shared memory (the rest are read from global)

// PARAM: the layer list travels in the kernel parameter block (constant bank): the per-tile culling and the
// per-pixel loop read it with no global round trip and no shared-memory copy; used whenever it fits.
#define PARAM_LAYERS kCompositeParamLayers
#define MAX_LUT 4          // translucent colour layers of a tile that get a blend table (FAST_LUT)
struct CompositeParams {
    CompositeJob job;
    LayerDev layers[PARAM_LAYERS];
};

template <bool PARAM>
__device__ __forceinline__ void composite_body(const CompositeJob &J, const LayerDev *__restrict__ LAYERS) {
    __shared__ Tables T;
    __shared__ unsigned short s_list[MAX_TILE_LAYERS];
    __shared__ int s_count;
    __shared__ LayerDev s_layers[PARAM ? 1 : SM_LAYERS];
    static_assert(CB_X * CT_W == kDirectTileW && CB_Y * CT_H * CT_ITERS == kDirectTileH, "direct tiles are the block tiles");
    // the fused resample kernel has written this tile's output bytes already (block-uniform, before any barrier)
    int tile_x = blockIdx.x, tile_y = blockIdx.y;
    if (J.tile_list != nullptr) {   // compacted launch: the direct tiles have no block at all
        if ((int)blockIdx.x >= J.n_tiles || blockIdx.y != 0) return;
        const uint32_t t = __ldg(J.tile_list + blockIdx.x);
        tile_x = (int)(t & 0xffffu); tile_y = (int)(t >> 16);
    } else if (J.direct_map != nullptr && __ldg(J.direct_map + tile_y * J.map_w + tile_x)) return;
    load_tables(T);
    const int tile_x0 = tile_x * (CB_X * CT_W), tile_y0 = tile_y * (CB_Y * CT_H * CT_ITERS);
    const int tile_x1 = min(tile_x0 + CB_X * CT_W, J.width), tile_y1 = min(tile_y0 + CB_Y * CT_H * CT_ITERS, J.height);
    // per-tile layer culling, painter's order preserved.  One layer per thread (a serial loop over the layer
    // list costs one dependent global-load latency per layer while the whole block waits), ordered compaction
    // with ballots.
    {
        __shared__ int s_wc[CB_Y];
        const int tid = threadIdx.y * CB_X + threadIdx.x;
        int base_count = 0;
        for (int base = 0; base < J.n_layers; base += CB_X * CB_Y) {
            const int i = base + tid;
            bool hit = false;
            if (i < J.n_layers) {
                int4 bb;
                if (PARAM) bb = make_int4(LAYERS[i].px0, LAYERS[i].px1, LAYERS[i].py0, LAYERS[i].py1);
                else bb = __ldg(reinterpret_cast<const int4 *>(&LAYERS[i].px0));
                hit = bb.x < tile_x1 && bb.y > tile_x0 && bb.z < tile_y1 && bb.w > tile_y0;
            }
            const unsigned m = __ballot_sync(0xffffffffu, hit);
            if (threadIdx.x == 0) s_wc[threadIdx.y] = __popc(m);
            __syncthreads();
            int before = base_count, total = base_count;
            for (int w = 0; w < CB_Y; w++) {
                if (w < (int)threadIdx.y) before += s_wc[w];
                total += s_wc[w];
            }
            const int pos = before + __popc(m & ((1u << threadIdx.x) - 1u));
            if (hit && pos < MAX_TILE_LAYERS) s_list[pos] = (unsigned short)i;
            base_count = min(total, MAX_TILE_LAYERS);
            __syncthreads();
        }
        if (tid == 0) s_count = base_count;
    }
    __syncthreads();
    if (!PARAM) {
        const int nsm = min(s_count, SM_LAYERS);
        const int words = (int)(sizeof(LayerDev) / 4);
        const int tid = threadIdx.y * CB_X + threadIdx.x;
        for (int i = tid; i < nsm * words; i += CB_X * CB_Y) {
            int l = i / words, w = i - l * words;
            reinterpret_cast<unsigned int *>(&s_layers[l])[w] =
                __ldg(reinterpret_cast<const unsigned int *>(&LAYERS[s_list[l]]) + w);
        }
    }
    __syncthreads();

    // FAST_LUT layers of this tile: blend() of the layer's constant source over each possible target byte, one
    // entry per thread (the four channels of blend() are independent, so one call fills all four maps)
    __shared__ uchar4 s_lut[MAX_LUT][CB_X * CB_Y];
    __shared__ uchar4 s_px[CB_Y][CB_X * CT_W * CT_H];          // per-warp scratch of the cooperative general path
    __shared__ unsigned char s_items[CB_Y][CB_X * CT_W * CT_H];
    static_assert(CB_X == 32 && CB_X * CT_W * CT_H <= 256, "one warp per tile row, items fit a byte");
    static_assert(CB_X * CB_Y == 256, "one table entry per thread");
    {
        const int tid = threadIdx.y * CB_X + threadIdx.x;
        int nl = 0;
        for (int li = 0; li < s_count && nl < MAX_LUT; li++) {
            const LayerDev &L = PARAM ? LAYERS[s_list[li]] : (li < SM_LAYERS ? s_layers[li] : LAYERS[s_list[li]]);
            if (L.fast & FAST_LUT) {
                s_lut[nl][tid] = blend(T, J.mode, make_uchar4(tid, tid, tid, tid),
                                       make_float4(L.color[0], L.color[1], L.color[2], L.color[3]));
                nl++;
            }
        }
        if (nl) __syncthreads();
    }

    for (int it = 0; it < CT_ITERS; it++) {
    const int x0 = tile_x0 + threadIdx.x * CT_W, y0 = tile_y0 + (it * CB_Y + threadIdx.y) * CT_H;
    uchar4 px[CT_H][CT_W];
#pragma unroll
    for (int j = 0; j < CT_H; j++)
#pragma unroll
        for (int i = 0; i < CT_W; i++) px[j][i] = make_uchar4(0, 0, 0, 0);  // LoadOp::Clear(TRANSPARENT)

    const int n = s_count;
    // occlusion: the last layer that replaces this thread's whole 4x2 block makes everything painted before it
    // invisible -- start there (exact: those layers' bytes do not depend on the target)
    int first = 0;
    for (int li = n - 1; li > 0; li--) {
        const LayerDev &L = PARAM ? LAYERS[s_list[li]] : (li < SM_LAYERS ? s_layers[li] : LAYERS[s_list[li]]);
        if (!(L.fast & FAST_OPAQUE)) continue;
        if ((x0 >= L.ix0 && x0 + CT_W <= L.ix1 && y0 >= L.iy0 && y0 + CT_H <= L.iy1) ||
            (x0 >= L.jx0 && x0 + CT_W <= L.jx1 && y0 >= L.jy0 && y0 + CT_H <= L.jy1)) { first = li; break; }
    }
    int lut_next = 0;
    for (int li = 0; li < n; li++) {
        const LayerDev &L = PARAM ? LAYERS[s_list[li]] : (li < SM_LAYERS ? s_layers[li] : LAYERS[s_list[li]]);
        const int lut_i = (L.fast & FAST_LUT) ? lut_next++ : MAX_LUT;   // same numbering as the table build above
        // fast classes first (per thread); `general` survives for blocks that need the full fragment path
        bool general = false;
        do {
            if (li < first) break;
            if (L.px0 >= x0 + CT_W || L.px1 <= x0 || L.py0 >= y0 + CT_H || L.py1 <= y0) break;
            const bool all_in = (x0 >= L.ix0 && x0 + CT_W <= L.ix1 && y0 >= L.iy0 && y0 + CT_H <= L.iy1) ||
                                (x0 >= L.jx0 && x0 + CT_W <= L.jx1 && y0 >= L.jy0 && y0 + CT_H <= L.jy1);
            if (all_in && (L.fast & FAST_CONST)) {  // opaque colour interior: the layer leaves constant bytes
                const uchar4 cb = *reinterpret_cast<const uchar4 *>(&L.const_bytes);
    #pragma unroll
                for (int j = 0; j < CT_H; j++)
    #pragma unroll
                    for (int i = 0; i < CT_W; i++) px[j][i] = cb;
                break;
            }
            if (all_in && lut_i < MAX_LUT) {  // translucent colour interior: four byte lookups per pixel
                const uchar4 *lut = s_lut[lut_i];
    #pragma unroll
                for (int j = 0; j < CT_H; j++)
    #pragma unroll
                    for (int i = 0; i < CT_W; i++) {
                        const uchar4 p = px[j][i];
                        px[j][i] = make_uchar4(lut[p.x].x, lut[p.y].y, lut[p.z].z, lut[p.w].w);
                    }
                break;
            }
            if (all_in && (L.fast & FAST_HALF)) {
                // exact 2:1 planar 4:2:0 / NV12 child (CpuOptimized): this thread's 4 x 2 pixels are the weight-1/2 taps of an
                // aligned 8 x 4 texel block; away from the texture border K1/K2 runs on pixel pairs with packed FP32
                const Tex &S = J.textures[L.tex];
                const int sx = 2 * (x0 + L.tx_off), sy = 2 * (y0 + L.ty_off);
                if (sx >= 2 && sx + 9 <= S.width - 1 && sy >= 2 && sy + 5 <= S.height - 1) {
                    // one copy of the tile's conversion per matrix: the coefficients are immediates, as in the fused kernels
                    auto half_tile = [&](auto mat) {
                        constexpr YuvCoef kc = yuv_coef(decltype(mat)::value);
                        const bool fr = S.full_range != 0;
                        const float nk16 = fr ? 0.0f : -K16, rcp_y = fr ? 1.0f : RCP_Y, rcp_c = fr ? 1.0f : RCP_C;
#pragma unroll
                        for (int j = 0; j < CT_H; j++) {
                            int sums[4][3];
#pragma unroll
                            for (int i = 0; i < 4; i++) sums[i][0] = sums[i][1] = sums[i][2] = 0;
                            if (S.kind == TEX_NV12 && (S.pitch1 & 3) == 0 && ((size_t)S.p1 & 3) == 0) {
                                half_pair_sums_nv12(S, sx, sy + 2 * j, nk16, rcp_y, rcp_c, kc, sums);
                            } else if (S.kind == TEX_NV12) {
                                half_row_sums<true>(S, sx, sy + 2 * j, nk16, rcp_y, rcp_c, kc, sums);
                                half_row_sums<true>(S, sx, sy + 2 * j + 1, nk16, rcp_y, rcp_c, kc, sums);
                            } else {
                                half_row_sums<false>(S, sx, sy + 2 * j, nk16, rcp_y, rcp_c, kc, sums);
                                half_row_sums<false>(S, sx, sy + 2 * j + 1, nk16, rcp_y, rcp_c, kc, sums);
                            }
#pragma unroll
                            for (int i = 0; i < CT_W; i++) {
                                // filter_u8 at weights (128, 128): N = 16384 (t00 + t10 + t01 + t11), NC-6u, stored through NC-2
                                px[j][i] = make_uchar4((unsigned char)unorm8(div255((float)(sums[i][0] << 14), 1.0f / 65536.0f)),
                                                       (unsigned char)unorm8(div255((float)(sums[i][1] << 14), 1.0f / 65536.0f)),
                                                       (unsigned char)unorm8(div255((float)(sums[i][2] << 14), 1.0f / 65536.0f)), 255);
                            }
                        }
                    };
                    if (S.matrix == 1) half_tile(std::integral_constant<int, 1>());
                    else half_tile(std::integral_constant<int, 0>());
                    break;
                }
            }
            if (all_in && (L.fast & FAST_SAMPLE)) {
                // opaque RGBA8 child sampled at a fractional position / size, axis-aligned: the taps depend on the
                // column (x) and the row (y) alone, and with alpha exactly 1 blend() ignores the target
                const Tex &S = J.textures[L.tex];
                LinTap ax[CT_W], ay[CT_H];
#pragma unroll
                for (int i = 0; i < CT_W; i++) {
                    const float u = (((float)(x0 + i) + 0.5f) - L.left) / L.width;
                    ax[i] = linear_tap(u * L.crop_sx + L.crop_ox, S.width);
                    if (ax[i].f == 1.0f) { ax[i].i0 = ax[i].i1; ax[i].f = 0.0f; }
                }
#pragma unroll
                for (int j = 0; j < CT_H; j++) {
                    const float v = (((float)(y0 + j) + 0.5f) - L.top) / L.height;
                    ay[j] = linear_tap(v * L.crop_sy + L.crop_oy, S.height);
                    if (ay[j].f == 1.0f) { ay[j].i0 = ay[j].i1; ay[j].f = 0.0f; }
                }
                if (S.kind != TEX_RGBA8) {
                    // planar 4:2:0 / NV12 child scaled by the layout shader itself (CpuOptimized): the four taps of a
                    // pixel are texels of the virtual node texture; when they form one chroma-aligned quad (e.g. an
                    // exact 2:1 grid) K1/K2 shares the chroma interpolation between them
#pragma unroll 1
                    for (int j = 0; j < CT_H; j++) {
                        const float fy = ay[j].f;
#pragma unroll 1
                        for (int i = 0; i < CT_W; i++) {
                            const float fx = ax[i].f;
                            uchar4 p00, p10, p01, p11;
                            if (ax[i].i1 == ax[i].i0 + 1 && ay[j].i1 == ay[j].i0 + 1 && yuv_quad_ok(S, ax[i].i0, ay[j].i0)) {
                                yuv_quad(T, S, ax[i].i0, ay[j].i0, p00, p10, p01, p11);
                            } else {
                                p00 = node_texel(T, S, ax[i].i0, ay[j].i0);
                                p10 = fx != 0.0f ? node_texel(T, S, ax[i].i1, ay[j].i0) : p00;
                                p01 = fy != 0.0f ? node_texel(T, S, ax[i].i0, ay[j].i1) : p00;
                                p11 = (fx != 0.0f && fy != 0.0f) ? node_texel(T, S, ax[i].i1, ay[j].i1) : (fx != 0.0f ? p10 : p01);
                            }
                            uchar4 o;
                            if (fx == 0.0f && fy == 0.0f) o = p00;
                            else {
                                o.x = (unsigned char)unorm8(filter_u8(p00.x, p10.x, p01.x, p11.x, fx, fy));
                                o.y = (unsigned char)unorm8(filter_u8(p00.y, p10.y, p01.y, p11.y, fx, fy));
                                o.z = (unsigned char)unorm8(filter_u8(p00.z, p10.z, p01.z, p11.z, fx, fy));
                            }
                            o.w = 255;
                            if (j == 0) { if (i == 0) px[0][0] = o; else if (i == 1) px[0][1] = o; else if (i == 2) px[0][2] = o; else px[0][3] = o; }
                            else { if (i == 0) px[1][0] = o; else if (i == 1) px[1][1] = o; else if (i == 2) px[1][2] = o; else px[1][3] = o; }
                        }
                    }
                    break;
                }
#pragma unroll
                for (int j = 0; j < CT_H; j++) {
                    const uchar4 *r0 = reinterpret_cast<const uchar4 *>(S.p0 + (size_t)ay[j].i0 * S.pitch0);
                    const uchar4 *r1 = reinterpret_cast<const uchar4 *>(S.p0 + (size_t)ay[j].i1 * S.pitch0);
                    const float fy = ay[j].f;
#pragma unroll
                    for (int i = 0; i < CT_W; i++) {
                        const float fx = ax[i].f;
                        const uchar4 p00 = __ldg(r0 + ax[i].i0);
                        if (fx == 0.0f && fy == 0.0f) { px[j][i] = p00; continue; }   // exact texel, alpha 255
                        const uchar4 p10 = fx != 0.0f ? __ldg(r0 + ax[i].i1) : p00;
                        const uchar4 p01 = fy != 0.0f ? __ldg(r1 + ax[i].i0) : p00;
                        const uchar4 p11 = (fx != 0.0f && fy != 0.0f) ? __ldg(r1 + ax[i].i1) : (fx != 0.0f ? p10 : p01);
                        uchar4 o;
                        if (J.mode != 0) {
                            o.x = (unsigned char)unorm8(filter_u8(p00.x, p10.x, p01.x, p11.x, fx, fy));
                            o.y = (unsigned char)unorm8(filter_u8(p00.y, p10.y, p01.y, p11.y, fx, fy));
                            o.z = (unsigned char)unorm8(filter_u8(p00.z, p10.z, p01.z, p11.z, fx, fy));
                        } else {
                            o.x = (unsigned char)srgb_encode(T, bilerp(T.dec[p00.x], T.dec[p10.x], T.dec[p01.x], T.dec[p11.x], fx, fy));
                            o.y = (unsigned char)srgb_encode(T, bilerp(T.dec[p00.y], T.dec[p10.y], T.dec[p01.y], T.dec[p11.y], fx, fy));
                            o.z = (unsigned char)srgb_encode(T, bilerp(T.dec[p00.z], T.dec[p10.z], T.dec[p01.z], T.dec[p11.z], fx, fy));
                        }
                        o.w = 255;
                        px[j][i] = o;
                    }
                }
                break;
            }
            if (all_in && (L.fast & FAST_IDENT)) {  // 1:1 texture interior: exact texel per pixel
                const Tex &S = J.textures[L.tex];
                const int sx = x0 + L.tx_off, sy = y0 + L.ty_off;
                if (yuv_quad_ok(S, sx, sy) && yuv_quad_ok(S, sx + 2, sy)) {  // YUV source: two chroma-aligned quads
                    yuv_quad(T, S, sx, sy, px[0][0], px[0][1], px[1][0], px[1][1]);       // alpha is 255: bytes pass through
                    yuv_quad(T, S, sx + 2, sy, px[0][2], px[0][3], px[1][2], px[1][3]);
                    break;
                }
                if (S.kind == TEX_RGBA8 && (sx & 3) == 0 && (S.pitch0 & 15) == 0 && ((size_t)S.p0 & 15) == 0) {
                    // RGBA8 source (e.g. a resampled child): one 16-byte load per row
                    const uint4 r0 = __ldg(reinterpret_cast<const uint4 *>(S.p0 + (size_t)sy * S.pitch0) + (sx >> 2));
                    const uint4 r1 = __ldg(reinterpret_cast<const uint4 *>(S.p0 + (size_t)(sy + 1) * S.pitch0) + (sx >> 2));
                    if ((r0.x & r0.y & r0.z & r0.w & r1.x & r1.y & r1.z & r1.w) >= 0xff000000u) {  // all 8 alphas are 255
                        *reinterpret_cast<unsigned int *>(&px[0][0]) = r0.x; *reinterpret_cast<unsigned int *>(&px[0][1]) = r0.y;
                        *reinterpret_cast<unsigned int *>(&px[0][2]) = r0.z; *reinterpret_cast<unsigned int *>(&px[0][3]) = r0.w;
                        *reinterpret_cast<unsigned int *>(&px[1][0]) = r1.x; *reinterpret_cast<unsigned int *>(&px[1][1]) = r1.y;
                        *reinterpret_cast<unsigned int *>(&px[1][2]) = r1.z; *reinterpret_cast<unsigned int *>(&px[1][3]) = r1.w;
                        break;
                    }
                }
    #pragma unroll
                for (int j = 0; j < CT_H; j++)
    #pragma unroll
                    for (int i = 0; i < CT_W; i++) {
                        uchar4 t = node_texel(T, S, x0 + i + L.tx_off, y0 + j + L.ty_off);
                        if (t.w == 255) px[j][i] = t;  // encode(decode(b)) == b
                        else {
                            const float *lut = J.mode == 0 ? T.dec : T.u8n;
                            px[j][i] = blend(T, J.mode, px[j][i], make_float4(lut[t.x], lut[t.y], lut[t.z], T.u8n[t.w]));
                        }
                    }
                break;
            }
            general = true;
        } while (0);
        // general path, warp-cooperative: the pixels that need the full fragment shader + blend are usually a thin
        // band (anti-aliased edges, corner squares), a few lanes' worth per warp.  They are gathered into a
        // per-warp list and shaded 32 at a time instead of 8 rounds with most lanes idle.
        unsigned need = 0;
        if (general) {
#pragma unroll 1
            for (int k = 0; k < CT_W * CT_H; k++) {
                const int X = x0 + (k & (CT_W - 1)), Y = y0 + k / CT_W;
                if (X < J.width && Y < J.height && quad_covers(L, X, Y)) need |= 1u << k;
            }
        }
        if (__ballot_sync(0xffffffffu, need != 0) == 0) continue;   // warp-uniform
        const int lane = threadIdx.x;
        const int cnt = __popc(need);
        int incl = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        const int total = __shfl_sync(0xffffffffu, incl, 31);
        if (total > 5 * 32) {   // dense (e.g. a resampled layer at a fractional position): every lane shades its own pixels
            for (int k = 0; k < CT_W * CT_H; k++) {  // deliberately not unrolled (code size)
                if (!((need >> k) & 1u)) continue;
                const int i = k & (CT_W - 1), j = k / CT_W;
                uchar4 cur = j == 0 ? (i == 0 ? px[0][0] : i == 1 ? px[0][1] : i == 2 ? px[0][2] : px[0][3])
                                    : (i == 0 ? px[1][0] : i == 1 ? px[1][1] : i == 2 ? px[1][2] : px[1][3]);
                uchar4 res = shade_blend(T, J, L, x0 + i, y0 + j, cur);
#pragma unroll
                for (int jj = 0; jj < CT_H; jj++)
#pragma unroll
                    for (int ii = 0; ii < CT_W; ii++)
                        if (jj == j && ii == i) px[jj][ii] = res;
            }
            continue;
        }
        unsigned char *items = s_items[threadIdx.y];
        uchar4 *spx = s_px[threadIdx.y];
        if (need) {
            int o = incl - cnt;
#pragma unroll
            for (int k = 0; k < CT_W * CT_H; k++) {
                spx[lane * (CT_W * CT_H) + k] = px[k / CT_W][k & (CT_W - 1)];
                if ((need >> k) & 1u) items[o++] = (unsigned char)(lane * (CT_W * CT_H) + k);
            }
        }
        __syncwarp();
        for (int base = 0; base < total; base += 32) {
            const int idx = base + lane;
            if (idx < total) {
                const int item = items[idx], k = item & (CT_W * CT_H - 1);
                const int X = tile_x0 + (item / (CT_W * CT_H)) * CT_W + (k & (CT_W - 1)), Y = y0 + k / CT_W;
                spx[item] = shade_blend(T, J, L, X, Y, spx[item]);
            }
        }
        __syncwarp();
        if (need) {
#pragma unroll
            for (int k = 0; k < CT_W * CT_H; k++) px[k / CT_W][k & (CT_W - 1)] = spx[lane * (CT_W * CT_H) + k];
        }
    }

    if (x0 >= J.width || y0 >= J.height) continue;
    if (J.out_format < 0 || J.out_format == 3) {  // RGBA8 node texture / RgbaWgpuTexture analogue
        // a caller's device plane is 4-byte aligned (host-checked), not necessarily 16: with x0 a multiple of 4 pixels,
        // every 16-byte store of the plane is aligned when its start and its pitch are
        const bool vec16 = (((uintptr_t)J.out0 | (uintptr_t)J.out_pitch0) & 15) == 0;
#pragma unroll
        for (int j = 0; j < CT_H; j++) {
            int Y = y0 + j;
            if (Y >= J.height) break;
            uchar4 *row = reinterpret_cast<uchar4 *>(J.out0 + (size_t)Y * J.out_pitch0);
            if (x0 + CT_W <= J.width && vec16) {
                uint4 v;
                v.x = *reinterpret_cast<unsigned int *>(&px[j][0]);
                v.y = *reinterpret_cast<unsigned int *>(&px[j][1]);
                v.z = *reinterpret_cast<unsigned int *>(&px[j][2]);
                v.w = *reinterpret_cast<unsigned int *>(&px[j][3]);
                *reinterpret_cast<uint4 *>(row + x0) = v;
            } else {
                for (int i = 0; i < CT_W && x0 + i < J.width; i++) row[x0 + i] = px[j][i];
            }
        }
        continue;
    }
    // fused K10/K11 (host guarantees even width/height): Y per pixel, chroma = 2x2 box of raw bytes
    unsigned char yv[CT_H][CT_W];
#pragma unroll
    for (int j = 0; j < CT_H; j++)
#pragma unroll
        for (int i = 0; i < CT_W; i++)
            yv[j][i] = (unsigned char)unorm8(to_y(T.u8n[px[j][i].x], T.u8n[px[j][i].y], T.u8n[px[j][i].z]));
    // YUV planes may start at any byte; x0 is a multiple of 4 (cx of 2), so a plane's vector stores are aligned when its
    // start and its pitch are
    const bool full = (x0 + CT_W <= J.width) && (((uintptr_t)J.out0 | (uintptr_t)J.out_pitch0) & 3) == 0;
#pragma unroll
    for (int j = 0; j < CT_H; j++) {
        int Y = y0 + j;
        if (Y >= J.height) break;
        unsigned char *row = J.out0 + (size_t)Y * J.out_pitch0;
        if (full) *reinterpret_cast<uchar4 *>(row + x0) = make_uchar4(yv[j][0], yv[j][1], yv[j][2], yv[j][3]);
        else
            for (int i = 0; i < CT_W && x0 + i < J.width; i++) row[x0 + i] = yv[j][i];
    }
    unsigned char uo[2], vo[2];
#pragma unroll
    for (int c = 0; c < 2; c++) {
        const uchar4 a = px[0][2 * c], b = px[0][2 * c + 1], d = px[1][2 * c], e = px[1][2 * c + 1];
        // NC-6u with the .5/.5 taps of an even-sized target: the exact mean of the four raw bytes
        float r = div255((float)((int)a.x + b.x + d.x + e.x), 0.25f);
        float g = div255((float)((int)a.y + b.y + d.y + e.y), 0.25f);
        float bb = div255((float)((int)a.z + b.z + d.z + e.z), 0.25f);
        uo[c] = (unsigned char)unorm8(to_u(r, g, bb));
        vo[c] = (unsigned char)unorm8(to_v(r, g, bb));
    }
    const int cx = x0 / 2, cy = y0 / 2, cw = J.width / 2;
    if (J.out_format == 4) {  // NV12
        unsigned char *row = J.out1 + (size_t)cy * J.out_pitch1 + cx * 2;
        if (cx + 1 < cw && (((uintptr_t)J.out1 | (uintptr_t)J.out_pitch1) & 3) == 0) *reinterpret_cast<uchar4 *>(row) = make_uchar4(uo[0], vo[0], uo[1], vo[1]);
        else
            for (int c = 0; c < 2 && cx + c < cw; c++) { row[2 * c] = uo[c]; row[2 * c + 1] = vo[c]; }
    } else {  // planar 4:2:0
        unsigned char *ru = J.out1 + (size_t)cy * J.out_pitch1 + cx, *rv = J.out2 + (size_t)cy * J.out_pitch2 + cx;
        if (cx + 1 < cw && (((uintptr_t)J.out1 | (uintptr_t)J.out2 | (uintptr_t)(J.out_pitch1 | J.out_pitch2)) & 1) == 0) {
            *reinterpret_cast<uchar2 *>(ru) = make_uchar2(uo[0], uo[1]);
            *reinterpret_cast<uchar2 *>(rv) = make_uchar2(vo[0], vo[1]);
        } else
            for (int c = 0; c < 2 && cx + c < cw; c++) { ru[c] = uo[c]; rv[c] = vo[c]; }
    }
    }  // it
}

__global__ void __launch_bounds__(CB_X *CB_Y, SMR_COMPOSITE_BLOCKS) k_composite_p(const __grid_constant__ CompositeParams P) {
    composite_body<true>(P.job, P.layers);
}

// all outputs of a tick in one launch (blockIdx.z = output): a 1080p frame alone is 2.3 waves of 444 resident
// blocks, eight of them back to back are 18.4 -- the per-launch tails disappear
__global__ void __launch_bounds__(CB_X *CB_Y, SMR_COMPOSITE_BLOCKS) k_composite_multi(const CompositeJob *__restrict__ jobs) {
    __shared__ CompositeJob J;
    {
        const int tid = threadIdx.y * CB_X + threadIdx.x;
        const unsigned int *src = reinterpret_cast<const unsigned int *>(jobs + blockIdx.z);
        if (tid < (int)(sizeof(CompositeJob) / 4)) reinterpret_cast<unsigned int *>(&J)[tid] = __ldg(src + tid);
    }
    __syncthreads();
    if (J.tile_list == nullptr &&
        ((int)blockIdx.x * (CB_X * CT_W) >= J.width || (int)blockIdx.y * (CB_Y * CT_H * CT_ITERS) >= J.height)) return;
    composite_body<false>(J, J.layers);
}

int launch_composite(const CompositeJob *jobs_dev, const CompositeJob *jobs_host, const LayerDev *layers0_host, int n, Stream s) {
    static_assert(sizeof(CompositeJob) % 4 == 0 && sizeof(CompositeJob) / 4 <= CB_X * CB_Y, "job copied by one block pass");
    int gx = 0, gy = 0;
    for (int i = 0; i < n; i++) {
        // a tile list leaves out the tiles the resample kernel has written already (all of them: no launch)
        if (jobs_host[i].tile_list != nullptr) { gx = max(gx, jobs_host[i].n_tiles); gy = max(gy, jobs_host[i].n_tiles > 0 ? 1 : 0); continue; }
        gx = max(gx, (jobs_host[i].width + CB_X * CT_W - 1) / (CB_X * CT_W));
        gy = max(gy, (jobs_host[i].height + CB_Y * CT_H * CT_ITERS - 1) / (CB_Y * CT_H * CT_ITERS));
    }
    if (n <= 0 || gx == 0 || gy == 0) return 0;
    if (n == 1 && jobs_host[0].n_layers <= PARAM_LAYERS) {
        CompositeParams P;   // ~26 KB on the host stack; the driver copies the parameter block at launch
        P.job = jobs_host[0];
        memcpy(P.layers, layers0_host, sizeof(LayerDev) * (size_t)P.job.n_layers);
        k_composite_p<<<dim3(gx, gy), dim3(CB_X, CB_Y), 0, (cudaStream_t)s>>>(P);
        return check_launch("k_composite_p") ? 1 : -1;
    }
    k_composite_multi<<<dim3(gx, gy, n), dim3(CB_X, CB_Y), 0, (cudaStream_t)s>>>(jobs_dev);
    return check_launch("k_composite_multi") ? 1 : -1;
}

// ------------------------------------------------------------------------------------------------
// K10/K11 stand-alone: the general form (linear sampler from a src of any size)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void sample_raw_rgb(const Tables &T, const Tex &S, float tx, float ty, float &r, float &g,
                                               float &b) {
    LinTap ax = linear_tap(tx, S.width), ay = linear_tap(ty, S.height);
    uchar4 p00 = node_texel(T, S, ax.i0, ay.i0);
    uchar4 p10 = ax.f != 0.0f ? node_texel(T, S, ax.i1, ay.i0) : p00;
    uchar4 p01 = ay.f != 0.0f ? node_texel(T, S, ax.i0, ay.i1) : p00;
    uchar4 p11 = (ax.f != 0.0f && ay.f != 0.0f) ? node_texel(T, S, ax.i1, ay.i1) : (ax.f != 0.0f ? p10 : p01);
    r = filter_u8(p00.x, p10.x, p01.x, p11.x, ax.f, ay.f);   // raw bytes through the Rgba8Unorm view: NC-6u
    g = filter_u8(p00.y, p10.y, p01.y, p11.y, ax.f, ay.f);
    b = filter_u8(p00.z, p10.z, p01.z, p11.z, ax.f, ay.f);
}

__global__ void __launch_bounds__(256) k_output(OutputJob J) {
    __shared__ Tables T;
    load_tables(T);
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= J.out_w || y >= J.out_h) return;
    if (J.out_format == 3) {  // RGBA copy of the root texture (size must match; host checks)
        reinterpret_cast<uchar4 *>(J.out0 + (size_t)y * J.out_pitch0)[x] = node_texel(T, J.src, x, y);
        return;
    }
    float r, g, b;
    sample_raw_rgb(T, J.src, ((float)x + 0.5f) / (float)J.out_w, ((float)y + 0.5f) / (float)J.out_h, r, g, b);
    J.out0[(size_t)y * J.out_pitch0 + x] = (unsigned char)unorm8(to_y(r, g, b));
    int cw, ch;
    chroma_dims(J.out_format, J.out_w, J.out_h, cw, ch);
    if (x < cw && y < ch) {  // chroma target texel (x, y)
        sample_raw_rgb(T, J.src, ((float)x + 0.5f) / (float)cw, ((float)y + 0.5f) / (float)ch, r, g, b);
        unsigned char u = (unsigned char)unorm8(to_u(r, g, b)), v = (unsigned char)unorm8(to_v(r, g, b));
        if (J.out_format == 4) {
            J.out1[(size_t)y * J.out_pitch1 + 2 * x] = u;
            J.out1[(size_t)y * J.out_pitch1 + 2 * x + 1] = v;
        } else {
            J.out1[(size_t)y * J.out_pitch1 + x] = u;
            J.out2[(size_t)y * J.out_pitch2 + x] = v;
        }
    }
}

int launch_output(const OutputJob &job, Stream s) {
    dim3 b(32, 8), g((job.out_w + 31) / 32, (job.out_h + 7) / 8);
    k_output<<<g, b, 0, (cudaStream_t)s>>>(job);
    return check_launch("k_output") ? 1 : -1;
}

// gpu-video's transcoder resize (smr_transcode_resize, NC-10)
#include "transcode.cuh"

// gpu-video's NV12 -> RGBA converter (smr_video_nv12_to_rgba, NC-11)
#include "video_convert.cuh"

// the deinterlacers of smr_set_input_deinterlace (NC-12)
#include "deinterlace.cuh"

// ------------------------------------------------------------------------------------------------
// FramePreProcessor (state/frame_pre_processor.rs): K1..K4 to RGBA8, optional rescale (rgba_rescale.wgsl, blend: None)
// ------------------------------------------------------------------------------------------------
// fs_main of add_premultiplied_alpha.wgsl:27-35 for one fragment: the sampled straight-alpha colour times max(alpha, 1e-5),
// clamped, stored through the target view (sRGB in GpuOptimized, plain UNORM8 in CpuOptimized)
__device__ __forceinline__ uchar4 premultiply_store(const Tables &T, int mode, float4 c) {
    const float am = fmaxf(c.w, 0.00001f);
    const float r = clamp01(c.x * am), g = clamp01(c.y * am), b = clamp01(c.z * am);
    if (mode == 0) return make_uchar4(srgb_encode(T, r), srgb_encode(T, g), srgb_encode(T, b), unorm8(c.w));
    return make_uchar4(unorm8(r), unorm8(g), unorm8(b), unorm8(c.w));
}

__global__ void __launch_bounds__(256) k_preprocess(Tex src, int mode, int rescale, uint8_t *out, int out_pitch, int ow, int oh) {
    __shared__ Tables T;
    load_tables(T);
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= ow || y >= oh) return;
    uchar4 o;
    if (!rescale) {
        o = node_texel(T, src, x, y);
    } else if (rescale == 2) {
        // add_premultiplied_alpha.wgsl:24-35: straight-alpha texel fetched through the source view (the full-screen quad
        // samples at texel centres: weight exactly 1), colour times max(alpha, 1e-5), clamped, stored through the target view
        const uchar4 t = node_texel(T, src, x, y);
        const float *lut = mode == 0 ? T.dec : T.u8n;
        o = premultiply_store(T, mode, make_float4(lut[t.x], lut[t.y], lut[t.z], T.u8n[t.w]));
    } else {
        bool exact;
        uchar4 texel;
        const float4 sm = sample_node(T, &src, mode, ((float)x + 0.5f) / (float)ow, ((float)y + 0.5f) / (float)oh, exact, texel);
        if (exact) o = texel;   // encode(decode(b)) == b, unorm8(b / 255) == b
        else if (mode == 0) o = make_uchar4(srgb_encode(T, sm.x), srgb_encode(T, sm.y), srgb_encode(T, sm.z), unorm8(sm.w));
        else o = make_uchar4(unorm8(sm.x), unorm8(sm.y), unorm8(sm.z), unorm8(sm.w));
    }
    reinterpret_cast<uchar4 *>(out + (size_t)y * out_pitch)[x] = o;
}

int launch_preprocess(const Tex &src, int mode, int rescale, uint8_t *out, int out_pitch, int out_w, int out_h, Stream s) {
    dim3 b(32, 8), g((out_w + 31) / 32, (out_h + 7) / 8);
    k_preprocess<<<g, b, 0, (cudaStream_t)s>>>(src, mode, rescale, out, out_pitch, out_w, out_h);
    return check_launch("k_preprocess") ? 1 : -1;
}

// ------------------------------------------------------------------------------------------------
// Text node texture (transformations/text_renderer.rs:72-167 + glyphon's glyph pipeline): LoadOp::Clear(background), then
// one quad per prepared glyph, wgpu::BlendState::ALPHA_BLENDING through the node texture's view, in list order.
// One thread per pixel of a 32 x 8 tile; the block walks the glyph list 256 entries at a time, keeps (in order) the
// ones whose quad touches the tile, and every pixel blends those that cover it.  Quads sit on whole pixels and whole
// atlas texels, so a covered pixel reads exactly one texel.  Rendered once per scene update, not per frame.
// Every text node of a tick is one launch: block b belongs to the job whose tile range [tile_begin[i], tile_begin[i + 1])
// holds it (a binary search by one thread), and the job is copied to shared memory.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_text(const TextJob *__restrict__ jobs, const int32_t *__restrict__ tile_begin, int n_jobs) {
    __shared__ Tables T;
    __shared__ int s_list[256];
    __shared__ int s_wc[8];
    __shared__ TextJob J;
    const int lane = threadIdx.x, warp = threadIdx.y, tid = warp * 32 + lane;
    // the tile's origin is handed over through s_wc before the glyph loop reuses it
    if (tid == 0) load_block_job(jobs, tile_begin, n_jobs, J, s_wc);
    load_tables(T);   // ends in __syncthreads
    const int x0 = s_wc[0], y0 = s_wc[1], px = x0 + lane, py = y0 + warp;
    __syncthreads();   // s_wc is rewritten by the glyph loop
    uchar4 d;
    if (J.dst.mode == 0) d = make_uchar4((unsigned char)srgb_encode(T, J.bg[0]), (unsigned char)srgb_encode(T, J.bg[1]), (unsigned char)srgb_encode(T, J.bg[2]), (unsigned char)unorm8(J.bg[3]));
    else d = make_uchar4((unsigned char)unorm8(J.bg[0]), (unsigned char)unorm8(J.bg[1]), (unsigned char)unorm8(J.bg[2]), (unsigned char)unorm8(J.bg[3]));
    const float *clut = J.color_mode == 0 ? T.dec : T.u8n;   // ColorMode::Accurate: glyph colours and colour-atlas texels -> linear
    const float *dlut = J.dst.mode == 0 ? T.dec : T.u8n;     // the node texture's view
    for (int base = 0; base < J.n_glyphs; base += 256) {
        const int gi = base + tid;
        bool hit = false;
        if (gi < J.n_glyphs) {
            const GlyphDev G = J.glyphs[gi];
            hit = G.w > 0 && G.h > 0 && G.x < x0 + 32 && G.x + (int)G.w > x0 && G.y < y0 + 8 && G.y + (int)G.h > y0;
        }
        const unsigned b = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) s_wc[warp] = __popc(b);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < 8; w++) { const int c = s_wc[w]; before += w < warp ? c : 0; total += c; }
        if (hit) s_list[before + __popc(b & ((1u << lane) - 1u))] = gi;   // list order is painter's order
        __syncthreads();
        for (int k = 0; k < total; k++) {
            const GlyphDev G = J.glyphs[s_list[k]];
            const int dx = px - G.x, dy = py - G.y;
            if ((unsigned)dx >= (unsigned)G.w || (unsigned)dy >= (unsigned)G.h) continue;
            const int ax = (int)G.ax + dx, ay = (int)G.ay + dy;
            float s0, s1, s2, a;
            if (G.content == 1) {      // ContentType::Mask: (colour.rgb, colour.a * coverage)
                const int cx = min(ax, J.mask_w - 1), cy = min(ay, J.mask_h - 1);
                const float cov = J.mask ? T.u8n[__ldg(J.mask + (size_t)cy * J.mask_pitch + cx)] : 0.0f;
                s0 = clut[G.color[0]]; s1 = clut[G.color[1]]; s2 = clut[G.color[2]];
                a = T.u8n[G.color[3]] * cov;
            } else {                   // ContentType::Color: the atlas texel
                if (J.color) {
                    const int cx = min(ax, J.color_w - 1), cy = min(ay, J.color_h - 1);
                    const uchar4 t = __ldg(reinterpret_cast<const uchar4 *>(J.color + (size_t)cy * J.color_pitch) + cx);
                    s0 = clut[t.x]; s1 = clut[t.y]; s2 = clut[t.z]; a = T.u8n[t.w];
                } else { s0 = s1 = s2 = a = 0.0f; }
            }
            s0 = clamp01(s0); s1 = clamp01(s1); s2 = clamp01(s2); a = clamp01(a);
            if (a == 0.0f) continue;   // dst * 1 + src * 0: encode(decode(b)) == b, unorm8(b / 255) == b
            const float ia = 1.0f - a;
            const float r0 = fmaf(dlut[d.x], ia, s0 * a), r1 = fmaf(dlut[d.y], ia, s1 * a), r2 = fmaf(dlut[d.z], ia, s2 * a);
            if (J.dst.mode == 0) { d.x = (unsigned char)srgb_encode(T, r0); d.y = (unsigned char)srgb_encode(T, r1); d.z = (unsigned char)srgb_encode(T, r2); }
            else { d.x = (unsigned char)unorm8(r0); d.y = (unsigned char)unorm8(r1); d.z = (unsigned char)unorm8(r2); }
            d.w = (unsigned char)unorm8(fmaf(T.u8n[d.w], ia, a));
        }
        __syncthreads();   // s_list / s_wc are rewritten by the next batch
    }
    if (px < J.dst.width && py < J.dst.height) reinterpret_cast<uchar4 *>(J.dst.out + (size_t)py * J.dst.out_pitch)[px] = d;
}

// ------------------------------------------------------------------------------------------------
// Image node texture (transformations/image.rs:178-187, add_premultiplied_alpha.wgsl): a full-target quad samples the
// asset frame (straight alpha) with the linear / clamp-to-edge sampler through the mode's source view, premultiplies and
// stores through the mode's target view.  When the node and the asset differ in size this pass is also the scaler.
// An SVG raster (svg_image.rs:144-180, 262-292: premultiplied, at the node's size) is stored unchanged in CpuOptimized;
// GpuOptimized runs the reference's two full-target passes per pixel:
//   1. remove_premultiplied_alpha.wgsl through UNORM views: the NC-6u sample, a = max(c.a, 1e-5), clamp(c.rgb / a) and
//      clamp(c.a), stored as UNORM8 (NC-2);
//   2. add_premultiplied_alpha.wgsl through sRGB views: pass 1's four bytes decoded as a straight-alpha texel (NC-3) and
//      premultiply_store.  Pass 2 samples a texture of the target's size at the pixel centre, as pass 1 does: the tap is
//      texel (x, y) with weight 1 at every size up to 16384 (tests/svg_oracle.c: orc_check_same_size_taps), so the
//      texel is the byte pass 1 stored for this pixel.
// Every image node a tick draws is one launch, block -> job as in k_text; one thread per pixel of a 32 x 8 tile.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_image(const ImageJob *__restrict__ jobs, const int32_t *__restrict__ tile_begin, int n_jobs) {
    __shared__ Tables T;
    __shared__ ImageJob J;
    __shared__ int s_origin[2];
    if (threadIdx.x == 0 && threadIdx.y == 0) load_block_job(jobs, tile_begin, n_jobs, J, s_origin);
    load_tables(T);   // ends in __syncthreads
    const int x = s_origin[0] + (int)threadIdx.x, y = s_origin[1] + (int)threadIdx.y;
    if (x >= J.dst.width || y >= J.dst.height) return;
    bool exact;
    uchar4 texel, o;
    const float tx = ((float)x + 0.5f) / (float)J.dst.width, ty = ((float)y + 0.5f) / (float)J.dst.height;
    if (!J.raster) {
        o = premultiply_store(T, J.dst.mode, sample_node(T, &J.src, J.dst.mode, tx, ty, exact, texel));
    } else if (J.dst.mode != 0) {
        o = node_texel(T, J.src, x, y);
    } else {
        const float4 c = sample_node(T, &J.src, 1, tx, ty, exact, texel);
        const float a = fmaxf(c.w, 0.00001f);
        const uchar4 s = make_uchar4(unorm8(c.x / a), unorm8(c.y / a), unorm8(c.z / a), unorm8(c.w));   // unorm8 clamps
        o = premultiply_store(T, 0, make_float4(T.dec[s.x], T.dec[s.y], T.dec[s.z], T.u8n[s.w]));
    }
    reinterpret_cast<uchar4 *>(J.dst.out + (size_t)y * J.dst.out_pitch)[x] = o;
}

// ------------------------------------------------------------------------------------------------
// Web view node texture (web_renderer/shader.rs:53-114, render_website.wgsl): one render pass per plane, the first one
// clearing to transparent.  A pass leaves the pixels its quad does not cover as they are and blends the bare sample into
// the others (PREMULTIPLIED_ALPHA_BLENDING through the target view), so each pixel walks the planes in order with its
// value quantised to 8 bits after every plane, as the texture holds it between passes.  The web nodes of one depth a tick
// draws are one launch, block -> job as in k_text; one thread per pixel of a 32 x 8 tile.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_web(const WebJob *__restrict__ jobs, const int32_t *__restrict__ tile_begin, int n_jobs) {
    __shared__ Tables T;
    __shared__ WebJob J;
    __shared__ int s_origin[2];
    if (threadIdx.x == 0 && threadIdx.y == 0) load_block_job(jobs, tile_begin, n_jobs, J, s_origin);
    load_tables(T);   // ends in __syncthreads
    const int x = s_origin[0] + (int)threadIdx.x, y = s_origin[1] + (int)threadIdx.y;
    if (x >= J.dst.width || y >= J.dst.height) return;
    const float pcx = (float)x + 0.5f, pcy = (float)y + 0.5f;
    uchar4 o = make_uchar4(0, 0, 0, 0);
    for (int i = 0; i < J.n_planes; i++) {
        const WebPlane &P = J.planes[i];
        if (x < P.px0 || x >= P.px1 || y < P.py0 || y >= P.py1) continue;
        bool exact;
        uchar4 texel;
        const float4 s = sample_node(T, &P.tex, J.dst.mode, (pcx - P.left) / P.width, (pcy - P.top) / P.height, exact, texel);
        o = blend(T, J.dst.mode, o, s);
    }
    reinterpret_cast<uchar4 *>(J.dst.out + (size_t)y * J.dst.out_pitch)[x] = o;
}

const void *node_kernel(NodeKernel k) {
    const void *const kernels[] = {(const void *)k_text, (const void *)k_image, (const void *)k_web};
    return kernels[k];
}

int launch_tile_jobs(const void *kernel, const void *jobs_dev, const int32_t *tile_begin_dev, int n_jobs, int n_tiles,
                     const char *name, Stream s) {
    if (n_jobs <= 0 || n_tiles <= 0) return 0;
    void *args[] = {(void *)&jobs_dev, (void *)&tile_begin_dev, (void *)&n_jobs};
    cudaLaunchKernel(kernel, dim3(n_tiles), dim3(32, 8), args, 0, (cudaStream_t)s);
    return check_launch(name) ? 1 : -1;
}

bool table_symbols(const void *ptr[5], size_t bytes[5]) {
    const void *sym[5] = {c_u8n, c_dec, c_thr, c_yl, c_enc1};
    const size_t n[5] = {sizeof(c_u8n), sizeof(c_dec), sizeof(c_thr), sizeof(c_yl), sizeof(c_enc1)};
    for (int i = 0; i < 5; i++) {
        void *p = nullptr;
        if (cudaGetSymbolAddress(&p, sym[i]) != cudaSuccess) return false;
        ptr[i] = p;
        bytes[i] = n[i];
    }
    return true;
}

// ------------------------------------------------------------------------------------------------
// K6: black frame (render_loop.rs:127-173)
// ------------------------------------------------------------------------------------------------
__global__ void k_fill(uint8_t *p0, uint8_t *p1, uint8_t *p2, int pitch0, int pitch1, int pitch2, int w, int h,
                       int fmt, uint8_t yv, uint8_t uv, uint8_t vv) {
    int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    if (fmt == 3) {
        reinterpret_cast<uchar4 *>(p0 + (size_t)y * pitch0)[x] = make_uchar4(0, 0, 0, 0);
        return;
    }
    p0[(size_t)y * pitch0 + x] = yv;
    int cw, ch;
    chroma_dims(fmt, w, h, cw, ch);
    if (x < cw && y < ch) {
        if (fmt == 4) {
            p1[(size_t)y * pitch1 + 2 * x] = uv;
            p1[(size_t)y * pitch1 + 2 * x + 1] = vv;
        } else {
            p1[(size_t)y * pitch1 + x] = uv;
            p2[(size_t)y * pitch2 + x] = vv;
        }
    }
}

int launch_fill_yuv(uint8_t *p0, uint8_t *p1, uint8_t *p2, int pitch0, int pitch1, int pitch2, int w, int h, int fmt,
                    uint8_t y, uint8_t u, uint8_t v, Stream s) {
    dim3 b(32, 8), g((w + 31) / 32, (h + 7) / 8);
    k_fill<<<g, b, 0, (cudaStream_t)s>>>(p0, p1, p2, pitch0, pitch1, pitch2, w, h, fmt, y, u, v);
    return check_launch("k_fill") ? 1 : -1;
}

}  // namespace dev
}  // namespace smr
