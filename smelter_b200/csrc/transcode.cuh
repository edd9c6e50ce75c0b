// transcode.cuh -- gpu-video's transcoder resize (vulkan_transcoder/shader.wgsl `main`): one NV12 frame to up to eight NV12
// renditions, each with its own size and ScalingAlgorithm, in one launch (NC-10).  Included by kernels.cu inside
// namespace smr::dev, after node_sample.cuh (c_u8n, unorm8).
//
// A block owns a 32 x 8 tile of one rendition's chroma plane, so the branch on the algorithm is uniform in the block; a
// thread owns one chroma sample and the 2 x 2 luma quad whose top-left pixel is the shader invocation that stores it.
// The per-axis coordinates and Lanczos weights come from host tables (TranscodeTap), so the device evaluates no
// transcendental; every remaining operation is the shader's, in its order, each rounded on its own (-fmad=false).

__device__ __forceinline__ float tc_mix(float a, float b, float t) { return a * (1.0f - t) + b * t; }   // WGSL mix

// one luma pixel of the rendition: the shader's sample_{nearest,bilinear,lanczos3}_y, stored NC-2
template <int ALGO>
__device__ __forceinline__ uint8_t tc_luma(const float *u8n, const TranscodeLaunch &L, const TranscodeTap *tx,
                                           const TranscodeTap *ty) {
    if (ALGO == 0)   // the texel's own byte: unorm8(v / 255) == v for every byte
        return __ldg(L.src_y + (size_t)__ldg(&ty->nearest) * L.pitch_y + __ldg(&tx->nearest));
    if (ALGO == 1) {
        const uint8_t *r0 = L.src_y + (size_t)__ldg(&ty->lo) * L.pitch_y, *r1 = L.src_y + (size_t)__ldg(&ty->hi) * L.pitch_y;
        const int x0 = __ldg(&tx->lo), x1 = __ldg(&tx->hi);
        const float fx = __ldg(&tx->frac), fy = __ldg(&ty->frac);
        const float v = tc_mix(tc_mix(u8n[__ldg(r0 + x0)], u8n[__ldg(r0 + x1)], fx),
                               tc_mix(u8n[__ldg(r1 + x0)], u8n[__ldg(r1 + x1)], fx), fy);
        return (uint8_t)unorm8(v);
    }
    const int cx = __ldg(&tx->center), cy = __ldg(&ty->center);
    int sx[6];
    float wx[6];
#pragma unroll
    for (int d = 0; d < 6; d++) {
        sx[d] = min(max(cx + d - 2, 0), L.width - 1);
        wx[d] = __ldg(&tx->w[d]);
    }
    float sum = 0.0f, wsum = 0.0f;
#pragma unroll
    for (int dy = 0; dy < 6; dy++) {
        const uint8_t *row = L.src_y + (size_t)min(max(cy + dy - 2, 0), L.height - 1) * L.pitch_y;
        const float wy = __ldg(&ty->w[dy]);
#pragma unroll
        for (int dx = 0; dx < 6; dx++) {
            const float w = wx[dx] * wy;
            sum = sum + u8n[__ldg(row + sx[dx])] * w;
            wsum = wsum + w;
        }
    }
    return (uint8_t)unorm8(sum / wsum);
}

// the chroma sample: sample_{nearest,bilinear,lanczos3}_uv on the {u, v} plane of (width / 2) x (height / 2)
template <int ALGO>
__device__ __forceinline__ uchar2 tc_chroma(const float *u8n, const TranscodeLaunch &L, const TranscodeTap *tx,
                                            const TranscodeTap *ty) {
    const uchar2 *src = reinterpret_cast<const uchar2 *>(L.src_uv);
    const int pitch = L.pitch_uv >> 1;   // in {u, v} pairs (the plane and its pitch are 2-byte aligned)
    if (ALGO == 0) return __ldg(src + (size_t)__ldg(&ty->nearest) * pitch + __ldg(&tx->nearest));
    if (ALGO == 1) {
        const uchar2 *r0 = src + (size_t)__ldg(&ty->lo) * pitch, *r1 = src + (size_t)__ldg(&ty->hi) * pitch;
        const int x0 = __ldg(&tx->lo), x1 = __ldg(&tx->hi);
        const float fx = __ldg(&tx->frac), fy = __ldg(&ty->frac);
        const uchar2 p00 = __ldg(r0 + x0), p10 = __ldg(r0 + x1), p01 = __ldg(r1 + x0), p11 = __ldg(r1 + x1);
        const float u = tc_mix(tc_mix(u8n[p00.x], u8n[p10.x], fx), tc_mix(u8n[p01.x], u8n[p11.x], fx), fy);
        const float v = tc_mix(tc_mix(u8n[p00.y], u8n[p10.y], fx), tc_mix(u8n[p01.y], u8n[p11.y], fx), fy);
        return make_uchar2((uint8_t)unorm8(u), (uint8_t)unorm8(v));
    }
    const int cw = L.width >> 1, ch = L.height >> 1;
    const int cx = __ldg(&tx->center), cy = __ldg(&ty->center);
    int sx[6];
    float wx[6];
#pragma unroll
    for (int d = 0; d < 6; d++) {
        sx[d] = min(max(cx + d - 2, 0), cw - 1);
        wx[d] = __ldg(&tx->w[d]);
    }
    float su = 0.0f, sv = 0.0f, wsum = 0.0f;
#pragma unroll
    for (int dy = 0; dy < 6; dy++) {
        const uchar2 *row = src + (size_t)min(max(cy + dy - 2, 0), ch - 1) * pitch;
        const float wy = __ldg(&ty->w[dy]);
#pragma unroll
        for (int dx = 0; dx < 6; dx++) {
            const float w = wx[dx] * wy;
            const uchar2 t = __ldg(row + sx[dx]);
            su = su + u8n[t.x] * w;
            sv = sv + u8n[t.y] * w;
            wsum = wsum + w;
        }
    }
    return make_uchar2((uint8_t)unorm8(su / wsum), (uint8_t)unorm8(sv / wsum));
}

template <int ALGO>
__device__ __forceinline__ void tc_quad(const float *u8n, const TranscodeLaunch &L, const TranscodeOut &O, int cx, int cy) {
#pragma unroll 1
    for (int q = 0; q < 4; q++) {
        const int x = 2 * cx + (q & 1), y = 2 * cy + (q >> 1);
        O.y[(size_t)y * O.pitch_y + x] = tc_luma<ALGO>(u8n, L, O.tx + x, O.ty + y);
    }
    const uchar2 c = tc_chroma<ALGO>(u8n, L, O.cx + cx, O.cy + cy);
    uint8_t *d = O.uv + (size_t)cy * O.pitch_uv + 2 * cx;
    d[0] = c.x;
    d[1] = c.y;
}

__global__ void __launch_bounds__(kTranscodeTileX * kTranscodeTileY) k_transcode(const __grid_constant__ TranscodeLaunch L) {
    __shared__ float u8n[256];   // NC-1
    const int tid = threadIdx.y * kTranscodeTileX + threadIdx.x;
    u8n[tid] = c_u8n[tid];
    __syncthreads();
    int r = 0;
    while (r + 1 < L.n && (int)blockIdx.x >= L.out[r + 1].tile_begin) r++;
    const TranscodeOut &O = L.out[r];
    const int t = (int)blockIdx.x - O.tile_begin;
    const int cx = (t % O.tiles_x) * kTranscodeTileX + threadIdx.x, cy = (t / O.tiles_x) * kTranscodeTileY + threadIdx.y;
    if (cx >= (O.width >> 1) || cy >= (O.height >> 1)) return;
    if (O.scaling == 2) tc_quad<2>(u8n, L, O, cx, cy);
    else if (O.scaling == 1) tc_quad<1>(u8n, L, O, cx, cy);
    else tc_quad<0>(u8n, L, O, cx, cy);
}

int launch_transcode(const TranscodeLaunch &L, int n_blocks, Stream s) {
    k_transcode<<<n_blocks, dim3(kTranscodeTileX, kTranscodeTileY), 0, (cudaStream_t)s>>>(L);
    return check_launch("k_transcode") ? 1 : -1;
}
