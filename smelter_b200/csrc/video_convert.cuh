// video_convert.cuh -- gpu-video's NV12 -> RGBA converter (WgpuNv12ToRgbaConverter, nv12_to_rgba.wgsl fs_main): one NV12
// crop to one Rgba8Unorm target of any size, BT.709 limited range (NC-11).  Included by kernels.cu inside namespace
// smr::dev, after node_sample.cuh, whose NC-6u sampler (linear_tap, sample_u8, quad_chroma_row / quad_chroma16, div255)
// it uses as the composite and k_preprocess do.  The reverse converter is K11 and runs as k_output.
//
// At the source size the taps are known (NC-6 at an even size: luma texel (x, y), the .25 / .75 chroma pair), so a thread
// owns a 2 x 2 luma quad and the 3 x 3 uv neighbourhood its chroma taps read, and stores two 8-byte RGBA runs.  At any
// other size a thread owns one target pixel and takes NC-6u's four taps per plane.

constexpr float kVcBiasY = 16.0f / 255.0f;    // f32(16 / 255): IEEE division of exact operands rounds the quotient once
constexpr float kVcScaleY = 255.0f / 219.0f;  // f32(255 / 219)
constexpr float kVcScaleC = 255.0f / 224.0f;  // f32(255 / 224)

// NC-11 steps 3-5 on the sampled (Y, Cb, Cr): offsets, scale, `s * M` (the x1 and x0 terms dropped: byte-identical), NC-2
// store, alpha 255.  Packed RGBA, r in the low byte.
__device__ __forceinline__ uint32_t vc_bt709_limited(float y, float cb, float cr) {
    const float s0 = (y - kVcBiasY) * kVcScaleY, s1 = (cb - 0.5f) * kVcScaleC, s2 = (cr - 0.5f) * kVcScaleC;
    constexpr YuvCoef k = yuv_coef(0);
    const uint32_t r = (uint32_t)unorm8(s0 + s2 * k.rv);
    const uint32_t g = (uint32_t)unorm8((s0 + s1 * k.gu) + s2 * k.gv);
    const uint32_t b = (uint32_t)unorm8(s0 + s1 * k.bu);
    return r | (g << 8) | (b << 16) | 0xff000000u;
}

template <bool SAME_SIZE>
__global__ void __launch_bounds__(kVideoConvertTileX * kVideoConvertTileY) k_video_nv12_to_rgba(const VideoConvertJob J) {
    const Tex &S = J.src;
    if constexpr (SAME_SIZE) {
        const int cw = S.width >> 1, ch = S.height >> 1;
        const int cx = blockIdx.x * kVideoConvertTileX + threadIdx.x, cy = blockIdx.y * kVideoConvertTileY + threadIdx.y;
        if (cx >= cw || cy >= ch) return;
        const int xm = max(cx - 1, 0), xp = min(cx + 1, cw - 1);   // the taps clamp to the edge
        unsigned he[3], ho[3];
#pragma unroll
        for (int i = 0; i < 3; i++) {
            const uchar2 *row = reinterpret_cast<const uchar2 *>(S.p1 + (size_t)min(max(cy - 1 + i, 0), ch - 1) * S.pitch1);
            const uchar2 a = __ldg(row + xm), b = __ldg(row + cx), d = __ldg(row + xp);
            quad_chroma_row(a.x | (a.y << 16), b.x | (b.y << 16), d.x | (d.y << 16), he[i], ho[i]);
        }
        unsigned n[4];
        quad_chroma16(he, ho, n[0], n[1], n[2], n[3]);
        const uint8_t *l0 = S.p0 + (size_t)(2 * cy) * S.pitch0 + 2 * cx;
        const uchar2 y0 = __ldg(reinterpret_cast<const uchar2 *>(l0)), y1 = __ldg(reinterpret_cast<const uchar2 *>(l0 + S.pitch0));
        const uint8_t luma[4] = {y0.x, y0.y, y1.x, y1.y};
        uint32_t px[4];
#pragma unroll
        for (int q = 0; q < 4; q++)   // NC-6u of one texel is NC-1; of the chroma taps, 16 x the value / (16 x 255)
            px[q] = vc_bt709_limited(div255((float)luma[q], 1.0f), div255((float)(n[q] & 0xffffu), 0.0625f),
                                     div255((float)(n[q] >> 16), 0.0625f));
        uint8_t *o0 = J.out + (size_t)(2 * cy) * J.out_pitch + 8 * cx, *o1 = o0 + J.out_pitch;
        if ((((uintptr_t)J.out | (uintptr_t)J.out_pitch) & 7) == 0) {
            *reinterpret_cast<uint2 *>(o0) = make_uint2(px[0], px[1]);
            *reinterpret_cast<uint2 *>(o1) = make_uint2(px[2], px[3]);
        } else {   // 4-byte aligned targets
            reinterpret_cast<uint32_t *>(o0)[0] = px[0]; reinterpret_cast<uint32_t *>(o0)[1] = px[1];
            reinterpret_cast<uint32_t *>(o1)[0] = px[2]; reinterpret_cast<uint32_t *>(o1)[1] = px[3];
        }
    } else {
        const int x = blockIdx.x * kVideoConvertTileX + threadIdx.x, y = blockIdx.y * kVideoConvertTileY + threadIdx.y;
        if (x >= J.out_w || y >= J.out_h) return;
        const float u = ((float)x + 0.5f) / (float)J.out_w, v = ((float)y + 0.5f) / (float)J.out_h;   // NC-11 step 1
        const LinTap ax = linear_tap(u, S.width), ay = linear_tap(v, S.height);
        const LinTap cx = linear_tap(u, S.width >> 1), cy = linear_tap(v, S.height >> 1);
        const float yy = sample_u8(S.p0, S.pitch0, 1, 0, ax, ay);
        const float cb = sample_u8(S.p1, S.pitch1, 2, 0, cx, cy), cr = sample_u8(S.p1, S.pitch1, 2, 1, cx, cy);
        reinterpret_cast<uint32_t *>(J.out + (size_t)y * J.out_pitch)[x] = vc_bt709_limited(yy, cb, cr);
    }
}

int launch_video_nv12_to_rgba(const VideoConvertJob &J, Stream s) {
    const dim3 b(kVideoConvertTileX, kVideoConvertTileY);
    if (J.out_w == J.src.width && J.out_h == J.src.height) {
        const dim3 g((J.out_w / 2 + kVideoConvertTileX - 1) / kVideoConvertTileX, (J.out_h / 2 + kVideoConvertTileY - 1) / kVideoConvertTileY);
        k_video_nv12_to_rgba<true><<<g, b, 0, (cudaStream_t)s>>>(J);
    } else {
        const dim3 g((J.out_w + kVideoConvertTileX - 1) / kVideoConvertTileX, (J.out_h + kVideoConvertTileY - 1) / kVideoConvertTileY);
        k_video_nv12_to_rgba<false><<<g, b, 0, (cudaStream_t)s>>>(J);
    }
    return check_launch("k_video_nv12_to_rgba") ? 1 : -1;
}
