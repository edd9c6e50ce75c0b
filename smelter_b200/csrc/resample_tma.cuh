// resample_tma.cuh -- K1/K2 + K8 (horizontal) + K8 (vertical) fused, TMA data movement (included by kernels.cu).
//
// Same arithmetic, same quantisation points and the same per-output accumulation order as k_resample_fused_int
// (resample.wgsl:42-86 twice, planar_yuv_to_rgba.wgsl / nv12_to_rgba.wgsl in front), so the bytes are identical;
// what changes is how the data moves and how the instructions are issued:
//
//   * the strip's source rows arrive by TMA: one elected thread issues cp.async.bulk.tensor.2d copies of a
//     (272 B x 32 rows) luma box and the matching chroma box per chunk into a double-buffered shared-memory
//     stage, completion on an mbarrier; the loads of chunk c+1 are in flight while chunk c is converted.  A box may
//     start at a negative coordinate but only at a 16-byte boundary of the row (the TMA unit's alignment rule for
//     the global address of a box), so the tile starts at the strip's first pixel rounded down
//     to 16 and every lane realigns its bytes with one funnel shift per word; out-of-image bytes (zero-filled by
//     the TMA unit) are replaced by the edge texels (resample.wgsl clamps the tap index);
//   * no shared-memory row buffer and no per-tap LDS in the horizontal pass: lane l owns the 8 consecutive source
//     pixels X0 + 8l .. X0 + 8l + 7 of a row, converts them once (K1/K2 -> u8 -> sRGB decode) and keeps the 24
//     decoded floats in registers.  The accumulators of an output column travel through the lanes that own its
//     taps: they start in the lane that owns tap 0, take that lane's pixels in tap order, hop to lane + 1 with
//     SHFL.UP, and so on (4 lanes for the 25 taps of a 4:1 pass) -- a systolic array along the warp.  Every
//     accumulator still sees its taps in the order t = 0 .. TAPS-1, one fma each, so the sum is bit-identical;
//   * FP32 pairs (fma2 / mul2 / add2, two scalar IEEE operations each on sm_90) hold two pixels (conversion), the
//     r and g channel of one output, or two output columns;
//   * integer -> float without the conversion unit: a byte or a 16-bit field is PRMT-ed under the exponent of 2^23
//     and 2^23 is subtracted (exact); float -> index by adding 1.5 * 2^23 (round-to-nearest-even, exactly
//     __float2int_rn for |x| < 2^22); the clamp of NC-2 is folded into a decode table that is extended on both sides;
//   * the horizontal results of a row (f16-quantised, NC-5) go to a ring of rows in shared memory as f32, each lane
//     into its own slot, and the vertical pass reads them back with LDS.64 / LDS.128 + FMA pairs.
//
// Template parameter S in {2, 4}: integer horizontal ratio with zero crop offset (first(o) = S * o + const).
// SRC: 0 planar 4:2:0, 1 NV12.
#pragma once

namespace v5 {

constexpr int kWarps = 8;
constexpr int kChunkRows = 32;                       // source rows per TMA chunk
// box widths in BYTES: 256 pixels + up to 14 bytes of alignment slack (luma); 6 chroma texels per lane + slack
constexpr int kLumaBox = 272, kNv12Box = 288, kPlanarBox = 160, kChromaRows = 18;
constexpr int kLumaBytes = kLumaBox * kChunkRows;                                    // 8704
constexpr int kChromaBytesNv12 = ((kNv12Box * kChromaRows + 127) / 128) * 128;      // 5248
constexpr int kChromaBytesPlanar = ((kPlanarBox * kChromaRows + 127) / 128) * 128;  // 2944 (per plane)
constexpr int kStageBytes = kLumaBytes + 2 * kChromaBytesPlanar;                    // 14592 >= luma + NV12 chroma
static_assert(kLumaBytes % 128 == 0, "chroma destination alignment");
static_assert(kStageBytes >= kLumaBytes + kChromaBytesNv12, "stage size");
constexpr int kDecLo = 240, kDecN = 736;             // extended decode table: entry i + kDecLo for i in [-240, 495]
constexpr float kMagicRound = 12582912.0f;           // 1.5 * 2^23
constexpr uint32_t kMagicBits = 0x4B400000u;

template <int S>
struct Cfg {
    static constexpr int P = 8;                      // source pixels per lane and row
    static constexpr int OUT = P / S;                // output columns started per lane
    static constexpr int TAPS = 6 * S + 1;
    static constexpr int A = S == 2 ? 1 : 0;         // X0 = first(O0) - A is even
    static constexpr int NST = (A + S * (OUT - 1) + TAPS + P - 1) / P;   // lanes an accumulator visits
    static __host__ __device__ constexpr int last_stage(int j) { return (A + S * j + TAPS - 1) / P; }
    // first strip-relative column no lane completes
    static __host__ __device__ constexpr int nout() {
        int m = 1 << 30;
        for (int j = 0; j < OUT; j++) {
            int c = OUT * (32 - last_stage(j)) + j;
            m = c < m ? c : m;
        }
        return m;
    }
    static constexpr int NOUT = nout();              // output columns per strip: 58 (S = 4), 122 (S = 2)
    static constexpr int RROWS = S == 4 ? 54 : 28;   // ring rows >= taps_v + ceil(7 * scale_v) + 1
    static constexpr int RROW_BYTES = 32 * 3 * OUT * 4;
    static constexpr int RING_BYTES = RROWS * RROW_BYTES;
    static constexpr int SMEM = 2 * kStageBytes + RING_BYTES + kDecN * 4 + 256 * 4 + 448 + 16;
};

struct Chunk {      // warp-uniform description of one pipeline step
    int valid;      // 0: the block has no more work
    int job, ox0;   // job index, first output column of the strip
    int x0;         // first source pixel of the strip's tile
    int r0, nrows;  // source rows [r0, r0 + nrows) to convert in this step (nrows may be 0)
    int last;       // the group's rows are complete after this chunk: run the vertical pass
    int o0, oy_end; // the group's output rows [o0, min(o0 + 8, oy_end))
};

template <int S>
struct ChunkIter {
    const FusedJob *jobs;
    const FusedPiece *pieces;
    int pi, pend;
    int job, ox0, x0, oy_end, onext, ocur;
    int produced_hi, rnext, rhi;
    int H, tv, fv0;   // of the current piece's job; fv0 = first_v[0] when the vertical mapping is the integer ratio
    bool in_group, vs;
    __device__ void init(const FusedJob *j, const FusedPiece *p, int b, int e) {
        jobs = j; pieces = p; pi = b - 1; pend = e; in_group = false; onext = 0; oy_end = 0;
        job = ox0 = x0 = ocur = 0; produced_hi = rnext = rhi = 0; H = tv = fv0 = 0; vs = false;
    }
    __device__ Chunk next() {
        Chunk c;
        c.valid = 0; c.job = c.ox0 = c.x0 = c.r0 = c.nrows = c.last = c.o0 = c.oy_end = 0;
        if (!(in_group && rnext <= rhi)) {   // next group of 8 output rows (possibly of the next piece)
            if (onext >= oy_end) {
                pi++;
                if (pi >= pend) return c;
                const FusedPiece P = pieces[pi];
                job = P.job; ox0 = P.strip * Cfg<S>::NOUT; onext = P.oy_begin; oy_end = P.oy_end;
                const FusedJob &J = jobs[job];
                x0 = __ldg(J.first_h + ox0) - Cfg<S>::A;
                H = J.src.height; tv = J.taps_v; vs = J.v_same != 0;
                fv0 = __ldg(J.first_v);
                produced_hi = -0x40000000;
            }
            ocur = onext;
            const int o_l = min(ocur + kWarps - 1, oy_end - 1);
            // same integer ratio vertically: first_v(o) = first_v(0) + S * o (resample.wgsl:45-50 in exact arithmetic), no
            // dependent global loads on the way to the next TMA issue
            const int f_lo = vs ? fv0 + S * ocur : __ldg(jobs[job].first_v + ocur);
            const int f_hi = vs ? fv0 + S * o_l : __ldg(jobs[job].first_v + o_l);
            const int need_lo = min(max(f_lo, 0), H - 1);
            const int need_hi = min(max(f_hi + tv - 1, 0), H - 1);
            rnext = max(produced_hi + 1, need_lo);
            rhi = need_hi;
            produced_hi = max(produced_hi, need_hi);
            onext += kWarps;
            in_group = true;
        }
        c.valid = 1; c.job = job; c.ox0 = ox0; c.x0 = x0; c.o0 = ocur; c.oy_end = oy_end;
        c.r0 = rnext;
        c.nrows = max(0, min(kChunkRows, rhi - rnext + 1));
        rnext += kChunkRows;
        c.last = rnext > rhi;
        return c;
    }
};

template <int S, int SRC>
__global__ void __launch_bounds__(32 * kWarps, 3) k_resample_tma(const FusedJob *jobs, const FusedPiece *pieces, const int *piece_begin) {
    using K = Cfg<S>;
    constexpr int P = K::P, OUT = K::OUT, TAPS = K::TAPS, A = K::A, NST = K::NST;
    constexpr bool NV12 = SRC == 1;
    extern __shared__ __align__(128) unsigned char smem[];
    const uint32_t stage0 = smem_u32(smem);
    float *ring = reinterpret_cast<float *>(smem + 2 * kStageBytes);
    float *s_dec = reinterpret_cast<float *>(smem + 2 * kStageBytes + K::RING_BYTES);
    float *s_thr = s_dec + kDecN;
    unsigned char *s_enc0 = reinterpret_cast<unsigned char *>(s_thr + 256);
    const uint32_t bar0 = smem_u32(s_enc0 + 448);
    volatile uint32_t *s_kaddr = reinterpret_cast<volatile uint32_t *>(s_enc0 + 424);
    const int lane = threadIdx.x, warp = threadIdx.y, tid = warp * 32 + lane;

    for (int i = tid; i < kDecN; i += 32 * kWarps) s_dec[i] = c_dec[min(max(i - kDecLo, 0), 255)];
    for (int i = tid; i < 256; i += 32 * kWarps) s_thr[i] = c_thr[i];
    if (tid == 0) {
        // table address such that entry i = [(float bits of (i + 1.5 * 2^23)) << 2 + kaddr]  (mod 2^32); it takes a
        // round trip through shared memory so that it stays ONE register and the lookup address ONE LEA
        *s_kaddr = smem_u32(s_dec) + 4u * (uint32_t)kDecLo - (kMagicBits << 2);
        mbar_init(bar0, 1);
        mbar_init(bar0 + 8, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const uint32_t kaddr = *s_kaddr;

    ChunkIter<S> it;
    it.init(jobs, pieces, __ldg(piece_begin + blockIdx.x), __ldg(piece_begin + blockIdx.x + 1));

    auto issue = [&](const Chunk &c, int buf) {   // one thread: TMA loads of the chunk's boxes
        if (!c.valid || c.nrows == 0) return;
        const FusedJob &J = jobs[c.job];
        const uint32_t bar = bar0 + 8u * (uint32_t)buf, dst = stage0 + (uint32_t)buf * kStageBytes;
        const int cyb = (c.r0 >> 1) - 1;
        const int xt = c.x0 & ~15;                         // luma tile: first byte, 16-byte boundary (may be negative)
        if (NV12) {
            const int xc = (c.x0 - 2) & ~15;               // chroma tile: texel cx - 1 of the first pair sits at byte x0 - 2
            mbar_expect_tx(bar, kLumaBox * kChunkRows + kNv12Box * kChromaRows);
            tma_load_2d(dst, J.tm0, xt >> 1, c.r0, bar);   // both planes are addressed in 2-byte elements
            tma_load_2d(dst + kLumaBytes, J.tm1, xc >> 1, cyb, bar);
        } else {
            const int xc = ((c.x0 >> 1) - 1) & ~15;
            mbar_expect_tx(bar, kLumaBox * kChunkRows + 2 * kPlanarBox * kChromaRows);
            tma_load_2d(dst, J.tm0, xt >> 1, c.r0, bar);
            tma_load_2d(dst + kLumaBytes, J.tm1, xc, cyb, bar);
            tma_load_2d(dst + kLumaBytes + kChromaBytesPlanar, J.tm2, xc, cyb, bar);
        }
    };

    Chunk cur = it.next();
    if (!cur.valid) return;
    if (tid == 0) issue(cur, 0);
    uint32_t nchunk = 0;        // chunks that carried a TMA load so far (stage / parity bookkeeping)

    while (cur.valid) {
        Chunk nxt = it.next();
        // every warp is done with the stage the next load overwrites (it was read two chunks ago) and with the
        // previous group's vertical pass (the ring rows it read may be overwritten now)
        __syncthreads();
        const bool cur_tma = cur.nrows > 0;
        const int buf = (int)(nchunk & 1u);
        if (tid == 0) issue(nxt, cur_tma ? buf ^ 1 : buf);
        const FusedJob &J = jobs[cur.job];
        const int W = J.src.width, H = J.src.height, chei = H >> 1;
        const bool full_range = J.src.full_range != 0;
        const float nk16 = full_range ? 0.0f : -K16, rcp_y = full_range ? 1.0f : RCP_Y, rcp_c = full_range ? 1.0f : RCP_C;
        const uint32_t sb = stage0 + (uint32_t)buf * kStageBytes;
        if (cur_tma) {
            mbar_wait(bar0 + 8u * (uint32_t)buf, (nchunk >> 1) & 1u);
            // ---- image borders: the tap index is clamped (resample.wgsl), the TMA unit zero-fills ----------------
            const int x0 = cur.x0;
            const int cyb = (cur.r0 >> 1) - 1;
            const int xt = x0 & ~15, xc = NV12 ? ((x0 - 2) & ~15) : (((x0 >> 1) - 1) & ~15);
            const int cw = W >> 1;
            if (xt < 0 || xt + kLumaBox > W || xc < 0 || (NV12 ? xc + kNv12Box > W : xc + kPlanarBox > cw)) {
                unsigned char *st = smem + (size_t)buf * kStageBytes;
                const int sub = tid & 7;
                {   // luma: tile byte b <-> pixel xt + b; valid bytes [bl, br)
                    const int bl = min(max(0, -xt), kLumaBox - 1), br = min(max(W - xt, 1), kLumaBox);
                    for (int row = tid >> 3; row < cur.nrows; row += 32) {
                        unsigned char *lr = st + row * kLumaBox;
                        const unsigned char vl = lr[bl], vr = lr[br - 1];
                        for (int j = sub; j < bl; j += 8) lr[j] = vl;
                        for (int j = br + sub; j < kLumaBox; j += 8) lr[j] = vr;
                    }
                }
                if (NV12) {   // texel = (u, v) pair; tile texel tt <-> chroma column xc / 2 + tt
                    const int c0 = xc >> 1, nt = kNv12Box / 2;
                    const int tl = min(max(0, -c0), nt - 1), tr = min(max(cw - c0, 1), nt);   // valid texels [tl, tr)
                    for (int row = tid >> 3; row < kChromaRows; row += 32) {
                        unsigned short *cr = reinterpret_cast<unsigned short *>(st + kLumaBytes + row * kNv12Box);
                        const unsigned short vl = cr[tl], vr = cr[tr - 1];
                        for (int j = sub; j < tl; j += 8) cr[j] = vl;
                        for (int j = tr + sub; j < nt; j += 8) cr[j] = vr;
                    }
                } else {
                    const int nt = kPlanarBox;
                    const int tl = min(max(0, -xc), nt - 1), tr = min(max(cw - xc, 1), nt);
                    for (int row = tid >> 3; row < 2 * kChromaRows; row += 32) {
                        unsigned char *cr = st + kLumaBytes + (row >= kChromaRows ? kChromaBytesPlanar + (row - kChromaRows) * kPlanarBox : row * kPlanarBox);
                        const unsigned char vl = cr[tl], vr = cr[tr - 1];
                        for (int j = sub; j < tl; j += 8) cr[j] = vl;
                        for (int j = tr + sub; j < nt; j += 8) cr[j] = vr;
                    }
                }
                fence_proxy_async();
                __syncthreads();
            }
            // this lane's bytes inside the tiles: word address and the funnel shift that realigns them
            const int dl = x0 - xt, dc = (NV12 ? x0 - 2 : (x0 >> 1) - 1) - xc;
            const uint32_t l_off = (uint32_t)((dl & ~3) + lane * 8), l_sh = (uint32_t)(dl & 3) * 8u;
            const uint32_t c_off = (uint32_t)((dc & ~3) + lane * (NV12 ? 8 : 4)), c_sh = (uint32_t)(dc & 3) * 8u;
            // ---- phase A: one source row per warp step ------------------------------------------------------------
            for (int r = cur.r0 + warp; r < cur.r0 + cur.nrows; r += kWarps) {
                // raw bytes of this lane's 8 pixels: 12 bytes from a 4-byte aligned address; the half that is 8-byte aligned
                // (warp-uniform) goes as one LDS.64 (lanes 8 bytes apart: conflict-free, an LDS.32 is 2-way)
                uint32_t yw[2];
                {
                    const uint32_t la = sb + (uint32_t)((r - cur.r0) * kLumaBox) + l_off;
                    uint32_t w0, w1, w2;
                    if (l_off & 4u) { w0 = lds32v(la); lds64v(la + 4, w1, w2); }
                    else { lds64v(la, w0, w1); w2 = lds32v(la + 8); }
                    yw[0] = __funnelshift_r(w0, w1, l_sh);
                    yw[1] = __funnelshift_r(w1, w2, l_sh);
                }
                const int ch = r >> 1;                                              // weight 3/4
                const int cl = (r & 1) ? min(ch + 1, chei - 1) : max(ch - 1, 0);    // weight 1/4
                uint32_t v[6];   // vertically combined chroma texels cx-1 .. cx+4: u in bits 0..15, v in bits 16..31 (4x)
                if (NV12) {
                    const uint32_t bh = sb + kLumaBytes + (uint32_t)((ch - cyb) * kNv12Box) + c_off;
                    const uint32_t bl = sb + kLumaBytes + (uint32_t)((cl - cyb) * kNv12Box) + c_off;
                    uint32_t h0, h1, h2, h3, l0, l1, l2, l3;
                    if (c_off & 4u) {
                        h0 = lds32v(bh); lds64v(bh + 4, h1, h2); h3 = lds32v(bh + 12);
                        l0 = lds32v(bl); lds64v(bl + 4, l1, l2); l3 = lds32v(bl + 12);
                    } else {
                        lds64v(bh, h0, h1); lds64v(bh + 8, h2, h3);
                        lds64v(bl, l0, l1); lds64v(bl + 8, l2, l3);
                    }
                    // words of two texels each: (cx-1, cx), (cx+1, cx+2), (cx+3, cx+4)
                    const uint32_t ph0 = __funnelshift_r(h0, h1, c_sh), ph1 = __funnelshift_r(h1, h2, c_sh), ph2 = __funnelshift_r(h2, h3, c_sh);
                    const uint32_t pl0 = __funnelshift_r(l0, l1, c_sh), pl1 = __funnelshift_r(l1, l2, c_sh), pl2 = __funnelshift_r(l2, l3, c_sh);
                    v[0] = 3u * __byte_perm(ph0, 0, 0x4140) + __byte_perm(pl0, 0, 0x4140);
                    v[1] = 3u * __byte_perm(ph0, 0, 0x4342) + __byte_perm(pl0, 0, 0x4342);
                    v[2] = 3u * __byte_perm(ph1, 0, 0x4140) + __byte_perm(pl1, 0, 0x4140);
                    v[3] = 3u * __byte_perm(ph1, 0, 0x4342) + __byte_perm(pl1, 0, 0x4342);
                    v[4] = 3u * __byte_perm(ph2, 0, 0x4140) + __byte_perm(pl2, 0, 0x4140);
                    v[5] = 3u * __byte_perm(ph2, 0, 0x4342) + __byte_perm(pl2, 0, 0x4342);
                } else {
                    const uint32_t uh = sb + kLumaBytes + (uint32_t)((ch - cyb) * kPlanarBox) + c_off;
                    const uint32_t ul = sb + kLumaBytes + (uint32_t)((cl - cyb) * kPlanarBox) + c_off;
                    const uint32_t vh = uh + kChromaBytesPlanar, vl = ul + kChromaBytesPlanar;
                    // 8 bytes from the lane's first texel (cx - 1): texels cx-1 .. cx+4 are bytes 0 .. 5
                    auto eight = [&](uint32_t a, uint32_t &q0, uint32_t &q1) {
                        const uint32_t w0 = lds32v(a), w1 = lds32v(a + 4), w2 = lds32v(a + 8);
                        q0 = __funnelshift_r(w0, w1, c_sh); q1 = __funnelshift_r(w1, w2, c_sh);
                    };
                    uint32_t uh0, uh1, ul0, ul1, vh0, vh1, vl0, vl1;
                    eight(uh, uh0, uh1); eight(ul, ul0, ul1); eight(vh, vh0, vh1); eight(vl, vl0, vl1);
                    v[0] = 3u * (__byte_perm(uh0, vh0, 0x0400) & 0x00ff00ffu) + (__byte_perm(ul0, vl0, 0x0400) & 0x00ff00ffu);
                    v[1] = 3u * (__byte_perm(uh0, vh0, 0x0501) & 0x00ff00ffu) + (__byte_perm(ul0, vl0, 0x0501) & 0x00ff00ffu);
                    v[2] = 3u * (__byte_perm(uh0, vh0, 0x0602) & 0x00ff00ffu) + (__byte_perm(ul0, vl0, 0x0602) & 0x00ff00ffu);
                    v[3] = 3u * (__byte_perm(uh0, vh0, 0x0703) & 0x00ff00ffu) + (__byte_perm(ul0, vl0, 0x0703) & 0x00ff00ffu);
                    v[4] = 3u * (__byte_perm(uh1, vh1, 0x0400) & 0x00ff00ffu) + (__byte_perm(ul1, vl1, 0x0400) & 0x00ff00ffu);
                    v[5] = 3u * (__byte_perm(uh1, vh1, 0x0501) & 0x00ff00ffu) + (__byte_perm(ul1, vl1, 0x0501) & 0x00ff00ffu);
                }
                // A1: K1/K2 -> u8 -> sRGB decode, two pixels per instruction
                float2 prg[P];   // (r, g) of pixel i
                float pb[P];     // b of pixel i
#pragma unroll
                for (int p = 0; p < P / 2; p++) {
                    // 16 x chroma of the even / odd pixel of the pair (NC-6u with the .25 / .75 taps)
                    const uint32_t ne = v[p] + 3u * v[p + 1], no = 3u * v[p + 1] + v[p + 2];
                    const float m23 = -8388608.0f;
                    float2 nu = add2(make_float2(__uint_as_float(__byte_perm(ne, 0x4B000000u, 0x7610)),
                                                 __uint_as_float(__byte_perm(no, 0x4B000000u, 0x7610))), splat(m23));
                    float2 nv = add2(make_float2(__uint_as_float(__byte_perm(ne, 0x4B000000u, 0x7632)),
                                                 __uint_as_float(__byte_perm(no, 0x4B000000u, 0x7632))), splat(m23));
                    const uint32_t ywd = yw[p >> 1];
                    float2 ny = add2(make_float2(__uint_as_float(__byte_perm(ywd, 0x4B000000u, (p & 1) ? 0x7642 : 0x7640)),
                                                 __uint_as_float(__byte_perm(ywd, 0x4B000000u, (p & 1) ? 0x7643 : 0x7641))), splat(m23));
                    // exact n / 255 and n / (255 * 16): fma(n, c, n * lo)
                    const float c1 = __uint_as_float(0x3b808081u), lo1 = __uint_as_float(0xaf7efeffu);
                    const float c16 = __uint_as_float(0x39808081u), lo16 = __uint_as_float(0xad7efeffu);
                    float2 y = fma2(ny, splat(c1), mul2(ny, splat(lo1)));
                    float2 u = fma2(nu, splat(c16), mul2(nu, splat(lo16)));
                    float2 w = fma2(nv, splat(c16), mul2(nv, splat(lo16)));
                    // limited range: clamp01((x - 16/255) * rcp); full range: (x - 0) * 1 and the clamp are identities on [0, 1]
                    y = add2(y, splat(nk16)); u = add2(u, splat(nk16)); w = add2(w, splat(nk16));
                    y = make_float2(__saturatef(y.x * rcp_y), __saturatef(y.y * rcp_y));
                    u = make_float2(__saturatef(u.x * rcp_c), __saturatef(u.y * rcp_c));
                    w = make_float2(__saturatef(w.x * rcp_c), __saturatef(w.y * rcp_c));
                    const float2 um = add2(u, splat(-0.5f)), vm = add2(w, splat(-0.5f));
                    const float2 rr = fma2(splat(1.5748f), vm, y);
                    const float2 gg = fma2(splat(-0.4681f), vm, fma2(splat(-0.1873f), um, y));
                    const float2 bb = fma2(splat(1.8556f), um, y);
                    // NC-2 (clamp folded into the extended table) and the sRGB decode of the node-texture fetch (NC-3)
                    const float2 qr = add2_after_mul(mul2(rr, splat(255.0f)), splat(kMagicRound));
                    const float2 qg = add2_after_mul(mul2(gg, splat(255.0f)), splat(kMagicRound));
                    const float2 qb = add2_after_mul(mul2(bb, splat(255.0f)), splat(kMagicRound));
                    prg[2 * p] = make_float2(lds_tab((__float_as_uint(qr.x) << 2) + kaddr), lds_tab((__float_as_uint(qg.x) << 2) + kaddr));
                    prg[2 * p + 1] = make_float2(lds_tab((__float_as_uint(qr.y) << 2) + kaddr), lds_tab((__float_as_uint(qg.y) << 2) + kaddr));
                    pb[2 * p] = lds_tab((__float_as_uint(qb.x) << 2) + kaddr);
                    pb[2 * p + 1] = lds_tab((__float_as_uint(qb.y) << 2) + kaddr);
                }
                // A2: horizontal Lanczos along the warp.  acc j of the lane that owns tap 0 of output OUT * lane + j
                float2 arg[OUT];          // (r, g)
                float ab[OUT];            // b
#pragma unroll
                for (int j = 0; j < OUT; j++) { arg[j] = make_float2(0.f, 0.f); ab[j] = 0.f; }
#pragma unroll
                for (int s = 0; s < NST; s++) {
#pragma unroll
                    for (int i = 0; i < P; i++) {
#pragma unroll
                        for (int j = 0; j < OUT; j++) {
                            const int t = P * s + i - A - S * j;   // compile-time after unrolling
                            if (t >= 0 && t < TAPS) arg[j] = fma2(prg[i], splat(c_wint[S][t]), arg[j]);
                        }
#pragma unroll
                        for (int j = 0; j < OUT; j += 2) {
                            const int t0 = P * s + i - A - S * j, t1 = t0 - S;
                            const bool a0 = t0 >= 0 && t0 < TAPS, a1 = t1 >= 0 && t1 < TAPS;
                            if (a0 && a1) {
                                const float2 d = fma2(splat(pb[i]), c_wpair[S][a0 ? t0 : 0], make_float2(ab[j], ab[j + 1]));
                                ab[j] = d.x; ab[j + 1] = d.y;
                            } else if (a0) {
                                ab[j] = fmaf(pb[i], c_wint[S][a0 ? t0 : 0], ab[j]);
                            } else if (a1) {
                                ab[j + 1] = fmaf(pb[i], c_wint[S][a1 ? t1 : 0], ab[j + 1]);
                            }
                        }
                    }
                    if (s + 1 < NST) {
#pragma unroll
                        for (int j = 0; j < OUT; j++)
                            if (K::last_stage(j) > s) {   // still collecting taps: on to the lane that owns the next ones
                                arg[j].x = __shfl_up_sync(0xffffffffu, arg[j].x, 1);
                                arg[j].y = __shfl_up_sync(0xffffffffu, arg[j].y, 1);
                                ab[j] = __shfl_up_sync(0xffffffffu, ab[j], 1);
                            }
                    }
                }
                // normalise, quantise to f16 (NC-5) and park the row in the ring: [row][lane][channel][j]
                {
                    const float inv = c_winv[S];
                    float *dst = ring + (size_t)(r % K::RROWS) * (K::RROW_BYTES / 4) + lane * 3 * OUT;
#pragma unroll
                    for (int j = 0; j < OUT; j += 2) {
                        const float2 fr = __half22float2(__floats2half2_rn(arg[j].x * inv, arg[j + 1].x * inv));
                        const float2 fg = __half22float2(__floats2half2_rn(arg[j].y * inv, arg[j + 1].y * inv));
                        const float2 fb = __half22float2(__floats2half2_rn(ab[j] * inv, ab[j + 1] * inv));
                        *reinterpret_cast<float2 *>(dst + j) = fr;
                        *reinterpret_cast<float2 *>(dst + OUT + j) = fg;
                        *reinterpret_cast<float2 *>(dst + 2 * OUT + j) = fb;
                    }
                }
            }
            nchunk++;
        }
        if (cur.last) {
            __syncthreads();
            // ---- phase B: vertical pass, one output row per warp, OUT columns per lane -----------------------------
            const int oy = cur.o0 + warp;
            if (oy < min(cur.o0 + kWarps, cur.oy_end)) {
                const int tv = J.taps_v;
                const int fv = __ldg(J.first_v + oy);
                const float *wv = J.w_v + (size_t)oy * tv;
                float2 acc[3 * OUT / 2];
#pragma unroll
                for (int k = 0; k < 3 * OUT / 2; k++) acc[k] = make_float2(0.f, 0.f);
                const bool inside = fv >= 0 && fv + tv - 1 <= H - 1;
                const float *lbase = ring + lane * 3 * OUT;
                constexpr int ROWF = K::RROW_BYTES / 4;
                if (inside && J.v_same) {
                    // same integer ratio vertically: the weights are the constant-bank row, the tap loop unrolls; the ring
                    // wraps at most once inside the window (warp-uniform tap index)
                    const int slot0 = fv % K::RROWS, nwrap = K::RROWS - slot0;
                    const float *p0 = lbase + slot0 * ROWF;
#pragma unroll
                    for (int t = 0; t < TAPS; t++) {
                        const float *p = p0 + (t >= nwrap ? (t - K::RROWS) * ROWF : t * ROWF);
#pragma unroll
                        for (int k = 0; k < 3 * OUT / 2; k++) acc[k] = fma2(*reinterpret_cast<const float2 *>(p + 2 * k), splat(c_wint[S][t]), acc[k]);
                    }
                } else if (inside) {
                    int slot = fv % K::RROWS;
                    for (int t = 0; t < tv; t++) {
                        const float wt = __ldg(wv + t);
                        const float *p = lbase + slot * ROWF;
#pragma unroll
                        for (int k = 0; k < 3 * OUT / 2; k++) acc[k] = fma2(*reinterpret_cast<const float2 *>(p + 2 * k), splat(wt), acc[k]);
                        slot = slot + 1 == K::RROWS ? 0 : slot + 1;
                    }
                } else {
                    for (int t = 0; t < tv; t++) {
                        const float wt = __ldg(wv + t);
                        const int row = min(max(fv + t, 0), H - 1);
                        const float *p = lbase + (row % K::RROWS) * ROWF;
#pragma unroll
                        for (int k = 0; k < 3 * OUT / 2; k++) acc[k] = fma2(*reinterpret_cast<const float2 *>(p + 2 * k), splat(wt), acc[k]);
                    }
                }
                const float inv_v = __ldg(J.inv_v + oy);
                // this lane's slot j holds strip column OUT * (lane - last_stage(j)) + j
                uint32_t px[OUT];
#pragma unroll
                for (int j = 0; j < OUT; j++) {
                    const float rv = (j & 1) ? acc[j / 2].y : acc[j / 2].x;
                    const float gv = (j & 1) ? acc[(OUT + j) / 2].y : acc[(OUT + j) / 2].x;
                    const float bv = (j & 1) ? acc[(2 * OUT + j) / 2].y : acc[(2 * OUT + j) / 2].x;
                    auto enc = [&](float lin) -> uint32_t {   // NC-4: count of thresholds <= x = bucket count + one comparison
                        const float x = clamp01(lin);
                        const int k = max((__float_as_int(x) >> 15) - ENC1_KEY0, 0);
                        const uint32_t e = __ldg(c_enc1 + k);
                        return e + (x >= s_thr[e] ? 1u : 0u);
                    };
                    px[j] = enc(rv * inv_v) | (enc(gv * inv_v) << 8) | (enc(bv * inv_v) << 16) | 0xff000000u;
                }
                uint32_t *drow = reinterpret_cast<uint32_t *>(J.dst + (size_t)oy * J.dst_pitch);
                const int ncols = min(K::NOUT, J.dst_w - cur.ox0);
#pragma unroll
                for (int j = 0; j < OUT; j += 2) {   // slots (j, j + 1) are adjacent columns
                    const int col = OUT * (lane - K::last_stage(j)) + j;
                    if (col >= 0 && col + 1 < ncols) {
                        *reinterpret_cast<uint2 *>(drow + cur.ox0 + col) = make_uint2(px[j], px[j + 1]);
                    } else if (col >= 0 && col < ncols) {
                        drow[cur.ox0 + col] = px[j];
                    }
                }
            }
        }
        cur = nxt;
    }
}

}  // namespace v5
