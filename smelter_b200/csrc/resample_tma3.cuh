// resample_tma3.cuh -- the INTEGER-RATIO (2:1 or 4:1 horizontally, zero crop offset) form of the TMA-staged fused resample
// (included by kernels.cu after resample_tma.cuh, which holds the front end: TMA tiles, edges, K1/K2, decode, encode).
//
//   * no shared-memory row buffer and no per-tap LDS in the horizontal pass: lane l keeps the 24 decoded floats of its 8
//     source pixels in registers.  The accumulators of an output column travel through the lanes that own its taps: they
//     start in the lane that owns tap 0, take that lane's pixels in tap order, hop to lane + 1 with SHFL.UP, and so on
//     (4 lanes for the 25 taps of a 4:1 pass) -- a systolic array along the warp.  Every accumulator still sees its taps
//     in the order t = 0 .. TAPS-1, one fma each, so the sum is bit-identical; FP32 pairs hold the r and g channel of one
//     output, or two output columns;
//   * the horizontal results of a row (f16-quantised, NC-5) go to a ring of rows in shared memory as f32, each lane into
//     its own slot, and the vertical pass reads them back with LDS.64 / LDS.128 + FMA pairs;
//   * one block of 24 warps per SM, three 8-warp groups; ONE 32-row TMA stage per group (a whole 8-output-row step of a
//     4:1 pass), refilled while the vertical pass runs: three groups' stages + rings fit in 227 KB;
//   * the vertical pass of a same-ratio job runs on four warps (one per scheduler) that produce TWO output rows each:
//     consecutive output rows share TAPS - S of their ring rows, every row is loaded once for both.
//
// Template parameter S in {2, 4}: integer horizontal ratio with zero crop offset (first(o) = S * o + const).
// SRC: 0 planar 4:2:0, 1 NV12.  FULL, MAT: the range and the matrix (Tex::matrix) of every source of the launch (the host
// keys the launches by both), so the range constants and the matrix coefficients of K1/K2 are immediates of the row loop
// and take no registers there.  The luma table depends on the range alone.
#pragma once

namespace tma_int {
using namespace tma;

constexpr int kGroups = 3;                            // independent 8-warp groups per block (one block per SM)

// x as a value the compiler knows nothing about: it stays in ONE register across the row loop -- at the kernel's register
// limit the compiler otherwise recomputes a loop-invariant value inside the loop, or folds a constant out of it and adds
// that constant back at every use
__device__ __forceinline__ uint32_t held(uint32_t x) {
    asm("" : "+r"(x));
    return x;
}

template <int S>
struct Cfg {
    static constexpr int P = 8;                      // source pixels per lane and row
    static constexpr int OUT = P / S;                // output columns started per lane
    static constexpr int TAPS = 6 * S + 1;
    // Taps in front of the trailing run of weights that are exactly zero: at an integer ratio with zero offset the Lanczos
    // window covers 6 S pixels, and the last weight of int_weights.h is +0.  No fma is issued for it, in either pass,
    // because there it is an identity:
    //   * every multiplicand is finite (decoded sRGB values in [0, 1]; ring values are f16-rounded finite floats), so
    //     the skipped product is +0 or -0;
    //   * the accumulator is never -0: it starts at +0, and under round-to-nearest fma(x, w, acc) is -0 only if x * w is
    //     -0 and acc is -0, or by underflow -- and x * w is a multiple of 2^-68 (pixels are multiples of 2^-35, ring
    //     values of 2^-24, weights of 2^-33), so x * w + acc is a multiple of the smallest float and rounds to zero only
    //     when it is zero, which gives +0;
    //   * acc + (+-0) == acc bit for bit for every acc other than -0.
    static __host__ __device__ constexpr int taps_nz() {
        int n = TAPS;
        while (n > 0 && int_weight<S>(n - 1) == 0.0f) n--;
        return n;
    }
    static constexpr int TAPS_NZ = taps_nz();
    static_assert(TAPS_NZ == 6 * S, "the integer-ratio weight rows end in exactly one zero");
    static constexpr int A = kLead<S>;               // X0 = first(O0) - A is even
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
    static constexpr int GROUP_BYTES = kStageBytes + RING_BYTES;   // ONE stage: it is refilled while the vertical pass runs
    static constexpr int SMEM = kGroups * GROUP_BYTES + kTailBytes + kLumaTabBytes;
};

template <int S, int SRC, bool FULL, int MAT>
__global__ void __launch_bounds__(32 * kWarps * kGroups, 1) k_resample_tma3(const FusedJob *jobs, const FusedPiece *pieces, const int *piece_begin,
                                                                            int n_virtual_blocks) {
    using K = Cfg<S>;
    using It = ChunkIter<S, 1>;
    constexpr int P = K::P, OUT = K::OUT, TAPS = K::TAPS, A = K::A, NST = K::NST;
    constexpr bool NV12 = SRC == 1;
    extern __shared__ __align__(128) unsigned char smem_all[];
    const int lane = threadIdx.x, warp = threadIdx.y % kWarps, grp = threadIdx.y / kWarps, tid = warp * 32 + lane;
    unsigned char *tail = smem_all + kGroups * K::GROUP_BYTES;
    const float *s_thr = reinterpret_cast<const float *>(tail + kThrOff);
    unsigned char *smem = smem_all + (size_t)grp * K::GROUP_BYTES;          // this group's stage + ring
    const uint32_t stage0 = smem_u32(smem);
    float *ring = reinterpret_cast<float *>(smem + kStageBytes);
    const uint32_t bar0 = smem_u32(tail + kBarOff) + 16u * (uint32_t)grp;
    // every source of the launch has the range FULL: the luma table is the block's
    constexpr float nk16 = FULL ? 0.0f : -K16, rcp_y = FULL ? 1.0f : RCP_Y, rcp_c = FULL ? 1.0f : RCP_C;
    constexpr YuvCoef kc = yuv_coef(MAT);
    const uint32_t kaddr = setup_block<kGroups>(tail, [&] { fill_luma_table(tail, nk16, rcp_y); });
    const uint32_t ybase = luma_base(tail);
    const int vb = blockIdx.x * kGroups + grp;         // the host cut the launch for SMs x 3 eight-warp blocks
    if (vb >= n_virtual_blocks) return;

    Stash<It> *stash = stash_slots<It, kGroups>(tail, grp);
    uint32_t phase = 0;         // bit 0: parity of the chunks that carried a TMA load so far (mbarrier parity); bit 1: of the steps
    It it;
    it.init(jobs, pieces, __ldg(piece_begin + vb), __ldg(piece_begin + vb + 1));

    Chunk cur = it.next();
    if (!cur.valid) return;
    if (tid == 0) issue<NV12, 1>(jobs, cur, stage0, bar0);

    while (cur.valid) {
        Stash<It> *const parked = stash + (phase >> 1);
        {
            const Chunk nxt = it.next();
            if (tid == 0) { parked->it = it; parked->nxt = nxt; }
        }
        const bool cur_tma = cur.nrows > 0;
        const FusedJob &J = jobs[cur.job];
        const int W = J.src.width, H = J.src.height, chei = H >> 1;
        const uint32_t sb = stage0;
        if (cur_tma) {
            mbar_wait(bar0, phase & 1u);
            replicate_edges<NV12>(smem, cur.x0, cur.nrows, W, tid, grp);
            LaneWords<NV12> lw(cur.x0, lane);
            lw.c_off = held(lw.c_off);
            // ---- phase A: one source row per warp step ------------------------------------------------------------
            // A warp's rows r are kWarps apart, so what the loop needs of a row is carried, not recomputed: the row's stage
            // addresses (fetch_row) advance by a constant -- the parity of r, hence which neighbour is the light chroma
            // row, stays -- and so does its ring slot, which wraps by a subtraction.  The row's luma address la counts the
            // rows.  The light chroma row's clamp to the image can bite in one row only, the image's first (even r) or
            // last (odd r), and makes it the heavy row there; la_clamp is that row's la (no row's, if it is not one of
            // this warp's rows of the chunk: the rows' la are whole steps of kWarps * kLumaBox from the first).
            constexpr int CBOX = NV12 ? kNv12Box : kPlanarBox;
            const int r_first = cur.r0 + warp;
            uint32_t la = sb + (uint32_t)(warp * kLumaBox) + lw.l_off;
            const uint32_t la_end = sb + (uint32_t)(cur.nrows * kLumaBox) + lw.l_off;
            const uint32_t la_clamp = la + (uint32_t)((((r_first & 1) ? 2 * chei - 1 : 0) - r_first) * kLumaBox);
            uint32_t bh = sb + kLumaBytes + (uint32_t)(((r_first >> 1) - (cur.r0 >> 1) + 1) * CBOX) + lw.c_off;
            const uint32_t dlight = held((r_first & 1) ? (uint32_t)CBOX : (uint32_t)-CBOX);
            uint32_t slot_off = (uint32_t)(r_first % K::RROWS) * K::RROW_BYTES;
            for (; la < la_end; la += kWarps * kLumaBox, bh += (kWarps / 2) * CBOX) {
                uint32_t yw[2], v[6];
                fetch_luma<NV12>(la, lw, yw);
                fetch_chroma<NV12>(bh, la == la_clamp ? bh : bh + dlight, lw, v);
                // A1: K1/K2 -> u8 -> sRGB decode, two pixels per instruction, luma from the luma table
                float2 prg[P];   // (r, g) of pixel i
                float pb[P];     // b of pixel i
                convert_run<true>(yw, v, nk16, rcp_y, rcp_c, kc, kaddr, prg, pb, ybase);
                // A2: horizontal Lanczos along the warp.  acc j of the lane that owns tap 0 of output OUT * lane + j.
                // The weights are compile-time constants (int_weights.h): every FFMA takes its weight as an immediate.
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
                            if (t >= 0 && t < K::TAPS_NZ) {
                                arg[j] = fma2(prg[i], splat(int_weight<S>(t)), arg[j]);
                                ab[j] = __fmaf_rn(pb[i], int_weight<S>(t), ab[j]);
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
                    constexpr float inv = int_inv<S>();
                    float *dst = reinterpret_cast<float *>(reinterpret_cast<unsigned char *>(ring) + slot_off) + lane * 3 * OUT;
                    slot_off += kWarps * K::RROW_BYTES;
                    slot_off = min(slot_off, slot_off - (uint32_t)K::RING_BYTES);   // unsigned: the difference is huge unless it wrapped
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
            phase ^= 1u;
        }
        // every warp has read its rows of the stage (and, for a last chunk, stored them in the ring): the next chunk's
        // loads refill the stage while the vertical pass runs
        group_sync(grp);
        if (tid == 0) issue<NV12, 1>(jobs, parked->nxt, stage0, bar0);
        if (cur.last) {
            // ---- phase B: vertical pass ------------------------------------------------------------------------------
            const int tv = J.taps_v;
            const float *lbase = ring + lane * 3 * OUT;
            constexpr int ROWF = K::RROW_BYTES / 4;
            const int row_end = min(cur.o0 + kWarps, cur.oy_end);
            auto col_of = [&](int j) { return OUT * (lane - K::last_stage(j)) + j; };   // strip column of this lane's slot j
            // direct tiles (FusedJob.direct_map): rows oa, oa + 1 are final rows of the output frame -- K10 / K11 of this lane's
            // 2 x 2 blocks from the encoded bytes still in registers; frame position and sizes are even (host)
            // does this lane's 2 x 2 block (columns j, j + 1 of rows oa, oa + 1) lie in a direct tile of this job?  Asked BEFORE the
            // tap loop: the map byte is a global load, and the vertical pass is the latency-bound leg of the step
            auto owned = [&](int oa, bool (&own)[OUT / 2]) {
                const int ncols = min(K::NOUT, J.dst_w - cur.ox0);
#pragma unroll
                for (int j = 0; j < OUT; j += 2) {
                    const int col = col_of(j);
                    own[j / 2] = false;
                    if (J.direct_map == nullptr || col < 0 || col >= ncols || oa >= row_end) continue;
                    const int X = J.fx + cur.ox0 + col, Y = J.fy + oa;
                    own[j / 2] = (int)__ldg(J.direct_map + (Y / kDirectTileH) * J.map_w + X / kDirectTileW) == J.direct_id;
                }
            };
            auto emit = [&](const uint32_t (&pa)[OUT], const uint32_t (&pb)[OUT], int oa, const bool (&own)[OUT / 2]) {
#pragma unroll
                for (int j = 0; j < OUT; j += 2) {
                    if (!own[j / 2]) continue;
                    emit_yuv_2x2(J, J.fx + cur.ox0 + col_of(j), J.fy + oa, pa[j], pa[j + 1], pb[j], pb[j + 1]);
                }
            };
            // one output row the general way: weights from global memory, tap rows clamped to the image
            auto one_row = [&](int oy, uint32_t (&px)[OUT]) {
                const int fv = __ldg(J.first_v + oy);
                const float *wv = J.w_v + (size_t)oy * tv;
                float2 acc[3 * OUT / 2];
#pragma unroll
                for (int k = 0; k < 3 * OUT / 2; k++) acc[k] = make_float2(0.f, 0.f);
                for (int t = 0; t < tv; t++) {
                    const float wt = __ldg(wv + t);
                    const int row = min(max(fv + t, 0), H - 1);
                    const float *p = lbase + (row % K::RROWS) * ROWF;
#pragma unroll
                    for (int k = 0; k < 3 * OUT / 2; k++) acc[k] = fma2(*reinterpret_cast<const float2 *>(p + 2 * k), splat(wt), acc[k]);
                }
                encode_store<OUT>(J, acc, oy, s_thr, cur.ox0, K::NOUT, col_of, px);
            };
            if (J.v_same) {
                // same integer ratio vertically: rows o and o + 1 share TAPS_NZ - S of their TAPS_NZ ring rows (the zero tap
                // is skipped: Cfg::TAPS_NZ).  Four warps (one per scheduler) take two output rows each: every ring row is
                // loaded once for both, the weights are the compile-time row of int_weights.h, the loop unrolls; the ring
                // wraps at most once inside the window.
                if (warp < kWarps / 2) {
                    const int oa = cur.o0 + 2 * warp, ob = oa + 1;
                    const int fa = __ldg(J.first_v) + S * oa;               // first_v(oa); first_v(ob) = fa + S
                    bool own[OUT / 2];
                    owned(oa, own);
                    if (ob < row_end && fa >= 0 && fa + S + TAPS - 1 <= H - 1) {
                        float2 aa[3 * OUT / 2], bb2[3 * OUT / 2];
#pragma unroll
                        for (int k = 0; k < 3 * OUT / 2; k++) { aa[k] = make_float2(0.f, 0.f); bb2[k] = make_float2(0.f, 0.f); }
                        const int slot0 = fa % K::RROWS, nwrap = K::RROWS - slot0;
                        const float *p0 = lbase + slot0 * ROWF;
#pragma unroll
                        for (int u = 0; u < K::TAPS_NZ + S; u++) {
                            const float *p = p0 + (u >= nwrap ? (u - K::RROWS) * ROWF : u * ROWF);
                            float2 v[3 * OUT / 2];
#pragma unroll
                            for (int k = 0; k < 3 * OUT / 2; k++) v[k] = *reinterpret_cast<const float2 *>(p + 2 * k);
                            if (u < K::TAPS_NZ) {
#pragma unroll
                                for (int k = 0; k < 3 * OUT / 2; k++) aa[k] = fma2(v[k], splat(int_weight<S>(u < K::TAPS_NZ ? u : 0)), aa[k]);
                            }
                            if (u >= S) {
#pragma unroll
                                for (int k = 0; k < 3 * OUT / 2; k++) bb2[k] = fma2(v[k], splat(int_weight<S>(u >= S ? u - S : 0)), bb2[k]);
                            }
                        }
                        uint32_t pa[OUT], pb[OUT];
                        encode_store<OUT>(J, aa, oa, s_thr, cur.ox0, K::NOUT, col_of, pa);
                        encode_store<OUT>(J, bb2, ob, s_thr, cur.ox0, K::NOUT, col_of, pb);
                        emit(pa, pb, oa, own);
                    } else {
                        uint32_t pa[OUT], pb[OUT];
                        if (oa < row_end) one_row(oa, pa);
                        if (ob < row_end) { one_row(ob, pb); emit(pa, pb, oa, own); }   // pieces of a direct job hold whole row pairs
                    }
                }
            } else {
                const int oy = cur.o0 + warp;
                uint32_t pz[OUT];
                if (oy < row_end) one_row(oy, pz);   // no direct output without the integer vertical ratio (host)
            }
            group_sync(grp);   // the ring rows this pass read may be overwritten by the next step's horizontal pass
        }
        cur = parked->nxt; it = parked->it; phase ^= 2u;   // written before this step's group_sync
    }
}

}  // namespace tma_int
