// resample_tma0.cuh -- the ANY-RATIO (<= 4:1 per axis) form of the TMA-staged fused resample (included by kernels.cu after
// resample_tma.cuh, which holds the front end: TMA tiles, edges, K1/K2, decode, encode).
//
// K1/K2 + K8 + K8 for mappings whose horizontal ratio is not 2 or 4 with zero offset: fractional ratios (grids with
// margins, transitions), ratio 3, crops.  The horizontal pass cannot be systolic here -- every output column has its own
// weights and window -- so each warp parks the decoded row in a shared-memory row buffer and every lane runs the union
// window of its two adjacent output columns out of it, one LDS.128 per source pixel feeding six FFMA, with the
// lane's weights held in registers for the whole strip (54 of the 128 registers of this kernel: two 8-warp groups per
// SM).  Strips are at most 64 columns and are narrowed by the host so that a strip's source span fits the 256 pixels
// a warp converts per row.  The vertical pass is the general one (per-row weights from global memory).
#pragma once

namespace tma_any {
using namespace tma;

constexpr int kGroups = 2;                            // independent 8-warp groups per block (one block per SM, 128 registers)

struct Cfg {
    static constexpr int P = 8;                      // source pixels per lane and row
    static constexpr int COLS = 64;                  // at most: the host narrows a job's strips so that its span fits 256 px
    static constexpr int MAXT = 25;                  // taps of a 4:1 pass
    static constexpr int WIN = MAXT + 4;             // union of the windows of a lane's two columns
    static constexpr int RROWS = 54;                 // ring rows >= taps_v + ceil(7 * scale_v) + 1
    static constexpr int RROW_BYTES = 32 * 3 * 2 * 4;
    static constexpr int RING_BYTES = RROWS * RROW_BYTES;
    // row buffer: pixel p of the strip's span sits in 16-byte slot p + p / 8 -- one pad slot after every lane's 8 pixels, so
    // that the 8 lanes of a quarter-warp storing pixel i of their runs hit 8 different bank groups (a stride of 128 bytes
    // would be an 8-way conflict).  Pad slots and the tail hold zeros for ever; a lane's window walks SLOTS, with weight 0
    // on the pads.
    static constexpr int WINP_MAX = WIN + 4;         // slots a window of WIN pixels can span (it crosses at most 4 pads)
    static constexpr int ROWBUF_PX = 320;            // 288 slots of the 256 converted pixels + the zero tail
    static constexpr int ROWBUF_BYTES = ROWBUF_PX * 16;   // (r, g, b, b) per pixel: one LDS.128 per tap
    static constexpr int GROUP_BYTES = kStageBytes + RING_BYTES + kWarps * ROWBUF_BYTES;
    static constexpr int SMEM = kGroups * GROUP_BYTES + kTailBytes;
};

// WINP: slots of a lane's window the tap loop walks (host: >= taps + widest distance of two adjacent columns + pads)
// BOX: the source is box-reduced 2:1 on both axes first (downsample.wgsl:28-41, one pre-decimation level of resampler.rs:56-67):
// the two source rows of a reduced row are converted back to back, summed in the shader's order, quantised to f16
// MAT: the matrix (Tex::matrix) of every source of the launch (the host keys the launches by it); the range is read per job
template <int SRC, int WINP, int BOX, int MAT>
__global__ void __launch_bounds__(32 * kWarps * kGroups, 1) k_resample_tma0(const FusedJob *jobs, const FusedPiece *pieces, const int *piece_begin,
                                                                            int n_virtual_blocks) {
    using K = Cfg;
    constexpr int P = K::P, OUT = 2;
    constexpr bool NV12 = SRC == 1;
    constexpr int BX = BOX ? 2 : 1;
    using It = ChunkIter<0, BX>;
    extern __shared__ __align__(128) unsigned char smem_all[];
    const int lane = threadIdx.x, warp = threadIdx.y % kWarps, grp = threadIdx.y / kWarps, tid = warp * 32 + lane;
    unsigned char *tail = smem_all + kGroups * K::GROUP_BYTES;
    const float *s_thr = reinterpret_cast<const float *>(tail + kThrOff);
    unsigned char *smem = smem_all + (size_t)grp * K::GROUP_BYTES;          // this group's stage, ring and row buffers
    const uint32_t stage0 = smem_u32(smem);
    float *ring = reinterpret_cast<float *>(smem + kStageBytes);
    float4 *rowbuf = reinterpret_cast<float4 *>(smem + kStageBytes + K::RING_BYTES) + (size_t)warp * K::ROWBUF_PX;
    const uint32_t bar0 = smem_u32(tail + kBarOff) + 16u * (uint32_t)grp;
    const uint32_t kaddr = setup_block<kGroups>(tail, [&] {
        for (int i = lane; i < K::ROWBUF_PX; i += 32) rowbuf[i] = make_float4(0.f, 0.f, 0.f, 0.f);   // pads and tail: never written again
    });
    const int vb = blockIdx.x * kGroups + grp;         // the host cut the launch for SMs x 2 eight-warp blocks
    if (vb >= n_virtual_blocks) return;

    Stash<It> *stash = stash_slots<It, kGroups>(tail, grp);
    uint32_t step = 0;
    It it;
    it.init(jobs, pieces, __ldg(piece_begin + vb), __ldg(piece_begin + vb + 1));

    static_assert(WINP <= K::WINP_MAX, "window");
    unsigned long long wq[WINP];      // registers (every index is a compile-time constant after unrolling): (weight of column 2 lane,
                            // weight of column 2 lane + 1) for source pixel j of the lane's union window
    float inv0 = 0.f, inv1 = 0.f;
    int rel0 = 0, w_job = -1, w_ox0 = -1;
    int pl = lane;               // the pair of columns this lane owns in the current strip (J.lane_perm)

    Chunk cur = it.next();
    if (!cur.valid) return;
    if (tid == 0) issue<NV12, BX>(jobs, cur, stage0, bar0);
    uint32_t nchunk = 0;        // chunks that carried a TMA load so far (mbarrier parity)

    while (cur.valid) {
        Stash<It> *const parked = stash + (step & 1u);
        {
            const Chunk nxt = it.next();
            if (tid == 0) { parked->it = it; parked->nxt = nxt; }
        }
        const bool cur_tma = cur.nrows > 0;
        const FusedJob &J = jobs[cur.job];
        const int W = J.src.width, H = J.src.height, chei = H >> 1, HR = H / BX;
        const bool full_range = J.src.full_range != 0;
        const float nk16 = full_range ? 0.0f : -K16, rcp_y = full_range ? 1.0f : RCP_Y, rcp_c = full_range ? 1.0f : RCP_C;
        const uint32_t sb = stage0;
        if (cur.job != w_job || cur.ox0 != w_ox0) {   // a new strip: this lane's two columns, their weights and window
            w_job = cur.job; w_ox0 = cur.ox0;
            const int th = J.taps_h;
            // which pair: the host deals the strip's 32 pairs to lanes so that the 8 lanes of a quarter-warp start their
            // windows in 8 different 16-byte bank groups wherever the geometry allows (the LDS.128 of a tap is then one
            // wavefront per quarter instead of two or three)
            pl = J.lane_perm ? (int)__ldg(J.lane_perm + (size_t)(cur.ox0 / J.strip_cols) * 32 + lane) : lane;
            const int oc0 = min(cur.ox0 + 2 * pl, J.dst_w - 1), oc1 = min(cur.ox0 + 2 * pl + 1, J.dst_w - 1);
            const int f0 = __ldg(J.first_h + oc0), f1 = __ldg(J.first_h + oc1);
            const int gD = f1 - f0;                       // 0 (clamped duplicate) .. 4
            const int rel = min(max(f0 - cur.x0, 0), 255);   // host: span <= 256
            rel0 = rel + (rel >> 3);                         // first SLOT of the lane's window
            inv0 = __ldg(J.inv_h + oc0); inv1 = __ldg(J.inv_h + oc1);
            {   // the host sized WINP for this job; a window that does not fit would silently lose taps
                const int last = rel + gD + th - 1;
                if (last + (last >> 3) - rel0 >= WINP) __trap();
            }
#pragma unroll
            for (int jj = 0; jj < WINP; jj++) {
                const int slot = rel0 + jj, q = slot / 9;
                const bool pad = slot - 9 * q == 8;
                const int j = slot - q - rel, t = j - gD;     // pixel of the window, tap of the second column
                wq[jj] = pk(make_float2((!pad && j < th) ? __ldg(J.w_h + (size_t)oc0 * th + j) : 0.0f,
                                        (!pad && t >= 0 && t < th) ? __ldg(J.w_h + (size_t)oc1 * th + t) : 0.0f));
            }
        }
        if (cur_tma) {
            mbar_wait(bar0, nchunk & 1u);
            const int x0 = cur.x0 * BX, sr0 = cur.r0 * BX;   // source pixel / row of the tile's origin
            replicate_edges<NV12>(smem, x0, cur.nrows * BX, W, tid, grp);
            const LaneWords<NV12> lw(x0, lane);
            // ---- phase A: one (reduced) row per warp step ---------------------------------------------------------
            for (int R = cur.r0 + warp; R < cur.r0 + cur.nrows; R += kWarps) {
                float2 prg[P];   // (r, g) of pixel i of the row handed to the horizontal pass (BOX: the first P / 2)
                float pb[P];     // b of pixel i
                float2 hrg[P / 2];   // BOX: (t00 + t01) of the 2 x 2 block, kept while the block's second row is converted
                float hb[P / 2];
#pragma unroll
                for (int k = 0; k < BX; k++) {
                    uint32_t yw[2], v[6];
                    fetch_row<NV12>(sb, lw, R * BX + k, sr0, chei, yw, v);
                    // A1: K1/K2 -> u8 -> sRGB decode, two pixels per instruction
                    float2 crg[P];   // (r, g) of source pixel i of this row
                    float cb[P];     // b
                    convert_run(yw, v, nk16, rcp_y, rcp_c, yuv_coef(MAT), kaddr, crg, cb);
                    if (!BOX) {
#pragma unroll
                        for (int i = 0; i < P; i++) { prg[i] = crg[i]; pb[i] = cb[i]; }
                    } else if (k == 0) {
#pragma unroll
                        for (int i = 0; i < P / 2; i++) { hrg[i] = add2(crg[2 * i], crg[2 * i + 1]); hb[i] = cb[2 * i] + cb[2 * i + 1]; }
                    } else {
                        // downsample.wgsl:28-41: sum in the order (0,0) (1,0) (0,1) (1,1), / 4, stored in the Rgba16Float reduced texture
#pragma unroll
                        for (int i = 0; i < P / 2; i++) {
                            const float2 srg = add2(add2(hrg[i], crg[2 * i]), crg[2 * i + 1]);
                            const float sb4 = (hb[i] + cb[2 * i]) + cb[2 * i + 1];
                            prg[i] = __half22float2(__floats2half2_rn(srg.x * 0.25f, srg.y * 0.25f));
                            pb[i] = __half2float(__float2half_rn(sb4 * 0.25f));
                        }
                    }
                }   // k: the source rows of R
                // park the pixels in this warp's row buffer: pixel X0 + n at slot n + n / 8 (n = 8 lane + i, BOX: 4 lane + i)
                if (!BOX) {
#pragma unroll
                    for (int i = 0; i < P; i++) rowbuf[lane * (P + 1) + i] = make_float4(prg[i].x, prg[i].y, pb[i], pb[i]);
                } else {
                    float4 *mine = rowbuf + 4 * lane + (lane >> 1);
#pragma unroll
                    for (int i = 0; i < P / 2; i++) mine[i] = make_float4(prg[i].x, prg[i].y, pb[i], pb[i]);
                    // The Lanczos pass clamps its taps to the REDUCED texture: a pixel outside it is the nearest reduced pixel
                    // (the replicate padding of the staged source tile stands for source pixels, not for their 2 x 2 means)
                    const int RW = W / 2;
                    if (cur.x0 < 0 || cur.x0 + 128 > RW) {
                        __syncwarp();
                        float4 fix[P / 2];
#pragma unroll
                        for (int i = 0; i < P / 2; i++) {
                            const int n = min(max(cur.x0 + 4 * lane + i, 0), RW - 1) - cur.x0;
                            fix[i] = rowbuf[n + (n >> 3)];
                        }
                        __syncwarp();
#pragma unroll
                        for (int i = 0; i < P / 2; i++) mine[i] = fix[i];
                    }
                }
                __syncwarp();
                // A2: horizontal Lanczos, two adjacent output columns per lane.  The lane's weights live in registers for
                // the whole piece: wq[j] = (weight of column 2 lane, weight of column 2 lane + 1 shifted by the distance of the
                // two windows), zeros outside -- one LDS.128 per source pixel (r, g, b, b) of the union window feeds four FFMA
                // and one FMA pair (the weight pair is the packed operand as it stands; a splat pair per weight would not fit the
                // register file); the nonzero taps of a column are taken in the shader's order t = 0 .. taps-1, a zero tap
                // leaves the sum alone
                {
                    float r0 = 0.f, r1 = 0.f, g0 = 0.f, g1 = 0.f;
                    unsigned long long abq = 0ull;
                    const uint32_t wa = smem_u32(rowbuf + rel0);
                    // three loads in flight: a tap's LDS.128 is issued three taps ahead of its five FMAs
                    constexpr int DEPTH = 3;
                    unsigned long long brg[DEPTH], bbb[DEPTH];
#pragma unroll
                    for (int j = 0; j < DEPTH; j++) lds128q(wa + 16u * j, brg[j], bbb[j]);
#pragma unroll
                    for (int j = 0; j < WINP; j++) {
                        const float2 rg = upk(brg[j % DEPTH]);   // (r, g) | (b, b); a pad / tail slot holds zeros under weight 0
                        const unsigned long long bb = bbb[j % DEPTH];
                        const float2 w = upk(wq[j]);
                        r0 = fmaf(rg.x, w.x, r0); r1 = fmaf(rg.x, w.y, r1);
                        g0 = fmaf(rg.y, w.x, g0); g1 = fmaf(rg.y, w.y, g1);
                        abq = fma2q(bb, wq[j], abq);
                        if (j + DEPTH < WINP) lds128q(wa + 16u * (j + DEPTH), brg[j % DEPTH], bbb[j % DEPTH]);
                    }
                    const float2 a0 = make_float2(r0, g0), a1 = make_float2(r1, g1), ab = upk(abq);
                    // normalise, quantise to f16 (NC-5) and park the row in the ring: [row][lane][channel][column]
                    float *dst = ring + (size_t)(R % K::RROWS) * (K::RROW_BYTES / 4) + lane * 6;
                    *reinterpret_cast<float2 *>(dst) = __half22float2(__floats2half2_rn(a0.x * inv0, a1.x * inv1));
                    *reinterpret_cast<float2 *>(dst + 2) = __half22float2(__floats2half2_rn(a0.y * inv0, a1.y * inv1));
                    *reinterpret_cast<float2 *>(dst + 4) = __half22float2(__floats2half2_rn(ab.x * inv0, ab.y * inv1));
                }
                __syncwarp();   // the row buffer is rewritten by the warp's next row
            }
            nchunk++;
        }
        // every warp has read its rows of the stage (and, for a last chunk, stored them in the ring): the next chunk's
        // loads refill the stage while the vertical pass runs
        group_sync(grp);
        if (tid == 0) issue<NV12, BX>(jobs, parked->nxt, stage0, bar0);
        if (cur.last) {
            // ---- phase B: vertical pass, one output row per warp ------------------------------------------------------
            // lane t fetches tap t's weight (one coalesced load per row), the tap loop takes it by shuffle; away from the
            // top / bottom image edge the ring slot of tap t is (first + t) mod RROWS, stepped, not divided
            const int tv = J.taps_v;
            const float *lbase = ring + lane * 6;
            constexpr int ROWF = K::RROW_BYTES / 4;
            const int oy = cur.o0 + warp;
            if (oy < min(cur.o0 + kWarps, cur.oy_end)) {
                const int fv = __ldg(J.first_v + oy);
                const float wl = lane < tv ? __ldg(J.w_v + (size_t)oy * tv + lane) : 0.0f;
                float2 acc[3 * OUT / 2];
#pragma unroll
                for (int k = 0; k < 3 * OUT / 2; k++) acc[k] = make_float2(0.f, 0.f);
                if (fv >= 0 && fv + tv <= HR) {
                    int slot = fv % K::RROWS;
#pragma unroll
                    for (int t = 0; t < K::MAXT; t++) {
                        if (t >= tv) break;
                        const float wt = __shfl_sync(0xffffffffu, wl, t);
                        const float *p = lbase + slot * ROWF;
#pragma unroll
                        for (int k = 0; k < 3 * OUT / 2; k++) acc[k] = fma2(*reinterpret_cast<const float2 *>(p + 2 * k), splat(wt), acc[k]);
                        slot = slot + 1 == K::RROWS ? 0 : slot + 1;
                    }
                } else {
                    for (int t = 0; t < tv; t++) {   // tap rows clamped to the image (resample.wgsl)
                        const float wt = __shfl_sync(0xffffffffu, wl, t);
                        const int row = min(max(fv + t, 0), HR - 1);
                        const float *p = lbase + (row % K::RROWS) * ROWF;
#pragma unroll
                        for (int k = 0; k < 3 * OUT / 2; k++) acc[k] = fma2(*reinterpret_cast<const float2 *>(p + 2 * k), splat(wt), acc[k]);
                    }
                }
                uint32_t px[OUT];
                encode_store<OUT>(J, acc, oy, s_thr, cur.ox0, J.strip_cols, [&](int) { return 2 * pl; }, px);
            }
            group_sync(grp);   // the ring rows this pass read may be overwritten by the next step's horizontal pass
        }
        cur = parked->nxt; it = parked->it; step++;   // written before this step's group_sync
    }
}

}  // namespace tma_any
