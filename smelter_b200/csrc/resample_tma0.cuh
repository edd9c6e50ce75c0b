// resample_tma0.cuh -- the ANY-RATIO (<= 4:1 per axis) form of the TMA-staged fused resample (included by kernels.cu).
//
// K1/K2 + K8 + K8 for mappings whose horizontal ratio is not 2 or 4 with zero offset: fractional ratios (grids with
// margins, transitions), ratio 3, crops.  Everything up to the decoded pixels is k_resample_tma3 (TMA tiles, packed FP32
// K1/K2, lane-replicated decode table); the horizontal pass cannot be systolic here -- every output column has its own
// weights and window -- so each warp parks the decoded row in a shared-memory row buffer and every lane runs the union
// window of its two adjacent output columns out of it, one LDS.128 per source pixel feeding six FFMA, with the
// lane's weights held in registers for the whole strip (54 of the 128 registers of this kernel: two 8-warp groups per
// SM).  Strips are at most 64 columns and are narrowed by the host so that a strip's source span fits the 256 pixels
// a warp converts per row.  The vertical pass is the general one (per-row weights from global memory).
#pragma once

namespace v7 {


constexpr int kWarps = 8;
constexpr int kGroups = 2;                            // independent 8-warp groups per block (one block per SM, 128 registers)
constexpr int kChunkRows = 32;                       // source rows per TMA chunk: one 8-output-row step of a 4:1 pass
// box widths in BYTES: 256 pixels + up to 14 bytes of alignment slack (luma); 6 chroma texels per lane + slack
constexpr int kLumaBox = 272, kNv12Box = 288, kPlanarBox = 160, kChromaRows = 18;
constexpr int kLumaBytes = kLumaBox * kChunkRows;                                    
constexpr int kChromaBytesNv12 = ((kNv12Box * kChromaRows + 127) / 128) * 128;      
constexpr int kChromaBytesPlanar = ((kPlanarBox * kChromaRows + 127) / 128) * 128;  
constexpr int kStageBytes = kLumaBytes + 2 * kChromaBytesPlanar;                    
static_assert(kLumaBytes % 128 == 0, "chroma destination alignment");
static_assert(kStageBytes >= kLumaBytes + kChromaBytesNv12, "stage size");
constexpr int kDecRep = 32;                          // decode table: one copy per lane (entry i of lane l in bank l)
constexpr float kMagicRound = 12582912.0f;           // 1.5 * 2^23
constexpr uint32_t kMagicBits = 0x4B400000u;

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
    static constexpr int STASH_BYTES = 1024;         // per group and parity: the chunk iterator + the next chunk, parked during the phases
    static constexpr int SMEM = kGroups * GROUP_BYTES + 256 * kDecRep * 4 + 256 * 4 + 128 + STASH_BYTES;
};

struct Chunk {      // warp-uniform description of one pipeline step
    int valid;      // 0: the block has no more work
    int job, ox0;   // job index, first output column of the strip
    int x0;         // first source pixel of the strip's tile
    int r0, nrows;  // source rows [r0, r0 + nrows) to convert in this step (nrows may be 0)
    int last;       // the group's rows are complete after this chunk: run the vertical pass
    int o0, oy_end; // the group's output rows [o0, min(o0 + 8, oy_end))
};

struct ChunkIter {
    const FusedJob *jobs;
    const FusedPiece *pieces;
    int pi, pend;
    int job, ox0, x0, oy_end, onext, ocur;
    int produced_hi, rnext, rhi;
    int H, tv, fv0;   // of the current piece's job; fv0 = first_v[0] when the vertical mapping is the integer ratio
    int bx;           // 1, or 2 when the kernel box-reduces the source 2:1 on the fly: rows, x0 and H are then in reduced units
    bool in_group, vs;
    __device__ void init(const FusedJob *j, const FusedPiece *p, int b, int e, int box) {
        bx = box;
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
                const FusedJob &J = jobs[P.job];
                job = P.job; ox0 = P.strip * J.strip_cols; onext = P.oy_begin; oy_end = P.oy_end;
                x0 = __ldg(J.first_h + ox0) & ~1;   // chroma-aligned
                H = J.src.height / bx; tv = J.taps_v; vs = J.v_same != 0;
                fv0 = __ldg(J.first_v);
                produced_hi = -0x40000000;
            }
            ocur = onext;
            const int o_l = min(ocur + kWarps - 1, oy_end - 1);
            // same integer ratio vertically: first_v(o) = first_v(0) + S * o (resample.wgsl:45-50 in exact arithmetic), no
            // dependent global loads on the way to the next TMA issue
            const int f_lo = __ldg(jobs[job].first_v + ocur);
            const int f_hi = __ldg(jobs[job].first_v + o_l);
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
        c.nrows = max(0, min(kChunkRows / bx, rhi - rnext + 1));
        rnext += kChunkRows / bx;
        c.last = rnext > rhi;
        return c;
    }
};

// bar.sync on a named barrier: the 8 warps of one group
__device__ __forceinline__ void group_sync(int g) { asm volatile("bar.sync %0, 256;" ::"r"(g + 1) : "memory"); }

// WINP: slots of a lane's window the tap loop walks (host: >= taps + widest distance of two adjacent columns + pads)
// BOX: the source is box-reduced 2:1 on both axes first (downsample.wgsl:28-41, one pre-decimation level of resampler.rs:56-67):
// the two source rows of a reduced row are converted back to back, summed in the shader's order, quantised to f16
template <int SRC, int WINP, int BOX>
__global__ void __launch_bounds__(32 * kWarps * kGroups, 1) k_resample_tma0(const FusedJob *jobs, const FusedPiece *pieces, const int *piece_begin,
                                                                            int n_virtual_blocks) {
    using K = Cfg;
    constexpr int P = K::P, OUT = 2;
    constexpr bool NV12 = SRC == 1;
    constexpr int BX = BOX ? 2 : 1;
    extern __shared__ __align__(128) unsigned char smem_all[];
    const int lane = threadIdx.x, warp = threadIdx.y % kWarps, grp = threadIdx.y / kWarps, tid = warp * 32 + lane;
    float *s_dec = reinterpret_cast<float *>(smem_all + kGroups * K::GROUP_BYTES);
    float *s_thr = s_dec + 256 * kDecRep;
    unsigned char *smem = smem_all + (size_t)grp * K::GROUP_BYTES;          // this group's stages + ring
    const uint32_t stage0 = v5::smem_u32(smem);
    float *ring = reinterpret_cast<float *>(smem + kStageBytes);
    float4 *rowbuf = reinterpret_cast<float4 *>(smem + kStageBytes + K::RING_BYTES) + (size_t)warp * K::ROWBUF_PX;
    const uint32_t bar0 = v5::smem_u32(s_thr + 256) + 16u * (uint32_t)grp;
    volatile uint32_t *s_kaddr = reinterpret_cast<volatile uint32_t *>(reinterpret_cast<unsigned char *>(s_thr + 256) + 64);
    {
        const int btid = threadIdx.y * 32 + lane, bn = 32 * kWarps * kGroups;
        for (int i = btid; i < 256 * kDecRep; i += bn) s_dec[i] = c_dec[i / kDecRep];   // word i * 32 + l: bank l
        for (int i = btid; i < 256; i += bn) s_thr[i] = c_thr[i];
        if (btid == 0) {
            // entry i of lane l = [(float bits of (i + 1.5 * 2^23)) << 7 + kaddr + 4 l]  (mod 2^32); through shared memory so
            // that it stays ONE register and the lookup address ONE LEA
            *s_kaddr = v5::smem_u32(s_dec) - (kMagicBits << 7);
            for (int g = 0; g < kGroups; g++) {
                v5::mbar_init(v5::smem_u32(s_thr + 256) + 16u * (uint32_t)g, 1);
                v5::mbar_init(v5::smem_u32(s_thr + 256) + 16u * (uint32_t)g + 8, 1);
            }
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
    }
    for (int i = lane; i < K::ROWBUF_PX; i += 32) rowbuf[i] = make_float4(0.f, 0.f, 0.f, 0.f);   // pads and tail: never written again
    __syncthreads();
    const uint32_t kaddr = *s_kaddr + 4u * (uint32_t)lane;
    const int vb = blockIdx.x * kGroups + grp;         // the host cut the launch for SMs x 3 eight-warp blocks
    if (vb >= n_virtual_blocks) return;

    // The iterator (20 registers) and the next chunk (9) are not needed while a chunk is being processed: thread 0 of the
    // group parks them in shared memory, everybody reloads them at the end of the step -- the tap loop gets the registers
    struct Stash { ChunkIter it; Chunk nxt; };
    static_assert(sizeof(Stash) * 2 * kGroups <= K::STASH_BYTES, "stash");
    Stash *stash = reinterpret_cast<Stash *>(reinterpret_cast<unsigned char *>(s_thr + 256) + 128) + 2 * grp;
    uint32_t step = 0;
    ChunkIter it;
    it.init(jobs, pieces, __ldg(piece_begin + vb), __ldg(piece_begin + vb + 1), BX);

    auto issue = [&](const Chunk &c) {   // one thread: TMA loads of the chunk's boxes into the group's stage
        if (!c.valid || c.nrows == 0) return;
        const FusedJob &J = jobs[c.job];
        const uint32_t bar = bar0, dst = stage0;
        const int cyb = ((c.r0 * BX) >> 1) - 1;
        const int xt = (c.x0 * BX) & ~15;                         // luma tile: first byte, 16-byte boundary (may be negative)
        if (NV12) {
            const int xc = (c.x0 * BX - 2) & ~15;               // chroma tile: texel cx - 1 of the first pair sits at byte x0 - 2
            v5::mbar_expect_tx(bar, kLumaBox * kChunkRows + kNv12Box * kChromaRows);
            v5::tma_load_2d(dst, J.tm0, xt >> 1, c.r0 * BX, bar);   // both planes are addressed in 2-byte elements
            v5::tma_load_2d(dst + kLumaBytes, J.tm1, xc >> 1, cyb, bar);
        } else {
            const int xc = (((c.x0 * BX) >> 1) - 1) & ~15;
            v5::mbar_expect_tx(bar, kLumaBox * kChunkRows + 2 * kPlanarBox * kChromaRows);
            v5::tma_load_2d(dst, J.tm0, xt >> 1, c.r0 * BX, bar);
            v5::tma_load_2d(dst + kLumaBytes, J.tm1, xc, cyb, bar);
            v5::tma_load_2d(dst + kLumaBytes + kChromaBytesPlanar, J.tm2, xc, cyb, bar);
        }
    };

    static_assert(WINP <= K::WINP_MAX, "window");
    unsigned long long wq[WINP];      // registers (every index is a compile-time constant after unrolling): (weight of column 2 lane,
                            // weight of column 2 lane + 1) for source pixel j of the lane's union window
    float inv0 = 0.f, inv1 = 0.f;
    int rel0 = 0, w_job = -1, w_ox0 = -1;
    int pl = lane;               // the pair of columns this lane owns in the current strip (J.lane_perm)

    Chunk cur = it.next();
    if (!cur.valid) return;
    if (tid == 0) issue(cur);
    uint32_t nchunk = 0;        // chunks that carried a TMA load so far (mbarrier parity)

    while (cur.valid) {
        Stash *const parked = stash + (step & 1u);   // the slot of step k is rewritten in step k + 2: a group_sync lies between
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
                wq[jj] = v5::pk(make_float2((!pad && j < th) ? __ldg(J.w_h + (size_t)oc0 * th + j) : 0.0f,
                                            (!pad && t >= 0 && t < th) ? __ldg(J.w_h + (size_t)oc1 * th + t) : 0.0f));
            }
        }
        if (cur_tma) {
            v5::mbar_wait(bar0, nchunk & 1u);
            // ---- image borders: the tap index is clamped (resample.wgsl), the TMA unit zero-fills ----------------
            const int x0 = cur.x0 * BX, sr0 = cur.r0 * BX;   // source pixel / row of the tile's origin
            const int cyb = (sr0 >> 1) - 1;
            const int xt = x0 & ~15, xc = NV12 ? ((x0 - 2) & ~15) : (((x0 >> 1) - 1) & ~15);
            const int cw = W >> 1;
            if (xt < 0 || xt + kLumaBox > W || xc < 0 || (NV12 ? xc + kNv12Box > W : xc + kPlanarBox > cw)) {
                unsigned char *st = smem;
                const int sub = tid & 7;
                {   // luma: tile byte b <-> pixel xt + b; valid bytes [bl, br)
                    const int bl = min(max(0, -xt), kLumaBox - 1), br = min(max(W - xt, 1), kLumaBox);
                    for (int row = tid >> 3; row < cur.nrows * BX; row += 32) {
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
                v5::fence_proxy_async();
                group_sync(grp);
            }
            // this lane's bytes inside the tiles: word address and the funnel shift that realigns them
            const int dl = x0 - xt, dc = (NV12 ? x0 - 2 : (x0 >> 1) - 1) - xc;
            const uint32_t l_off = (uint32_t)((dl & ~3) + lane * 8), l_sh = (uint32_t)(dl & 3) * 8u;
            const uint32_t c_off = (uint32_t)((dc & ~3) + lane * (NV12 ? 8 : 4)), c_sh = (uint32_t)(dc & 3) * 8u;
            // ---- phase A: one (reduced) row per warp step ---------------------------------------------------------
            for (int R = cur.r0 + warp; R < cur.r0 + cur.nrows; R += kWarps) {
                float2 prg[P];   // (r, g) of pixel i of the row handed to the horizontal pass (BOX: the first P / 2)
                float pb[P];     // b of pixel i
                float2 hrg[P / 2];   // BOX: (t00 + t01) of the 2 x 2 block, kept while the block's second row is converted
                float hb[P / 2];
#pragma unroll
                for (int k = 0; k < BX; k++) {
                const int r = R * BX + k;   // source row
                // raw bytes of this lane's 8 pixels: 12 bytes from a 4-byte aligned address; the half that is 8-byte aligned
                // (warp-uniform) goes as one LDS.64 (lanes 8 bytes apart: conflict-free, an LDS.32 is 2-way)
                uint32_t yw[2];
                {
                    const uint32_t la = sb + (uint32_t)((r - sr0) * kLumaBox) + l_off;
                    uint32_t w0, w1, w2;
                    if (l_off & 4u) { w0 = v5::lds32v(la); v5::lds64v(la + 4, w1, w2); }
                    else { v5::lds64v(la, w0, w1); w2 = v5::lds32v(la + 8); }
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
                        h0 = v5::lds32v(bh); v5::lds64v(bh + 4, h1, h2); h3 = v5::lds32v(bh + 12);
                        l0 = v5::lds32v(bl); v5::lds64v(bl + 4, l1, l2); l3 = v5::lds32v(bl + 12);
                    } else {
                        v5::lds64v(bh, h0, h1); v5::lds64v(bh + 8, h2, h3);
                        v5::lds64v(bl, l0, l1); v5::lds64v(bl + 8, l2, l3);
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
                        const uint32_t w0 = v5::lds32v(a), w1 = v5::lds32v(a + 4), w2 = v5::lds32v(a + 8);
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
                float2 crg[P];   // (r, g) of source pixel i of this row
                float cb[P];     // b
#pragma unroll
                for (int p = 0; p < P / 2; p++) {
                    // 16 x chroma of the even / odd pixel of the pair (NC-6u with the .25 / .75 taps)
                    const uint32_t ne = v[p] + 3u * v[p + 1], no = 3u * v[p + 1] + v[p + 2];
                    const float m23 = -8388608.0f;
                    float2 nu = v5::add2(make_float2(__uint_as_float(__byte_perm(ne, 0x4B000000u, 0x7610)),
                                                 __uint_as_float(__byte_perm(no, 0x4B000000u, 0x7610))), v5::splat(m23));
                    float2 nv = v5::add2(make_float2(__uint_as_float(__byte_perm(ne, 0x4B000000u, 0x7632)),
                                                 __uint_as_float(__byte_perm(no, 0x4B000000u, 0x7632))), v5::splat(m23));
                    const uint32_t ywd = yw[p >> 1];
                    float2 ny = v5::add2(make_float2(__uint_as_float(__byte_perm(ywd, 0x4B000000u, (p & 1) ? 0x7642 : 0x7640)),
                                                 __uint_as_float(__byte_perm(ywd, 0x4B000000u, (p & 1) ? 0x7643 : 0x7641))), v5::splat(m23));
                    // exact n / 255 and n / (255 * 16): fma(n, c, n * lo)
                    const float c1 = __uint_as_float(0x3b808081u), lo1 = __uint_as_float(0xaf7efeffu);
                    const float c16 = __uint_as_float(0x39808081u), lo16 = __uint_as_float(0xad7efeffu);
                    float2 y = v5::fma2(ny, v5::splat(c1), v5::mul2(ny, v5::splat(lo1)));
                    float2 u = v5::fma2(nu, v5::splat(c16), v5::mul2(nu, v5::splat(lo16)));
                    float2 w = v5::fma2(nv, v5::splat(c16), v5::mul2(nv, v5::splat(lo16)));
                    // limited range: clamp01((x - 16/255) * rcp); full range: (x - 0) * 1 and the clamp are identities on [0, 1]
                    y = v5::add2(y, v5::splat(nk16)); u = v5::add2(u, v5::splat(nk16)); w = v5::add2(w, v5::splat(nk16));
                    y = make_float2(__saturatef(y.x * rcp_y), __saturatef(y.y * rcp_y));
                    u = make_float2(__saturatef(u.x * rcp_c), __saturatef(u.y * rcp_c));
                    w = make_float2(__saturatef(w.x * rcp_c), __saturatef(w.y * rcp_c));
                    const float2 um = v5::add2(u, v5::splat(-0.5f)), vm = v5::add2(w, v5::splat(-0.5f));
                    // clamp01 (NC-2) as the .SAT of the matrix row's last fma: the table has exactly the 256 entries
                    const float2 gi = v5::fma2(v5::splat(-0.1873f), um, y);
                    const float2 rr = make_float2(__saturatef(fmaf(1.5748f, vm.x, y.x)), __saturatef(fmaf(1.5748f, vm.y, y.y)));
                    const float2 gg = make_float2(__saturatef(fmaf(-0.4681f, vm.x, gi.x)), __saturatef(fmaf(-0.4681f, vm.y, gi.y)));
                    const float2 bb = make_float2(__saturatef(fmaf(1.8556f, um.x, y.x)), __saturatef(fmaf(1.8556f, um.y, y.y)));
                    // NC-2 rounding and the sRGB decode of the node-texture fetch (NC-3): lane-private table copy, no bank conflicts
                    const float2 qr = v5::add2_after_mul(v5::mul2(rr, v5::splat(255.0f)), v5::splat(kMagicRound));
                    const float2 qg = v5::add2_after_mul(v5::mul2(gg, v5::splat(255.0f)), v5::splat(kMagicRound));
                    const float2 qb = v5::add2_after_mul(v5::mul2(bb, v5::splat(255.0f)), v5::splat(kMagicRound));
                    crg[2 * p] = make_float2(v5::lds_tab((__float_as_uint(qr.x) << 7) + kaddr), v5::lds_tab((__float_as_uint(qg.x) << 7) + kaddr));
                    crg[2 * p + 1] = make_float2(v5::lds_tab((__float_as_uint(qr.y) << 7) + kaddr), v5::lds_tab((__float_as_uint(qg.y) << 7) + kaddr));
                    cb[2 * p] = v5::lds_tab((__float_as_uint(qb.x) << 7) + kaddr);
                    cb[2 * p + 1] = v5::lds_tab((__float_as_uint(qb.y) << 7) + kaddr);
                }
                if (!BOX) {
#pragma unroll
                    for (int i = 0; i < P; i++) { prg[i] = crg[i]; pb[i] = cb[i]; }
                } else if (k == 0) {
#pragma unroll
                    for (int i = 0; i < P / 2; i++) { hrg[i] = v5::add2(crg[2 * i], crg[2 * i + 1]); hb[i] = cb[2 * i] + cb[2 * i + 1]; }
                } else {
                    // downsample.wgsl:28-41: sum in the order (0,0) (1,0) (0,1) (1,1), / 4, stored in the Rgba16Float reduced texture
#pragma unroll
                    for (int i = 0; i < P / 2; i++) {
                        const float2 srg = v5::add2(v5::add2(hrg[i], crg[2 * i]), crg[2 * i + 1]);
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
                    const uint32_t wa = v5::smem_u32(rowbuf + rel0);
                    // three loads in flight: a tap's LDS.128 is issued three taps ahead of its five FMAs
                    constexpr int DEPTH = 3;
                    unsigned long long brg[DEPTH], bbb[DEPTH];
#pragma unroll
                    for (int j = 0; j < DEPTH; j++) v5::lds128q(wa + 16u * j, brg[j], bbb[j]);
#pragma unroll
                    for (int j = 0; j < WINP; j++) {
                        const float2 rg = v5::upk(brg[j % DEPTH]);   // (r, g) | (b, b); a pad / tail slot holds zeros under weight 0
                        const unsigned long long bb = bbb[j % DEPTH];
                        const float2 w = v5::upk(wq[j]);
                        r0 = fmaf(rg.x, w.x, r0); r1 = fmaf(rg.x, w.y, r1);
                        g0 = fmaf(rg.y, w.x, g0); g1 = fmaf(rg.y, w.y, g1);
                        abq = v5::fma2q(bb, wq[j], abq);
                        if (j + DEPTH < WINP) v5::lds128q(wa + 16u * (j + DEPTH), brg[j % DEPTH], bbb[j % DEPTH]);
                    }
                    const float2 a0 = make_float2(r0, g0), a1 = make_float2(r1, g1), ab = v5::upk(abq);
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
        if (tid == 0) issue(parked->nxt);
        if (cur.last) {
            // ---- phase B: vertical pass ------------------------------------------------------------------------------
            const int tv = J.taps_v;
            const float *lbase = ring + lane * 6;
            constexpr int ROWF = K::RROW_BYTES / 4;
            const int row_end = min(cur.o0 + kWarps, cur.oy_end);
            // one output row: encode (NC-4) and store this lane's OUT columns
            auto finish = [&](const float2 *acc, int oy) {
                const float inv_v = __ldg(J.inv_v + oy);
                uint32_t px[OUT];
#pragma unroll
                for (int j = 0; j < OUT; j++) {
                    const float rv = (j & 1) ? acc[j / 2].y : acc[j / 2].x;
                    const float gv = (j & 1) ? acc[(OUT + j) / 2].y : acc[(OUT + j) / 2].x;
                    const float bv = (j & 1) ? acc[(2 * OUT + j) / 2].y : acc[(2 * OUT + j) / 2].x;
                    auto enc = [&](float lin) -> uint32_t {   // count of thresholds <= x = bucket count + one comparison
                        const float x = clamp01(lin);
                        const int k = max((__float_as_int(x) >> 15) - ENC1_KEY0, 0);
                        const uint32_t e = __ldg(c_enc1 + k);
                        return e + (x >= s_thr[e] ? 1u : 0u);
                    };
                    px[j] = enc(rv * inv_v) | (enc(gv * inv_v) << 8) | (enc(bv * inv_v) << 16) | 0xff000000u;
                }
                uint32_t *drow = reinterpret_cast<uint32_t *>(J.dst + (size_t)oy * J.dst_pitch);
                const int ncols = min(J.strip_cols, J.dst_w - cur.ox0);
                const int col = 2 * pl;
                if (col + 1 < ncols) {
                    *reinterpret_cast<uint2 *>(drow + cur.ox0 + col) = make_uint2(px[0], px[1]);
                } else if (col < ncols) {
                    drow[cur.ox0 + col] = px[0];
                }
            };
            // one output row: lane t fetches tap t's weight (one coalesced load per row), the tap loop takes it by shuffle;
            // away from the top / bottom image edge the ring slot of tap t is (first + t) mod RROWS, stepped, not divided
            auto one_row = [&](int oy) {
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
                        for (int k = 0; k < 3 * OUT / 2; k++) acc[k] = v5::fma2(*reinterpret_cast<const float2 *>(p + 2 * k), v5::splat(wt), acc[k]);
                        slot = slot + 1 == K::RROWS ? 0 : slot + 1;
                    }
                } else {
                    for (int t = 0; t < tv; t++) {   // tap rows clamped to the image (resample.wgsl)
                        const float wt = __shfl_sync(0xffffffffu, wl, t);
                        const int row = min(max(fv + t, 0), HR - 1);
                        const float *p = lbase + (row % K::RROWS) * ROWF;
#pragma unroll
                        for (int k = 0; k < 3 * OUT / 2; k++) acc[k] = v5::fma2(*reinterpret_cast<const float2 *>(p + 2 * k), v5::splat(wt), acc[k]);
                    }
                }
                finish(acc, oy);
            };
            {
                const int oy = cur.o0 + warp;
                if (oy < row_end) one_row(oy);
            }
            group_sync(grp);   // the ring rows this pass read may be overwritten by the next step's horizontal pass
        }
        cur = parked->nxt; it = parked->it; step++;   // written before this step's group_sync
    }
}



}  // namespace v7
