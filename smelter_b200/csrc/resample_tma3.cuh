// resample_tma3.cuh -- k_resample_tma (resample_tma.cuh) re-cut for ONE block per SM (included by kernels.cu).
//
// Same arithmetic and data movement as k_resample_tma; what changes is the use of the SM:
//   * one block of 24 warps per SM, three independent 8-warp groups (named barriers 1..3, own TMA stages, own
//     mbarriers, own ring, own list of pieces -- each group is what a block of k_resample_tma was), so that the
//     sRGB decode table can be shared by all of them and REPLICATED per lane: entry i of lane l sits at word
//     32 i + l, i.e. in bank l, and the 24 data-dependent lookups of a row never conflict (they were 3-way on average,
//     a large share of the shared-memory wavefronts of k_resample_tma).  The table has exactly 256 entries, so
//     the clamp of NC-2 moves back in front of the rounding as the .SAT of the matrix row's last fma;
//   * ONE 32-row TMA stage per group (a whole 8-output-row step of a 4:1 pass): it is refilled right after the
//     horizontal pass has consumed it, i.e. while the vertical pass runs; three groups' stages + rings fit in 227 KB;
//   * the vertical pass of a same-ratio job runs on four warps (one per scheduler) that produce TWO output rows each:
//     consecutive output rows share TAPS - S of their ring rows, every row is loaded once for both.
#pragma once

namespace v6 {

constexpr int kWarps = 8;
constexpr int kGroups = 3;                            // independent 8-warp groups per block (one block per SM)
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
    static constexpr int GROUP_BYTES = kStageBytes + RING_BYTES;   // ONE stage: it is refilled while the vertical pass runs
    static constexpr int STASH_BYTES = 1024;   // per group and parity: the chunk iterator + the next chunk, parked during the phases
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

// bar.sync on a named barrier: the 8 warps of one group
__device__ __forceinline__ void group_sync(int g) { asm volatile("bar.sync %0, 256;" ::"r"(g + 1) : "memory"); }

template <int S, int SRC>
__global__ void __launch_bounds__(32 * kWarps * kGroups, 1) k_resample_tma3(const FusedJob *jobs, const FusedPiece *pieces, const int *piece_begin,
                                                                            int n_virtual_blocks) {
    using K = Cfg<S>;
    constexpr int P = K::P, OUT = K::OUT, TAPS = K::TAPS, A = K::A, NST = K::NST;
    constexpr bool NV12 = SRC == 1;
    extern __shared__ __align__(128) unsigned char smem_all[];
    const int lane = threadIdx.x, warp = threadIdx.y % kWarps, grp = threadIdx.y / kWarps, tid = warp * 32 + lane;
    float *s_dec = reinterpret_cast<float *>(smem_all + kGroups * K::GROUP_BYTES);
    float *s_thr = s_dec + 256 * kDecRep;
    unsigned char *smem = smem_all + (size_t)grp * K::GROUP_BYTES;          // this group's stages + ring
    const uint32_t stage0 = v5::smem_u32(smem);
    float *ring = reinterpret_cast<float *>(smem + kStageBytes);
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
    __syncthreads();
    const uint32_t kaddr = *s_kaddr + 4u * (uint32_t)lane;
    const int vb = blockIdx.x * kGroups + grp;         // the host cut the launch for SMs x 3 eight-warp blocks
    if (vb >= n_virtual_blocks) return;

    // The iterator and the next chunk are not needed while a chunk is being processed: thread 0 of the group parks them in
    // shared memory, everybody reloads them at the end of the step -- some 30 registers less across the phases
    struct Stash { ChunkIter<S> it; Chunk nxt; };
    static_assert(sizeof(Stash) * 2 * kGroups <= K::STASH_BYTES, "stash");
    Stash *stash = reinterpret_cast<Stash *>(reinterpret_cast<unsigned char *>(s_thr + 256) + 128) + 2 * grp;
    uint32_t step = 0;
    ChunkIter<S> it;
    it.init(jobs, pieces, __ldg(piece_begin + vb), __ldg(piece_begin + vb + 1));

    auto issue = [&](const Chunk &c) {   // one thread: TMA loads of the chunk's boxes into the group's stage
        if (!c.valid || c.nrows == 0) return;
        const FusedJob &J = jobs[c.job];
        const uint32_t bar = bar0, dst = stage0;
        const int cyb = (c.r0 >> 1) - 1;
        const int xt = c.x0 & ~15;                         // luma tile: first byte, 16-byte boundary (may be negative)
        if (NV12) {
            const int xc = (c.x0 - 2) & ~15;               // chroma tile: texel cx - 1 of the first pair sits at byte x0 - 2
            v5::mbar_expect_tx(bar, kLumaBox * kChunkRows + kNv12Box * kChromaRows);
            v5::tma_load_2d(dst, J.tm0, xt >> 1, c.r0, bar);   // both planes are addressed in 2-byte elements
            v5::tma_load_2d(dst + kLumaBytes, J.tm1, xc >> 1, cyb, bar);
        } else {
            const int xc = ((c.x0 >> 1) - 1) & ~15;
            v5::mbar_expect_tx(bar, kLumaBox * kChunkRows + 2 * kPlanarBox * kChromaRows);
            v5::tma_load_2d(dst, J.tm0, xt >> 1, c.r0, bar);
            v5::tma_load_2d(dst + kLumaBytes, J.tm1, xc, cyb, bar);
            v5::tma_load_2d(dst + kLumaBytes + kChromaBytesPlanar, J.tm2, xc, cyb, bar);
        }
    };

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
        const int W = J.src.width, H = J.src.height, chei = H >> 1;
        const bool full_range = J.src.full_range != 0;
        const float nk16 = full_range ? 0.0f : -K16, rcp_y = full_range ? 1.0f : RCP_Y, rcp_c = full_range ? 1.0f : RCP_C;
        const uint32_t sb = stage0;
        if (cur_tma) {
            v5::mbar_wait(bar0, nchunk & 1u);
            // ---- image borders: the tap index is clamped (resample.wgsl), the TMA unit zero-fills ----------------
            const int x0 = cur.x0;
            const int cyb = (cur.r0 >> 1) - 1;
            const int xt = x0 & ~15, xc = NV12 ? ((x0 - 2) & ~15) : (((x0 >> 1) - 1) & ~15);
            const int cw = W >> 1;
            if (xt < 0 || xt + kLumaBox > W || xc < 0 || (NV12 ? xc + kNv12Box > W : xc + kPlanarBox > cw)) {
                unsigned char *st = smem;
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
                v5::fence_proxy_async();
                group_sync(grp);
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
                float2 prg[P];   // (r, g) of pixel i
                float pb[P];     // b of pixel i
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
#ifdef SMR_EXP_NO_CONV   // what-if build: no K1/K2 arithmetic (bytes -> float only), no decode
                    prg[2 * p] = make_float2(ny.x, nu.x); prg[2 * p + 1] = make_float2(ny.y, nu.y); pb[2 * p] = nv.x; pb[2 * p + 1] = nv.y;
                    continue;
#endif
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
#ifdef SMR_EXP_NO_DEC    // what-if build: no sRGB decode lookups
                    prg[2 * p] = make_float2(qr.x, qg.x); prg[2 * p + 1] = make_float2(qr.y, qg.y); pb[2 * p] = qb.x; pb[2 * p + 1] = qb.y;
#else
                    prg[2 * p] = make_float2(v5::lds_tab((__float_as_uint(qr.x) << 7) + kaddr), v5::lds_tab((__float_as_uint(qg.x) << 7) + kaddr));
                    prg[2 * p + 1] = make_float2(v5::lds_tab((__float_as_uint(qr.y) << 7) + kaddr), v5::lds_tab((__float_as_uint(qg.y) << 7) + kaddr));
                    pb[2 * p] = v5::lds_tab((__float_as_uint(qb.x) << 7) + kaddr);
                    pb[2 * p + 1] = v5::lds_tab((__float_as_uint(qb.y) << 7) + kaddr);
#endif
                }
                // A2: horizontal Lanczos along the warp.  acc j of the lane that owns tap 0 of output OUT * lane + j
                float2 arg[OUT];          // (r, g)
                float ab[OUT];            // b
#pragma unroll
                for (int j = 0; j < OUT; j++) { arg[j] = make_float2(0.f, 0.f); ab[j] = 0.f; }
#ifdef SMR_EXP_NO_A2     // what-if build: no horizontal taps -- measures the systolic pass
#pragma unroll
                for (int j = 0; j < OUT; j++) {   // every converted pixel stays live, at one add each
                    arg[j] = prg[j]; ab[j] = pb[j];
#pragma unroll
                    for (int i = OUT + j; i < P; i += OUT) { arg[j] = v5::add2(arg[j], prg[i]); ab[j] += pb[i]; }
                }
#else
#pragma unroll
                for (int s = 0; s < NST; s++) {
#pragma unroll
                    for (int i = 0; i < P; i++) {
#pragma unroll
                        for (int j = 0; j < OUT; j++) {
                            const int t = P * s + i - A - S * j;   // compile-time after unrolling
                            if (t >= 0 && t < TAPS) arg[j] = v5::fma2(prg[i], v5::splat(c_wint[S][t]), arg[j]);
                        }
#pragma unroll
                        for (int j = 0; j < OUT; j += 2) {
                            const int t0 = P * s + i - A - S * j, t1 = t0 - S;
                            const bool a0 = t0 >= 0 && t0 < TAPS, a1 = t1 >= 0 && t1 < TAPS;
                            if (a0 && a1) {
                                const float2 d = v5::fma2(v5::splat(pb[i]), c_wpair[S][a0 ? t0 : 0], make_float2(ab[j], ab[j + 1]));
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
#endif
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
        // every warp has read its rows of the stage (and, for a last chunk, stored them in the ring): the next chunk's
        // loads refill the stage while the vertical pass runs
        group_sync(grp);
        if (tid == 0) issue(parked->nxt);
#ifdef SMR_EXP_NO_B      // what-if build (-DSMR_EXP_NO_B): no vertical pass -- measures what phase B costs; output is garbage
        if (false) {
#else
        if (cur.last) {
#endif
            // ---- phase B: vertical pass ------------------------------------------------------------------------------
            const int tv = J.taps_v;
            const float *lbase = ring + lane * 3 * OUT;
            constexpr int ROWF = K::RROW_BYTES / 4;
            const int row_end = min(cur.o0 + kWarps, cur.oy_end);
            // one output row: encode (NC-4) and store this lane's OUT columns
            auto finish = [&](const float2 *acc, int oy, uint32_t *px) {
                const float inv_v = __ldg(J.inv_v + oy);
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
                const int ncols = min(K::NOUT, J.dst_w - cur.ox0);
#pragma unroll
                for (int j = 0; j < OUT; j += 2) {   // slots (j, j + 1) are adjacent columns
                    const int col = OUT * (lane - K::last_stage(j)) + j;   // this lane's slot j holds strip column `col`
                    if (col >= 0 && col + 1 < ncols) {
                        *reinterpret_cast<uint2 *>(drow + cur.ox0 + col) = make_uint2(px[j], px[j + 1]);
                    } else if (col >= 0 && col < ncols) {
                        drow[cur.ox0 + col] = px[j];
                    }
                }
            };
            // direct tiles (FusedJob.direct_map): rows oa, oa + 1 are final rows of the output frame -- K10 / K11 of this lane's
            // 2 x 2 blocks from the encoded bytes still in registers; frame position and sizes are even (host)
            // does this lane's 2 x 2 block (columns j, j + 1 of rows oa, oa + 1) lie in a direct tile of this job?  Asked BEFORE the
            // tap loop: the map byte is a global load, and the vertical pass is the latency-bound leg of the step
            auto owned = [&](int oa, bool *own) {
                const int ncols = min(K::NOUT, J.dst_w - cur.ox0);
#pragma unroll
                for (int j = 0; j < OUT; j += 2) {
                    const int col = OUT * (lane - K::last_stage(j)) + j;
                    own[j / 2] = false;
                    if (J.direct_map == nullptr || col < 0 || col >= ncols || oa >= row_end) continue;
                    const int X = J.fx + cur.ox0 + col, Y = J.fy + oa;
                    own[j / 2] = (int)__ldg(J.direct_map + (Y / kDirectTileH) * J.map_w + X / kDirectTileW) == J.direct_id;
                }
            };
            auto emit = [&](const uint32_t *pa, const uint32_t *pb, int oa, const bool *own) {
#pragma unroll
                for (int j = 0; j < OUT; j += 2) {
                    if (!own[j / 2]) continue;
                    const int col = OUT * (lane - K::last_stage(j)) + j;
                    emit_yuv_2x2(J, J.fx + cur.ox0 + col, J.fy + oa, pa[j], pa[j + 1], pb[j], pb[j + 1]);
                }
            };
            // one output row the general way: weights from global memory, tap rows clamped to the image
            auto one_row = [&](int oy, uint32_t *px) {
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
                    for (int k = 0; k < 3 * OUT / 2; k++) acc[k] = v5::fma2(*reinterpret_cast<const float2 *>(p + 2 * k), v5::splat(wt), acc[k]);
                }
                finish(acc, oy, px);
            };
            if (J.v_same) {
                // same integer ratio vertically: rows o and o + 1 share TAPS - S of their TAPS ring rows.  Four warps (one
                // per scheduler) take two output rows each: every ring row is loaded once for both, the weights are the
                // constant-bank row, the loop unrolls; the ring wraps at most once inside the window.
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
                        for (int u = 0; u < TAPS + S; u++) {
                            const float *p = p0 + (u >= nwrap ? (u - K::RROWS) * ROWF : u * ROWF);
                            float2 v[3 * OUT / 2];
#pragma unroll
                            for (int k = 0; k < 3 * OUT / 2; k++) v[k] = *reinterpret_cast<const float2 *>(p + 2 * k);
                            if (u < TAPS) {
#pragma unroll
                                for (int k = 0; k < 3 * OUT / 2; k++) aa[k] = v5::fma2(v[k], v5::splat(c_wint[S][u < TAPS ? u : 0]), aa[k]);
                            }
                            if (u >= S) {
#pragma unroll
                                for (int k = 0; k < 3 * OUT / 2; k++) bb2[k] = v5::fma2(v[k], v5::splat(c_wint[S][u >= S ? u - S : 0]), bb2[k]);
                            }
                        }
                        uint32_t pa[OUT], pb[OUT];
                        finish(aa, oa, pa);
                        finish(bb2, ob, pb);
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
        cur = parked->nxt; it = parked->it; step++;   // written before this step's group_sync
    }
}


}  // namespace v6
