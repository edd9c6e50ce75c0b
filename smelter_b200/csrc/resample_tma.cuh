// resample_tma.cuh -- the front end shared by the TMA-staged fused resample kernels (included by kernels.cu):
// k_resample_tma3 (resample_tma3.cuh, integer ratio 2 / 4) and k_resample_tma0 (resample_tma0.cuh, any ratio <= 4:1).
//
// K1/K2 + K8 (horizontal) + K8 (vertical) with the arithmetic, quantisation points and per-output accumulation order of
// k_resample_fused_int (resample.wgsl:42-86 twice, planar_yuv_to_rgba.wgsl / nv12_to_rgba.wgsl in front), so the bytes
// are identical; what this file holds is how the source data moves and how it is converted:
//
//   * a block is one per SM and runs independent 8-warp groups (named barriers 1.., own TMA stage, own mbarriers, own
//     ring, own list of pieces); the tables behind the groups' memory are the block's;
//   * a chunk's source rows arrive by TMA: one elected thread issues cp.async.bulk.tensor.2d copies of a (272 B x 32 rows)
//     luma box and the matching chroma box into the group's stage, completion on an mbarrier; the stage is refilled
//     while the vertical pass runs.  A box may start at a negative coordinate but only at a 16-byte boundary of the row
//     (the TMA unit's alignment rule for the global address of a box), so the tile starts at the strip's first pixel
//     rounded down to 16 and every lane realigns its bytes with one funnel shift per word; out-of-image bytes
//     (zero-filled by the TMA unit) are replaced by the edge texels (resample.wgsl clamps the tap index);
//   * lane l converts the 8 consecutive source pixels X0 + 8l .. X0 + 8l + 7 of a row once (K1/K2 -> u8 -> sRGB decode),
//     FP32 pairs (fma2 / mul2 / add2, two scalar IEEE operations each on sm_90) holding two pixels;
//   * integer -> float without the conversion unit: a byte or a 16-bit field is PRMT-ed under the exponent of 2^23
//     and 2^23 is subtracted (exact); float -> index by adding 1.5 * 2^23 (round-to-nearest-even, exactly
//     __float2int_rn for |x| < 2^22);
//   * the sRGB decode table is REPLICATED per lane: entry i of lane l sits at word 32 i + l, i.e. in bank l, and the 24
//     data-dependent lookups of a row never conflict.  The table has exactly 256 entries, so the clamp of NC-2 sits in
//     front of the rounding as the .SAT of the matrix row's last fma.
#pragma once

namespace tma {

constexpr int kWarps = 8;                            // warps of one group
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
// the block's shared memory behind its groups' stages and rings ("tail"): the decode table, the 256 encode thresholds,
// two mbarriers per group (16 bytes per group), the decode table's lookup base, the iterator stash
constexpr int kThrOff = 256 * kDecRep * 4;
constexpr int kBarOff = kThrOff + 256 * 4;
constexpr int kKaddrOff = kBarOff + 64;
constexpr int kYbaseOff = kKaddrOff + 4;
constexpr int kStashOff = kBarOff + 128;
constexpr int kStashBytes = 1024;
constexpr int kTailBytes = kStashOff + kStashBytes;
// the luma table of the integer-ratio kernel, behind the tail: K1/K2 luma of every byte for the launch's range, 16
// copies (entry n of copy c at word 16 n + c, lane l reads copy l % 16), so two lanes at most share a bank
constexpr int kLumaRep = 16;
constexpr int kLumaTabBytes = 256 * kLumaRep * 4;

// strips of the integer-ratio kernel: output columns per strip, and the offset that makes the tile's first source pixel
// first_h(strip) - kLead<S> even
template <int S> constexpr int kStripCols = S == 4 ? kTmaStripCols4 : kTmaStripCols2;
template <int S> constexpr int kLead = S == 2 ? 1 : 0;

struct Chunk {      // warp-uniform description of one pipeline step
    int valid;      // 0: the group has no more work
    int job, ox0;   // job index, first output column of the strip
    int x0;         // first source pixel of the strip's tile
    int r0, nrows;  // source rows [r0, r0 + nrows) to convert in this step (nrows may be 0)
    int last;       // the group's rows are complete after this chunk: run the vertical pass
    int o0, oy_end; // the group's output rows [o0, min(o0 + 8, oy_end))
};

// The walk over a group's pieces, 8 output rows and up to kChunkRows / BX source rows at a time.
// S = 2, 4: the integer-ratio kernel (strips of kStripCols<S> columns); S = 0: the any-ratio kernel (strips of the job's
// strip_cols columns, tile starting at the even pixel at or below the first tap).  BX = 2: the kernel box-reduces the
// source 2:1 on the fly, and rows, x0 and H are in reduced units.
template <int S, int BX>
struct ChunkIter {
    const FusedJob *jobs;
    const FusedPiece *pieces;
    int pi, pend;
    int job, ox0, x0, oy_end, onext, ocur;
    int produced_hi, rnext, rhi;
    int H, tv, fv0;   // of the current piece's job; fv0 = first_v[0] when the vertical mapping is the integer ratio
    int in_group, vs;   // flags; int, not bool: the layout of the stashed copy (Stash) is what the register budget was tuned with
    __device__ __forceinline__ void init(const FusedJob *j, const FusedPiece *p, int b, int e) {
        jobs = j; pieces = p; pi = b - 1; pend = e; in_group = false; onext = 0; oy_end = 0;
        job = ox0 = x0 = ocur = 0; produced_hi = rnext = rhi = 0; H = tv = fv0 = 0; vs = false;
    }
    __device__ __forceinline__ Chunk next() {
        constexpr int rows = kChunkRows / BX;
        Chunk c;
        c.valid = 0; c.job = c.ox0 = c.x0 = c.r0 = c.nrows = c.last = c.o0 = c.oy_end = 0;
        if (!(in_group && rnext <= rhi)) {   // next group of 8 output rows (possibly of the next piece)
            if (onext >= oy_end) {
                pi++;
                if (pi >= pend) return c;
                const FusedPiece P = pieces[pi];
                const FusedJob &J = jobs[P.job];
                job = P.job; ox0 = P.strip * (S ? kStripCols<S> : J.strip_cols); onext = P.oy_begin; oy_end = P.oy_end;
                x0 = S ? __ldg(J.first_h + ox0) - kLead<S> : __ldg(J.first_h + ox0) & ~1;   // S = 0: chroma-aligned
                H = J.src.height / BX; tv = J.taps_v; vs = J.v_same != 0;
                fv0 = __ldg(J.first_v);
                produced_hi = -0x40000000;
            }
            ocur = onext;
            const int o_l = min(ocur + kWarps - 1, oy_end - 1);
            // same integer ratio vertically: first_v(o) = first_v(0) + S * o (resample.wgsl:45-50 in exact arithmetic), no
            // dependent global loads on the way to the next TMA issue
            const int f_lo = (S && vs) ? fv0 + S * ocur : __ldg(jobs[job].first_v + ocur);
            const int f_hi = (S && vs) ? fv0 + S * o_l : __ldg(jobs[job].first_v + o_l);
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
        c.nrows = max(0, min(rows, rhi - rnext + 1));
        rnext += rows;
        c.last = rnext > rhi;
        return c;
    }
};

// The iterator and the next chunk are not needed while a chunk is being processed: thread 0 of the group parks them in
// shared memory, everybody reloads them at the end of the step -- registers for the phases.  Two slots per group: the slot
// of step k is rewritten in step k + 2, and a group_sync lies between.
template <class It>
struct Stash { It it; Chunk nxt; };
template <class It, int GROUPS>
__device__ __forceinline__ Stash<It> *stash_slots(unsigned char *tail, int grp) {
    static_assert(sizeof(Stash<It>) * 2 * GROUPS <= kStashBytes, "stash");
    return reinterpret_cast<Stash<It> *>(tail + kStashOff) + 2 * grp;
}

// bar.sync on a named barrier: the 8 warps of one group
__device__ __forceinline__ void group_sync(int g) { asm volatile("bar.sync %0, 256;" ::"r"(g + 1) : "memory"); }

// Fills the tail (decode table, thresholds, mbarriers) and returns this lane's decode-table base: entry i of lane l is
// [(float bits of (i + 1.5 * 2^23)) << 7 + base]  (mod 2^32).  The base takes a round trip through shared memory so that
// it stays ONE register and the lookup address ONE LEA.  extra(): the kernel's own set-up, run before the closing
// __syncthreads.
template <int GROUPS, class Extra>
__device__ __forceinline__ uint32_t setup_block(unsigned char *tail, Extra extra) {
    float *s_dec = reinterpret_cast<float *>(tail), *s_thr = reinterpret_cast<float *>(tail + kThrOff);
    volatile uint32_t *s_kaddr = reinterpret_cast<volatile uint32_t *>(tail + kKaddrOff);
    const int btid = threadIdx.y * 32 + threadIdx.x, bn = 32 * kWarps * GROUPS;
    for (int i = btid; i < 256 * kDecRep; i += bn) s_dec[i] = c_dec[i / kDecRep];   // word i * 32 + l: bank l
    for (int i = btid; i < 256; i += bn) s_thr[i] = c_thr[i];
    if (btid == 0) {
        *s_kaddr = smem_u32(s_dec) - (kMagicBits << 7);
        for (int g = 0; g < GROUPS; g++) {
            mbar_init(smem_u32(tail + kBarOff) + 16u * (uint32_t)g, 1);
            mbar_init(smem_u32(tail + kBarOff) + 16u * (uint32_t)g + 8, 1);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    extra();
    __syncthreads();
    return *s_kaddr + 4u * (uint32_t)threadIdx.x;
}

// first byte of the luma tile / chroma tile (NV12: byte, planar: texel) of a tile whose first source pixel is x0:
// 16-byte boundaries, possibly negative.  NV12: texel cx - 1 of the first pair sits at byte x0 - 2.
__device__ __forceinline__ int luma_tile_x(int x0) { return x0 & ~15; }
template <bool NV12>
__device__ __forceinline__ int chroma_tile_x(int x0) { return NV12 ? ((x0 - 2) & ~15) : (((x0 >> 1) - 1) & ~15); }

// one thread: the TMA loads of chunk c's boxes into the stage at dst, completion on bar
template <bool NV12, int BX>
__device__ __forceinline__ void issue(const FusedJob *jobs, const Chunk &c, uint32_t dst, uint32_t bar) {
    if (!c.valid || c.nrows == 0) return;
    const FusedJob &J = jobs[c.job];
    const int x0 = c.x0 * BX, sr0 = c.r0 * BX;   // source pixel / row of the tile's origin
    const int cyb = (sr0 >> 1) - 1;
    const int xt = luma_tile_x(x0), xc = chroma_tile_x<NV12>(x0);
    if (NV12) {
        mbar_expect_tx(bar, kLumaBox * kChunkRows + kNv12Box * kChromaRows);
        tma_load_2d(dst, J.tm0, xt >> 1, sr0, bar);   // both planes are addressed in 2-byte elements
        tma_load_2d(dst + kLumaBytes, J.tm1, xc >> 1, cyb, bar);
    } else {
        mbar_expect_tx(bar, kLumaBox * kChunkRows + 2 * kPlanarBox * kChromaRows);
        tma_load_2d(dst, J.tm0, xt >> 1, sr0, bar);
        tma_load_2d(dst + kLumaBytes, J.tm1, xc, cyb, bar);
        tma_load_2d(dst + kLumaBytes + kChromaBytesPlanar, J.tm2, xc, cyb, bar);
    }
}

// Image borders: the tap index is clamped (resample.wgsl), the TMA unit zero-fills.  When a tile (origin x0, lrows luma
// rows) reaches outside the W-pixel-wide image, the group replaces the out-of-image bytes of its stage st by the edge
// texels and hands the stage back to the async proxy.
template <bool NV12>
__device__ __forceinline__ void replicate_edges(unsigned char *st, int x0, int lrows, int W, int tid, int grp) {
    const int xt = luma_tile_x(x0), xc = chroma_tile_x<NV12>(x0);
    const int cw = W >> 1;
    if (!(xt < 0 || xt + kLumaBox > W || xc < 0 || (NV12 ? xc + kNv12Box > W : xc + kPlanarBox > cw))) return;
    const int sub = tid & 7;
    {   // luma: tile byte b <-> pixel xt + b; valid bytes [bl, br)
        const int bl = min(max(0, -xt), kLumaBox - 1), br = min(max(W - xt, 1), kLumaBox);
        for (int row = tid >> 3; row < lrows; row += 32) {
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
    group_sync(grp);
}

// This lane's bytes inside the tiles of a tile whose first source pixel is x0: word offsets and the funnel shifts that
// realign them.
template <bool NV12>
struct LaneWords {
    uint32_t l_off, l_sh, c_off, c_sh;
    __device__ __forceinline__ LaneWords(int x0, int lane) {
        const int dl = x0 - luma_tile_x(x0), dc = (NV12 ? x0 - 2 : (x0 >> 1) - 1) - chroma_tile_x<NV12>(x0);
        l_off = (uint32_t)((dl & ~3) + lane * 8); l_sh = (uint32_t)(dl & 3) * 8u;
        c_off = (uint32_t)((dc & ~3) + lane * (NV12 ? 8 : 4)); c_sh = (uint32_t)(dc & 3) * 8u;
    }
};

// yw = the lane's 8 luma bytes of a source row, la: the shared address of the lane's words of it (stage + row + lw.l_off)
template <bool NV12>
__device__ __forceinline__ void fetch_luma(uint32_t la, const LaneWords<NV12> &lw, uint32_t (&yw)[2]) {
    // raw bytes of this lane's 8 pixels: 12 bytes from a 4-byte aligned address; the half that is 8-byte aligned
    // (warp-uniform) goes as one LDS.64 (lanes 8 bytes apart: conflict-free, an LDS.32 is 2-way)
    uint32_t w0, w1, w2;
    if (lw.l_off & 4u) { w0 = lds32v(la); lds64v(la + 4, w1, w2); }
    else { lds64v(la, w0, w1); w2 = lds32v(la + 8); }
    yw[0] = __funnelshift_r(w0, w1, lw.l_sh);
    yw[1] = __funnelshift_r(w1, w2, lw.l_sh);
}

// v[k] = 3 * heavy + light chroma texel cx - 1 + k (u in bits 0..15, v in bits 16..31) of a source row; bh, bl: the shared
// addresses of the lane's words (chroma tile + row + lw.c_off) of the chroma row that weighs 3/4 and of the one that weighs
// 1/4; planar: in the u plane, the v plane lies kChromaBytesPlanar behind
template <bool NV12>
__device__ __forceinline__ void fetch_chroma(uint32_t bh, uint32_t bl, const LaneWords<NV12> &lw, uint32_t (&v)[6]) {
    const uint32_t c_off = lw.c_off, c_sh = lw.c_sh;
    if (NV12) {
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
        const uint32_t uh = bh, ul = bl;
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
}

// Source row r of the stage sb whose tile starts at source row sr0 (chei chroma rows in the image): fetch_luma and
// fetch_chroma at the row's addresses
template <bool NV12>
__device__ __forceinline__ void fetch_row(uint32_t sb, const LaneWords<NV12> &lw, int r, int sr0, int chei, uint32_t (&yw)[2],
                                          uint32_t (&v)[6]) {
    constexpr int box = NV12 ? kNv12Box : kPlanarBox;
    fetch_luma<NV12>(sb + (uint32_t)((r - sr0) * kLumaBox) + lw.l_off, lw, yw);
    const int cyb = (sr0 >> 1) - 1;                                     // chroma row of the tile's first row
    const int ch = r >> 1;                                              // weight 3/4
    const int cl = (r & 1) ? min(ch + 1, chei - 1) : max(ch - 1, 0);    // weight 1/4
    fetch_chroma<NV12>(sb + kLumaBytes + (uint32_t)((ch - cyb) * box) + lw.c_off,
                       sb + kLumaBytes + (uint32_t)((cl - cyb) * box) + lw.c_off, lw, v);
}

// exact n / 255 of a byte n held as a float: fma(n, c, n * lo)
constexpr uint32_t kDiv255C = 0x3b808081u, kDiv255Lo = 0xaf7efeffu;

// K1/K2 luma of byte n (ny = n as a float): clamp01((n / 255 - 16/255) * rcp_y), or n / 255 for a full range source
// (nk16 = 0, rcp_y = 1) -- each operation is one component of convert_pair's pair arithmetic
__device__ __forceinline__ float luma_of(float ny, float nk16, float rcp_y) {
    const float y = __fmaf_rn(ny, __uint_as_float(kDiv255C), __fmul_rn(ny, __uint_as_float(kDiv255Lo)));
    return __saturatef(__fmul_rn(__fadd_rn(y, nk16), rcp_y));
}

// The luma table behind the tail (kLumaTabBytes, filled by the block before its first __syncthreads) and this lane's
// lookup base: the entry of byte n is [(float bits of (n + 2^23)) << 6 + base]  (mod 2^32), so that the PRMT which puts
// the byte under the exponent of 2^23 plus one LEA make the address.  Like the decode table's base (setup_block) the base
// takes a round trip through shared memory: known to the compiler it is a constant too wide for the load's address
// field, and every lookup pays an extra add for its upper half.
__device__ __forceinline__ void fill_luma_table(unsigned char *tail, float nk16, float rcp_y) {
    float *s_y = reinterpret_cast<float *>(tail + kTailBytes);
    const int btid = threadIdx.y * 32 + threadIdx.x, bn = blockDim.x * blockDim.y;
    for (int i = btid; i < 256 * kLumaRep; i += bn) s_y[i] = luma_of((float)(i / kLumaRep), nk16, rcp_y);
    if (btid == 0) *reinterpret_cast<volatile uint32_t *>(tail + kYbaseOff) = smem_u32(s_y) - (0x4B000000u << 6);
}
// after the __syncthreads that follows fill_luma_table
__device__ __forceinline__ uint32_t luma_base(unsigned char *tail) {
    return *reinterpret_cast<volatile uint32_t *>(tail + kYbaseOff) + 4u * (threadIdx.x % kLumaRep);
}

// K1/K2 -> u8 of pixels 2p and 2p + 1 of an 8-pixel run (yw: its luma bytes, v: its combined chroma as fetch_row makes it),
// two pixels per instruction: q = 1.5 * 2^23 + the byte.  nk16, rcp_y, rcp_c: -16/255 and the limited-range scales, or
// 0, 1, 1 for a full-range source; k: the matrix's coefficients (yuv_coef).  YTAB: the luma comes from the luma table (ybase from luma_base, filled for the same
// nk16 and rcp_y) instead of the arithmetic.
template <bool YTAB = false>
__device__ __forceinline__ void convert_pair(const uint32_t (&yw)[2], const uint32_t (&v)[6], int p, float nk16, float rcp_y,
                                             float rcp_c, const YuvCoef &k, float2 &qr, float2 &qg, float2 &qb, uint32_t ybase = 0) {
    // 16 x chroma of the even / odd pixel of the pair (NC-6u with the .25 / .75 taps)
    const uint32_t ne = v[p] + 3u * v[p + 1], no = 3u * v[p + 1] + v[p + 2];
    const float m23 = -8388608.0f;
    float2 nu = add2(make_float2(__uint_as_float(__byte_perm(ne, 0x4B000000u, 0x7610)),
                                 __uint_as_float(__byte_perm(no, 0x4B000000u, 0x7610))), splat(m23));
    float2 nv = add2(make_float2(__uint_as_float(__byte_perm(ne, 0x4B000000u, 0x7632)),
                                 __uint_as_float(__byte_perm(no, 0x4B000000u, 0x7632))), splat(m23));
    const uint32_t ywd = yw[p >> 1];
    const uint32_t by0 = __byte_perm(ywd, 0x4B000000u, (p & 1) ? 0x7642 : 0x7640);
    const uint32_t by1 = __byte_perm(ywd, 0x4B000000u, (p & 1) ? 0x7643 : 0x7641);
    // exact n / 255 and n / (255 * 16): fma(n, c, n * lo)
    const float c1 = __uint_as_float(kDiv255C), lo1 = __uint_as_float(kDiv255Lo);
    const float c16 = __uint_as_float(0x39808081u), lo16 = __uint_as_float(0xad7efeffu);
    float2 y;
    if (YTAB) {
        y = make_float2(lds_tab((by0 << 6) + ybase), lds_tab((by1 << 6) + ybase));
    } else {
        const float2 ny = add2(make_float2(__uint_as_float(by0), __uint_as_float(by1)), splat(m23));
        y = fma2(ny, splat(c1), mul2(ny, splat(lo1)));
    }
    float2 u = fma2(nu, splat(c16), mul2(nu, splat(lo16)));
    float2 w = fma2(nv, splat(c16), mul2(nv, splat(lo16)));
    // limited range: clamp01((x - 16/255) * rcp); full range: (x - 0) * 1 and the clamp are identities on [0, 1]
    if (!YTAB) y = add2(y, splat(nk16));
    u = add2(u, splat(nk16)); w = add2(w, splat(nk16));
    if (!YTAB) y = make_float2(__saturatef(y.x * rcp_y), __saturatef(y.y * rcp_y));
    u = make_float2(__saturatef(u.x * rcp_c), __saturatef(u.y * rcp_c));
    w = make_float2(__saturatef(w.x * rcp_c), __saturatef(w.y * rcp_c));
    const float2 um = add2(u, splat(-0.5f)), vm = add2(w, splat(-0.5f));
    // clamp01 (NC-2) as the .SAT of the matrix row's last fma
    const float2 gi = fma2(splat(k.gu), um, y);
    const float2 rr = make_float2(__saturatef(fmaf(k.rv, vm.x, y.x)), __saturatef(fmaf(k.rv, vm.y, y.y)));
    const float2 gg = make_float2(__saturatef(fmaf(k.gv, vm.x, gi.x)), __saturatef(fmaf(k.gv, vm.y, gi.y)));
    const float2 bb = make_float2(__saturatef(fmaf(k.bu, um.x, y.x)), __saturatef(fmaf(k.bu, um.y, y.y)));
    // NC-2 rounding: the add rounds to the nearest-even integer
    qr = add2_after_mul(mul2(rr, splat(255.0f)), splat(kMagicRound));
    qg = add2_after_mul(mul2(gg, splat(255.0f)), splat(kMagicRound));
    qb = add2_after_mul(mul2(bb, splat(255.0f)), splat(kMagicRound));
}

// K1/K2 -> u8 -> sRGB decode of the node-texture fetch (NC-3) of an 8-pixel run: (r, g) and b of pixel i, looked up in
// this lane's copy of the decode table (kaddr from setup_block); k, YTAB, ybase: as in convert_pair
template <bool YTAB = false>
__device__ __forceinline__ void convert_run(const uint32_t (&yw)[2], const uint32_t (&v)[6], float nk16, float rcp_y, float rcp_c,
                                            const YuvCoef &k, uint32_t kaddr, float2 (&prg)[8], float (&pb)[8], uint32_t ybase = 0) {
#pragma unroll
    for (int p = 0; p < 4; p++) {
        float2 qr, qg, qb;
        convert_pair<YTAB>(yw, v, p, nk16, rcp_y, rcp_c, k, qr, qg, qb, ybase);
        prg[2 * p] = make_float2(lds_tab((__float_as_uint(qr.x) << 7) + kaddr), lds_tab((__float_as_uint(qg.x) << 7) + kaddr));
        prg[2 * p + 1] = make_float2(lds_tab((__float_as_uint(qr.y) << 7) + kaddr), lds_tab((__float_as_uint(qg.y) << 7) + kaddr));
        pb[2 * p] = lds_tab((__float_as_uint(qb.x) << 7) + kaddr);
        pb[2 * p + 1] = lds_tab((__float_as_uint(qb.y) << 7) + kaddr);
    }
}

// NC-4 of one output row's OUT columns of a lane -- acc: r of the columns, then g, then b, two columns per float2 -- scaled
// by inv_v, into RGBA8 words px; then the store of each pair (j, j + 1), which are adjacent columns col_of(j), col_of(j) + 1
// of the strip that starts at output column ox0 and is strip_cols wide
template <int OUT, class ColOf>
__device__ __forceinline__ void encode_store(const FusedJob &J, const float2 (&acc)[3 * OUT / 2], int oy, const float *s_thr,
                                             int ox0, int strip_cols, ColOf col_of, uint32_t (&px)[OUT]) {
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
    const int ncols = min(strip_cols, J.dst_w - ox0);
#pragma unroll
    for (int j = 0; j < OUT; j += 2) {
        const int col = col_of(j);
        if (col >= 0 && col + 1 < ncols) {
            *reinterpret_cast<uint2 *>(drow + ox0 + col) = make_uint2(px[j], px[j + 1]);
        } else if (col >= 0 && col < ncols) {
            drow[ox0 + col] = px[j];
        }
    }
}

}  // namespace tma
