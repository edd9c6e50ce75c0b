// deinterlace.cuh -- k_deinterlace: the field and motion-adaptive deinterlacers of smr_set_input_deinterlace (NC-12), on
// the planes of the tick's deinterlaced inputs before anything reads them.  Included by kernels.cu inside namespace
// smr::dev.
//
// Every plane is bytes along rows, whatever the frame format, so one job is one plane and the kernel never looks at a
// pixel's layout.  A thread owns a 16-byte column of a run of kDeinterlaceRun row pairs: walking down, the kept row below
// one rebuilt row is the kept row above the next, so each kept row is loaded once for its two neighbours.  The arithmetic
// is per byte, four lanes to a 32-bit word (__vavgu4 is the rounded-up average (a + b + 1) >> 1 of NC-12).
// Memory-bound: the library's planes (out, history) have 16-byte aligned rows and take 16-byte stores; a caller's plane
// takes 16-byte loads where its row is 16-byte aligned and byte loads elsewhere.

// 16 bytes of a row from byte x.  PADDED: a library plane, whose pitch covers the 16-byte column past the row's end
template <bool PADDED>
__device__ __forceinline__ uint4 di_load(const uint8_t *p, int pitch, int y, int x, int row_bytes) {
    const uint8_t *q = p + (size_t)y * pitch + x;
    if (PADDED || (x + 16 <= row_bytes && ((uintptr_t)q & 15) == 0)) return __ldg(reinterpret_cast<const uint4 *>(q));
    uint32_t w[4] = {0, 0, 0, 0};
    const int n = min(16, row_bytes - x);   // bytes past the row are never read
#pragma unroll
    for (int i = 0; i < 16; i++)
        if (i < n) w[i >> 2] |= (uint32_t)__ldg(q + i) << (8 * (i & 3));
    return make_uint4(w[0], w[1], w[2], w[3]);
}

__device__ __forceinline__ void di_store(uint8_t *p, int pitch, int y, int x, uint4 v) {
    *reinterpret_cast<uint4 *>(p + (size_t)y * pitch + x) = v;
}

// NC-12 on one word: FIELD is avg(a, b); MOTION_ADAPTIVE keeps c where max(|c - p|, |a - pa|, |b - pb|) <= T
__device__ __forceinline__ uint32_t di_word(uint32_t c, uint32_t a, uint32_t b, uint32_t p, uint32_t pa, uint32_t pb, bool motion,
                                            uint32_t t4) {
    const uint32_t avg = __vavgu4(a, b);
    if (!motion) return avg;
    const uint32_t m = __vmaxu4(__vmaxu4(__vabsdiffu4(c, p), __vabsdiffu4(a, pa)), __vabsdiffu4(b, pb));
    const uint32_t still = __vcmpleu4(m, t4);   // 0xff in each byte lane where m <= T
    return (c & still) | (avg & ~still);
}

__global__ void __launch_bounds__(kDeinterlaceTileX * kDeinterlaceTileY)
k_deinterlace(const DeinterlaceJob *__restrict__ jobs, const int32_t *__restrict__ tile_begin, int n_jobs) {
    const int blk = (int)blockIdx.x;
    int lo = 0, hi = n_jobs - 1;   // the job whose block range holds this block
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(tile_begin + mid) <= blk) lo = mid;
        else hi = mid - 1;
    }
    const DeinterlaceJob J = jobs[lo];
    const int t = blk - __ldg(tile_begin + lo);
    const int x = ((t % J.tiles_x) * kDeinterlaceTileX + (int)threadIdx.x) * 16;
    const int j0 = ((t / J.tiles_x) * kDeinterlaceTileY + (int)threadIdx.y) * kDeinterlaceRun;
    const int pairs = (J.rows + 1) >> 1;
    if (x >= J.row_bytes || j0 >= pairs) return;
    // pair j is rows 2j and 2j + 1: its rebuilt row y = 2j + rb, its kept row 2j + kb.  The rebuilt row's neighbours are the
    // kept rows of pairs j + rb - 1 (above) and j + rb (below)
    const int rb = J.rebuild, kb = 1 - rb;
    const bool motion = J.prev != nullptr;
    const uint32_t t4 = J.threshold * 0x01010101u;
    auto kept_row = [&](int i) { return 2 * i + kb; };
    auto valid = [&](int r) { return r >= 0 && r < J.rows; };
    const uint4 zero = make_uint4(0, 0, 0, 0);
    uint4 A = zero, PA = zero;   // the kept row above (and its history)
    bool va = valid(kept_row(j0 + rb - 1));
    if (va) {
        A = di_load<false>(J.cur, J.cur_pitch, kept_row(j0 + rb - 1), x, J.row_bytes);
        if (motion) PA = di_load<true>(J.prev, J.prev_pitch, kept_row(j0 + rb - 1), x, J.row_bytes);
    }
    const int j1 = min(j0 + kDeinterlaceRun, pairs);
    for (int j = j0; j < j1; j++) {
        const int rbelow = kept_row(j + rb), y = 2 * j + rb, k = 2 * j + kb;
        const bool vb = valid(rbelow);
        uint4 B = zero, PB = zero;   // the kept row below
        if (vb) {
            B = di_load<false>(J.cur, J.cur_pitch, rbelow, x, J.row_bytes);
            if (motion) PB = di_load<true>(J.prev, J.prev_pitch, rbelow, x, J.row_bytes);
        }
        if (valid(k)) {   // the kept row of this pair is the one above (rb = 1) or below (rb = 0)
            const uint4 K = rb ? A : B;
            di_store(J.out, J.out_pitch, k, x, K);
            if (J.hist) di_store(J.hist, J.hist_pitch, k, x, K);
        }
        if (valid(y)) {
            uint4 c = zero, p = zero, o;
            if (motion || J.hist || (!va && !vb)) c = di_load<false>(J.cur, J.cur_pitch, y, x, J.row_bytes);
            if (motion) p = di_load<true>(J.prev, J.prev_pitch, y, x, J.row_bytes);
            if (!va && !vb) {   // a plane of one row
                o = c;
            } else {            // an edge row takes its one neighbour for both
                const uint4 a = va ? A : B, b = vb ? B : A, pa = va ? PA : PB, pb = vb ? PB : PA;
                o.x = di_word(c.x, a.x, b.x, p.x, pa.x, pb.x, motion, t4);
                o.y = di_word(c.y, a.y, b.y, p.y, pa.y, pb.y, motion, t4);
                o.z = di_word(c.z, a.z, b.z, p.z, pa.z, pb.z, motion, t4);
                o.w = di_word(c.w, a.w, b.w, p.w, pa.w, pb.w, motion, t4);
            }
            di_store(J.out, J.out_pitch, y, x, o);
            if (J.hist) di_store(J.hist, J.hist_pitch, y, x, c);
        }
        A = B; PA = PB; va = vb;
    }
}

int launch_deinterlace(const DeinterlaceJob *jobs_dev, const int32_t *tile_begin_dev, int n_jobs, int n_tiles, Stream s) {
    if (n_jobs <= 0 || n_tiles <= 0) return 0;
    k_deinterlace<<<n_tiles, dim3(kDeinterlaceTileX, kDeinterlaceTileY), 0, (cudaStream_t)s>>>(jobs_dev, tile_begin_dev, n_jobs);
    return check_launch("k_deinterlace") ? 1 : -1;
}
