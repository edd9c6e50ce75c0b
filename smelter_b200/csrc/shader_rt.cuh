// shader_rt.cuh -- what a registered shader's CUDA C++ source is compiled against, by NVRTC at smr_register_shader.
// Never compiled by nvcc: renderer.cpp embeds it as a string.  The module is, in this order: kernels.h and
// node_sample.cuh inside namespace smr::dev, the SMR_SHADER_API part below, the user's source, the SMR_SHADER_MAIN part.
// For a WGSL shader the user's source is wgsl_rt.cuh followed by the translation, and the main part is the rasteriser.
// It stands in for the reference's shader header (transformations/shader/validation/shader_header.wgsl).
#ifdef SMR_SHADER_API
// VertexOutput of the full-target plane: tex_coords (0, 0) at the top-left corner, position the pixel centre in target
// pixels (@builtin(position): x + .5, y + .5, z 0, w 1).  There is no user vertex stage: every plane is the full target
// under the identity transform, as the reference's example shaders draw it.
struct smr_fragment_in {
    float2 tex_coords;
    float4 position;
};
// BaseShaderParameters (base_params.rs), same fields, types and values
struct smr_base_params {
    int plane_id;                  // 0 .. texture_count - 1, or -1 when the node has no child
    float time;                    // pts in seconds (Duration::as_secs_f32)
    unsigned output_resolution[2]; // the node texture's width and height
    unsigned texture_count;        // the number of children
};
// The child textures (binding group 0) through the reference's sampler (group 2: linear filtering, clamp to edge).  A
// sample is what wgpu's view returns: sRGB-decoded colour in GpuOptimized mode, the raw bytes over 255 in CpuOptimized
// mode, premultiplied alpha.  An index at or above texture_count, or a child input without a live frame, samples the
// empty view (0, 0, 0, 0).
struct smr_textures {
    const smr::dev::Tables *T;
    const smr::dev::Tex *tex;
    unsigned count;
    int mode;
    __device__ float4 sample(unsigned i, float2 uv) const {
        bool exact;
        uchar4 texel;
        return smr::dev::sample_node(*T, i < count ? tex + i : nullptr, mode, uv.x, uv.y, exact, texel);
    }
};
__device__ float4 smr_fragment(smr_fragment_in in, const smr_base_params &base, const void *params, const smr_textures &tex);
#endif

#if defined(SMR_SHADER_MAIN) && defined(SMR_WGSL)
// A WGSL shader (wgsl.cpp, wgsl_rt.cuh): ShaderPipeline::render with the user's vertex stage.  Every node of this shader
// in one launch, one thread per pixel of a 32 x 8 tile, as below.  The contract, restated in include/smelter_b200.h:
//  - The block's prologue runs vs_main for the 4 plane-mesh vertices of each of the max(1, texture_count) planes into
//    shared memory, then sets up the plane's two triangles (indices 0,1,2 and 2,3,0).
//  - A plane with a vertex whose w is not above 0, or whose window coordinate is not finite or beyond 2^20 px, is not
//    drawn.  Window coordinates: x = fmaf(x_c / w, W / 2, W / 2), y = fmaf(-(y_c / w), H / 2, H / 2), snapped to
//    1/256 px (rint(v * 256)); the depth is z_c / w.
//  - A triangle's doubled area A from the snapped vertices (int64) decides its face: A < 0 (counter-clockwise in clip
//    space, as the reference plane is) is front; A > 0 is culled; A == 0 draws nothing.
//  - A pixel (centre x + 1/2, y + 1/2 in 1/256 units) is covered when its three int64 edge functions are positive, or 0
//    on a top or left edge (interior below, or to the right): a pixel on a shared edge is drawn once.
//  - Barycentrics b_i = (float)E_i / (float)A (E_i the edge function opposite vertex i).  The fragment's depth is
//    (b0 z0 + b1 z1) + b2 z2; a depth outside [0, 1] is not drawn.  With p_i = b_i / w_i and s = (p0 + p1) + p2, a
//    perspective varying is ((p0 v0 + p1 v1) + p2 v2) / s, a linear one (b0 v0 + b1 v1) + b2 v2, a flat one the first
//    vertex's.  @builtin(position) is (x + 1/2, y + 1/2, depth, s).
//  - Each covered fragment runs fs_main; unless it discards, its value is blended (PREMULTIPLIED_ALPHA_BLENDING) and
//    stored as 8 bits, in plane order and, within a plane, triangle order.
// Two blocks per SM are enough to hide the prologue's barriers; asking for no more lets ptxas keep a vertex stage that
// samples textures (textureSampleLevel / Grad) and a gather-heavy fragment stage in registers, without spills.
struct wg_tri {
    long long x[3], y[3];   // snapped window coordinates, 1/256 px
    long long area;         // doubled, of the front-facing (sign-normalised) triangle: > 0
    int v[3];               // the vertices, in the shared arrays
    int bx0, by0, bx1, by1; // pixel bounding box, inclusive
    bool live;
};
__device__ inline bool wg_window(const float *p, int W, int H, long long &x, long long &y, float &z) {
    const float w = p[3];
    if (!(w > 0.0f)) return false;
    const float xw = fmaf(p[0] / w, (float)W / 2.0f, (float)W / 2.0f), yw = fmaf(-(p[1] / w), (float)H / 2.0f, (float)H / 2.0f);
    if (!(fabsf(xw) <= 1048576.0f && fabsf(yw) <= 1048576.0f)) return false;   // also false for NaN
    x = (long long)rintf(xw * 256.0f);
    y = (long long)rintf(yw * 256.0f);
    z = p[2] / w;
    return true;
}
// E(p) for the edge a -> b, oriented by the triangle's sign so that the interior is positive
__device__ inline long long wg_edge(const wg_tri &t, int a, int b, long long px, long long py, long long sgn) {
    return sgn * ((t.x[b] - t.x[a]) * (py - t.y[a]) - (t.y[b] - t.y[a]) * (px - t.x[a]));
}

extern "C" __global__ void __launch_bounds__(256, 2) smr_shader_main(const smr::dev::ShaderJob *__restrict__ jobs,
                                                                     const int *__restrict__ tile_begin, int n_jobs) {
    constexpr int NV = WG_NVARY > 0 ? WG_NVARY : 1;
    __shared__ smr::dev::Tables T;
    __shared__ smr::dev::ShaderJob J;
    __shared__ int s_origin[2];
    __shared__ float s_pos[64][4];
    __shared__ float s_z[64];
    __shared__ float s_vary[64][NV];
    __shared__ wg_tri s_tri[32];
    const int tid = (int)threadIdx.y * 32 + (int)threadIdx.x;
    if (tid == 0) smr::dev::load_block_job(jobs, tile_begin, n_jobs, J, s_origin);
    smr::dev::load_tables(T);   // ends in __syncthreads
    const int W = J.dst.width, H = J.dst.height;
    const int planes = J.n_tex > 0 ? J.n_tex : 1;
    wg_ctx ctx;
    ctx.params = J.params;
    ctx.tex.T = &T; ctx.tex.tex = J.tex; ctx.tex.count = (unsigned)J.n_tex; ctx.tex.mode = J.dst.mode;
    if (tid < 4 * planes) {   // vs_main, one vertex per thread
        wg_base(ctx, J.n_tex > 0 ? tid / 4 : -1, J.time, (unsigned)W, (unsigned)H, (unsigned)J.n_tex);
        ctx.discarded = false;
        float vary[NV];
        wg_vertex(ctx, tid % 4, s_pos[tid], vary);
        for (int k = 0; k < WG_NVARY; k++) s_vary[tid][k] = vary[k];
    }
    __syncthreads();
    if (tid < 2 * planes) {   // triangle set-up
        const int pl = tid / 2;
        const int idx[2][3] = {{0, 1, 2}, {2, 3, 0}};
        wg_tri t;
        t.live = true;
        for (int k = 0; k < 4; k++) {   // the plane is drawn only if all four vertices are
            long long x, y;
            float z;
            if (!wg_window(s_pos[pl * 4 + k], W, H, x, y, z)) t.live = false;
        }
        for (int k = 0; k < 3 && t.live; k++) {
            t.v[k] = pl * 4 + idx[tid % 2][k];
            wg_window(s_pos[t.v[k]], W, H, t.x[k], t.y[k], s_z[t.v[k]]);
        }
        if (t.live) {
            const long long a = (t.x[1] - t.x[0]) * (t.y[2] - t.y[0]) - (t.y[1] - t.y[0]) * (t.x[2] - t.x[0]);
            t.live = a < 0;   // front-facing; back faces and degenerate triangles are not drawn
            t.area = -a;
            long long x0 = t.x[0], x1 = t.x[0], y0 = t.y[0], y1 = t.y[0];
            for (int k = 1; k < 3; k++) {
                x0 = min(x0, t.x[k]); x1 = max(x1, t.x[k]); y0 = min(y0, t.y[k]); y1 = max(y1, t.y[k]);
            }
            // pixels whose centre (256 p + 128) can lie in [x0, x1]
            t.bx0 = (int)max(0LL, (x0 - 128 + 255) >> 8); t.bx1 = (int)min((long long)W - 1, (x1 - 128) >> 8);
            t.by0 = (int)max(0LL, (y0 - 128 + 255) >> 8); t.by1 = (int)min((long long)H - 1, (y1 - 128) >> 8);
            if (t.bx0 > t.bx1 || t.by0 > t.by1) t.live = false;
        }
        s_tri[tid] = t;
    }
    __syncthreads();
    const int x = s_origin[0] + (int)threadIdx.x, y = s_origin[1] + (int)threadIdx.y;
    if (x >= W || y >= H) return;
    const int tx0 = s_origin[0], ty0 = s_origin[1], tx1 = s_origin[0] + 31, ty1 = s_origin[1] + 7;
    const long long px = 256LL * x + 128, py = 256LL * y + 128;
    uchar4 o = make_uchar4(0, 0, 0, 0);   // the target is cleared to transparent
    for (int i = 0; i < 2 * planes; i++) {
        const wg_tri &t = s_tri[i];
        if (!t.live || t.bx1 < tx0 || t.bx0 > tx1 || t.by1 < ty0 || t.by0 > ty1) continue;   // the same for the whole block
        long long E[3];
        bool in = true;
        for (int k = 0; k < 3; k++) {   // E[k]: the edge opposite vertex k, from vertex k+1 to k+2 (front faces are clockwise here)
            const int a = (k + 1) % 3, b = (k + 2) % 3;
            E[k] = wg_edge(t, a, b, px, py, -1);
            // inward normal (-(dy), dx) * -1: top-left when it points right, or straight down
            const long long nx = t.y[b] - t.y[a], ny = -(t.x[b] - t.x[a]);
            const bool top_left = nx > 0 || (nx == 0 && ny > 0);
            in = in && (E[k] > 0 || (E[k] == 0 && top_left));
        }
        if (!in) continue;
        const float A = (float)t.area;
        const float b0 = (float)E[0] / A, b1 = (float)E[1] / A, b2 = (float)E[2] / A;
        const int v0 = t.v[0], v1 = t.v[1], v2 = t.v[2];
        const float depth = (b0 * s_z[v0] + b1 * s_z[v1]) + b2 * s_z[v2];
        if (!(depth >= 0.0f && depth <= 1.0f)) continue;
        const float p0 = b0 / s_pos[v0][3], p1 = b1 / s_pos[v1][3], p2 = b2 / s_pos[v2][3];
        const float sum = (p0 + p1) + p2;
        float vary[NV];
        for (int k = 0; k < WG_NVARY; k++) {
            const float a0 = s_vary[v0][k], a1 = s_vary[v1][k], a2 = s_vary[v2][k];
            vary[k] = wg_interp[k] == 2 ? a0 : wg_interp[k] == 1 ? (b0 * a0 + b1 * a1) + b2 * a2 : ((p0 * a0 + p1 * a1) + p2 * a2) / sum;
        }
        const float pos[4] = {(float)x + 0.5f, (float)y + 0.5f, depth, sum};
        wg_base(ctx, J.n_tex > 0 ? i / 2 : -1, J.time, (unsigned)W, (unsigned)H, (unsigned)J.n_tex);
        float4 c;
        if (wg_fragment(ctx, pos, vary, c)) o = smr::dev::blend(T, J.dst.mode, o, c);
    }
    reinterpret_cast<uchar4 *>(J.dst.out + (size_t)y * J.dst.out_pitch)[x] = o;
}
#elif defined(SMR_SHADER_MAIN)
// Every node of this shader in one launch (block -> job as in k_web); one thread per pixel of a 32 x 8 tile.  Each
// plane is a render pass over the whole target, so a pixel walks the planes in order and its value is quantised to 8
// bits after each one, as the texture holds it between passes.
extern "C" __global__ void __launch_bounds__(256) smr_shader_main(const smr::dev::ShaderJob *__restrict__ jobs,
                                                                  const int *__restrict__ tile_begin, int n_jobs) {
    __shared__ smr::dev::Tables T;
    __shared__ smr::dev::ShaderJob J;
    __shared__ int s_origin[2];
    if (threadIdx.x == 0 && threadIdx.y == 0) smr::dev::load_block_job(jobs, tile_begin, n_jobs, J, s_origin);
    smr::dev::load_tables(T);   // ends in __syncthreads
    const int x = s_origin[0] + (int)threadIdx.x, y = s_origin[1] + (int)threadIdx.y;
    if (x >= J.dst.width || y >= J.dst.height) return;
    smr_fragment_in in;
    in.position = make_float4((float)x + 0.5f, (float)y + 0.5f, 0.0f, 1.0f);
    in.tex_coords = make_float2(in.position.x / (float)J.dst.width, in.position.y / (float)J.dst.height);
    smr_base_params base;
    base.time = J.time;
    base.output_resolution[0] = (unsigned)J.dst.width;
    base.output_resolution[1] = (unsigned)J.dst.height;
    base.texture_count = (unsigned)J.n_tex;
    smr_textures tex;
    tex.T = &T; tex.tex = J.tex; tex.count = (unsigned)J.n_tex; tex.mode = J.dst.mode;
    uchar4 o = make_uchar4(0, 0, 0, 0);
    const int planes = J.n_tex > 0 ? J.n_tex : 1;
    for (int p = 0; p < planes; p++) {
        base.plane_id = J.n_tex > 0 ? p : -1;
        o = smr::dev::blend(T, J.dst.mode, o, smr_fragment(in, base, J.params, tex));
    }
    reinterpret_cast<uchar4 *>(J.dst.out + (size_t)y * J.dst.out_pitch)[x] = o;
}
#endif
