// shader_rt.cuh -- what a registered shader's CUDA C++ source is compiled against, by NVRTC at smr_register_shader.
// Never compiled by nvcc: renderer.cpp embeds it as a string.  The module is, in this order: kernels.h and
// node_sample.cuh inside namespace smr::dev, the SMR_SHADER_API part below, the user's source, the SMR_SHADER_MAIN part.
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

#ifdef SMR_SHADER_MAIN
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
