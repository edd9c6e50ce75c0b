// renderer.cpp -- the Renderer behind the C ABI (include/smelter_b200.h).
//
// Replaces smelter-render/src/state.rs (Renderer/InnerRenderer), state/render_loop.rs
// (populate_inputs / run_transforms / read_outputs), state/render_graph.rs, state/{input,node,output}_texture.rs
// and transformations/layout.rs (LayoutNode::render, resample_scaled_children) + layout/params.rs.
//
// Design: no per-node textures and no per-pass submits.  Per tick the host flattens every
// output's scene (CPU, as in the reference), packs ALL device-side descriptors of the tick into one
// pinned arena, ships it with one async copy, and issues a fixed short sequence of launches on one
// stream: [convert inputs that feed a Lanczos pass] -> [weights for new mappings] -> [box passes] ->
// [first passes] -> [last passes] -> one composite(+YUV writeback) launch per output.  All transient
// textures live in a frame arena in HBM that is recycled every tick.
#include <cuda.h>
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/smelter_b200.h"
#include "interior.h"
#include "kernels.h"
#include "scene.h"

namespace smr {

#define CUDA_OK(expr)                                                                        \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess) {                                                             \
            set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));                   \
            return SMR_ERR_CUDA;                                                             \
        }                                                                                    \
    } while (0)

static const float kPiF = 3.14159265359f;

// ------------------------------------------------------------------------------------------------
// resampler planning (transformations/layout/resampler.rs:43-145)
// ------------------------------------------------------------------------------------------------
// Ticks the host may have submitted ahead of the GPU (smr_render_begin without smr_render_end): each owns a parameter
// block, an input staging set and its events.  Four absorb a host hiccup of some milliseconds at the 0.25-0.5 ms ticks of
// the benchmark configurations; the kernels of all of them run in submission order on one stream.
constexpr int kTicksInFlight = SMR_TICKS_IN_FLIGHT;

struct AxisMapping {
    int axis;  // 0 horizontal, 1 vertical
    float crop_offset, crop_len;
    int dst_len;
    float scale() const { return crop_len / (float)dst_len; }
    int predecimate_levels() const {  // :56-58
        float l = std::ceil(std::log2(scale() / 4.0f));
        l = (l > 0.0f) ? l : 0.0f;
        uint32_t lv = (l >= 4294967296.0f) ? 0xffffffffu : (uint32_t)l;
        return (int)std::min<uint32_t>(lv, 16u);
    }
    AxisMapping on_reduced_source(int levels) const {  // :60-67
        float factor = (float)(1u << levels);
        AxisMapping m = *this;
        m.crop_offset = crop_offset / factor;
        m.crop_len = crop_len / factor;
        return m;
    }
    bool as_direct(int &off) const {  // :72-76
        auto same = [](float a, float b) { return std::fabs(a - b) < 0.001f; };
        float r = std::round(crop_offset);
        if (same(crop_len, (float)dst_len) && same(crop_offset, r)) {
            off = (int)r;
            return true;
        }
        return false;
    }
};

struct KernelPass {
    AxisMapping mapping;
    int perp_offset;
};

// returns number of passes (0 = direct)
static int plan_passes(const AxisMapping &h, const AxisMapping &v, KernelPass out[2]) {  // :122-145
    int ho = 0, vo = 0;
    bool hd = h.as_direct(ho), vd = v.as_direct(vo);
    if (hd && vd) return 0;
    if (!hd && vd) { out[0] = {h, vo}; return 1; }
    if (hd && !vd) { out[0] = {v, ho}; return 1; }
    if (v.scale() > h.scale()) { out[0] = {v, 0}; out[1] = {h, 0}; }
    else { out[0] = {h, 0}; out[1] = {v, 0}; }
    return 2;
}

static int resample_taps(float scale) {  // resample.wgsl:43-48
    float ks = std::fmax(scale, 1.0f);
    return (int)std::ceil(2.0f * (3.0f * ks)) + 1;
}

// ------------------------------------------------------------------------------------------------
// small RAII helpers
// ------------------------------------------------------------------------------------------------
// Balanced partition of a launch of the fused resample kernel (kernels.cu: k_resample_fused_int): the output rows of
// every (job, 64-column strip) are concatenated and cut into `max_blocks` equal contiguous shares (a multiple of the 8
// output rows a block produces per step).  Block b owns pieces [begin[b], begin[b+1]); every output row of every
// strip belongs to exactly one piece.
void partition_fused_rows(const int *job_index, const int *dst_w, const int *dst_h, int n_jobs, int max_blocks,
                          std::vector<dev::FusedPiece> &pieces, std::vector<int> &begin, int strip_cols_all = dev::kFusedStripCols,
                          const int *strip_cols_per_job = nullptr, int gran = 8) {
    pieces.clear(); begin.clear();
    long long total = 0;
    auto cols_of = [&](int i) { return strip_cols_per_job ? strip_cols_per_job[i] : strip_cols_all; };
    for (int i = 0; i < n_jobs; i++)
        if (dst_w[i] > 0 && dst_h[i] > 0) total += (long long)((dst_w[i] + cols_of(i) - 1) / cols_of(i)) * dst_h[i];
    if (total <= 0 || max_blocks <= 0) return;
    const int nblocks = (int)std::min<long long>((long long)max_blocks, (total + 7) / 8);
    // share per block: a multiple of `gran` rows.  8 = whole steps of the kernels; the grouped TMA kernel takes 2 (whole row
    // pairs): with 444 groups a share of 330.8 rows rounds to 332 instead of 336 -- every SM gets work (336 left two idle) and
    // the critical path is half a step shorter
    const long long g = gran > 0 ? gran : 8;
    const long long per_block = ((total + nblocks - 1) / nblocks + g - 1) / g * g;
    begin.push_back(0);
    long long room = per_block;
    for (int i = 0; i < n_jobs; i++) {
        if (dst_w[i] <= 0 || dst_h[i] <= 0) continue;
        const int strips = (dst_w[i] + cols_of(i) - 1) / cols_of(i);
        for (int st = 0; st < strips; st++) {
            int y = 0;
            while (y < dst_h[i]) {
                const int take = (int)std::min<long long>(room, dst_h[i] - y);
                pieces.push_back({job_index[i], st, y, y + take});
                y += take; room -= take;
                if (room == 0) { begin.push_back((int)pieces.size()); room = per_block; }
            }
        }
    }
    if (begin.back() != (int)pieces.size()) begin.push_back((int)pieces.size());
}

struct DevBuf {
    uint8_t *p = nullptr;
    size_t cap = 0;
    ~DevBuf() { if (p) cudaFree(p); }
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    cudaError_t ensure(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = n + n / 4 + 4096;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
};

struct PinnedBuf {
    uint8_t *p = nullptr;
    size_t cap = 0;
    ~PinnedBuf() { if (p) cudaFreeHost(p); }
    cudaError_t ensure(size_t n) {
        if (n <= cap) return cudaSuccess;
        uint8_t *np = nullptr;
        size_t want = n * 2 + 4096;
        cudaError_t e = cudaMallocHost(&np, want);
        if (e != cudaSuccess) return e;
        if (p) { memcpy(np, p, cap); cudaFreeHost(p); }
        p = np; cap = want;
        return cudaSuccess;
    }
};

struct NcclId { char b[128]; };
typedef int (*nccl_init_fn)(void **, int, NcclId, int);
static struct {
    void *lib = nullptr;
    int (*GetUniqueId)(NcclId *) = nullptr;
    nccl_init_fn CommInitRank = nullptr;
    int (*CommDestroy)(void *) = nullptr;
    int (*Broadcast)(const void *, void *, size_t, int, int, void *, cudaStream_t) = nullptr;
    int (*Send)(const void *, size_t, int, int, void *, cudaStream_t) = nullptr;
    int (*Recv)(void *, size_t, int, int, void *, cudaStream_t) = nullptr;
    int (*AllReduce)(const void *, void *, size_t, int, int, void *, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
} g_nccl;

static bool nccl_load(std::string &err) {
    if (g_nccl.lib) return true;
    // RTLD_NOLOAD first: reuse the NCCL already in the process (e.g. the one torch.distributed loaded)
    void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) { err = std::string("cannot load libnccl: ") + dlerror(); return false; }
    g_nccl.GetUniqueId = (int (*)(NcclId *))dlsym(h, "ncclGetUniqueId");
    g_nccl.CommInitRank = (nccl_init_fn)dlsym(h, "ncclCommInitRank");
    g_nccl.CommDestroy = (int (*)(void *))dlsym(h, "ncclCommDestroy");
    g_nccl.Broadcast = (int (*)(const void *, void *, size_t, int, int, void *, cudaStream_t))dlsym(h, "ncclBroadcast");
    g_nccl.Send = (int (*)(const void *, size_t, int, int, void *, cudaStream_t))dlsym(h, "ncclSend");
    g_nccl.Recv = (int (*)(void *, size_t, int, int, void *, cudaStream_t))dlsym(h, "ncclRecv");
    g_nccl.AllReduce = (int (*)(const void *, void *, size_t, int, int, void *, cudaStream_t))dlsym(h, "ncclAllReduce");
    g_nccl.GroupStart = (int (*)())dlsym(h, "ncclGroupStart");
    g_nccl.GroupEnd = (int (*)())dlsym(h, "ncclGroupEnd");
    g_nccl.GetErrorString = (const char *(*)(int))dlsym(h, "ncclGetErrorString");
    if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.CommDestroy || !g_nccl.Broadcast || !g_nccl.GroupStart ||
        !g_nccl.GroupEnd || !g_nccl.Send || !g_nccl.Recv || !g_nccl.AllReduce) { err = "libnccl lacks required symbols"; return false; }
    g_nccl.lib = h;
    return true;
}

// TMA descriptors of the input planes (k_resample_tma3 / k_resample_tma0): cuTensorMapEncodeTiled through the runtime's driver entry
// point, so libcuda is not a link-time dependency.  2-D, no swizzle, zero fill outside the plane.
typedef CUresult (*tmap_encode_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                   const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static tmap_encode_fn tmap_encoder() {
    static std::once_flag once;
    static tmap_encode_fn fn = nullptr;
    std::call_once(once, [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (tmap_encode_fn)p;
        else
            cudaGetLastError();
    });
    return fn;
}
// elem_bytes 1 (u8 planes) or 2 (the NV12 chroma plane as (u, v) texels); width in elements
static bool encode_plane_tmap(const uint8_t *p, int pitch, int width_elems, int rows, int elem_bytes, int box_w, int box_h,
                              CUtensorMap *out) {
    tmap_encode_fn enc = tmap_encoder();
    if (!enc || ((uintptr_t)p & 15) || (pitch & 15) || width_elems <= 0 || rows <= 0) return false;
    cuuint64_t dims[2] = {(cuuint64_t)width_elems, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)pitch};
    cuuint32_t box[2] = {(cuuint32_t)box_w, (cuuint32_t)box_h};
    cuuint32_t estr[2] = {1, 1};
    return enc(out, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_UINT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, (void *)p, dims, strides, box,
               estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// A caller's smr_input_frame once Renderer::read_frame has checked it.  Nothing is uploaded: tex holds the caller's plane
// pointers and pitches, which a reader of host frames replaces with those of its device copies.
struct FrameView {
    dev::Tex tex;
    struct Plane {
        const uint8_t *p = nullptr;   // nullptr: the format has no such plane
        size_t pitch = 0, row_bytes = 0, rows = 0;
        size_t span() const { return pitch * (rows - 1) + row_bytes; }   // first to last byte of the plane
    } plane[3];
};

// ------------------------------------------------------------------------------------------------
class Renderer {
  public:
    explicit Renderer(const smr_options &o) : opts_(o) {}
    ~Renderer();
    smr_status init();

    smr_status register_input(const char *id);
    smr_status unregister_input(const char *id);
    smr_status update_scene(const char *output_id, uint32_t w, uint32_t h, int32_t fmt, const smr_component *root);
    smr_status unregister_output(const char *id);
    smr_status set_layouts(const char *output_id, uint32_t w, uint32_t h, int32_t fmt, uint32_t root_w, uint32_t root_h,
                           const char *const *child_ids, uint32_t n_children, const smr_render_layout *layouts, uint32_t n);
    smr_status render_begin(uint64_t pts, const smr_input_frame *in, uint32_t n_in, smr_output_frame *out, uint32_t n_out);
    smr_status render_end();
    smr_status render_end_all();
    smr_status preprocess_frame(const smr_input_frame *f, uint32_t ow, uint32_t oh, void *rgba, uint32_t pitch, int32_t mem_kind,
                                bool premultiply = false);
    smr_status render_text(uint32_t w, uint32_t h, smr_rgba bg, const smr_glyph *glyphs, uint32_t n, const smr_atlas *mask,
                           const smr_atlas *color, int32_t color_mode, void *rgba, uint32_t pitch, int32_t mem_kind);
    smr_status debug_set_inputs(uint64_t pts, const smr_input_frame *in, uint32_t n_in);
    smr_status debug_layouts(const char *output_id, uint64_t pts, smr_render_layout *out, uint32_t cap, uint32_t *n,
                             uint32_t *rw, uint32_t *rh);
    smr_status debug_fused_jobs(smr_fused_job_info *out, uint32_t cap, uint32_t *n);
    smr_status debug_composite_layers(smr_composite_layer_info *out, uint32_t cap, uint32_t *n);
    smr_status debug_resample_stages(smr_resample_stage_info *out, uint32_t cap, uint32_t *n, int32_t *convert_kinds,
                                     uint32_t convert_cap, uint32_t *n_convert);
    void stats(smr_stats *s) { std::lock_guard<std::mutex> g(mu_); *s = stats_; }
    void *stream() { return (void *)stream_; }
    const char *last_error() { return err_.c_str(); }
    void set_error(const std::string &e) { err_ = e; }
    std::mutex mu_;

  private:
    struct Input {
        bool has_frame = false;
        dev::Tex tex;           // planes as they sit in HBM
        DevBuf planes[kTicksInFlight][3];    // owned copies of host frames, one set per tick in flight
        Resolution res;
        int node_tex = -1;      // index in the tick's texture table of the materialised RGBA8 node texture
        int raw_tex = -1;       // index of the virtual (fused K1/K2) texture
    };
    struct Output {
        OutputNode node;
        int32_t format = 0;
        Resolution res;
        DevBuf planes[kTicksInFlight][3];       // device staging for host outputs, one set per tick in flight: the read-back of
                                                // tick k runs on its own stream while tick k + 1 composes into the next set
        // smr_set_layouts: the caller flattened the scene itself (the reference's scene/** stays in Rust); used instead
        // of `node` until the next smr_update_scene of this output
        // tile plan of the composite (direct-tile owners + cost-sorted list of the tiles that are left), kept while the
        // flattened layers and the resamples feeding them stay the same (a static scene plans once)
        uint64_t tile_key = 0;
        bool tile_key_valid = false;
        std::vector<int> tile_owner_layer;       // per tile: index of the layer whose child is shown there 1:1 and alone, or -1
        std::vector<uint32_t> tile_list;         // tiles that are left for the composite, most expensive first
        bool flat = false;
        Resolution flat_root;
        std::vector<std::string> flat_children;
        std::vector<RenderLayout> flat_layouts;
    };
    struct WeightKey {
        uint32_t scale_bits, offset_bits;
        int32_t n_out;
        bool operator<(const WeightKey &o) const {
            return std::tie(scale_bits, offset_bits, n_out) < std::tie(o.scale_bits, o.offset_bits, o.n_out);
        }
    };
    struct WeightEntry {
        float *weights = nullptr, *inv = nullptr;
        int32_t *first = nullptr;
        int taps = 0;
        uint64_t last_used = 0;
    };

    // arenas ----------------------------------------------------------------------------------
    size_t param_alloc(size_t bytes) {  // returns offset in the param arena (256-byte aligned: tensor maps need 64)
        size_t off = (param_used_ + 255) & ~(size_t)255;
        param_used_ = off + bytes;
        if (param_host_.size() < param_used_) param_host_.resize(param_used_ * 2);
        return off;
    }
    size_t param_put(const void *p, size_t bytes) {
        size_t off = param_alloc(bytes);
        if (bytes) memcpy(param_host_.data() + off, p, bytes);
        return off;
    }
    // the device structs of a list of host records as one array
    template <class Rec, class Dev> size_t param_put_all(const std::vector<Rec> &recs, Dev Rec::*dev) {
        size_t off = param_alloc(sizeof(Dev) * recs.size());
        for (size_t i = 0; i < recs.size(); i++) memcpy(param_host_.data() + off + i * sizeof(Dev), &(recs[i].*dev), sizeof(Dev));
        return off;
    }
    size_t frame_alloc(size_t bytes) {
        size_t off = (frame_used_ + 511) & ~(size_t)511;
        frame_used_ = off + bytes;
        return off;
    }

    smr_status check_output(uint32_t w, uint32_t h, int32_t fmt);
    smr_status read_frame(const smr_input_frame &f, FrameView &v);
    template <class Use> smr_status select_inputs(uint64_t pts, const smr_input_frame *in, uint32_t n_in, Use use);
    smr_status upload_input(Input &I, const smr_input_frame &f);
    Resolution output_children(const Output &o, const OutputNode &node, uint64_t pts, std::vector<Input *> &child_in,
                               std::vector<std::optional<Resolution>> &child_res);
    std::vector<RenderLayout> output_layouts(const Output &o, OutputNode &node, uint64_t pts,
                                             const std::vector<std::optional<Resolution>> &child_res, Resolution root);
    smr_status plan_output(Output &o, smr_output_frame &of, uint64_t pts);
    smr_status child_texture(Input &in, RenderLayout &l, int &tex_index, int &tex_w, int &tex_h);
    template <class Launch> smr_status write_rgba(void *rgba, uint32_t pitch, int32_t mem_kind, uint32_t w, uint32_t h, Launch launch);
    smr_status get_weights(const KernelPass &p, WeightEntry &out);
    int materialised_input(Input &in);
    int try_fused_resample(Input &in, const struct AxisMapping &hm, const struct AxisMapping &vm, int dw, int dh);
    int source_tmaps(const dev::Tex &t, int src_class);
    int add_texture(const dev::Tex &t, bool opaque, size_t frame_off = SIZE_MAX, int fused_job = -1) {
        plan_.tex.push_back({t, opaque, frame_off, fused_job});
        return (int)plan_.tex.size() - 1;
    }
    void prepare_layer(const RenderLayout &l, int W, int H, int tex_index, int tex_w, int tex_h, dev::LayerDev &d, bool &skip);
    void shader_color(const RGBA &c, float out[4]) const;

    smr_options opts_;
    cudaStream_t stream_ = nullptr;
    SceneState scene_;
    std::map<std::string, Input> inputs_;
    std::map<std::string, Output> outputs_;
    std::string err_;
    smr_stats stats_ = {};
    uint64_t tick_ = 0;

    // per-tick plan: host records; frame-arena and parameter-arena offsets become device addresses in render_begin once
    // both arenas are sized
    struct TexRec {             // one entry of the tick's texture table
        dev::Tex tex;
        bool opaque;            // every texel's alpha is 255 by construction
        size_t frame_off;       // p0 lives in the frame arena at this offset (SIZE_MAX: tex.p0 is a device pointer already)
        int fused_job;          // the fused resample that writes it, or -1
    };
    struct FusedRec {
        dev::FusedJob job;
        dev::FusedKernel kernel;
        int src_tex;            // the job's source (texture table)
        size_t dst_off;         // frame-arena offset of its RGBA8 output
        int tmap_idx;           // first of its three entries in `tmaps`, or -1
        size_t direct_off;      // param-arena offset of the direct-tile map it writes for (SIZE_MAX: none)
    };
    struct StageRec {           // one generic resample pass
        dev::ResampleJob job;
        int src_tex;            // source from the texture table, or -1: the frame-arena f16 at src_off
        size_t src_off, dst_off;
    };
    struct OutputRec { dev::OutputJob job; int src_tex; };
    struct CompositeRec {
        dev::CompositeJob job; size_t layers_off, masks_off;
        size_t out_frame_off = SIZE_MAX;  // the target is an RGBA8 frame-arena texture (SIZE_MAX: the caller's planes)
        size_t direct_off = SIZE_MAX;     // param-arena offset of the direct-tile map (SIZE_MAX: none)
        std::vector<int> direct_owner;    // per tile: the fused job that writes its output bytes, or -1
        bool use_list = false;            // compacted launch over `list` (tiles left for the composite, most expensive first)
        std::vector<uint32_t> list;
        size_t list_off = SIZE_MAX;       // param-arena offset of `list`
    };
    struct PendingCopy { void *dst; size_t dpitch; const void *src; size_t spitch; size_t width, height; };
    struct Fill { uint8_t *p[3]; int pitch[3]; int w, h, fmt; uint8_t yuv[3]; };
    struct TickPlan {
        std::vector<TexRec> tex;
        std::vector<StageRec> stages[3];      // box passes, first passes, last passes
        std::vector<FusedRec> fused;
        std::vector<CUtensorMap> tmaps;       // three per TMA job
        std::vector<dev::WeightJob> weight_jobs;
        std::vector<std::pair<int, size_t>> convert_jobs;  // (raw tex index, frame offset of RGBA8)
        std::vector<CompositeRec> composites;
        std::vector<OutputRec> outputs;
        std::vector<Fill> fills;
        std::vector<PendingCopy> d2h;
        std::map<std::tuple<int, uint32_t, uint32_t, uint32_t, uint32_t, int, int>, int> resample_cache;
        void clear() {   // keeps the vectors' capacity
            tex.clear();
            for (auto &s : stages) s.clear();
            fused.clear(); tmaps.clear(); weight_jobs.clear(); convert_jobs.clear();
            composites.clear(); outputs.clear(); fills.clear(); d2h.clear(); resample_cache.clear();
        }
    } plan_;
    void plan_tiles(Output &o, CompositeRec &pc, const std::vector<dev::LayerDev> &layers, int W, int H);
    std::vector<WeightKey> new_weight_keys_;   // cache entries whose k_weights launch is not enqueued yet
    void rollback_weights();                   // a tick that fails before that launch must not leave them behind
    // TMA kernels of the fused resample: descriptors of the source planes, cached per (pointer, pitch, size, kind)
    struct TmapKey {
        uintptr_t p; int pitch, w, h, kind;
        bool operator<(const TmapKey &o) const { return std::tie(p, pitch, w, h, kind) < std::tie(o.p, o.pitch, o.w, o.h, o.kind); }
    };
    std::map<TmapKey, CUtensorMap> tmap_cache_;
    // any-ratio TMA kernel: per (horizontal mapping, strip width) the lane <-> column-pair deal of every strip
    std::map<std::tuple<uint32_t, uint32_t, int32_t, int32_t>, uint8_t *> lane_perms_;
    const uint8_t *lane_perm(float scale, float offset, int n_out, int cols);
    bool plane_tmap(const uint8_t *p, int pitch, int w, int h, int kind, CUtensorMap *out);
    bool direct_k11_ = true;                   // SMR_DIRECT_K11=0: A/B switch, every tile goes through the composite

    std::vector<uint8_t> param_host_;  // built here, copied to pinned, then to device
    size_t param_used_ = 0;
    PinnedBuf param_pinned_[kTicksInFlight];   // one per tick in flight: tick n+1 .. n+3 are prepared and uploaded
    DevBuf param_dev_[kTicksInFlight];         // while tick n is still executing
    size_t frame_used_ = 0;
    DevBuf frame_dev_;
    std::map<WeightKey, WeightEntry> weights_;
    // up to two ticks in flight: uploads of tick n+1 (copy stream) overlap the kernels of tick n
    cudaStream_t copy_stream_ = nullptr, copy_stream2_ = nullptr;   // uploads alternate between two streams (two DMA engines)
    cudaStream_t d2h_stream_ = nullptr;      // read-back of host outputs: overlaps the next tick's kernels
    cudaEvent_t kernels_done_[kTicksInFlight] = {};
    cudaEvent_t h2d_done2_[kTicksInFlight] = {};
    int upload_rr_ = 0;
    cudaEvent_t h2d_done_[kTicksInFlight] = {}, tick_done_[kTicksInFlight] = {};
    // the tick's exchange step overlaps the previous tick's kernels: NCCL runs on its own stream, ordered after
    // everything submitted BEFORE the most recent tick and before the next one
    cudaStream_t comm_stream_ = nullptr;
    cudaEvent_t comm_done_ = nullptr, tick_start_ = nullptr;
    bool comm_pending_ = false, tick_started_ = false;
    std::deque<int> inflight_;
    int slot_ = 0;
    bool uploaded_ = false;
    int sm_count_ = 132;
    void drain() {
        if (stream_) cudaStreamSynchronize(stream_);
        if (copy_stream_) cudaStreamSynchronize(copy_stream_);
        if (copy_stream2_) cudaStreamSynchronize(copy_stream2_);
        if (d2h_stream_) cudaStreamSynchronize(d2h_stream_);
        if (comm_stream_) cudaStreamSynchronize(comm_stream_);
        fold_profile();
        inflight_.clear();
    }
    void fold_profile();
    bool host_only_ = false;
    DevBuf pre_planes_[3], pre_out_;   // FramePreProcessor scratch (input_texture / rescale_texture / download_buffer)
    // optional per-kernel-class device timing (cudaEvents on the launching stream)
    void prof_mark(int kernel_class);
    bool profiling_ = false;
    std::vector<cudaEvent_t> prof_events_;
    size_t prof_next_event_ = 0;
    std::vector<std::pair<cudaEvent_t, int>> prof_marks_;
    smr_kernel_times prof_ = {};
    // NCCL communicator for shared-input replication (SURVEY 8e); libnccl is dlopen'ed on first use
    void *nccl_comm_ = nullptr;
    int comm_rank_ = 0, comm_size_ = 1;
    int32_t *barrier_word_ = nullptr;            // 4 device bytes the per-tick all-reduce of the peer modes runs on
    std::vector<void *> peer_own_, peer_opened_; // pools of smr_peer_pool_alloc / smr_peer_pool_open still alive
  public:
    smr_status comm_init(const uint8_t *id, int rank, int nranks);
    smr_status comm_exchange(const smr_input_frame *frames, uint32_t n, const int32_t *roots, const uint64_t *consumers,
                             uint32_t flags);
    smr_status comm_destroy();
    smr_status comm_pull(const smr_input_frame *frames, const smr_input_frame *peer_frames, uint32_t n, const int32_t *roots,
                         const uint64_t *consumers);
    smr_status comm_tick_barrier();   // caller holds mu_
    smr_status peer_pool_alloc(size_t bytes, void **dev_ptr, uint8_t handle[64]);
    smr_status peer_pool_open(const uint8_t handle[64], void **dev_ptr);
    smr_status peer_pool_close(void *dev_ptr);
    smr_status peer_pool_free(void *dev_ptr);
    smr_status set_profiling(int enabled);
    void kernel_times(smr_kernel_times *out) { std::lock_guard<std::mutex> g(mu_); *out = prof_; }
};

Renderer::~Renderer() {
    if (stream_) {
        cudaSetDevice(opts_.cuda_device);
        cudaStreamSynchronize(stream_);
        if (copy_stream_) { cudaStreamSynchronize(copy_stream_); cudaStreamDestroy(copy_stream_); }
        if (copy_stream2_) { cudaStreamSynchronize(copy_stream2_); cudaStreamDestroy(copy_stream2_); }
        if (d2h_stream_) { cudaStreamSynchronize(d2h_stream_); cudaStreamDestroy(d2h_stream_); }
        for (int i = 0; i < kTicksInFlight; i++) if (kernels_done_[i]) cudaEventDestroy(kernels_done_[i]);
        for (int i = 0; i < kTicksInFlight; i++) if (h2d_done2_[i]) cudaEventDestroy(h2d_done2_[i]);
        if (comm_stream_) { cudaStreamSynchronize(comm_stream_); cudaStreamDestroy(comm_stream_); }
        if (comm_done_) cudaEventDestroy(comm_done_);
        if (tick_start_) cudaEventDestroy(tick_start_);
        for (int i = 0; i < kTicksInFlight; i++) { if (h2d_done_[i]) cudaEventDestroy(h2d_done_[i]); if (tick_done_[i]) cudaEventDestroy(tick_done_[i]); }
        if (nccl_comm_) { g_nccl.CommDestroy(nccl_comm_); nccl_comm_ = nullptr; }
        for (auto &kv : weights_) {
            cudaFree(kv.second.weights); cudaFree(kv.second.inv); cudaFree(kv.second.first);
        }
        for (auto &kv : lane_perms_) cudaFree(kv.second);
        for (void *p : peer_opened_) cudaIpcCloseMemHandle(p);
        for (void *p : peer_own_) cudaFree(p);
        if (barrier_word_) cudaFree(barrier_word_);
        cudaStreamDestroy(stream_);
    }
}

static double eotf_f64(double c) { return c <= 0.04045 ? c / 12.92 : std::pow((c + 0.055) / 1.055, 2.4); }  // wgpu/utils.rs:74-81
// sRGB encode thresholds (numeric contract NC-4): byte k + 1 starts where linear light reaches eotf((k + 0.5) / 255); the
// device table and the host encoder use the same values
static const std::array<float, 255> kSrgbEncodeThr = [] {
    std::array<float, 255> thr;
    for (int k = 0; k < 255; k++) thr[k] = (float)eotf_f64(((double)k + 0.5) / 255.0);
    return thr;
}();

smr_status Renderer::init() {
    if (opts_.max_layouts_count == 0) opts_.max_layouts_count = 100;  // DEFAULT_MAX_LAYOUTS_COUNT
    if (opts_.max_layouts_count > 1024) opts_.max_layouts_count = 1024;
    if (opts_.cuda_device == -1) { host_only_ = true; return SMR_OK; }  // scene/layout inspection only
    if (const char *e = getenv("SMR_DIRECT_K11")) direct_k11_ = e[0] != '0';
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        set_error("no CUDA device: the H100 compositor has no CPU fallback");
        return SMR_ERR_CUDA;
    }
    if (opts_.cuda_device < 0 || opts_.cuda_device >= n) {
        set_error("cuda_device out of range");
        return SMR_ERR_INVALID_ARGUMENT;
    }
    int cc_major = 0, cc_minor = 0;
    CUDA_OK(cudaDeviceGetAttribute(&cc_major, cudaDevAttrComputeCapabilityMajor, opts_.cuda_device));
    CUDA_OK(cudaDeviceGetAttribute(&cc_minor, cudaDevAttrComputeCapabilityMinor, opts_.cuda_device));
    if (cc_major != 9 || cc_minor != 0) {  // sm_90a code loads on compute capability 9.0 alone: say so up front
        set_error("device has compute capability " + std::to_string(cc_major) + "." + std::to_string(cc_minor) +
                  "; this library is built for sm_90a (H100) only");
        return SMR_ERR_UNSUPPORTED;
    }
    CUDA_OK(cudaSetDevice(opts_.cuda_device));
    CUDA_OK(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
    CUDA_OK(cudaStreamCreateWithFlags(&copy_stream_, cudaStreamNonBlocking));
    CUDA_OK(cudaStreamCreateWithFlags(&copy_stream2_, cudaStreamNonBlocking));
    CUDA_OK(cudaStreamCreateWithFlags(&d2h_stream_, cudaStreamNonBlocking));
    for (int i = 0; i < kTicksInFlight; i++) CUDA_OK(cudaEventCreateWithFlags(&kernels_done_[i], cudaEventDisableTiming));
    for (int i = 0; i < kTicksInFlight; i++) CUDA_OK(cudaEventCreateWithFlags(&h2d_done2_[i], cudaEventDisableTiming));
    CUDA_OK(cudaStreamCreateWithFlags(&comm_stream_, cudaStreamNonBlocking));
    CUDA_OK(cudaEventCreateWithFlags(&comm_done_, cudaEventDisableTiming));
    CUDA_OK(cudaEventCreateWithFlags(&tick_start_, cudaEventDisableTiming));
    CUDA_OK(cudaDeviceGetAttribute(&sm_count_, cudaDevAttrMultiProcessorCount, opts_.cuda_device));
    for (int i = 0; i < kTicksInFlight; i++) {
        CUDA_OK(cudaEventCreateWithFlags(&h2d_done_[i], cudaEventDisableTiming));
        CUDA_OK(cudaEventCreateWithFlags(&tick_done_[i], cudaEventDisableTiming));
    }
    float u8n[256], dec[256];
    for (int b = 0; b < 256; b++) {
        u8n[b] = (float)b / 255.0f;
        dec[b] = (float)eotf_f64((double)b / 255.0);
    }
    dev::upload_tables(u8n, dec, kSrgbEncodeThr.data());
    CUDA_OK(cudaGetLastError());
    return SMR_OK;
}

smr_status Renderer::register_input(const char *id) {
    if (!id) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    inputs_.emplace(std::piecewise_construct, std::forward_as_tuple(id), std::forward_as_tuple());
    return SMR_OK;
}

smr_status Renderer::unregister_input(const char *id) {
    if (!id) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    if (!host_only_) { cudaSetDevice(opts_.cuda_device); drain(); }
    inputs_.erase(id);
    return SMR_OK;
}

smr_status Renderer::unregister_output(const char *id) {
    if (!id) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    if (!host_only_) { cudaSetDevice(opts_.cuda_device); drain(); }
    outputs_.erase(id);
    scene_.unregister_output(id);
    return SMR_OK;
}

smr_status Renderer::check_output(uint32_t w, uint32_t h, int32_t fmt) {
    if (fmt < SMR_OUT_PLANAR_YUV420 || fmt > SMR_OUT_NV12) { set_error("unsupported output format"); return SMR_ERR_UNSUPPORTED; }
    if (w == 0 || h == 0 || w > 16384 || h > 16384) { set_error("output resolution out of range"); return SMR_ERR_INVALID_ARGUMENT; }
    return SMR_OK;
}

smr_status Renderer::update_scene(const char *output_id, uint32_t w, uint32_t h, int32_t fmt, const smr_component *root) {
    if (!output_id || !root) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    if (smr_status st = check_output(w, h, fmt); st != SMR_OK) return st;
    Component c;
    std::string err;
    if (!component_from_c(root, c, err)) {
        set_error(err);
        return err.find("outside") != std::string::npos ? SMR_ERR_UNSUPPORTED : SMR_ERR_INVALID_ARGUMENT;
    }
    OutputNode node;
    if (!scene_.update_scene(output_id, c, {w, h}, node, err)) {
        set_error(err);
        return SMR_ERR_SCENE;
    }
    Output &o = outputs_[output_id];
    o.node = std::move(node);
    o.format = fmt;
    o.res = {w, h};
    o.flat = false; o.flat_layouts.clear(); o.flat_children.clear();
    return SMR_OK;
}

// One smr_render_layout (type and masks_len checked by the caller)
static RenderLayout layout_from_c(const smr_render_layout &d) {
    RenderLayout l;
    l.kind = (RenderLayout::Kind)d.type;
    l.top = d.top; l.left = d.left; l.width = d.width; l.height = d.height; l.rotation_degrees = d.rotation_degrees;
    l.border_radius = {d.border_radius[0], d.border_radius[1], d.border_radius[2], d.border_radius[3]};
    l.color = {d.color.r, d.color.g, d.color.b, d.color.a};
    l.border_color = {d.border_color.r, d.border_color.g, d.border_color.b, d.border_color.a};
    l.border_width = d.border_width; l.blur_radius = d.blur_radius;
    l.index = (size_t)std::max(d.child_index, 0);
    l.crop = {d.crop_top, d.crop_left, d.crop_width, d.crop_height};
    for (int m = 0; m < d.masks_len; m++) {
        Mask mk;
        mk.radius = {d.masks[m].radius[0], d.masks[m].radius[1], d.masks[m].radius[2], d.masks[m].radius[3]};
        mk.top = d.masks[m].top; mk.left = d.masks[m].left; mk.width = d.masks[m].width; mk.height = d.masks[m].height;
        l.masks.push_back(mk);
    }
    return l;
}

// The flattened boundary (SURVEY 8b, second form): RenderLayout[] exactly as NestedLayout::flatten returns them and
// LayoutNodeParams consumes them (transformations/layout/params.rs:169-333), child node indices resolved through
// `child_ids` (the node's children in DFS order, scene/layout.rs:84-93).
smr_status Renderer::set_layouts(const char *output_id, uint32_t w, uint32_t h, int32_t fmt, uint32_t root_w, uint32_t root_h,
                                 const char *const *child_ids, uint32_t n_children, const smr_render_layout *layouts, uint32_t n) {
    if (!output_id || (n && !layouts) || (n_children && !child_ids)) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    if (smr_status st = check_output(w, h, fmt); st != SMR_OK) return st;
    std::vector<RenderLayout> ls(n);
    for (uint32_t i = 0; i < n; i++) {
        const smr_render_layout &d = layouts[i];
        RenderLayout &l = ls[i];
        if (d.type < 0 || d.type > 2 || d.masks_len < 0 || d.masks_len > SMR_MAX_MASKS) { set_error("malformed layout"); return SMR_ERR_INVALID_ARGUMENT; }
        if (d.type == 0 && (d.child_index < 0 || (uint32_t)d.child_index >= n_children)) { set_error("child index outside child_ids"); return SMR_ERR_INVALID_ARGUMENT; }
        if (d.type == 0 && !(std::isfinite(d.crop_top) && std::isfinite(d.crop_left) && std::isfinite(d.crop_width) &&
                             std::isfinite(d.crop_height))) {
            set_error("texture layout crop is not finite");
            return SMR_ERR_INVALID_ARGUMENT;
        }
        l = layout_from_c(d);
    }
    Output &o = outputs_[output_id];
    o.format = fmt;
    o.res = {w, h};
    o.flat = true;
    o.flat_root = {root_w, root_h};
    o.flat_children.clear();
    for (uint32_t i = 0; i < n_children; i++) o.flat_children.push_back(child_ids[i] ? child_ids[i] : "");
    o.flat_layouts = std::move(ls);
    return SMR_OK;
}

// ------------------------------------------------------------------------------------------------
// populate_inputs (state/render_loop.rs:19-42, state/input_texture.rs:69-201)
// ------------------------------------------------------------------------------------------------
static bool plane_layout(int fmt, uint32_t w, uint32_t h, int plane, size_t &row_bytes, size_t &rows) {
    uint32_t cw = w / 2, ch = h / 2;
    switch (fmt) {
        case SMR_FRAME_PLANAR_YUV420:
        case SMR_FRAME_PLANAR_YUVJ420:
            if (plane == 0) { row_bytes = w; rows = h; return true; }
            if (plane <= 2) { row_bytes = cw; rows = ch; return true; }
            return false;
        case SMR_FRAME_NV12:
            if (plane == 0) { row_bytes = w; rows = h; return true; }
            if (plane == 1) { row_bytes = (size_t)cw * 2; rows = ch; return true; }
            return false;
        case SMR_FRAME_PLANAR_YUV422:   // texture/planar_yuv.rs:72-77
            if (plane == 0) { row_bytes = w; rows = h; return true; }
            if (plane <= 2) { row_bytes = cw; rows = h; return true; }
            return false;
        case SMR_FRAME_PLANAR_YUV444:   // texture/planar_yuv.rs:78-83
            if (plane <= 2) { row_bytes = w; rows = h; return true; }
            return false;
        case SMR_FRAME_UYVY422:
        case SMR_FRAME_YUYV422:         // texture/interleaved_yuv422.rs:12-36: (w/2) x h texels of 4 bytes
            if (plane == 0) { row_bytes = (size_t)cw * 4; rows = h; return true; }
            return false;
        case SMR_FRAME_BGRA:
        case SMR_FRAME_ARGB:
        case SMR_FRAME_RGBA8:
            if (plane == 0) { row_bytes = (size_t)w * 4; rows = h; return true; }
            return false;
        default: return false;
    }
}

static bool tex_kind_of_format(int fmt, dev::Tex &t) {   // FrameData variant -> texture kind (input_texture.rs:69-150)
    switch (fmt) {
        case SMR_FRAME_PLANAR_YUV420: t.kind = dev::TEX_YUV420; return true;
        case SMR_FRAME_PLANAR_YUVJ420: t.kind = dev::TEX_YUV420; t.full_range = 1; return true;
        case SMR_FRAME_NV12: t.kind = dev::TEX_NV12; return true;
        case SMR_FRAME_BGRA: t.kind = dev::TEX_BGRA; return true;
        case SMR_FRAME_ARGB: t.kind = dev::TEX_ARGB; return true;
        case SMR_FRAME_RGBA8: t.kind = dev::TEX_RGBA8; return true;
        case SMR_FRAME_PLANAR_YUV422: t.kind = dev::TEX_YUV422; return true;
        case SMR_FRAME_PLANAR_YUV444: t.kind = dev::TEX_YUV444; return true;
        case SMR_FRAME_UYVY422: t.kind = dev::TEX_UYVY; return true;
        case SMR_FRAME_YUYV422: t.kind = dev::TEX_YUYV; return true;
        default: return false;
    }
}

static void set_tex_plane(dev::Tex &t, int p, const uint8_t *ptr, size_t pitch) {
    (p == 0 ? t.p0 : p == 1 ? t.p1 : t.p2) = ptr;
    (p == 0 ? t.pitch0 : p == 1 ? t.pitch1 : t.pitch2) = (int)pitch;
}

// The largest input frame side.  The kernels' fixed .25 / .75 chroma taps for even 4:2:0 sizes are proved up to this bound
// (tests/test_oracle_kat.py reads it from here).
static constexpr uint32_t kMaxFrameDim = 16384;
static bool frame_size_ok(const smr_input_frame &f) {
    return f.width >= 2 && f.height >= 2 && f.width <= kMaxFrameDim && f.height <= kMaxFrameDim;
}

// The checks every reader of a caller's frame applies (smr_render, smr_preprocess_frame, the exchange calls)
smr_status Renderer::read_frame(const smr_input_frame &f, FrameView &v) {
    if (!frame_size_ok(f)) { set_error("input frame resolution out of range"); return SMR_ERR_INVALID_ARGUMENT; }
    v = FrameView();
    if (!tex_kind_of_format(f.format, v.tex)) { set_error("unsupported input frame format"); return SMR_ERR_UNSUPPORTED; }
    v.tex.width = (int)f.width; v.tex.height = (int)f.height;
    // the kernels read these as one 4-byte word per texel
    const bool texel4 = f.format == SMR_FRAME_UYVY422 || f.format == SMR_FRAME_YUYV422 || f.format == SMR_FRAME_RGBA8 ||
                        f.format == SMR_FRAME_BGRA || f.format == SMR_FRAME_ARGB;
    // 4:2:0 luma is read a pixel pair (2 bytes) at a time, NV12 chroma a {u, v} pair at a time (node_texel, yuv_quad,
    // k_resample_fused_int, half_row_sums); planar U / V are read byte by byte
    const bool yuv420 = f.format == SMR_FRAME_PLANAR_YUV420 || f.format == SMR_FRAME_PLANAR_YUVJ420 || f.format == SMR_FRAME_NV12;
    for (int p = 0; p < 3; p++) {
        FrameView::Plane &P = v.plane[p];
        if (!plane_layout(f.format, f.width, f.height, p, P.row_bytes, P.rows)) continue;
        if (!f.planes[p]) { set_error("input plane pointer is null"); return SMR_ERR_INVALID_ARGUMENT; }
        P.pitch = f.pitch[p] ? f.pitch[p] : P.row_bytes;
        if (P.pitch < P.row_bytes) { set_error("input plane pitch is smaller than a row"); return SMR_ERR_INVALID_ARGUMENT; }
        if (f.mem_kind == SMR_MEM_DEVICE && texel4 && (((uintptr_t)f.planes[p] | P.pitch) & 3)) {
            set_error("4-byte texel planes must be 4-byte aligned (pointer and pitch)");
            return SMR_ERR_INVALID_ARGUMENT;
        }
        if (f.mem_kind == SMR_MEM_DEVICE && yuv420 && (p == 0 || f.format == SMR_FRAME_NV12) && (((uintptr_t)f.planes[p] | P.pitch) & 1)) {
            set_error("4:2:0 luma and NV12 chroma planes must be 2-byte aligned (pointer and pitch)");
            return SMR_ERR_INVALID_ARGUMENT;
        }
        P.p = (const uint8_t *)f.planes[p];
        set_tex_plane(v.tex, p, P.p, P.pitch);
    }
    return SMR_OK;
}

// A frame set as the scene and the render loop see it: the scene records the input resolutions (state.rs:233-239), and a
// registered input has a live frame when the set holds one with its id -- the last such -- that is not stale
// (Duration::saturating_sub(frame_set.pts, timeout) > frame.pts, render_loop.rs:29-32).  `use(input, frame or nullptr)` runs
// for every registered input before it is marked live; the first status other than SMR_OK ends the walk.
template <class Use> smr_status Renderer::select_inputs(uint64_t pts, const smr_input_frame *in, uint32_t n_in, Use use) {
    std::map<std::string, Resolution> res_map;
    for (uint32_t i = 0; i < n_in; i++)
        if (in[i].input_id) res_map[in[i].input_id] = {in[i].width, in[i].height};
    scene_.register_render_event(pts, std::move(res_map));
    const uint64_t lim = pts > opts_.stream_fallback_timeout_ns ? pts - opts_.stream_fallback_timeout_ns : 0;
    for (auto &kv : inputs_) {
        Input &I = kv.second;
        const smr_input_frame *f = nullptr;
        for (uint32_t i = 0; i < n_in; i++)
            if (in[i].input_id && kv.first == in[i].input_id) f = &in[i];
        if (f && lim > f->pts_ns) f = nullptr;
        I.has_frame = false;
        if (smr_status st = use(I, f); st != SMR_OK) return st;
        if (f) { I.has_frame = true; I.res = {f->width, f->height}; }
    }
    return SMR_OK;
}

// a live frame, checked and uploaded: host planes go to the slot's buffers on alternating copy streams
smr_status Renderer::upload_input(Input &I, const smr_input_frame &f) {
    FrameView v;
    if (smr_status st = read_frame(f, v); st != SMR_OK) return st;
    for (int p = 0; p < 3 && f.mem_kind != SMR_MEM_DEVICE; p++) {
        const FrameView::Plane &P = v.plane[p];
        if (!P.p) continue;
        DevBuf &buf = I.planes[slot_][p];
        CUDA_OK(buf.ensure(P.row_bytes * P.rows));
        cudaStream_t cs = (upload_rr_++ & 1) ? copy_stream2_ : copy_stream_;
        if (P.pitch == P.row_bytes)   // tightly packed (the reference's bytes::Bytes planes): one linear DMA
            CUDA_OK(cudaMemcpyAsync(buf.p, P.p, P.row_bytes * P.rows, cudaMemcpyHostToDevice, cs));
        else
            CUDA_OK(cudaMemcpy2DAsync(buf.p, P.row_bytes, P.p, P.pitch, P.row_bytes, P.rows, cudaMemcpyHostToDevice, cs));
        uploaded_ = true;
        stats_.h2d_bytes += P.row_bytes * P.rows;
        set_tex_plane(v.tex, p, buf.p, P.row_bytes);
    }
    I.tex = v.tex;
    I.raw_tex = add_texture(v.tex, v.tex.kind == dev::TEX_YUV420 || v.tex.kind == dev::TEX_NV12 || v.tex.kind >= dev::TEX_YUV422);
    return SMR_OK;
}

// K1/K2 materialised once per tick for inputs that feed a resampler pass (taps x conversion is wasteful)
int Renderer::materialised_input(Input &in) {
    if (in.node_tex >= 0) return in.node_tex;
    if (in.tex.kind == dev::TEX_RGBA8) { in.node_tex = in.raw_tex; return in.node_tex; }
    size_t pitch = (size_t)in.tex.width * 4;
    size_t off = frame_alloc(pitch * in.tex.height);
    dev::Tex t;
    t.kind = dev::TEX_RGBA8;
    t.width = in.tex.width; t.height = in.tex.height;
    t.pitch0 = (int)pitch;
    in.node_tex = add_texture(t, plan_.tex[in.raw_tex].opaque, off);
    plan_.convert_jobs.push_back({in.raw_tex, off});
    return in.node_tex;
}

// The common case -- a YUV input scaled on both axes, horizontal pass first, no box pre-pass -- runs as ONE
// kernel (k_resample_fused).  Returns the texture-table index of the result, -1 when not eligible
// (the generic multi-pass path is used), -2 on error.
int Renderer::try_fused_resample(Input &in, const AxisMapping &hm_in, const AxisMapping &vm_in, int dw, int dh) {
    const dev::Tex &t = in.tex;
    const int src_class = dev::fused_source_class(t.kind);
    if (src_class < 0) return -1;
    if (src_class < 2 && ((t.width | t.height) & 1)) return -1;
    // interleaved 4:2:2: texel-centre fast form holds for even widths >= 8 and 4-byte aligned rows
    if (src_class >= 2 && ((t.width & 1) || t.width < 8 || (t.pitch0 & 3) || ((uintptr_t)t.p0 & 3))) return -1;
    // one box pre-decimation level on both axes (ratios in (4, 8], resampler.rs:56-67): the any-ratio TMA kernel reduces
    // the source 2:1 on the fly and resamples the reduced texture; other level combinations take the generic passes
    const int lv_h = hm_in.predecimate_levels(), lv_v = vm_in.predecimate_levels();
    const bool box = lv_h == 1 && lv_v == 1;
    if (!box && (lv_h != 0 || lv_v != 0)) return -1;
    if (box && (src_class >= 2 || (dw & 1))) return -1;
    const AxisMapping hm = box ? hm_in.on_reduced_source(1) : hm_in, vm = box ? vm_in.on_reduced_source(1) : vm_in;
    KernelPass passes[2];
    if (plan_passes(hm, vm, passes) != 2 || passes[0].mapping.axis != 0) return -1;
    float sh = hm.scale(), sv = vm.scale();
    if (!(sh > 0.0f) || !(sv > 0.0f) || !(sh <= 4.001f) || !(sv <= 4.001f)) return -1;
    int th = resample_taps(sh), tv = resample_taps(sv);
    // at most kFusedMaxTaps taps keeps both ratios <= 4, where the LDG kernel takes any job (kernels.cu asserts its bounds)
    if (th > dev::kFusedMaxTaps || tv > dev::kFusedMaxTaps) return -1;
    // the kernel is chosen before anything is allocated for it.  TMA-staged kernels: planar 4:2:0 / NV12 planes a
    // descriptor can address (16-byte aligned rows), even target width, the vertical footprint of 8 output rows inside the ring
    const bool tma = src_class < 2 && (dw & 1) == 0;
    const int rows8 = (int)std::ceil((dev::kFusedWarps - 1) * sv) + tv + 1;
    dev::FusedKernel k;   // LDG, weights from smem
    int tmap_idx = -1, cols = 64;
    if (!box && hm.crop_offset == 0.0f && (sh == 2.0f || sh == 3.0f || sh == 4.0f)) k.ratio = (int)sh;   // LDG, int_weights.h
    if (tma && (k.ratio == 2 || k.ratio == 4) && rows8 <= (k.ratio == 4 ? dev::kTmaRing4 : dev::kTmaRing2) &&
        (tmap_idx = source_tmaps(t, src_class)) >= 0) {
        k.kind = dev::FusedKernel::TMA_INT;
    } else if (tma && th <= dev::kTma0MaxTaps && rows8 <= dev::kTmaRing4) {
        // any other ratio <= 4 (fractional, 3, with a crop offset, box-reduced): the any-ratio TMA kernel; its strips are
        // narrowed so that a strip's source span fits the 256 pixels a warp converts per row (= 128 reduced ones)
        const int max_span = box ? dev::kTma0MaxSpan / 2 : dev::kTma0MaxSpan;
        auto span = [&](int c) { return (int)std::ceil((c - 1) * sh) + th + 3; };
        while (cols > 2 && span(cols) > max_span) cols -= 2;
        // slots of a lane's window: taps + the widest distance of two adjacent columns' first taps + the pad slots crossed
        // (an integer ratio without offset is exact in f32: the distance is the ratio; otherwise floor + 1 bounds it, and the
        // kernel traps rather than drop a tap should rounding ever exceed that)
        const int gmax = (sh == std::floor(sh) && hm.crop_offset == 0.0f) ? (int)sh : (int)std::floor(sh) + 1;
        const int win = th + gmax, winp = win + ((7 + win - 1) >> 3);
        int bucket = 0;
        while (bucket < 4 && dev::kTma0Window[bucket] < winp) bucket++;
        if (bucket < 4 && span(cols) <= max_span && (tmap_idx = source_tmaps(t, src_class)) >= 0)
            k = {dev::FusedKernel::TMA_ANY, 0, bucket, box ? 1 : 0};
    }
    if (box && k.kind != dev::FusedKernel::TMA_ANY) return -1;   // no other fused kernel reduces: generic passes
    WeightEntry wh, wv;
    if (get_weights(passes[0], wh) != SMR_OK || get_weights(passes[1], wv) != SMR_OK) return -2;
    size_t dst_off = frame_alloc((size_t)dw * dh * 4);
    dev::FusedJob j{};
    j.dst_w = dw; j.dst_h = dh; j.dst_pitch = dw * 4;
    j.taps_h = wh.taps; j.taps_v = wv.taps;
    j.w_h = wh.weights; j.inv_h = wh.inv; j.first_h = wh.first;
    j.w_v = wv.weights; j.inv_v = wv.inv; j.first_v = wv.first;
    if (k.kind == dev::FusedKernel::TMA_INT) j.v_same = vm.crop_offset == 0.0f && sv == sh && tv == th;
    if (k.kind == dev::FusedKernel::TMA_ANY) {
        j.strip_cols = cols;
        j.lane_perm = lane_perm(sh, hm.crop_offset, dw, cols);   // nullptr (identity) if the table could not be made
    }
    plan_.fused.push_back({j, k, in.raw_tex, dst_off, tmap_idx, SIZE_MAX});
    dev::Tex out;
    out.kind = dev::TEX_RGBA8; out.width = dw; out.height = dh; out.pitch0 = dw * 4;
    return add_texture(out, true, dst_off, (int)plan_.fused.size() - 1);   // the fused kernel reads YUV and writes alpha 255
}

// The tensor maps of a planar 4:2:0 / NV12 source (luma; NV12 chroma, or U and V) for the TMA kernels, added to the tick's
// list: the index of the first of the three, or -1 when a plane cannot be described
int Renderer::source_tmaps(const dev::Tex &t, int src_class) {
    CUtensorMap m[3];
    memset(m, 0, sizeof(m));
    bool ok = plane_tmap(t.p0, t.pitch0, t.width, t.height, 0, &m[0]);
    if (src_class == 1) ok = ok && plane_tmap(t.p1, t.pitch1, t.width / 2, t.height / 2, 1, &m[1]);
    else ok = ok && plane_tmap(t.p1, t.pitch1, t.width / 2, t.height / 2, 2, &m[1]) &&
              plane_tmap(t.p2, t.pitch2, t.width / 2, t.height / 2, 2, &m[2]);
    if (!ok) return -1;
    plan_.tmaps.insert(plan_.tmaps.end(), m, m + 3);
    return (int)plan_.tmaps.size() - 3;
}

// The deal of a strip's 32 column pairs to the 32 lanes (resample_tma0.cuh): a tap of the horizontal pass is one LDS.128
// per lane at the lane's window start + tap, served a quarter-warp (8 lanes) at a time; two lanes of a quarter whose
// starts fall in the same 16-byte bank group cost an extra wavefront.  Sorting the pairs by bank group and dealing them
// round-robin to the four quarters gives every quarter ceil(n_k / 4) lanes of group k at most -- the minimum.  Only the
// speed depends on this table: the first-tap indices are recomputed here the way k_weights computes them, and a pair
// owned by the "wrong" lane is still resampled exactly.
const uint8_t *Renderer::lane_perm(float scale, float offset, int n_out, int cols) {
    uint32_t sb, ob;
    memcpy(&sb, &scale, 4); memcpy(&ob, &offset, 4);
    auto key = std::make_tuple(sb, ob, (int32_t)n_out, (int32_t)cols);
    auto it = lane_perms_.find(key);
    if (it != lane_perms_.end()) return it->second;
    if (lane_perms_.size() > 4096) {
        cudaStreamSynchronize(stream_);
        for (auto &e : lane_perms_) cudaFree(e.second);
        lane_perms_.clear();
    }
    const float ks = std::fmax(scale, 1.0f);
    auto first = [&](int o) {
        volatile float c = offset + ((float)o + 0.5f) * scale;
        volatile float d = c - 0.5f;
        return (int)std::ceil(d - 3.0f * ks);
    };
    const int strips = (n_out + cols - 1) / cols;
    std::vector<uint8_t> perm((size_t)strips * 32);
    for (int st = 0; st < strips; st++) {
        const int ox0 = st * cols, x0 = first(ox0) & ~1;
        int order[32], group[32];
        for (int p = 0; p < 32; p++) {
            const int rel = std::max(first(std::min(ox0 + 2 * p, n_out - 1)) - x0, 0);
            group[p] = (rel + (rel >> 3)) & 7;
            order[p] = p;
        }
        std::stable_sort(order, order + 32, [&](int a, int b) { return group[a] < group[b]; });
        for (int i = 0; i < 32; i++) perm[(size_t)st * 32 + (i & 3) * 8 + (i >> 2)] = (uint8_t)order[i];
    }
    uint8_t *dev_perm = nullptr;
    if (cudaMalloc(&dev_perm, perm.size()) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    // pageable source: staged before the call returns
    if (cudaMemcpyAsync(dev_perm, perm.data(), perm.size(), cudaMemcpyHostToDevice, stream_) != cudaSuccess) {
        cudaGetLastError(); cudaFree(dev_perm); return nullptr;
    }
    cudaStreamSynchronize(stream_);   // once per geometry; keeps the pageable staging out of the steady state
    lane_perms_[key] = dev_perm;
    return dev_perm;
}

bool Renderer::plane_tmap(const uint8_t *p, int pitch, int w, int h, int kind, CUtensorMap *out) {
    TmapKey key{(uintptr_t)p, pitch, w, h, kind};
    auto it = tmap_cache_.find(key);
    if (it != tmap_cache_.end()) { *out = it->second; return true; }
    // kind: 0 luma, 1 NV12 chroma, 2 planar chroma
    bool ok = kind == 0   ? encode_plane_tmap(p, pitch, w / 2, h, 2, dev::kTmaLumaBoxW, dev::kTmaLumaBoxH, out)
              : kind == 1 ? encode_plane_tmap(p, pitch, w, h, 2, dev::kTmaNv12BoxW, dev::kTmaChromaBoxH, out)
                          : encode_plane_tmap(p, pitch, w, h, 1, dev::kTmaPlanarBoxW, dev::kTmaChromaBoxH, out);
    if (!ok) return false;
    if (tmap_cache_.size() > 2048) tmap_cache_.clear();
    tmap_cache_[key] = *out;
    return true;
}

// Weight tables created by a tick whose k_weights launch was never enqueued hold uninitialised memory: drop them so that
// the next tick computes them.
void Renderer::rollback_weights() {
    for (const WeightKey &k : new_weight_keys_) {
        auto it = weights_.find(k);
        if (it == weights_.end()) continue;
        cudaFree(it->second.weights); cudaFree(it->second.inv); cudaFree(it->second.first);
        weights_.erase(it);
    }
    new_weight_keys_.clear();
    plan_.weight_jobs.clear();
}

void Renderer::shader_color(const RGBA &c, float out[4]) const {  // wgpu/utils.rs:51-71 + params.rs:353-361
    double a = (double)c.a / 255.0;
    if (opts_.rendering_mode == SMR_MODE_GPU_OPTIMIZED) {
        out[0] = (float)(a * eotf_f64((double)c.r / 255.0));
        out[1] = (float)(a * eotf_f64((double)c.g / 255.0));
        out[2] = (float)(a * eotf_f64((double)c.b / 255.0));
    } else {
        out[0] = (float)(a * (double)c.r / 255.0);
        out[1] = (float)(a * (double)c.g / 255.0);
        out[2] = (float)(a * (double)c.b / 255.0);
    }
    out[3] = (float)a;
}

static uint8_t unorm8_host(float x) { return (uint8_t)std::rint(std::fmin(std::fmax(x, 0.0f), 1.0f) * 255.0f); }
static uint8_t srgb_encode_host(float lin) {  // numeric contract NC-4, same thresholds as the device table
    float x = std::fmin(std::fmax(lin, 0.0f), 1.0f);
    int lo = 0, hi = 255;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (x >= kSrgbEncodeThr[mid]) lo = mid + 1; else hi = mid;
    }
    return (uint8_t)lo;
}

static inline long long snap256(float v) { return (long long)std::rint(v * 256.0f); }
static inline long long ceil_div256(long long a) {  // ceil(a / 256)
    long long q = a / 256, r = a % 256;
    return q + (r > 0 ? 1 : 0);
}

// The geometry of a layer drawn into a W x H target: the vertex stage of apply_layouts.wgsl:174-243 + rasteriser (numeric
// contract NC-7) and the interior proof (interior.h).  Fills the geometric fields of `d` (pixel box, rect, radii, border
// width, the two bars); false when the layer covers no pixel.
static bool layer_geometry(const RenderLayout &l, int W, int H, dev::LayerDev &d) {
    memset(&d, 0, sizeof(d));
    float left = l.left, top = l.top, w = l.width, h = l.height;
    if (l.kind == RenderLayout::BoxShadow) {
        float bw = l.width + 2.0f * l.blur_radius, bh = l.height + 2.0f * l.blur_radius;
        left = l.left - l.blur_radius; top = l.top - l.blur_radius; w = bw; h = bh;
    }
    float rot = l.rotation_degrees;
    if (!(left == left) || !(top == top) || !(w == w) || !(h == h) || !(rot == rot)) return false;
    if (std::fabs(left) > 1e7f || std::fabs(top) > 1e7f || std::fabs(w) > 1e7f || std::fabs(h) > 1e7f) return false;
    d.type = (int)l.kind;
    d.left = left; d.top = top; d.width = w; d.height = h;
    d.content_w = l.width; d.content_h = l.height;
    float hw = w / 2.0f, hh = h / 2.0f;
    d.cx = left + hw; d.cy = top + hh;
    d.rotated = rot != 0.0f;
    float minx, maxx, miny, maxy;
    if (!d.rotated) {
        d.cs = 1.0f; d.sn = 0.0f;
        long long x0 = snap256(d.cx - hw), x1 = snap256(d.cx + hw), y0 = snap256(d.cy - hh), y1 = snap256(d.cy + hh);
        long long px0 = ceil_div256(x0 - 128), px1 = ceil_div256(x1 - 128);
        long long py0 = ceil_div256(y0 - 128), py1 = ceil_div256(y1 - 128);
        d.px0 = (int)std::max<long long>(px0, 0); d.px1 = (int)std::min<long long>(px1, W);
        d.py0 = (int)std::max<long long>(py0, 0); d.py1 = (int)std::min<long long>(py1, H);
    } else {
        float ang = rot * (kPiF / 180.0f);
        d.cs = (float)std::cos((double)ang); d.sn = (float)std::sin((double)ang);
        const float lx[4] = {-hw, hw, hw, -hw}, ly[4] = {hh, hh, -hh, -hh};
        minx = miny = 1e30f; maxx = maxy = -1e30f;
        for (int i = 0; i < 4; i++) {
            float xr = lx[i] * d.cs - ly[i] * d.sn, yr = lx[i] * d.sn + ly[i] * d.cs;
            float X = d.cx + xr, Y = d.cy - yr;
            d.vx[i] = snap256(X); d.vy[i] = snap256(Y);
            minx = std::fmin(minx, X); maxx = std::fmax(maxx, X);
            miny = std::fmin(miny, Y); maxy = std::fmax(maxy, Y);
        }
        float fx0 = std::floor(minx) - 1.0f, fx1 = std::ceil(maxx) + 1.0f;
        float fy0 = std::floor(miny) - 1.0f, fy1 = std::ceil(maxy) + 1.0f;
        d.px0 = (int)std::fmax(fx0, 0.0f); d.py0 = (int)std::fmax(fy0, 0.0f);
        d.px1 = (int)std::fmin(fx1, (float)W); d.py1 = (int)std::fmin(fy1, (float)H);
    }
    if (d.px0 >= d.px1 || d.py0 >= d.py1) return false;
    d.border_radius[0] = l.border_radius.top_left; d.border_radius[1] = l.border_radius.top_right;
    d.border_radius[2] = l.border_radius.bottom_right; d.border_radius[3] = l.border_radius.bottom_left;
    d.border_width = l.border_width;
    d.blur_radius = l.blur_radius;
    // ---- fast interior (see LayerDev): only where every alpha factor of fs_main is provably exactly 1 ----
    // The layer and each mask prove the pixel centres at least `edge` inside their straight edges and outside their
    // corner squares (interior.h).  The intersection of those regions contains two bars: core x range x edge y range,
    // and the transpose.
    dev::interior_margins(l.left, l.top, l.width, l.height, d.border_radius, d.border_width, d.int_edge, d.int_corner);
    if (d.rotated || l.kind == RenderLayout::BoxShadow) return true;
    dev::InteriorRect k;
    if (!dev::interior_rect(l.left, l.top, l.width, l.height, d.border_radius, d.border_width, k)) return true;
    float cx0 = l.left + k.core, cx1 = l.left + l.width - k.core, cy0 = l.top + k.core, cy1 = l.top + l.height - k.core;
    float ex0 = l.left + k.edge, ex1 = l.left + l.width - k.edge, ey0 = l.top + k.edge, ey1 = l.top + l.height - k.edge;
    size_t nm = std::min<size_t>(l.masks.size(), SMR_MAX_MASKS);
    for (size_t i = 0; i < nm; i++) {
        const Mask &mk = l.masks[i];
        const float r[4] = {mk.radius.top_left, mk.radius.top_right, mk.radius.bottom_right, mk.radius.bottom_left};
        if (!dev::interior_rect(mk.left, mk.top, mk.width, mk.height, r, 0.0f, k)) return true;
        cx0 = std::fmax(cx0, mk.left + k.core); cx1 = std::fmin(cx1, mk.left + mk.width - k.core);
        cy0 = std::fmax(cy0, mk.top + k.core); cy1 = std::fmin(cy1, mk.top + mk.height - k.core);
        ex0 = std::fmax(ex0, mk.left + k.edge); ex1 = std::fmin(ex1, mk.left + mk.width - k.edge);
        ey0 = std::fmax(ey0, mk.top + k.edge); ey1 = std::fmin(ey1, mk.top + mk.height - k.edge);
    }
    // pixel X is inside iff lo <= X + .5 <= hi
    auto bar = [&](float lx, float hx, float ly, float hy, int32_t &x0, int32_t &x1, int32_t &y0, int32_t &y1) {
        if (!(lx < hx && ly < hy)) return;
        int ax0 = std::max((int)std::ceil(lx - 0.5f), d.px0), ax1 = std::min((int)std::floor(hx - 0.5f) + 1, d.px1);
        int ay0 = std::max((int)std::ceil(ly - 0.5f), d.py0), ay1 = std::min((int)std::floor(hy - 0.5f) + 1, d.py1);
        if (ax0 >= ax1 || ay0 >= ay1) return;
        x0 = ax0; x1 = ax1; y0 = ay0; y1 = ay1;
    };
    bar(cx0, cx1, ey0, ey1, d.ix0, d.ix1, d.iy0, d.iy1);
    bar(ex0, ex1, cy0, cy1, d.jx0, d.jx1, d.jy0, d.jy1);
    return true;
}

// Appends the masks of `l` the shader sees (params.rs:284-294); returns their count
static int layer_masks(const RenderLayout &l, std::vector<dev::MaskDev> &masks) {
    size_t nm = std::min<size_t>(l.masks.size(), SMR_MAX_MASKS);
    for (size_t i = 0; i < nm; i++) {
        const Mask &m = l.masks[i];
        dev::MaskDev md;
        md.radius[0] = m.radius.top_left; md.radius[1] = m.radius.top_right;
        md.radius[2] = m.radius.bottom_right; md.radius[3] = m.radius.bottom_left;
        md.top = m.top; md.left = m.left; md.width = m.width; md.height = m.height;
        dev::interior_margins(md.left, md.top, md.width, md.height, md.radius, 0.0f, md.edge, md.corner);
        masks.push_back(md);
    }
    return (int)nm;
}

// One layer as the composite draws it: its geometry (layer_geometry), colours, texture mapping and fast class
void Renderer::prepare_layer(const RenderLayout &l, int W, int H, int tex_index, int tex_w, int tex_h,
                             dev::LayerDev &d, bool &skip) {
    skip = !layer_geometry(l, W, H, d);
    if (skip) return;
    shader_color(l.color, d.color);
    shader_color(l.border_color, d.border_color);
    d.tex = tex_index;
    if (l.kind == RenderLayout::ChildNode) {
        d.crop_sx = l.crop.width / (float)tex_w; d.crop_ox = l.crop.left / (float)tex_w;
        d.crop_sy = l.crop.height / (float)tex_h; d.crop_oy = l.crop.top / (float)tex_h;
    }
    if (d.ix0 >= d.ix1 && d.jx0 >= d.jx1) return;
    if (l.kind == RenderLayout::Color && l.color.a == 255) {
        // opaque colour: fma(dst, 0, src) == src, so the target bytes are a constant of the layer
        d.fast |= dev::FAST_CONST | dev::FAST_OPAQUE;
        uint8_t b[4];
        for (int c = 0; c < 3; c++)
            b[c] = opts_.rendering_mode == SMR_MODE_GPU_OPTIMIZED ? srgb_encode_host(d.color[c]) : unorm8_host(d.color[c]);
        b[3] = 255;
        memcpy(&d.const_bytes, b, 4);
    } else if (l.kind == RenderLayout::Color) {
        d.fast |= dev::FAST_LUT;
    }
    auto integral = [](float v) { return v == std::rint(v) && std::fabs(v) <= 4096.0f; };
    if (l.kind == RenderLayout::ChildNode && tex_index >= 0 && tex_w <= 4096 && tex_h <= 4096 &&
        l.width == (float)tex_w && l.crop.width == (float)tex_w && l.height == (float)tex_h &&
        l.crop.height == (float)tex_h && integral(l.left) && integral(l.top) && l.crop.left == 0.0f &&
        l.crop.top == 0.0f) {
        // 1:1 mapping on whole texels: the NC-6 tap is texel (px - left, py - top) with weight exactly 1
        // (|coordinate error| < 1e-3 << 1/512, the 8-bit weight rounds to 0 or 1)
        d.fast |= dev::FAST_IDENT;
        if (plan_.tex[tex_index].opaque) d.fast |= dev::FAST_OPAQUE;
        d.tx_off = -(int)l.left; d.ty_off = -(int)l.top;
    } else if (l.kind == RenderLayout::ChildNode && tex_index >= 0 && plan_.tex[tex_index].opaque && l.width > 0.0f &&
               l.height > 0.0f &&
               (plan_.tex[tex_index].tex.kind == dev::TEX_RGBA8 ||
                (opts_.rendering_mode == SMR_MODE_CPU_OPTIMIZED &&
                 (plan_.tex[tex_index].tex.kind == dev::TEX_NV12 || plan_.tex[tex_index].tex.kind == dev::TEX_YUV420)))) {
        // opaque child at a fractional position / size: filtered sample alone, target ignored.  RGBA8: a
        // resampled child; planar 4:2:0 / NV12 in CpuOptimized: the layout shader's own bilinear scaling of
        // the (virtual) node texture, K1/K2 evaluated per tap quad
        d.fast |= dev::FAST_SAMPLE | dev::FAST_OPAQUE;
        const dev::Tex &tt = plan_.tex[tex_index].tex;
        if (tt.kind != dev::TEX_RGBA8 && ((tex_w | tex_h) & 1) == 0 && tex_w <= 4096 && tex_h <= 4096 &&
            l.width * 2.0f == (float)tex_w && l.height * 2.0f == (float)tex_h && l.crop.left == 0.0f && l.crop.top == 0.0f &&
            l.crop.width == (float)tex_w && l.crop.height == (float)tex_h && integral(l.left) && integral(l.top) &&
            ((int)l.left & 1) == 0 && (tt.pitch0 & 3) == 0 && ((uintptr_t)tt.p0 & 3) == 0) {
            // exact 2:1 on whole pixels (a 2x2 grid of same-size inputs): sample coordinate = 2 k + 1/2 with an error
            // far below the 1/512 weight step, so the taps are the aligned texel quad at weights exactly 1/2
            d.fast |= dev::FAST_HALF;
            d.tx_off = -(int)l.left; d.ty_off = -(int)l.top;
        }
    }
}

// An RGBA8 result of w x h for the caller: `launch` writes it into `rgba` itself (device memory) or into pre_out_, which is
// copied back (host memory).  Returns once the result is complete, like the reference's device.poll
// (frame_pre_processor.rs:171-176); the caller's host buffers are borrowed for the call only.
template <class Launch>
smr_status Renderer::write_rgba(void *rgba, uint32_t pitch, int32_t mem_kind, uint32_t w, uint32_t h, Launch launch) {
    const size_t row = (size_t)w * 4, user_pitch = pitch ? pitch : row;
    if (user_pitch < row) { set_error("output pitch smaller than a row"); return SMR_ERR_BUFFER_TOO_SMALL; }
    uint8_t *dst = (uint8_t *)rgba;
    size_t dpitch = user_pitch;
    if (mem_kind != SMR_MEM_DEVICE) {
        if (row * h > pre_out_.cap) CUDA_OK(cudaStreamSynchronize(stream_));
        CUDA_OK(pre_out_.ensure(row * h));
        dst = pre_out_.p; dpitch = row;
    } else if ((dpitch & 3) || ((uintptr_t)dst & 3)) { set_error("device RGBA8 planes are 4-byte aligned"); return SMR_ERR_INVALID_ARGUMENT; }
    if (launch(dst, (int)dpitch) < 0) { set_error(dev::last_launch_error()); return SMR_ERR_CUDA; }
    stats_.kernel_launches++;
    if (mem_kind != SMR_MEM_DEVICE) {
        CUDA_OK(cudaMemcpy2DAsync(rgba, user_pitch, dst, dpitch, row, h, cudaMemcpyDeviceToHost, stream_));
        stats_.d2h_bytes += row * h;
    }
    CUDA_OK(cudaStreamSynchronize(stream_));
    return SMR_OK;
}

// FramePreProcessor::process_to_bytes / process_to_texture (state/frame_pre_processor.rs:60-100)
smr_status Renderer::preprocess_frame(const smr_input_frame *f, uint32_t ow, uint32_t oh, void *rgba, uint32_t pitch,
                                      int32_t mem_kind, bool premultiply) {
    if (!f || !rgba) return SMR_ERR_INVALID_ARGUMENT;
    if (premultiply && (f->format != SMR_FRAME_RGBA8 || ow != 0 || oh != 0)) {
        set_error("premultiply takes a straight-alpha RGBA8 frame at its own resolution");
        return SMR_ERR_INVALID_ARGUMENT;
    }
    std::lock_guard<std::mutex> g(mu_);
    if (host_only_) { set_error("host-only handle (cuda_device = -1) has no device: no CPU fallback"); return SMR_ERR_CUDA; }
    CUDA_OK(cudaSetDevice(opts_.cuda_device));
    const bool rescale = ow != 0 || oh != 0;
    // the output size is checked after the input size and before the rest of the frame
    if (rescale && frame_size_ok(*f) && (ow == 0 || oh == 0 || ow > 16384 || oh > 16384)) {
        set_error("output resolution out of range");
        return SMR_ERR_INVALID_ARGUMENT;
    }
    FrameView v;
    if (smr_status st = read_frame(*f, v); st != SMR_OK) return st;
    if (!rescale) { ow = f->width; oh = f->height; }
    for (int p = 0; p < 3 && f->mem_kind != SMR_MEM_DEVICE; p++) {
        const FrameView::Plane &P = v.plane[p];
        if (!P.p) continue;
        if (P.row_bytes * P.rows > pre_planes_[p].cap) CUDA_OK(cudaStreamSynchronize(stream_));
        CUDA_OK(pre_planes_[p].ensure(P.row_bytes * P.rows));
        CUDA_OK(cudaMemcpy2DAsync(pre_planes_[p].p, P.row_bytes, P.p, P.pitch, P.row_bytes, P.rows, cudaMemcpyHostToDevice, stream_));
        stats_.h2d_bytes += P.row_bytes * P.rows;
        set_tex_plane(v.tex, p, pre_planes_[p].p, P.row_bytes);
    }
    const int kind = premultiply ? 2 : (rescale ? 1 : 0);
    return write_rgba(rgba, pitch, mem_kind, ow, oh, [&](uint8_t *dst, int dpitch) {
        return dev::launch_preprocess(v.tex, opts_.rendering_mode, kind, dst, dpitch, (int)ow, (int)oh, stream_);
    });
}

// TextRendererNode::render (transformations/text_renderer.rs:72-167): clear + glyphon's glyph quads
smr_status Renderer::render_text(uint32_t w, uint32_t h, smr_rgba bg, const smr_glyph *glyphs, uint32_t n, const smr_atlas *mask,
                                 const smr_atlas *color, int32_t color_mode, void *rgba, uint32_t pitch, int32_t mem_kind) {
    static_assert(sizeof(smr_glyph) == sizeof(dev::GlyphDev), "smr_glyph is copied to the device as it is");
    if (!rgba || (n && !glyphs) || (color_mode != 0 && color_mode != 1)) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    if (host_only_) { set_error("host-only handle (cuda_device = -1) has no device: no CPU fallback"); return SMR_ERR_CUDA; }
    CUDA_OK(cudaSetDevice(opts_.cuda_device));
    // a zero-sized text texture is a transparent 1x1 one in the reference (text_renderer.rs:77-85); here the caller skips it
    if (w == 0 || h == 0 || w > 16384 || h > 16384) { set_error("text texture resolution out of range"); return SMR_ERR_INVALID_ARGUMENT; }
    if (n > (1u << 22)) { set_error("too many glyphs"); return SMR_ERR_INVALID_ARGUMENT; }
    bool need_mask = false, need_color = false;
    for (uint32_t i = 0; i < n; i++) {
        if (glyphs[i].content == SMR_GLYPH_MASK) need_mask = true;
        else if (glyphs[i].content == SMR_GLYPH_COLOR) need_color = true;
        else { set_error("glyph content type must be SMR_GLYPH_COLOR or SMR_GLYPH_MASK"); return SMR_ERR_INVALID_ARGUMENT; }
    }
    dev::TextJob J = {};
    J.width = (int)w; J.height = (int)h; J.mode = opts_.rendering_mode; J.color_mode = color_mode; J.n_glyphs = (int)n;
    shader_color(RGBA{bg.r, bg.g, bg.b, bg.a}, J.bg);
    const smr_atlas *atl[2] = {mask, color};
    const bool need[2] = {need_mask, need_color};
    for (int k = 0; k < 2; k++) {
        if (!need[k]) continue;
        const smr_atlas *a = atl[k];
        const size_t texel = k == 0 ? 1 : 4;
        if (!a || !a->data || a->width == 0 || a->height == 0 || a->width > 16384 || a->height > 16384) {
            set_error(k == 0 ? "mask glyphs need a mask atlas" : "colour glyphs need a colour atlas");
            return SMR_ERR_INVALID_ARGUMENT;
        }
        const size_t row = (size_t)a->width * texel, sp = a->pitch ? a->pitch : row;
        if (sp < row) { set_error("atlas pitch smaller than a row"); return SMR_ERR_INVALID_ARGUMENT; }
        if (row * a->height > pre_planes_[k].cap) CUDA_OK(cudaStreamSynchronize(stream_));
        CUDA_OK(pre_planes_[k].ensure(row * a->height));
        CUDA_OK(cudaMemcpy2DAsync(pre_planes_[k].p, row, a->data, sp, row, a->height, cudaMemcpyHostToDevice, stream_));
        stats_.h2d_bytes += row * a->height;
        if (k == 0) { J.mask = pre_planes_[0].p; J.mask_w = (int)a->width; J.mask_h = (int)a->height; J.mask_pitch = (int)row; }
        else { J.color = pre_planes_[1].p; J.color_w = (int)a->width; J.color_h = (int)a->height; J.color_pitch = (int)row; }
    }
    if (n) {
        const size_t bytes = sizeof(smr_glyph) * (size_t)n;
        if (bytes > pre_planes_[2].cap) CUDA_OK(cudaStreamSynchronize(stream_));
        CUDA_OK(pre_planes_[2].ensure(bytes));
        CUDA_OK(cudaMemcpyAsync(pre_planes_[2].p, glyphs, bytes, cudaMemcpyHostToDevice, stream_));
        stats_.h2d_bytes += bytes;
        J.glyphs = reinterpret_cast<const dev::GlyphDev *>(pre_planes_[2].p);
    }
    return write_rgba(rgba, pitch, mem_kind, w, h, [&](uint8_t *dst, int dpitch) {
        J.out = dst; J.out_pitch = dpitch;
        return dev::launch_text(J, stream_);
    });
}

smr_status Renderer::get_weights(const KernelPass &p, WeightEntry &out) {
    WeightKey key;
    float scale = p.mapping.scale(), offset = p.mapping.crop_offset;
    memcpy(&key.scale_bits, &scale, 4);
    memcpy(&key.offset_bits, &offset, 4);
    key.n_out = p.mapping.dst_len;
    auto it = weights_.find(key);
    if (it != weights_.end()) {
        it->second.last_used = tick_;
        out = it->second;
        return SMR_OK;
    }
    if (weights_.size() > 4096) {  // bound the cache: drop entries not used this tick
        cudaStreamSynchronize(stream_);
        for (auto i = weights_.begin(); i != weights_.end();) {
            if (i->second.last_used != tick_) {
                cudaFree(i->second.weights); cudaFree(i->second.inv); cudaFree(i->second.first);
                i = weights_.erase(i);
            } else ++i;
        }
    }
    WeightEntry e;
    e.taps = resample_taps(scale);
    if (e.taps < 1 || e.taps > 4096) { set_error("resampler tap count out of range"); return SMR_ERR_INVALID_ARGUMENT; }
    e.last_used = tick_;
    if (cudaMalloc(&e.weights, sizeof(float) * (size_t)e.taps * key.n_out) != cudaSuccess ||
        cudaMalloc(&e.inv, sizeof(float) * key.n_out) != cudaSuccess ||
        cudaMalloc(&e.first, sizeof(int32_t) * key.n_out) != cudaSuccess) {
        cudaFree(e.weights); cudaFree(e.inv); cudaFree(e.first);
        cudaGetLastError();
        set_error("out of device memory for resampler weight tables");
        return SMR_ERR_CUDA;
    }
    new_weight_keys_.push_back(key);
    dev::WeightJob j;
    j.scale = scale; j.offset = offset; j.n_out = key.n_out; j.taps = e.taps;
    j.weights = e.weights; j.inv_wsum = e.inv; j.first = e.first;
    plan_.weight_jobs.push_back(j);
    weights_[key] = e;
    out = e;
    return SMR_OK;
}

static void black_yuv(uint8_t out[3]) {  // RGBColor::BLACK.to_yuv() through an R8Unorm store
    float y = 0.0f, u = 0.0f, v = 0.0f;
    out[0] = unorm8_host((y * 0.85882354f) + (16.0f / 255.0f));
    out[1] = unorm8_host(((u + 0.5f) * 0.8784314f) + (16.0f / 255.0f));
    out[2] = unorm8_host(((v + 0.5f) * 0.8784314f) + (16.0f / 255.0f));
}

static void out_plane_layout(int fmt, uint32_t w, uint32_t h, size_t row_bytes[3], size_t rows[3]) {
    for (int i = 0; i < 3; i++) row_bytes[i] = rows[i] = 0;
    int icw, ich;
    dev::chroma_dims(fmt, (int)w, (int)h, icw, ich);
    uint32_t cw = (uint32_t)icw, ch = (uint32_t)ich;
    if (fmt == SMR_OUT_RGBA8) { row_bytes[0] = (size_t)w * 4; rows[0] = h; }
    else if (fmt == SMR_OUT_NV12) { row_bytes[0] = w; rows[0] = h; row_bytes[1] = (size_t)cw * 2; rows[1] = ch; }
    else { row_bytes[0] = w; rows[0] = h; row_bytes[1] = row_bytes[2] = cw; rows[1] = rows[2] = ch; }
}

// LayoutNode::render (transformations/layout.rs:169-278) + read_outputs (render_loop.rs:59-230) for one output
// Tile plan of a composite with fused K10 / K11 output.
//
// Direct tiles: a composite tile (128 x 16 output pixels) whose TOPMOST intersecting layer is the exact 1:1, opaque
// interior of a resampled child (FAST_IDENT | FAST_OPAQUE: host-proved, every alpha factor exactly 1) and covers the
// whole tile shows nothing but that child's texels -- whatever lies below is replaced, nothing lies above.  For such a
// tile K10 / K11 need only the child's encoded bytes, which the fused resample kernel still holds in registers at the end
// of its vertical pass: it writes the tile's Y / chroma bytes itself (FusedJob.direct_map) and the composite skips the
// tile.  Conditions on the job: the grouped TMA kernel with the integer vertical ratio (rows come out in pairs), even
// frame position and size (chroma blocks), one direct target per job (the first claimant).
//
// Tile list: the composite is launched over the tiles that are left, one block each, MOST EXPENSIVE FIRST.  Those tiles are
// few (2 - 3 waves of resident blocks in the BASELINE grids) and uneven -- edges, corners, overlays and shadows take the
// general fragment path, interiors do not -- so in row-major order the launch ends on whatever heavy tiles come last while
// most SMs idle; longest-first leaves a tail of cheap tiles.  Cost estimate per intersecting layer: 1 when the tile lies
// in one of the layer's exact-interior bars, 8 when some of its pixels run the fragment path.
//
// The plan depends only on the flattened layers and on which fused job feeds each of them: it is cached per output.
static inline void fnv1a(uint64_t &h, const void *p, size_t n) {
    const uint8_t *b = (const uint8_t *)p;
    for (size_t i = 0; i < n; i++) { h ^= b[i]; h *= 1099511628211ull; }
}
// The geometric core of the plan as a free function (device-free; smr_debug_tile_plan and the CPU tests call it too).
// boxes[i] = what the plan needs of layer i, painter's order: its pixel bounding box, its two exact-interior bars, whether
// the interior replaces the target (FAST_OPAQUE), and the fused job that could write its tiles directly (-1: none).
struct TileLayerBox { int32_t px0, px1, py0, py1, ix0, ix1, iy0, iy1, jx0, jx1, jy0, jy1, opaque, job; };
void plan_tiles_core(const TileLayerBox *boxes, int n_layers, int W, int H, bool sort, std::vector<int> &owner_layer,
                     std::vector<uint32_t> &list) {
    const int TW = dev::kDirectTileW, TH = dev::kDirectTileH;
    const int tx_n = (W + TW - 1) / TW, ty_n = (H + TH - 1) / TH;
    const size_t n_tiles = (size_t)tx_n * ty_n;
    owner_layer.assign(n_tiles, -1);
    std::vector<std::pair<int, uint32_t>> keyed;
    keyed.reserve(n_tiles);
    std::map<int, int> layer_of_job;   // one layer per job (a texture shown twice 1:1 would need two frame positions)
    for (int ty = 0; ty < ty_n; ty++)
        for (int tx = 0; tx < tx_n; tx++) {
            const int x0 = tx * TW, y0 = ty * TH, x1 = std::min(x0 + TW, W), y1 = std::min(y0 + TH, H);
            int cost = 0;
            bool top = true;
            int owner = -1;
            for (int li = n_layers - 1; li >= 0; li--) {
                const TileLayerBox &L = boxes[li];
                if (L.px0 >= x1 || L.px1 <= x0 || L.py0 >= y1 || L.py1 <= y0) continue;   // the composite's own culling test
                const bool in = (x0 >= L.ix0 && x1 <= L.ix1 && y0 >= L.iy0 && y1 <= L.iy1) || (x0 >= L.jx0 && x1 <= L.jx1 && y0 >= L.jy0 && y1 <= L.jy1);
                if (top) {   // the topmost intersecting layer decides about a direct tile
                    top = false;
                    if (in && L.job >= 0) {
                        auto ins = layer_of_job.emplace(L.job, li);
                        if (ins.first->second == li) { owner = li; break; }
                    }
                }
                cost += in ? 1 : 8;
                if (in && L.opaque) break;   // the kernel's occlusion start: nothing below is evaluated
            }
            if (owner >= 0) owner_layer[(size_t)ty * tx_n + tx] = owner;
            else keyed.push_back({-cost, (uint32_t)tx | ((uint32_t)ty << 16)});
        }
    if (sort)
        std::stable_sort(keyed.begin(), keyed.end(), [](const std::pair<int, uint32_t> &a, const std::pair<int, uint32_t> &b) { return a.first < b.first; });
    list.resize(keyed.size());
    for (size_t k = 0; k < keyed.size(); k++) list[k] = keyed[k].second;
}

void Renderer::plan_tiles(Output &o, CompositeRec &pc, const std::vector<dev::LayerDev> &layers, int W, int H) {
    const int TW = dev::kDirectTileW, TH = dev::kDirectTileH;
    const int tx_n = (W + TW - 1) / TW, ty_n = (H + TH - 1) / TH;
    if (tx_n > 0xffff || ty_n > 0xffff) return;
    const dev::CompositeJob &cj = pc.job;
    bool direct_ok = direct_k11_ && (cj.out_format == SMR_OUT_NV12 || cj.out_format == SMR_OUT_PLANAR_YUV420);
    if ((cj.out_pitch0 & 1) || ((uintptr_t)cj.out0 & 1) || (cj.out_format == SMR_OUT_NV12 && ((cj.out_pitch1 & 1) || ((uintptr_t)cj.out1 & 1)))) direct_ok = false;
    // which fused job could serve each layer
    std::vector<int> job_of(layers.size(), -1);
    if (direct_ok)
        for (size_t li = 0; li < layers.size(); li++) {
            const dev::LayerDev &L = layers[li];
            if (L.type != 0 || (L.fast & (dev::FAST_IDENT | dev::FAST_OPAQUE)) != (dev::FAST_IDENT | dev::FAST_OPAQUE)) continue;
            const int ji = plan_.tex[L.tex].fused_job;   // FAST_IDENT: L.tex >= 0
            if (ji < 0 || ji >= 255) continue;   // the map holds the owner as one byte
            const FusedRec &f = plan_.fused[ji];
            const dev::FusedJob &fj = f.job;
            // 4:1 only: per OUTPUT pixel the emission costs the resample kernel about what it saves the composite; at 2:1 a
            // quarter as many source pixels stand behind each output pixel and the vertical pass (four of a group's eight
            // warps) becomes the longer leg -- measured: 4:1 grid +4 %, 2:1 grid -2 %
            if (f.kernel.kind != dev::FusedKernel::TMA_INT || f.kernel.ratio != 4 || !fj.v_same || ((fj.dst_w | fj.dst_h) & 1)) continue;
            if ((L.tx_off & 1) || (L.ty_off & 1)) continue;   // frame position of texel (0, 0) = (-tx_off, -ty_off)
            // the whole child inside the frame: the kernel maps EVERY pixel of the job to a tile of the map, so a child hanging
            // over an edge (overflow: visible, absolute positions) would index tiles that do not exist
            if (L.tx_off > 0 || L.ty_off > 0 || -L.tx_off + fj.dst_w > W || -L.ty_off + fj.dst_h > H) continue;
            if (f.direct_off != SIZE_MAX) continue;   // serves another output (or an earlier layer) already
            job_of[li] = ji;
        }
    uint64_t key = 1469598103934665603ull;
    fnv1a(key, &W, sizeof(W)); fnv1a(key, &H, sizeof(H));
    if (!layers.empty()) fnv1a(key, layers.data(), sizeof(dev::LayerDev) * layers.size());
    if (!job_of.empty()) fnv1a(key, job_of.data(), sizeof(int) * job_of.size());
    const size_t n_tiles = (size_t)tx_n * ty_n;
    if (!(o.tile_key_valid && o.tile_key == key && o.tile_owner_layer.size() == n_tiles)) {
        std::vector<TileLayerBox> boxes(layers.size());
        for (size_t li = 0; li < layers.size(); li++) {
            const dev::LayerDev &L = layers[li];
            boxes[li] = {L.px0, L.px1, L.py0, L.py1, L.ix0, L.ix1, L.iy0, L.iy1, L.jx0, L.jx1, L.jy0, L.jy1,
                         (L.fast & dev::FAST_OPAQUE) ? 1 : 0, job_of[li]};
        }
        plan_tiles_core(boxes.data(), (int)boxes.size(), W, H, true, o.tile_owner_layer, o.tile_list);
        o.tile_key = key; o.tile_key_valid = true;
    }
    pc.use_list = true;
    pc.list = o.tile_list;
    pc.job.map_w = tx_n;
    // claim the fused jobs of the direct tiles
    std::map<int, int> claimed;   // job -> layer
    bool any = false;
    pc.direct_owner.assign(n_tiles, -1);
    for (size_t t = 0; t < n_tiles; t++) {
        const int li = o.tile_owner_layer[t];
        if (li < 0) continue;
        pc.direct_owner[t] = job_of[li];
        claimed[job_of[li]] = li;
        any = true;
    }
    if (!any) { pc.direct_owner.clear(); return; }
    pc.direct_off = param_alloc(n_tiles);
    for (auto &jl : claimed) {
        dev::FusedJob &fj = plan_.fused[jl.first].job;
        const dev::LayerDev &L = layers[jl.second];
        plan_.fused[jl.first].direct_off = pc.direct_off;
        fj.map_w = tx_n;
        fj.direct_id = jl.first + 1;
        fj.fx = -L.tx_off; fj.fy = -L.ty_off;
        fj.out_format = cj.out_format;
        fj.out0 = cj.out0; fj.out1 = cj.out1; fj.out2 = cj.out2;
        fj.out_pitch0 = cj.out_pitch0; fj.out_pitch1 = cj.out_pitch1; fj.out_pitch2 = cj.out_pitch2;
    }
}

// An output's children at `pts` (sources[i].resolution(), layout.rs:176-179): the input behind each (nullptr: no live frame)
// and its resolution.  Returns the root resolution.
Resolution Renderer::output_children(const Output &o, const OutputNode &node, uint64_t pts, std::vector<Input *> &child_in,
                                     std::vector<std::optional<Resolution>> &child_res) {
    for (const std::string &id : (o.flat ? o.flat_children : node.child_input_ids)) {
        auto it = inputs_.find(id);
        Input *in = it != inputs_.end() && it->second.has_frame ? &it->second : nullptr;
        child_in.push_back(in);
        child_res.push_back(in ? std::optional<Resolution>(in->res) : std::nullopt);
    }
    return o.flat ? o.flat_root : node.layout_resolution(pts);
}

// Its flattened layouts (layout.rs:180-181), untruncated.  Evaluating them advances Tiles::last_layout of `node`: o.node
// when rendering, a copy for inspection.
std::vector<RenderLayout> Renderer::output_layouts(const Output &o, OutputNode &node, uint64_t pts,
                                                   const std::vector<std::optional<Resolution>> &child_res, Resolution root) {
    return o.flat ? o.flat_layouts : node.layouts(pts, child_res).flatten(child_res, root);
}

// The texture a child layer samples: the input's own, or in GpuOptimized mode its copy resampled to the layer's size, whose
// crop then replaces the layer's (resample_scaled_children, layout.rs:238-278)
smr_status Renderer::child_texture(Input &in, RenderLayout &l, int &tex_index, int &tex_w, int &tex_h) {
    tex_index = in.raw_tex; tex_w = in.tex.width; tex_h = in.tex.height;
    if (opts_.rendering_mode != SMR_MODE_GPU_OPTIMIZED) return SMR_OK;
    float rw = std::round(l.width), rh = std::round(l.height);
    int dw = rw >= 1.0f ? (rw > 16384.0f ? 16384 : (int)rw) : 1;
    int dh = rh >= 1.0f ? (rh > 16384.0f ? 16384 : (int)rh) : 1;
    AxisMapping hm{0, l.crop.left, l.crop.width, dw}, vm{1, l.crop.top, l.crop.height, dh};
    KernelPass passes[2];
    if (plan_passes(hm, vm, passes) == 0) return SMR_OK;
    uint32_t cb[4];
    memcpy(&cb[0], &l.crop.left, 4); memcpy(&cb[1], &l.crop.top, 4);
    memcpy(&cb[2], &l.crop.width, 4); memcpy(&cb[3], &l.crop.height, 4);
    auto key = std::make_tuple(in.raw_tex, cb[0], cb[1], cb[2], cb[3], dw, dh);
    auto hit = plan_.resample_cache.find(key);
    if (hit != plan_.resample_cache.end()) {
        tex_index = hit->second;  // same input/crop/size already resampled this tick
    } else if (int fused_tex = try_fused_resample(in, hm, vm, dw, dh); fused_tex != -1) {
        if (fused_tex < -1) return SMR_ERR_CUDA;
        tex_index = fused_tex;
        plan_.resample_cache[key] = tex_index;
    } else {
        int levels[2] = {hm.predecimate_levels(), vm.predecimate_levels()};
        int fac[2] = {1 << levels[0], 1 << levels[1]};
        if ((uint64_t)fac[0] * (uint64_t)fac[1] > dev::kMaxBoxTexels) {
            set_error("texture layout crop is too large for its size: the box pass would average more than 2^24 texels");
            return SMR_ERR_INVALID_ARGUMENT;
        }
        int src_tex = materialised_input(in);
        int cur_w = in.tex.width, cur_h = in.tex.height;
        size_t cur_off = SIZE_MAX;  // SIZE_MAX: source is plan_.tex[src_tex]
        if (fac[0] != 1 || fac[1] != 1) {
            int rwid = (cur_w + fac[0] - 1) / fac[0], rhei = (cur_h + fac[1] - 1) / fac[1];
            size_t off = frame_alloc((size_t)rwid * rhei * 8);
            dev::ResampleJob j{};
            j.box_fx = fac[0]; j.box_fy = fac[1];
            j.dst_w = rwid; j.dst_h = rhei; j.dst_f16 = 1; j.dst_pitch = rwid * 8;
            plan_.stages[0].push_back({j, src_tex, SIZE_MAX, off});
            cur_w = rwid; cur_h = rhei; cur_off = off;
        }
        AxisMapping rh_ = hm.on_reduced_source(levels[0]), rv_ = vm.on_reduced_source(levels[1]);
        int np = plan_passes(rh_, rv_, passes);
        if (np == 0) { set_error("resampler planning failed"); return SMR_ERR_INVALID_ARGUMENT; }
        size_t dst_off = frame_alloc((size_t)dw * dh * 4);
        for (int pi = 0; pi < np; pi++) {
            const KernelPass &kp = passes[pi];
            bool last = pi == np - 1;
            WeightEntry we;
            smr_status st = get_weights(kp, we);
            if (st != SMR_OK) return st;
            dev::ResampleJob j{};
            j.axis = kp.mapping.axis; j.perp_offset = kp.perp_offset; j.taps = we.taps;
            j.weights = we.weights; j.inv_wsum = we.inv; j.first = we.first;
            j.box_fx = j.box_fy = 1;
            size_t out_off;
            if (last) {
                j.dst_w = dw; j.dst_h = dh; j.dst_f16 = 0; j.dst_pitch = dw * 4;
                out_off = dst_off;
            } else {
                j.dst_w = kp.mapping.axis == 0 ? kp.mapping.dst_len : cur_w;  // output_size
                j.dst_h = kp.mapping.axis == 1 ? kp.mapping.dst_len : cur_h;
                j.dst_f16 = 1; j.dst_pitch = j.dst_w * 8;
                out_off = frame_alloc((size_t)j.dst_w * j.dst_h * 8);
            }
            // f16 sources carry their geometry in the job; RGBA8/YUV sources come from the table
            if (cur_off != SIZE_MAX) {
                j.src.kind = dev::TEX_F16; j.src.width = cur_w; j.src.height = cur_h; j.src.pitch0 = cur_w * 8;
            }
            plan_.stages[last ? 2 : 1].push_back({j, cur_off == SIZE_MAX ? src_tex : -1, cur_off, out_off});
            if (!last) { cur_w = j.dst_w; cur_h = j.dst_h; cur_off = out_off; }
        }
        dev::Tex t;
        t.kind = dev::TEX_RGBA8; t.width = dw; t.height = dh; t.pitch0 = dw * 4;
        tex_index = add_texture(t, false, dst_off);
        plan_.resample_cache[key] = tex_index;
    }
    tex_w = dw; tex_h = dh;
    l.crop = {0.0f, 0.0f, (float)dw, (float)dh};  // ResampledChild::output_crop
    return SMR_OK;
}

smr_status Renderer::plan_output(Output &o, smr_output_frame &of, uint64_t pts) {
    const int mode = opts_.rendering_mode;
    of.width = (uint32_t)o.res.width; of.height = (uint32_t)o.res.height;
    of.format = o.format; of.pts_ns = pts;

    // where the kernels write: caller's device planes, or our device staging + D2H
    size_t row_bytes[3], rows[3];
    out_plane_layout(o.format, of.width, of.height, row_bytes, rows);
    uint8_t *dst[3] = {nullptr, nullptr, nullptr};
    int pitch[3] = {0, 0, 0};
    for (int p = 0; p < 3; p++) {
        if (!row_bytes[p]) continue;
        if (!of.planes[p]) { set_error("output plane pointer is null"); return SMR_ERR_INVALID_ARGUMENT; }
        size_t user_pitch = of.pitch[p] ? of.pitch[p] : row_bytes[p];
        if (user_pitch < row_bytes[p]) { set_error("output plane pitch is smaller than a row"); return SMR_ERR_INVALID_ARGUMENT; }
        if (of.mem_kind == SMR_MEM_DEVICE) {
            // every kernel that writes RGBA8 stores whole pixels (4-byte words); YUV planes may start at any byte
            if (o.format == SMR_OUT_RGBA8 && (((uintptr_t)of.planes[p] | user_pitch) & 3)) {
                set_error("device RGBA8 output planes are 4-byte aligned (pointer and pitch)");
                return SMR_ERR_INVALID_ARGUMENT;
            }
            dst[p] = (uint8_t *)of.planes[p];
            pitch[p] = (int)user_pitch;
        } else {
            size_t dp = (row_bytes[p] + 15) & ~(size_t)15;  // 16-B rows: vector stores
            DevBuf &stage = o.planes[slot_][p];   // the slot's previous tick was waited for in render_begin
            CUDA_OK(stage.ensure(dp * rows[p]));
            dst[p] = stage.p;
            pitch[p] = (int)dp;
            plan_.d2h.push_back({of.planes[p], user_pitch, dst[p], dp, row_bytes[p], rows[p]});
            stats_.d2h_bytes += row_bytes[p] * rows[p];
        }
    }
    auto push_fill = [&]() {
        Fill f;
        for (int p = 0; p < 3; p++) { f.p[p] = dst[p]; f.pitch[p] = pitch[p]; }
        f.w = (int)of.width; f.h = (int)of.height; f.fmt = o.format;
        black_yuv(f.yuv);
        plan_.fills.push_back(f);
    };
    auto push_output_job = [&](int src_tex) {
        dev::OutputJob j;
        j.out_w = (int)of.width; j.out_h = (int)of.height; j.out_format = o.format;
        j.out0 = dst[0]; j.out1 = dst[1]; j.out2 = dst[2];
        j.out_pitch0 = pitch[0]; j.out_pitch1 = pitch[1]; j.out_pitch2 = pitch[2];
        plan_.outputs.push_back({j, src_tex});
    };

    if (!o.flat && o.node.root_is_input) {  // pass-through: the root texture IS the input's node texture
        auto it = inputs_.find(o.node.root_input_id);
        if (it == inputs_.end() || !it->second.has_frame) { push_fill(); return SMR_OK; }
        Input &in = it->second;
        if (o.format == SMR_OUT_RGBA8 && (in.res.width != o.res.width || in.res.height != o.res.height)) {
            // the reference hands out a clone of the node texture at ITS resolution (render_loop.rs:81-103)
            set_error("RGBA output of a pass-through root must match the input resolution");
            return SMR_ERR_UNSUPPORTED;
        }
        const bool same = in.res.width == o.res.width && in.res.height == o.res.height;
        const bool fused_fmt = o.format == SMR_OUT_PLANAR_YUV420 || o.format == SMR_OUT_NV12;   // K10/K11 in the composite
        if (same && (o.format == SMR_OUT_RGBA8 || (fused_fmt && (of.width % 2 == 0) && (of.height % 2 == 0)))) {
            // Same size: K1 -> K10 runs as ONE composite launch with a single full-frame texture layer; an
            // unmodified opaque texel passes through the sRGB target byte-exactly, so the bytes K10 sees
            // are the node texture's.
            RenderLayout l;
            l.kind = RenderLayout::ChildNode;
            l.width = (float)of.width; l.height = (float)of.height;
            l.crop = {0.0f, 0.0f, (float)of.width, (float)of.height};
            dev::LayerDev d;
            bool skip;
            prepare_layer(l, (int)of.width, (int)of.height, in.raw_tex, (int)of.width, (int)of.height, d, skip);
            CompositeRec pc;
            memset(&pc.job, 0, sizeof(pc.job));
            pc.job.width = (int)of.width; pc.job.height = (int)of.height; pc.job.mode = mode;
            pc.job.n_layers = skip ? 0 : 1;
            pc.layers_off = param_put(&d, sizeof(d));
            pc.masks_off = param_alloc(sizeof(dev::MaskDev));
            pc.job.out_format = o.format;
            pc.job.out0 = dst[0]; pc.job.out1 = dst[1]; pc.job.out2 = dst[2];
            pc.job.out_pitch0 = pitch[0]; pc.job.out_pitch1 = pitch[1]; pc.job.out_pitch2 = pitch[2];
            plan_.composites.push_back(pc);
            return SMR_OK;
        }
        push_output_job(in.raw_tex);
        return SMR_OK;
    }

    std::vector<Input *> child_in;
    std::vector<std::optional<Resolution>> child_res;
    const Resolution root = output_children(o, o.node, pts, child_in, child_res);
    if (root.width == 0 || root.height == 0 || root.width > 16384 || root.height > 16384) { push_fill(); return SMR_OK; }
    std::vector<RenderLayout> layouts = output_layouts(o, o.node, pts, child_res, root);
    if (layouts.size() > opts_.max_layouts_count) layouts.resize(opts_.max_layouts_count);  // params.rs:176-182

    const int W = (int)root.width, H = (int)root.height;
    std::vector<dev::LayerDev> layers;
    std::vector<dev::MaskDev> masks;
    for (RenderLayout &l : layouts) {
        int tex_index = -1, tex_w = 1, tex_h = 1;
        Input *in = l.kind == RenderLayout::ChildNode && l.index < child_in.size() ? child_in[l.index] : nullptr;
        if (in) {
            smr_status st = child_texture(*in, l, tex_index, tex_w, tex_h);
            if (st != SMR_OK) return st;
        }
        dev::LayerDev d;
        bool skip;
        prepare_layer(l, W, H, tex_index, tex_w, tex_h, d, skip);
        if (skip) continue;
        d.mask_begin = (int)masks.size();
        d.mask_count = layer_masks(l, masks);
        layers.push_back(d);
    }

    CompositeRec pc;
    memset(&pc.job, 0, sizeof(pc.job));
    pc.job.width = W; pc.job.height = H; pc.job.mode = mode;
    pc.job.n_layers = (int)layers.size();
    pc.layers_off = param_put(layers.data(), sizeof(dev::LayerDev) * layers.size());
    pc.masks_off = param_put(masks.data(), sizeof(dev::MaskDev) * masks.size());

    bool same_size = (size_t)W == o.res.width && (size_t)H == o.res.height;
    bool fused_fmt = o.format == SMR_OUT_PLANAR_YUV420 || o.format == SMR_OUT_NV12;
    bool fusable = same_size && (o.format == SMR_OUT_RGBA8 || (fused_fmt && (W % 2 == 0) && (H % 2 == 0)));
    if (fusable) {
        pc.job.out_format = o.format;
        pc.job.out0 = dst[0]; pc.job.out1 = dst[1]; pc.job.out2 = dst[2];
        pc.job.out_pitch0 = pitch[0]; pc.job.out_pitch1 = pitch[1]; pc.job.out_pitch2 = pitch[2];
        if (fused_fmt) plan_tiles(o, pc, layers, W, H);
        plan_.composites.push_back(pc);
    } else {
        if (o.format == SMR_OUT_RGBA8) { set_error("RGBA output must match the root layout resolution"); return SMR_ERR_UNSUPPORTED; }
        pc.out_frame_off = frame_alloc((size_t)W * H * 4);
        pc.job.out_format = -1;
        pc.job.out_pitch0 = W * 4;
        plan_.composites.push_back(pc);
        dev::Tex t;
        t.kind = dev::TEX_RGBA8; t.width = W; t.height = H; t.pitch0 = W * 4;
        push_output_job(add_texture(t, false, pc.out_frame_off));
    }
    return SMR_OK;
}

smr_status Renderer::render_begin(uint64_t pts, const smr_input_frame *in, uint32_t n_in, smr_output_frame *out,
                                  uint32_t n_out) {
    if ((n_in && !in) || (n_out && !out)) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    if (host_only_) { set_error("host-only handle (cuda_device = -1) cannot render: no CPU fallback"); return SMR_ERR_CUDA; }
    CUDA_OK(cudaSetDevice(opts_.cuda_device));
    if (profiling_ && !inflight_.empty()) drain();   // per-kernel timing: one tick at a time
    tick_++;
    slot_ = (int)(tick_ % kTicksInFlight);
    // the slot's buffers (pinned params, input staging) belong to the tick kTicksInFlight ago: wait for it (without retiring it)
    for (int s : inflight_)
        if (s == slot_) CUDA_OK(cudaEventSynchronize(tick_done_[s]));
    while ((int)inflight_.size() >= kTicksInFlight) {   // never more than kTicksInFlight in flight: the oldest is retired here
        CUDA_OK(cudaEventSynchronize(tick_done_[inflight_.front()]));
        inflight_.pop_front();
    }
    uploaded_ = false;
    rollback_weights();   // leftovers of a tick that failed before its weight launch (normally empty)
    plan_.clear();
    param_used_ = 0; frame_used_ = 0;
    uint64_t launches = 0;
    cudaStream_t done_on = stream_;   // the stream the tick's last operation goes to

    struct WeightGuard {   // any return before the k_weights launch is enqueued drops this tick's new cache entries
        Renderer *r; bool armed = true;
        ~WeightGuard() { if (armed) r->rollback_weights(); }
    } weight_guard{this};
    smr_status st = select_inputs(pts, in, n_in, [&](Input &I, const smr_input_frame *f) {
        I.node_tex = I.raw_tex = -1;
        return f ? upload_input(I, *f) : SMR_OK;
    });
    if (st != SMR_OK) return st;
    for (uint32_t i = 0; i < n_out; i++) {
        if (!out[i].output_id) return SMR_ERR_INVALID_ARGUMENT;
        auto it = outputs_.find(out[i].output_id);
        if (it == outputs_.end()) {
            set_error(std::string("Output \"") + out[i].output_id + "\" does not exist, register it first");
            return SMR_ERR_OUTPUT_NOT_REGISTERED;
        }
        st = plan_output(it->second, out[i], pts);
        if (st != SMR_OK) return st;
    }

    // everything already on the stream belongs to earlier ticks: a broadcast issued after this call may overwrite any
    // buffer those ticks read once this event has fired
    CUDA_OK(cudaEventRecord(tick_start_, stream_));
    tick_started_ = true;
    if (comm_pending_) {   // this tick's shared inputs arrive on the communication stream
        CUDA_OK(cudaStreamWaitEvent(stream_, comm_done_, 0));
        comm_pending_ = false;
    }
    // ---- resolve frame-arena addresses --------------------------------------------------------
    if (uploaded_) {   // kernels of this tick start after its uploads; earlier ticks keep running meanwhile
        CUDA_OK(cudaEventRecord(h2d_done_[slot_], copy_stream_));
        CUDA_OK(cudaStreamWaitEvent(stream_, h2d_done_[slot_], 0));
        CUDA_OK(cudaEventRecord(h2d_done2_[slot_], copy_stream2_));
        CUDA_OK(cudaStreamWaitEvent(stream_, h2d_done2_[slot_], 0));
    }
    if (frame_used_ + 512 > frame_dev_.cap && !inflight_.empty()) CUDA_OK(cudaStreamSynchronize(stream_));
    CUDA_OK(frame_dev_.ensure(frame_used_ + 512));
    uint8_t *fb = frame_dev_.p;
    for (TexRec &t : plan_.tex)
        if (t.frame_off != SIZE_MAX) t.tex.p0 = fb + t.frame_off;
    for (auto &stage : plan_.stages)
        for (StageRec &r : stage) {
            if (r.src_tex >= 0) r.job.src = plan_.tex[r.src_tex].tex;
            else r.job.src.p0 = fb + r.src_off;
            r.job.dst = fb + r.dst_off;
        }
    for (OutputRec &r : plan_.outputs) r.job.src = plan_.tex[r.src_tex].tex;
    for (FusedRec &f : plan_.fused) {
        f.job.src = plan_.tex[f.src_tex].tex;
        f.job.dst = fb + f.dst_off;
    }
    for (CompositeRec &c : plan_.composites)
        if (c.out_frame_off != SIZE_MAX) c.job.out0 = fb + c.out_frame_off;

    // ---- pack the parameter arena and ship it in one copy -------------------------------------
    // partition the fused resamples of the tick over a persistent grid, one launch per kernel, source class and launch range
    struct FusedKey {
        dev::FusedKernel kernel; int src, range;
        bool operator==(const FusedKey &o) const { return kernel == o.kernel && src == o.src && range == o.range; }
    };
    auto key_of = [](const FusedRec &f) {
        return FusedKey{f.kernel, dev::fused_source_class(f.job.src.kind), dev::fused_launch_range(f.kernel, f.job)};
    };
    struct FusedLaunch { FusedKey key; size_t pieces_off, begin_off; int nblocks; };
    std::vector<FusedLaunch> fused_launches;
    {
        std::vector<FusedKey> keys;
        for (const FusedRec &f : plan_.fused)
            if (std::find(keys.begin(), keys.end(), key_of(f)) == keys.end()) keys.push_back(key_of(f));
        for (const FusedKey &v : keys) {
            std::vector<int> idx, widths, heights, cols;
            dev::FusedShape shape{};
            for (size_t ji = 0; ji < plan_.fused.size(); ji++) {
                const FusedRec &f = plan_.fused[ji];
                if (!(key_of(f) == v)) continue;
                shape = dev::fused_shape(f.kernel, f.job);
                idx.push_back((int)ji); widths.push_back(f.job.dst_w); heights.push_back(f.job.dst_h); cols.push_back(shape.strip_cols);
            }
            std::vector<dev::FusedPiece> pieces;
            std::vector<int> begin;
            partition_fused_rows(idx.data(), widths.data(), heights.data(), (int)idx.size(), sm_count_ * shape.groups_per_sm, pieces,
                                 begin, dev::kFusedStripCols, cols.data(), shape.row_gran);
            if (pieces.empty()) continue;
            // direct tiles: the vertical pass emits K10 / K11 per PAIR of output rows, so a job's pieces must hold whole pairs
            // (they do whenever every job of the launch has an even height); a job cut at an odd row writes nothing directly
            for (const dev::FusedPiece &pp : pieces)
                if (plan_.fused[pp.job].direct_off != SIZE_MAX && ((pp.oy_begin | pp.oy_end) & 1)) {
                    plan_.fused[pp.job].direct_off = SIZE_MAX;
                    for (CompositeRec &pc : plan_.composites)
                        for (size_t t = 0; t < pc.direct_owner.size(); t++)
                            if (pc.direct_owner[t] == pp.job) {   // back to the composite (cheap interior tiles: at the end of the list)
                                pc.direct_owner[t] = -1;
                                pc.list.push_back((uint32_t)(t % (size_t)pc.job.map_w) | ((uint32_t)(t / (size_t)pc.job.map_w) << 16));
                            }
                }
            fused_launches.push_back({v, param_put(pieces.data(), sizeof(dev::FusedPiece) * pieces.size()),
                                      param_put(begin.data(), sizeof(int) * begin.size()), (int)begin.size() - 1});
        }
    }
    const size_t tex_off = param_put_all(plan_.tex, &TexRec::tex);
    size_t stage_off[3];
    for (int s = 0; s < 3; s++) stage_off[s] = param_put_all(plan_.stages[s], &StageRec::job);
    const size_t wj_off = param_put(plan_.weight_jobs.data(), sizeof(dev::WeightJob) * plan_.weight_jobs.size());
    const size_t tm_off = param_put(plan_.tmaps.data(), sizeof(CUtensorMap) * plan_.tmaps.size());
    uint64_t direct_tiles = 0;
    for (CompositeRec &pc : plan_.composites) {   // direct-tile maps (one byte per tile: the owner's id) and tile lists
        if (pc.direct_off != SIZE_MAX) {
            bool any = false;
            for (size_t t = 0; t < pc.direct_owner.size(); t++) {
                param_host_[pc.direct_off + t] = pc.direct_owner[t] >= 0 ? (uint8_t)(pc.direct_owner[t] + 1) : 0;
                any = any || pc.direct_owner[t] >= 0;
                direct_tiles += pc.direct_owner[t] >= 0 ? 1 : 0;
            }
            if (!any) pc.direct_off = SIZE_MAX;
        }
        if (pc.use_list) {
            pc.list_off = param_put(pc.list.data(), sizeof(uint32_t) * pc.list.size());
            pc.job.n_tiles = (int)pc.list.size();
        }
    }
    const size_t fj_off = param_put_all(plan_.fused, &FusedRec::job);
    const size_t cj_off = param_put_all(plan_.composites, &CompositeRec::job);   // read by k_composite_multi
    // the arena is sized: its offsets become device pointers in the packed jobs
    CUDA_OK(param_pinned_[slot_].ensure(param_used_));
    CUDA_OK(param_dev_[slot_].ensure(param_used_));
    uint8_t *pd = param_dev_[slot_].p;
    auto dev_ptr = [&](size_t off) -> uint8_t * { return off != SIZE_MAX ? pd + off : nullptr; };
    dev::FusedJob *fj = reinterpret_cast<dev::FusedJob *>(param_host_.data() + fj_off);
    for (size_t i = 0; i < plan_.fused.size(); i++) {
        const FusedRec &f = plan_.fused[i];
        if (f.tmap_idx >= 0) {
            const uint8_t *m = pd + tm_off + sizeof(CUtensorMap) * (size_t)f.tmap_idx;
            fj[i].tm0 = m; fj[i].tm1 = m + sizeof(CUtensorMap); fj[i].tm2 = m + 2 * sizeof(CUtensorMap);
        }
        fj[i].direct_map = dev_ptr(f.direct_off);
    }
    dev::CompositeJob *cj = reinterpret_cast<dev::CompositeJob *>(param_host_.data() + cj_off);
    for (size_t i = 0; i < plan_.composites.size(); i++) {
        const CompositeRec &c = plan_.composites[i];
        cj[i].layers = (const dev::LayerDev *)(pd + c.layers_off);
        cj[i].masks = (const dev::MaskDev *)(pd + c.masks_off);
        cj[i].textures = (const dev::Tex *)(pd + tex_off);
        cj[i].direct_map = dev_ptr(c.direct_off);
        cj[i].tile_list = (const uint32_t *)dev_ptr(c.list_off);
    }
    memcpy(param_pinned_[slot_].p, param_host_.data(), param_used_);
    CUDA_OK(cudaMemcpyAsync(pd, param_pinned_[slot_].p, param_used_, cudaMemcpyHostToDevice, stream_));

    // ---- launches -----------------------------------------------------------------------------
    auto launched = [&](int n) -> bool { if (n < 0) return false; launches += (uint64_t)n; return true; };
    prof_mark(-1);
    for (auto &cv : plan_.convert_jobs) {
        const dev::Tex &src = plan_.tex[cv.first].tex;
        if (!launched(dev::launch_convert_to_rgba(src, fb + cv.second, src.width * 4, stream_))) goto fail;
        prof_mark(SMR_KERNEL_CONVERT);
    }
    if (!launched(dev::launch_weights((const dev::WeightJob *)(pd + wj_off), plan_.weight_jobs.data(), (int)plan_.weight_jobs.size(),
                                      stream_))) goto fail;
    if (!plan_.weight_jobs.empty()) prof_mark(SMR_KERNEL_WEIGHTS);
    new_weight_keys_.clear();
    weight_guard.armed = false;   // the tables are being computed on the stream: the cache entries are good
    for (const FusedLaunch &fl : fused_launches) {
        if (!launched(dev::launch_resample_fused(fl.key.kernel, fl.key.src, fl.key.range, (const dev::FusedJob *)(pd + fj_off),
                                                 (const dev::FusedPiece *)(pd + fl.pieces_off), (const int *)(pd + fl.begin_off),
                                                 fl.nblocks, stream_))) goto fail;
        prof_mark(SMR_KERNEL_RESAMPLE_FUSED);
    }
    for (int s = 0; s < 3; s++) {
        if (!launched(dev::launch_resample((const dev::ResampleJob *)(pd + stage_off[s]),
                                           (const dev::ResampleJob *)(param_host_.data() + stage_off[s]), (int)plan_.stages[s].size(),
                                           stream_))) goto fail;
        if (!plan_.stages[s].empty()) prof_mark(SMR_KERNEL_RESAMPLE_BOX + s);
    }
    if (!plan_.composites.empty()) {   // ONE launch for every output of the tick
        if (!launched(dev::launch_composite((const dev::CompositeJob *)(pd + cj_off), cj,
                                            (const dev::LayerDev *)(param_host_.data() + plan_.composites[0].layers_off),
                                            (int)plan_.composites.size(), stream_))) goto fail;
        prof_mark(SMR_KERNEL_COMPOSITE);
    }
    for (OutputRec &o : plan_.outputs) {
        if (!launched(dev::launch_output(o.job, stream_))) goto fail;
        prof_mark(SMR_KERNEL_OUTPUT);
    }
    for (Fill &f : plan_.fills) {
        if (!launched(dev::launch_fill_yuv(f.p[0], f.p[1], f.p[2], f.pitch[0], f.pitch[1], f.pitch[2], f.w, f.h, f.fmt,
                                           f.yuv[0], f.yuv[1], f.yuv[2], stream_))) goto fail;
        prof_mark(SMR_KERNEL_FILL);
    }
    // read-back on its own stream: the staging planes are per slot, so the next tick's kernels need not wait for it
    if (!plan_.d2h.empty() && !profiling_) {
        CUDA_OK(cudaEventRecord(kernels_done_[slot_], stream_));
        CUDA_OK(cudaStreamWaitEvent(d2h_stream_, kernels_done_[slot_], 0));
        done_on = d2h_stream_;
    }
    for (PendingCopy &c : plan_.d2h)
        if (c.dpitch == c.width && c.spitch == c.width)
            CUDA_OK(cudaMemcpyAsync(c.dst, c.src, c.width * c.height, cudaMemcpyDeviceToHost, done_on));
        else
            CUDA_OK(cudaMemcpy2DAsync(c.dst, c.dpitch, c.src, c.spitch, c.width, c.height, cudaMemcpyDeviceToHost, done_on));
    stats_.kernel_launches += launches;
    stats_.last_render_kernel_launches = launches;
    stats_.last_render_direct_tiles = direct_tiles;
    stats_.frames_rendered += n_out;
    CUDA_OK(cudaEventRecord(tick_done_[slot_], done_on));
    inflight_.push_back(slot_);
    return SMR_OK;
fail:
    set_error(dev::last_launch_error());
    cudaStreamSynchronize(stream_);
    return SMR_ERR_CUDA;
}

// inspection: what smr_render records for this FrameSet (select_inputs), without reading or copying the frames
smr_status Renderer::debug_set_inputs(uint64_t pts, const smr_input_frame *in, uint32_t n_in) {
    if (n_in && !in) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    return select_inputs(pts, in, n_in, [](Input &, const smr_input_frame *) { return SMR_OK; });
}

// inspection: the fused resample jobs of the last planned tick, as render_begin packed and launched them
smr_status Renderer::debug_fused_jobs(smr_fused_job_info *out, uint32_t cap, uint32_t *n) {
    if (!n) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    *n = (uint32_t)plan_.fused.size();
    if (!out) return SMR_OK;
    if (cap < plan_.fused.size()) return SMR_ERR_BUFFER_TOO_SMALL;
    for (size_t i = 0; i < plan_.fused.size(); i++) {
        const FusedRec &f = plan_.fused[i];
        const dev::FusedJob &j = f.job;
        smr_fused_job_info &o = out[i];
        o.kernel = f.kernel.kind == dev::FusedKernel::TMA_INT   ? SMR_FUSED_TMA_INT
                   : f.kernel.kind == dev::FusedKernel::TMA_ANY ? SMR_FUSED_TMA_ANY
                                                                : SMR_FUSED_LDG;
        o.ratio = f.kernel.ratio;
        o.window = f.kernel.kind == dev::FusedKernel::TMA_ANY ? dev::kTma0Window[f.kernel.window] : 0;
        o.box = f.kernel.box;
        o.src_class = dev::fused_source_class(j.src.kind);
        o.full_range = j.src.full_range;
        o.v_same = j.v_same;
        o.strip_cols = dev::fused_shape(f.kernel, j).strip_cols;
        o.src_width = (uint32_t)j.src.width; o.src_height = (uint32_t)j.src.height;
        o.dst_width = (uint32_t)j.dst_w; o.dst_height = (uint32_t)j.dst_h;
        o.taps_h = j.taps_h; o.taps_v = j.taps_v;
        o.direct = f.direct_off != SIZE_MAX ? 1 : 0;
    }
    return SMR_OK;
}

// inspection: the generic resample passes and k_convert jobs of the last planned tick
smr_status Renderer::debug_resample_stages(smr_resample_stage_info *out, uint32_t cap, uint32_t *n, int32_t *convert_kinds,
                                           uint32_t convert_cap, uint32_t *n_convert) {
    if (!n || !n_convert) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    size_t total = 0;
    for (const auto &stage : plan_.stages) total += stage.size();
    *n = (uint32_t)total;
    *n_convert = (uint32_t)plan_.convert_jobs.size();
    if ((out && cap < total) || (convert_kinds && convert_cap < plan_.convert_jobs.size())) return SMR_ERR_BUFFER_TOO_SMALL;
    if (convert_kinds)
        for (size_t i = 0; i < plan_.convert_jobs.size(); i++) convert_kinds[i] = plan_.tex[plan_.convert_jobs[i].first].tex.kind;
    if (!out) return SMR_OK;
    size_t k = 0;
    for (int s = 0; s < 3; s++)
        for (const StageRec &r : plan_.stages[s]) {
            const dev::ResampleJob &j = r.job;
            smr_resample_stage_info &o = out[k++];
            memset(&o, 0, sizeof(o));
            o.stage = s;
            o.axis = s == 0 ? -1 : j.axis;
            o.box_fx = j.box_fx; o.box_fy = j.box_fy;
            o.taps = s == 0 ? 0 : j.taps;
            o.perp_offset = j.perp_offset;
            dev::Tex src = j.src;   // the f16 intermediate's geometry is in the job
            o.source = SMR_STAGE_SRC_F16;
            if (r.src_tex >= 0) {
                src = plan_.tex[r.src_tex].tex;
                o.source = SMR_STAGE_SRC_RAW;
                for (const auto &cv : plan_.convert_jobs)
                    if (plan_.tex[r.src_tex].frame_off == cv.second) {
                        o.source = SMR_STAGE_SRC_CONVERTED;
                        src.kind = plan_.tex[cv.first].tex.kind;
                    }
            }
            o.src_kind = src.kind;
            o.src_width = (uint32_t)src.width; o.src_height = (uint32_t)src.height;
            o.dst_width = (uint32_t)j.dst_w; o.dst_height = (uint32_t)j.dst_h;
            o.dst_f16 = j.dst_f16;
        }
    return SMR_OK;
}

// inspection: the layers of the last planned tick's composite jobs, as render_begin packed and launched them
smr_status Renderer::debug_composite_layers(smr_composite_layer_info *out, uint32_t cap, uint32_t *n) {
    if (!n) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    size_t total = 0;
    for (const CompositeRec &c : plan_.composites) total += (size_t)c.job.n_layers;
    *n = (uint32_t)total;
    if (!out) return SMR_OK;
    if (cap < total) return SMR_ERR_BUFFER_TOO_SMALL;
    // launch_composite's choice
    const int kernel = plan_.composites.size() == 1 && plan_.composites[0].job.n_layers <= dev::kCompositeParamLayers
                           ? SMR_COMPOSITE_PARAM : SMR_COMPOSITE_MULTI;
    size_t k = 0;
    for (size_t ci = 0; ci < plan_.composites.size(); ci++) {
        const CompositeRec &c = plan_.composites[ci];
        const dev::LayerDev *layers = reinterpret_cast<const dev::LayerDev *>(param_host_.data() + c.layers_off);
        for (int li = 0; li < c.job.n_layers; li++, k++) {
            const dev::LayerDev &L = layers[li];
            smr_composite_layer_info &o = out[k];
            memset(&o, 0, sizeof(o));
            o.job = (int32_t)ci; o.kernel = kernel; o.layer = li;
            o.type = L.type; o.rotated = L.rotated; o.fast = L.fast;
            const int32_t box[12] = {L.px0, L.px1, L.py0, L.py1, L.ix0, L.ix1, L.iy0, L.iy1, L.jx0, L.jx1, L.jy0, L.jy1};
            memcpy(o.box, box, sizeof(box));
            o.tx_off = L.tx_off; o.ty_off = L.ty_off;
            o.mask_count = L.mask_count;
            if (L.type == 0 && L.tex >= 0) {
                const dev::Tex &t = plan_.tex[L.tex].tex;
                const uint8_t *p[3] = {t.p0, t.p1, t.p2};
                const int32_t pitch[3] = {t.pitch0, t.pitch1, t.pitch2};
                o.tex_kind = t.kind; o.tex_width = t.width; o.tex_height = t.height;
                for (int pl = 0; pl < 3; pl++) {
                    o.tex_pitch[pl] = p[pl] ? pitch[pl] : 0;
                    o.tex_align[pl] = (int32_t)((uintptr_t)p[pl] & 15);
                }
            }
            o.width = c.job.width; o.height = c.job.height;
            o.out_format = c.job.out_format;
        }
    }
    return SMR_OK;
}

smr_status Renderer::render_end() {   // retires the OLDEST tick in flight
    std::lock_guard<std::mutex> g(mu_);
    if (inflight_.empty()) return SMR_OK;
    CUDA_OK(cudaSetDevice(opts_.cuda_device));
    int s = inflight_.front();
    inflight_.pop_front();
    CUDA_OK(cudaEventSynchronize(tick_done_[s]));
    if (inflight_.empty()) fold_profile();
    return SMR_OK;
}

smr_status Renderer::render_end_all() {   // smr_render: "blocks until the output planes are complete" -- of THIS tick
    std::lock_guard<std::mutex> g(mu_);
    if (inflight_.empty()) return SMR_OK;
    CUDA_OK(cudaSetDevice(opts_.cuda_device));
    while (!inflight_.empty()) {
        int s = inflight_.front();
        inflight_.pop_front();
        CUDA_OK(cudaEventSynchronize(tick_done_[s]));
    }
    fold_profile();
    return SMR_OK;
}

void Renderer::fold_profile() {
    // fold this tick's event pairs into the per-kernel-class totals
    for (size_t i = 1; i < prof_marks_.size(); i++) {
        int k = prof_marks_[i].second;
        if (k < 0) continue;
        float ms = 0.0f;
        if (cudaEventElapsedTime(&ms, prof_marks_[i - 1].first, prof_marks_[i].first) == cudaSuccess) {
            prof_.total_ms[k] += ms;
            prof_.launches[k] += 1;
        }
    }
    prof_marks_.clear();
}

void Renderer::prof_mark(int kernel_class) {
    if (!profiling_) return;
    if (kernel_class == -1) { prof_marks_.clear(); prof_next_event_ = 0; }
    if (prof_next_event_ >= prof_events_.size()) {
        cudaEvent_t e;
        if (cudaEventCreate(&e) != cudaSuccess) return;
        prof_events_.push_back(e);
    }
    cudaEvent_t e = prof_events_[prof_next_event_++];
    cudaEventRecord(e, stream_);
    prof_marks_.push_back({e, kernel_class});
}

// ------------------------------------------------------------------------------------------------
// Multi-GPU: outputs shard across GPUs with no data-path collective; the only exchange is replicating an
// input frame to every GPU that hosts an output referencing it (ncclBroadcast over NVLink, grouped per tick,
// enqueued on the render stream so the following smr_render is ordered after it).
// ------------------------------------------------------------------------------------------------
smr_status Renderer::comm_init(const uint8_t *id, int rank, int nranks) {
    std::lock_guard<std::mutex> g(mu_);
    if (host_only_) { set_error("host-only handle has no device"); return SMR_ERR_CUDA; }
    if (!id || nranks < 1 || rank < 0 || rank >= nranks) return SMR_ERR_INVALID_ARGUMENT;
    std::string err;
    if (!nccl_load(err)) { set_error(err); return SMR_ERR_UNSUPPORTED; }
    CUDA_OK(cudaSetDevice(opts_.cuda_device));
    NcclId nid;
    memcpy(nid.b, id, 128);
    int rc = g_nccl.CommInitRank(&nccl_comm_, nranks, nid, rank);
    if (rc != 0) { set_error(std::string("ncclCommInitRank: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error")); return SMR_ERR_CUDA; }
    comm_rank_ = rank; comm_size_ = nranks;
    return SMR_OK;
}

// consumers[i]: bit k set = rank k hosts an output that reads frame i (NULL: every rank).  A frame every rank needs
// goes out as ncclBroadcast (ring / tree / NVLS inside NCCL); a frame only some ranks need is sent point to point to
// exactly those ranks, so a rank that does not consume it neither receives nor stores it.
smr_status Renderer::comm_exchange(const smr_input_frame *frames, uint32_t n, const int32_t *roots, const uint64_t *consumers,
                                   uint32_t flags) {
    std::lock_guard<std::mutex> g(mu_);
    if (!nccl_comm_) { set_error("smr_comm_init was not called"); return SMR_ERR_INVALID_ARGUMENT; }
    if (n && (!frames || !roots)) return SMR_ERR_INVALID_ARGUMENT;
    if (comm_size_ > 64 && consumers) { set_error("consumer masks cover at most 64 ranks"); return SMR_ERR_UNSUPPORTED; }
    CUDA_OK(cudaSetDevice(opts_.cuda_device));
    // Runs on its own stream so that it overlaps the kernels of the tick submitted last; it is ordered after every
    // EARLIER tick (whose buffers the caller may be recycling) and before the next smr_render_begin.
    if (tick_started_) CUDA_OK(cudaStreamWaitEvent(comm_stream_, tick_start_, 0));
    if (flags & SMR_COMM_PEER_DIRECT) {
        // nothing moves: the frames rooted elsewhere are read in place over NVLink by the tick's kernels (the TMA loads of the
        // fused resample kernel); the step is the cross-rank ordering alone
        smr_status st = comm_tick_barrier();
        if (st != SMR_OK) return st;
        CUDA_OK(cudaEventRecord(comm_done_, comm_stream_));
        comm_pending_ = true;
        return SMR_OK;
    }
    const uint64_t all = comm_size_ >= 64 ? ~0ull : ((1ull << comm_size_) - 1ull);
    // SMR_COMM_POOLED: the caller declares that the planes are laid out identically on every rank (e.g. one frame pool
    // per ingest GPU), so consecutive planes with the same root and consumers that are contiguous HERE are contiguous
    // everywhere and go out as one message.  Without the declaration nothing is merged: the sequence of collectives
    // must not depend on a rank's allocator.
    struct Run { uint8_t *p; size_t bytes; int root; uint64_t mask; };
    std::vector<Run> runs;
    for (uint32_t i = 0; i < n; i++) {
        const smr_input_frame &f = frames[i];
        if (f.mem_kind != SMR_MEM_DEVICE) { set_error("the exchange needs device-resident planes"); return SMR_ERR_INVALID_ARGUMENT; }
        if (roots[i] < 0 || roots[i] >= comm_size_) return SMR_ERR_INVALID_ARGUMENT;
        const uint64_t mask = ((consumers ? consumers[i] : all) | (1ull << roots[i])) & all;
        FrameView v;
        if (smr_status st = read_frame(f, v); st != SMR_OK) return st;
        for (const FrameView::Plane &P : v.plane) {
            if (!P.p) continue;
            const size_t bytes = P.span();
            uint8_t *ptr = (uint8_t *)P.p;
            if ((flags & SMR_COMM_POOLED) && !runs.empty() && runs.back().root == roots[i] && runs.back().mask == mask &&
                runs.back().p + runs.back().bytes == ptr)
                runs.back().bytes += bytes;
            else
                runs.push_back({ptr, bytes, roots[i], mask});
        }
    }
    int rc = g_nccl.GroupStart();
    for (size_t i = 0; i < runs.size() && rc == 0; i++) {
        const Run &R = runs[i];
        if (R.mask == all) {
            rc = g_nccl.Broadcast(R.p, R.p, R.bytes, /*ncclUint8*/ 1, R.root, nccl_comm_, comm_stream_);
        } else if (comm_rank_ == R.root) {
            for (int k = 0; k < comm_size_ && rc == 0; k++)
                if (k != R.root && ((R.mask >> k) & 1ull)) rc = g_nccl.Send(R.p, R.bytes, 1, k, nccl_comm_, comm_stream_);
        } else if ((R.mask >> comm_rank_) & 1ull) {
            rc = g_nccl.Recv(R.p, R.bytes, 1, R.root, nccl_comm_, comm_stream_);
        }
    }
    int rc2 = g_nccl.GroupEnd();
    if (rc == 0) rc = rc2;
    if (rc != 0) { set_error(std::string("NCCL exchange: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error")); return SMR_ERR_CUDA; }
    CUDA_OK(cudaEventRecord(comm_done_, comm_stream_));
    comm_pending_ = true;
    return SMR_OK;
}

// A 4-byte all-reduce on the communication stream: when it completes here, every rank's communication stream has reached
// the same tick, i.e. every rank has finished the ticks before its last submitted one and has its frames of this tick in
// place.  The only cross-GPU traffic of SMR_COMM_PEER_DIRECT besides the tile loads themselves.
smr_status Renderer::comm_tick_barrier() {
    if (!barrier_word_) {
        CUDA_OK(cudaMalloc(&barrier_word_, 256));
        CUDA_OK(cudaMemsetAsync(barrier_word_, 0, 256, comm_stream_));
    }
    int rc = g_nccl.AllReduce(barrier_word_, barrier_word_, 1, /*ncclInt32*/ 2, /*ncclSum*/ 0, nccl_comm_, comm_stream_);
    if (rc != 0) { set_error(std::string("NCCL barrier: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error")); return SMR_ERR_CUDA; }
    return SMR_OK;
}

// Pull form of the exchange: after the tick barrier each consumer copies the frames rooted elsewhere out of the root's pool
// (opened with smr_peer_pool_open) with the copy engines -- cudaMemcpyAsync over NVLink, no SM is spent on the transfer.
smr_status Renderer::comm_pull(const smr_input_frame *frames, const smr_input_frame *peer_frames, uint32_t n, const int32_t *roots,
                               const uint64_t *consumers) {
    std::lock_guard<std::mutex> g(mu_);
    if (!nccl_comm_) { set_error("smr_comm_init was not called"); return SMR_ERR_INVALID_ARGUMENT; }
    if (n && (!frames || !peer_frames || !roots)) return SMR_ERR_INVALID_ARGUMENT;
    CUDA_OK(cudaSetDevice(opts_.cuda_device));
    if (tick_started_) CUDA_OK(cudaStreamWaitEvent(comm_stream_, tick_start_, 0));
    smr_status st = comm_tick_barrier();
    if (st != SMR_OK) return st;
    struct Run { uint8_t *dst; const uint8_t *src; size_t bytes; };
    std::vector<Run> runs;
    for (uint32_t i = 0; i < n; i++) {
        const smr_input_frame &f = frames[i], &pf = peer_frames[i];
        if (roots[i] < 0 || roots[i] >= comm_size_) return SMR_ERR_INVALID_ARGUMENT;
        if (roots[i] == comm_rank_) continue;
        if (consumers && !((consumers[i] >> comm_rank_) & 1ull)) continue;
        if (f.mem_kind != SMR_MEM_DEVICE || pf.mem_kind != SMR_MEM_DEVICE) { set_error("the exchange needs device-resident planes"); return SMR_ERR_INVALID_ARGUMENT; }
        if (pf.format != f.format || pf.width != f.width || pf.height != f.height) { set_error("peer frame geometry differs"); return SMR_ERR_INVALID_ARGUMENT; }
        FrameView v, pv;
        st = read_frame(f, v);
        if (st == SMR_OK) st = read_frame(pf, pv);
        if (st != SMR_OK) return st;
        for (int p = 0; p < 3; p++) {
            if (!v.plane[p].p) continue;
            if (v.plane[p].pitch != pv.plane[p].pitch) { set_error("peer frame pitch differs"); return SMR_ERR_INVALID_ARGUMENT; }
            const size_t bytes = v.plane[p].span();
            uint8_t *d = (uint8_t *)v.plane[p].p;
            const uint8_t *sp = pv.plane[p].p;
            if (!runs.empty() && runs.back().dst + runs.back().bytes == d && runs.back().src + runs.back().bytes == sp) runs.back().bytes += bytes;
            else runs.push_back({d, sp, bytes});
        }
    }
    for (const Run &R : runs) CUDA_OK(cudaMemcpyAsync(R.dst, R.src, R.bytes, cudaMemcpyDeviceToDevice, comm_stream_));
    CUDA_OK(cudaEventRecord(comm_done_, comm_stream_));
    comm_pending_ = true;
    return SMR_OK;
}

smr_status Renderer::peer_pool_alloc(size_t bytes, void **dev_ptr, uint8_t handle[64]) {
    std::lock_guard<std::mutex> g(mu_);
    if (!dev_ptr || !handle || !bytes) return SMR_ERR_INVALID_ARGUMENT;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size of the C ABI");
    CUDA_OK(cudaSetDevice(opts_.cuda_device));
    void *p = nullptr;
    CUDA_OK(cudaMalloc(&p, bytes));   // its own allocation: an IPC handle names a whole cudaMalloc block
    cudaIpcMemHandle_t h;
    if (cudaIpcGetMemHandle(&h, p) != cudaSuccess) { cudaGetLastError(); cudaFree(p); set_error("cudaIpcGetMemHandle failed"); return SMR_ERR_CUDA; }
    memcpy(handle, &h, 64);
    peer_own_.push_back(p);
    *dev_ptr = p;
    return SMR_OK;
}

smr_status Renderer::peer_pool_open(const uint8_t handle[64], void **dev_ptr) {
    std::lock_guard<std::mutex> g(mu_);
    if (!dev_ptr || !handle) return SMR_ERR_INVALID_ARGUMENT;
    CUDA_OK(cudaSetDevice(opts_.cuda_device));
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    void *p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) { cudaGetLastError(); set_error(std::string("cudaIpcOpenMemHandle: ") + cudaGetErrorString(e)); return SMR_ERR_CUDA; }
    peer_opened_.push_back(p);
    *dev_ptr = p;
    return SMR_OK;
}

smr_status Renderer::peer_pool_close(void *dev_ptr) {
    std::lock_guard<std::mutex> g(mu_);
    auto it = std::find(peer_opened_.begin(), peer_opened_.end(), dev_ptr);
    if (it == peer_opened_.end()) return SMR_ERR_INVALID_ARGUMENT;
    CUDA_OK(cudaSetDevice(opts_.cuda_device));
    cudaStreamSynchronize(stream_);
    if (comm_stream_) cudaStreamSynchronize(comm_stream_);
    tmap_cache_.clear();   // descriptors of planes inside the mapping
    cudaIpcCloseMemHandle(dev_ptr);
    peer_opened_.erase(it);
    return SMR_OK;
}

smr_status Renderer::peer_pool_free(void *dev_ptr) {
    std::lock_guard<std::mutex> g(mu_);
    auto it = std::find(peer_own_.begin(), peer_own_.end(), dev_ptr);
    if (it == peer_own_.end()) return SMR_ERR_INVALID_ARGUMENT;
    CUDA_OK(cudaSetDevice(opts_.cuda_device));
    cudaStreamSynchronize(stream_);
    if (comm_stream_) cudaStreamSynchronize(comm_stream_);
    tmap_cache_.clear();
    cudaFree(dev_ptr);
    peer_own_.erase(it);
    return SMR_OK;
}

smr_status Renderer::comm_destroy() {
    std::lock_guard<std::mutex> g(mu_);
    if (nccl_comm_) {
        cudaSetDevice(opts_.cuda_device);
        cudaStreamSynchronize(comm_stream_);   // the collectives run here
        cudaStreamSynchronize(stream_);
        g_nccl.CommDestroy(nccl_comm_);
        nccl_comm_ = nullptr;
    }
    return SMR_OK;
}

smr_status Renderer::set_profiling(int enabled) {
    std::lock_guard<std::mutex> g(mu_);
    if (!host_only_) { cudaSetDevice(opts_.cuda_device); drain(); }
    profiling_ = enabled != 0;
    memset(&prof_, 0, sizeof(prof_));
    return SMR_OK;
}

smr_status Renderer::debug_layouts(const char *output_id, uint64_t pts, smr_render_layout *out, uint32_t cap,
                                   uint32_t *n, uint32_t *rw, uint32_t *rh) {
    if (!output_id || !n) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    auto it = outputs_.find(output_id);
    if (it == outputs_.end()) { set_error("output not registered"); return SMR_ERR_OUTPUT_NOT_REGISTERED; }
    Output &o = it->second;
    *n = 0;
    if (!o.flat && o.node.root_is_input) { if (rw) *rw = 0; if (rh) *rh = 0; return SMR_OK; }
    OutputNode copy = o.node;  // do not advance Tiles::last_layout
    std::vector<Input *> child_in;
    std::vector<std::optional<Resolution>> child_res;
    const Resolution root = output_children(o, copy, pts, child_in, child_res);
    if (rw) *rw = (uint32_t)root.width;
    if (rh) *rh = (uint32_t)root.height;
    std::vector<RenderLayout> layouts = output_layouts(o, copy, pts, child_res, root);
    *n = (uint32_t)layouts.size();
    if (!out) return SMR_OK;
    if (cap < layouts.size()) return SMR_ERR_BUFFER_TOO_SMALL;
    for (size_t i = 0; i < layouts.size(); i++) {
        const RenderLayout &l = layouts[i];
        smr_render_layout &d = out[i];
        memset(&d, 0, sizeof(d));
        d.type = (int)l.kind;
        d.top = l.top; d.left = l.left; d.width = l.width; d.height = l.height;
        d.rotation_degrees = l.rotation_degrees;
        d.border_radius[0] = l.border_radius.top_left; d.border_radius[1] = l.border_radius.top_right;
        d.border_radius[2] = l.border_radius.bottom_right; d.border_radius[3] = l.border_radius.bottom_left;
        d.color = {l.color.r, l.color.g, l.color.b, l.color.a};
        d.border_color = {l.border_color.r, l.border_color.g, l.border_color.b, l.border_color.a};
        d.border_width = l.border_width; d.blur_radius = l.blur_radius;
        d.child_index = (int)l.index;
        d.crop_top = l.crop.top; d.crop_left = l.crop.left; d.crop_width = l.crop.width; d.crop_height = l.crop.height;
        d.masks_len = (int)std::min<size_t>(l.masks.size(), SMR_MAX_MASKS);
        for (int m = 0; m < d.masks_len; m++) {
            const Mask &mk = l.masks[m];
            d.masks[m].radius[0] = mk.radius.top_left; d.masks[m].radius[1] = mk.radius.top_right;
            d.masks[m].radius[2] = mk.radius.bottom_right; d.masks[m].radius[3] = mk.radius.bottom_left;
            d.masks[m].top = mk.top; d.masks[m].left = mk.left; d.masks[m].width = mk.width; d.masks[m].height = mk.height;
        }
    }
    return SMR_OK;
}

}  // namespace smr

// ------------------------------------------------------------------------------------------------
// extern "C"
// ------------------------------------------------------------------------------------------------
struct smr_renderer {
    smr::Renderer impl;
    explicit smr_renderer(const smr_options &o) : impl(o) {}
};

static thread_local std::string g_create_error;

extern "C" {

smr_status smr_create(const smr_options *opts, smr_renderer **out) {
    if (!opts || !out) return SMR_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    smr_renderer *r = nullptr;
    try { r = new smr_renderer(*opts); } catch (...) { return SMR_ERR_OUT_OF_MEMORY; }
    smr_status st;
    try { st = r->impl.init(); } catch (...) { st = SMR_ERR_OUT_OF_MEMORY; }
    if (st != SMR_OK) {
        g_create_error = r->impl.last_error();
        delete r;
        return st;
    }
    *out = r;
    return SMR_OK;
}

void smr_destroy(smr_renderer *r) { delete r; }

#define SMR_GUARD(call)                                                       \
    if (!r) return SMR_ERR_INVALID_ARGUMENT;                                  \
    try { return call; }                                                      \
    catch (const std::bad_alloc &) { return SMR_ERR_OUT_OF_MEMORY; }          \
    catch (...) { r->impl.set_error("internal error"); return SMR_ERR_INVALID_ARGUMENT; }

smr_status smr_register_input(smr_renderer *r, const char *id) { SMR_GUARD(r->impl.register_input(id)) }
smr_status smr_unregister_input(smr_renderer *r, const char *id) { SMR_GUARD(r->impl.unregister_input(id)) }
smr_status smr_update_scene(smr_renderer *r, const char *output_id, uint32_t w, uint32_t h, int32_t fmt,
                            const smr_component *root) { SMR_GUARD(r->impl.update_scene(output_id, w, h, fmt, root)) }
smr_status smr_unregister_output(smr_renderer *r, const char *id) { SMR_GUARD(r->impl.unregister_output(id)) }
smr_status smr_set_layouts(smr_renderer *r, const char *output_id, uint32_t w, uint32_t h, int32_t fmt, uint32_t root_w,
                           uint32_t root_h, const char *const *child_ids, uint32_t n_children, const smr_render_layout *layouts,
                           uint32_t n) { SMR_GUARD(r->impl.set_layouts(output_id, w, h, fmt, root_w, root_h, child_ids, n_children, layouts, n)) }
smr_status smr_render_begin(smr_renderer *r, uint64_t pts, const smr_input_frame *in, uint32_t n_in,
                            smr_output_frame *out, uint32_t n_out) { SMR_GUARD(r->impl.render_begin(pts, in, n_in, out, n_out)) }
smr_status smr_render_end(smr_renderer *r) { SMR_GUARD(r->impl.render_end()) }
smr_status smr_debug_partition(const int32_t *dst_w, const int32_t *dst_h, uint32_t n_jobs, uint32_t max_blocks,
                               int32_t *pieces, uint32_t pieces_cap, uint32_t *n_pieces, int32_t *begin, uint32_t begin_cap,
                               uint32_t *n_blocks) {
    if ((n_jobs && (!dst_w || !dst_h)) || !n_pieces || !n_blocks) return SMR_ERR_INVALID_ARGUMENT;
    std::vector<int> idx(n_jobs);
    for (uint32_t i = 0; i < n_jobs; i++) idx[i] = (int)i;
    std::vector<smr::dev::FusedPiece> pc;
    std::vector<int> bg;
    smr::partition_fused_rows(idx.data(), dst_w, dst_h, (int)n_jobs, (int)max_blocks, pc, bg);
    *n_pieces = (uint32_t)pc.size();
    *n_blocks = bg.empty() ? 0 : (uint32_t)bg.size() - 1;
    if (pc.size() > pieces_cap || bg.size() > begin_cap) return SMR_ERR_BUFFER_TOO_SMALL;
    for (size_t i = 0; i < pc.size(); i++) {
        pieces[4 * i] = pc[i].job; pieces[4 * i + 1] = pc[i].strip; pieces[4 * i + 2] = pc[i].oy_begin; pieces[4 * i + 3] = pc[i].oy_end;
    }
    for (size_t i = 0; i < bg.size(); i++) begin[i] = bg[i];
    return SMR_OK;
}
smr_status smr_debug_weights(float scale, float offset, uint32_t n_out, float *weights, size_t cap, uint32_t *taps, float *inv,
                             int32_t *first) {
    if (!weights || !taps || !inv || !first || n_out == 0 || n_out > 16384 || !(scale > 0.0f && scale <= 1024.0f))
        return SMR_ERR_INVALID_ARGUMENT;
    int n = 0;
    const int rc = smr::dev::debug_weights(scale, offset, (int)n_out, weights, cap, &n, inv, first);
    *taps = (uint32_t)n;
    return rc > 0 ? SMR_OK : rc == 0 ? SMR_ERR_BUFFER_TOO_SMALL : SMR_ERR_CUDA;
}
smr_status smr_debug_sincos(const float *x, uint32_t n, float *s, float *c) {
    if ((n && (!x || !s || !c)) || n > (1u << 28)) return SMR_ERR_INVALID_ARGUMENT;
    if (n == 0) return SMR_OK;
    return smr::dev::debug_sincos(x, (int)n, s, c) > 0 ? SMR_OK : SMR_ERR_CUDA;
}
smr_status smr_debug_resample_stages(smr_renderer *r, smr_resample_stage_info *out, uint32_t cap, uint32_t *n,
                                     int32_t *convert_kinds, uint32_t convert_cap, uint32_t *n_convert) {
    SMR_GUARD(r->impl.debug_resample_stages(out, cap, n, convert_kinds, convert_cap, n_convert))
}
smr_status smr_preprocess_frame(smr_renderer *r, const smr_input_frame *f, uint32_t ow, uint32_t oh, void *rgba, uint32_t pitch,
                                int32_t mem_kind) { SMR_GUARD(r->impl.preprocess_frame(f, ow, oh, rgba, pitch, mem_kind)) }
smr_status smr_premultiply_rgba8(smr_renderer *r, const smr_input_frame *f, void *rgba, uint32_t pitch, int32_t mem_kind) {
    SMR_GUARD(r->impl.preprocess_frame(f, 0, 0, rgba, pitch, mem_kind, true))
}
smr_status smr_render_text(smr_renderer *r, uint32_t w, uint32_t h, smr_rgba bg, const smr_glyph *glyphs, uint32_t n,
                           const smr_atlas *mask, const smr_atlas *color, int32_t color_mode, void *rgba, uint32_t pitch, int32_t mem_kind) {
    SMR_GUARD(r->impl.render_text(w, h, bg, glyphs, n, mask, color, color_mode, rgba, pitch, mem_kind))
}
smr_status smr_render(smr_renderer *r, uint64_t pts, const smr_input_frame *in, uint32_t n_in, smr_output_frame *out,
                      uint32_t n_out) {
    if (!r) return SMR_ERR_INVALID_ARGUMENT;
    smr_status st = smr_render_begin(r, pts, in, n_in, out, n_out);
    if (st != SMR_OK) return st;
    SMR_GUARD(r->impl.render_end_all())   // every tick in flight, the one just submitted included
}
smr_status smr_debug_layouts(smr_renderer *r, const char *output_id, uint64_t pts, smr_render_layout *out, uint32_t cap,
                             uint32_t *n, uint32_t *rw, uint32_t *rh) { SMR_GUARD(r->impl.debug_layouts(output_id, pts, out, cap, n, rw, rh)) }
smr_status smr_debug_set_inputs(smr_renderer *r, uint64_t pts, const smr_input_frame *in, uint32_t n_in) { SMR_GUARD(r->impl.debug_set_inputs(pts, in, n_in)) }
smr_status smr_debug_fused_jobs(smr_renderer *r, smr_fused_job_info *out, uint32_t cap, uint32_t *n) { SMR_GUARD(r->impl.debug_fused_jobs(out, cap, n)) }
smr_status smr_debug_composite_layers(smr_renderer *r, smr_composite_layer_info *out, uint32_t cap, uint32_t *n) {
    SMR_GUARD(r->impl.debug_composite_layers(out, cap, n))
}
smr_status smr_debug_interior(const smr_render_layout *layout, uint32_t width, uint32_t height, int32_t box[12], uint8_t *shortcut) {
    if (!layout || !box || width == 0 || height == 0 || width > 16384 || height > 16384) return SMR_ERR_INVALID_ARGUMENT;
    if (layout->type < 0 || layout->type > 2 || layout->masks_len < 0 || layout->masks_len > SMR_MAX_MASKS) return SMR_ERR_INVALID_ARGUMENT;
    try {
        const smr::RenderLayout l = smr::layout_from_c(*layout);
        smr::dev::LayerDev d;
        const bool drawn = smr::layer_geometry(l, (int)width, (int)height, d);
        const int32_t b[12] = {d.px0, d.px1, d.py0, d.py1, d.ix0, d.ix1, d.iy0, d.iy1, d.jx0, d.jx1, d.jy0, d.jy1};
        for (int i = 0; i < 12; i++) box[i] = drawn ? b[i] : 0;
        if (shortcut) {
            memset(shortcut, 0, (size_t)width * height);
            std::vector<smr::dev::MaskDev> masks;
            d.mask_count = smr::layer_masks(l, masks);
            for (int y = drawn ? d.py0 : 0; y < (drawn ? d.py1 : 0); y++)
                for (int x = d.px0; x < d.px1; x++)   // an axis-aligned layer covers its whole box
                    shortcut[(size_t)y * width + x] = smr::dev::interior_shortcut(d, masks.data(), x, y) ? 1 : 0;
        }
        return SMR_OK;
    } catch (...) { return SMR_ERR_OUT_OF_MEMORY; }
}
smr_status smr_comm_get_unique_id(uint8_t id[128]) {
    if (!id) return SMR_ERR_INVALID_ARGUMENT;
    std::string err;
    if (!smr::nccl_load(err)) { g_create_error = err; return SMR_ERR_UNSUPPORTED; }
    smr::NcclId nid;
    if (smr::g_nccl.GetUniqueId(&nid) != 0) { g_create_error = "ncclGetUniqueId failed"; return SMR_ERR_CUDA; }
    memcpy(id, nid.b, 128);
    return SMR_OK;
}
smr_status smr_comm_init(smr_renderer *r, const uint8_t id[128], int32_t rank, int32_t nranks) { SMR_GUARD(r->impl.comm_init(id, rank, nranks)) }
smr_status smr_comm_broadcast_inputs(smr_renderer *r, const smr_input_frame *frames, uint32_t n, const int32_t *root_ranks) { SMR_GUARD(r->impl.comm_exchange(frames, n, root_ranks, nullptr, 0)) }
smr_status smr_comm_exchange_inputs(smr_renderer *r, const smr_input_frame *frames, uint32_t n, const int32_t *root_ranks,
                                    const uint64_t *consumer_masks, uint32_t flags) { SMR_GUARD(r->impl.comm_exchange(frames, n, root_ranks, consumer_masks, flags)) }
smr_status smr_comm_pull_inputs(smr_renderer *r, const smr_input_frame *frames, const smr_input_frame *peer_frames, uint32_t n,
                                const int32_t *root_ranks, const uint64_t *consumer_masks) { SMR_GUARD(r->impl.comm_pull(frames, peer_frames, n, root_ranks, consumer_masks)) }
smr_status smr_peer_pool_alloc(smr_renderer *r, size_t bytes, void **dev_ptr, uint8_t handle[64]) { SMR_GUARD(r->impl.peer_pool_alloc(bytes, dev_ptr, handle)) }
smr_status smr_peer_pool_open(smr_renderer *r, const uint8_t handle[64], void **dev_ptr) { SMR_GUARD(r->impl.peer_pool_open(handle, dev_ptr)) }
smr_status smr_peer_pool_close(smr_renderer *r, void *dev_ptr) { SMR_GUARD(r->impl.peer_pool_close(dev_ptr)) }
smr_status smr_peer_pool_free(smr_renderer *r, void *dev_ptr) { SMR_GUARD(r->impl.peer_pool_free(dev_ptr)) }
smr_status smr_comm_destroy(smr_renderer *r) { SMR_GUARD(r->impl.comm_destroy()) }
smr_status smr_set_profiling(smr_renderer *r, int32_t enabled) { SMR_GUARD(r->impl.set_profiling(enabled)) }
smr_status smr_get_kernel_times(smr_renderer *r, smr_kernel_times *out) {
    if (!r || !out) return SMR_ERR_INVALID_ARGUMENT;
    r->impl.kernel_times(out);
    return SMR_OK;
}
smr_status smr_get_stats(smr_renderer *r, smr_stats *out) {
    if (!r || !out) return SMR_ERR_INVALID_ARGUMENT;
    r->impl.stats(out);
    return SMR_OK;
}
void *smr_cuda_stream(smr_renderer *r) { return r ? r->impl.stream() : nullptr; }
// page-lock a caller-owned frame buffer once, so that every later upload / download of it is a direct DMA
smr_status smr_host_register(void *ptr, size_t bytes) {
    if (!ptr || !bytes) return SMR_ERR_INVALID_ARGUMENT;
    cudaError_t e = cudaHostRegister(ptr, bytes, cudaHostRegisterPortable);
    if (e == cudaErrorHostMemoryAlreadyRegistered) { cudaGetLastError(); return SMR_OK; }
    if (e != cudaSuccess) { cudaGetLastError(); return SMR_ERR_CUDA; }
    return SMR_OK;
}
smr_status smr_host_unregister(void *ptr) {
    if (!ptr) return SMR_ERR_INVALID_ARGUMENT;
    if (cudaHostUnregister(ptr) != cudaSuccess) { cudaGetLastError(); return SMR_ERR_CUDA; }
    return SMR_OK;
}
const char *smr_last_error(smr_renderer *r) { return r ? r->impl.last_error() : g_create_error.c_str(); }
const char *smr_version(void) { return "smelter_b200 0.1 (sm_90a)"; }

smr_status smr_debug_tile_plan(const int32_t *boxes, uint32_t n_layers, uint32_t width, uint32_t height, int32_t sorted,
                               int32_t *owner_layer, uint32_t owner_cap, uint32_t *tiles, uint32_t tiles_cap, uint32_t *n_tiles) {
    static_assert(sizeof(smr::TileLayerBox) == 14 * sizeof(int32_t), "14 ints per layer");
    if ((n_layers && !boxes) || !n_tiles || width == 0 || height == 0 || width > 16384 * 4 || height > 16384 * 4) return SMR_ERR_INVALID_ARGUMENT;
    try {
        std::vector<int> owner;
        std::vector<uint32_t> list;
        smr::plan_tiles_core(reinterpret_cast<const smr::TileLayerBox *>(boxes), (int)n_layers, (int)width, (int)height, sorted != 0, owner, list);
        *n_tiles = (uint32_t)list.size();
        if (owner_layer) {
            if (owner_cap < owner.size()) return SMR_ERR_BUFFER_TOO_SMALL;
            for (size_t i = 0; i < owner.size(); i++) owner_layer[i] = owner[i];
        }
        if (tiles) {
            if (tiles_cap < list.size()) return SMR_ERR_BUFFER_TOO_SMALL;
            memcpy(tiles, list.data(), sizeof(uint32_t) * list.size());
        }
        return SMR_OK;
    } catch (...) { return SMR_ERR_OUT_OF_MEMORY; }
}
smr_status smr_output_plane_sizes(uint32_t w, uint32_t h, int32_t fmt, size_t sizes[3]) {
    if (!sizes) return SMR_ERR_INVALID_ARGUMENT;
    if (fmt < SMR_OUT_PLANAR_YUV420 || fmt > SMR_OUT_NV12) return SMR_ERR_UNSUPPORTED;
    size_t rb[3], rows[3];
    smr::out_plane_layout(fmt, w, h, rb, rows);
    for (int i = 0; i < 3; i++) sizes[i] = rb[i] * rows[i];
    return SMR_OK;
}

void smr_component_default(int32_t type, smr_component *c) {  // components.rs:289-347
    if (!c) return;
    memset(c, 0, sizeof(*c));
    c->type = type;
    c->direction = SMR_DIRECTION_ROW;
    c->overflow = SMR_OVERFLOW_HIDDEN;
    c->rescale_mode = SMR_RESCALE_FIT;
    c->horizontal_align = SMR_HALIGN_CENTER;
    c->vertical_align = SMR_VALIGN_CENTER;
    c->tile_aspect_ratio_w = 16;
    c->tile_aspect_ratio_h = 9;
}

}  // extern "C"
