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
#include "wgsl.h"

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

// An owning CUDA handle, move-only: the resource is released when the handle is reset or destroyed, and a null handle
// releases nothing.  It converts to the raw handle, so calls that take one are written as with a raw member.
template <class H, auto Release> class Owned {
    H h_ = nullptr;
  public:
    Owned() = default;
    explicit Owned(H h) : h_(h) {}
    Owned(Owned &&o) noexcept : h_(o.release()) {}
    Owned &operator=(Owned &&o) noexcept { reset(o.release()); return *this; }
    ~Owned() { reset(); }
    operator H() const { return h_; }
    H release() { H h = h_; h_ = nullptr; return h; }
    void reset(H h = nullptr) { if (h_) Release(h_); h_ = h; }
};
using Stream = Owned<cudaStream_t, cudaStreamDestroy>;
using Event = Owned<cudaEvent_t, cudaEventDestroy>;
using MemPool = Owned<cudaMemPool_t, cudaMemPoolDestroy>;
using Library = Owned<cudaLibrary_t, cudaLibraryUnload>;
template <class T> using DevMem = Owned<T *, cudaFree>;
using IpcMapping = Owned<void *, cudaIpcCloseMemHandle>;

// `create`(&handle, args...) into `out`, with the status it returns
template <class H, auto R, class Create, class... Args> static cudaError_t make(Owned<H, R> &out, Create create, Args... args) {
    H h = nullptr;
    cudaError_t e = create(&h, args...);
    out.reset(e == cudaSuccess ? h : nullptr);
    return e;
}

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
static int nccl_comm_destroy(void *comm) { return g_nccl.CommDestroy(comm); }

// NVRTC (shader registration), also dlopen'ed on first use: the library does not link against it
static struct {
    void *lib = nullptr;
    int (*CreateProgram)(void **, const char *, const char *, int, const char *const *, const char *const *) = nullptr;
    int (*CompileProgram)(void *, int, const char *const *) = nullptr;
    int (*GetProgramLogSize)(void *, size_t *) = nullptr;
    int (*GetProgramLog)(void *, char *) = nullptr;
    int (*GetCUBINSize)(void *, size_t *) = nullptr;
    int (*GetCUBIN)(void *, char *) = nullptr;
    int (*AddNameExpression)(void *, const char *) = nullptr;
    int (*GetLoweredName)(void *, const char *, const char **) = nullptr;
    int (*DestroyProgram)(void **) = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
} g_nvrtc;

static bool nvrtc_load(std::string &err) {
    if (g_nvrtc.lib) return true;
    void *h = dlopen("libnvrtc.so.12", RTLD_NOW | RTLD_NOLOAD);   // the one already in the process (e.g. torch's)
    if (!h) h = dlopen("libnvrtc.so.12", RTLD_NOW);
    if (!h) h = dlopen("libnvrtc.so", RTLD_NOW);
    if (!h) {
        const char *home = getenv("CUDA_HOME");
        h = dlopen((std::string(home ? home : "/usr/local/cuda") + "/lib64/libnvrtc.so.12").c_str(), RTLD_NOW);
    }
    if (!h) { err = std::string("cannot load NVRTC (libnvrtc.so.12), which compiles shaders: ") + dlerror(); return false; }
    g_nvrtc.CreateProgram = (decltype(g_nvrtc.CreateProgram))dlsym(h, "nvrtcCreateProgram");
    g_nvrtc.CompileProgram = (decltype(g_nvrtc.CompileProgram))dlsym(h, "nvrtcCompileProgram");
    g_nvrtc.GetProgramLogSize = (decltype(g_nvrtc.GetProgramLogSize))dlsym(h, "nvrtcGetProgramLogSize");
    g_nvrtc.GetProgramLog = (decltype(g_nvrtc.GetProgramLog))dlsym(h, "nvrtcGetProgramLog");
    g_nvrtc.GetCUBINSize = (decltype(g_nvrtc.GetCUBINSize))dlsym(h, "nvrtcGetCUBINSize");
    g_nvrtc.GetCUBIN = (decltype(g_nvrtc.GetCUBIN))dlsym(h, "nvrtcGetCUBIN");
    g_nvrtc.AddNameExpression = (decltype(g_nvrtc.AddNameExpression))dlsym(h, "nvrtcAddNameExpression");
    g_nvrtc.GetLoweredName = (decltype(g_nvrtc.GetLoweredName))dlsym(h, "nvrtcGetLoweredName");
    g_nvrtc.DestroyProgram = (decltype(g_nvrtc.DestroyProgram))dlsym(h, "nvrtcDestroyProgram");
    g_nvrtc.GetErrorString = (decltype(g_nvrtc.GetErrorString))dlsym(h, "nvrtcGetErrorString");
    if (!g_nvrtc.CreateProgram || !g_nvrtc.CompileProgram || !g_nvrtc.GetProgramLogSize || !g_nvrtc.GetProgramLog ||
        !g_nvrtc.GetCUBINSize || !g_nvrtc.GetCUBIN || !g_nvrtc.AddNameExpression || !g_nvrtc.GetLoweredName ||
        !g_nvrtc.DestroyProgram || !g_nvrtc.GetErrorString) { err = "libnvrtc lacks required symbols"; return false; }
    g_nvrtc.lib = h;
    return true;
}

// the sources a shader module is compiled against (generated from kernels.h, node_sample.cuh, shader_rt.cuh by build.py)
#include "shader_sources.inc"
// the node_sample.cuh tables of a shader module, in table_symbols' order
static const char *const kShaderTables[5] = {"&smr::dev::c_u8n", "&smr::dev::c_dec", "&smr::dev::c_thr", "&smr::dev::c_yl",
                                             "&smr::dev::c_enc1"};

// CreateShaderError analogue: false with NVRTC's log in `err`; `names` receives the lowered names of kShaderTables
static bool compile_shader(const std::string &source, std::vector<char> &cubin, std::vector<std::string> &names, std::string &err) {
    static const char kCstddef[] = "typedef decltype(sizeof(0)) size_t;\nnamespace std { using ::size_t; }\n";
    static const char kCstdint[] =
        "typedef signed char int8_t; typedef short int16_t; typedef int int32_t; typedef long int64_t;\n"
        "typedef unsigned char uint8_t; typedef unsigned short uint16_t; typedef unsigned int uint32_t;\n"
        "typedef unsigned long uint64_t; typedef unsigned long uintptr_t;\n"
        "namespace std { using ::int8_t; using ::int16_t; using ::int32_t; using ::int64_t; using ::uint8_t; using ::uint16_t;\n"
        "using ::uint32_t; using ::uint64_t; using ::uintptr_t; }\n";
    const char *hdr[3] = {kSrc_kernels, kCstddef, kCstdint}, *hdr_names[3] = {"kernels.h", "cstddef", "cstdint"};
    const std::string src = std::string("#include \"kernels.h\"\nnamespace smr {\nnamespace dev {\n") + kSrc_node_sample +
                            "}  // namespace dev\n}  // namespace smr\n#define SMR_SHADER_API\n" + kSrc_shader_rt +
                            "#undef SMR_SHADER_API\n#line 1 \"shader\"\n" + source + "\n#define SMR_SHADER_MAIN\n" + kSrc_shader_rt;
    void *prog = nullptr;
    int rc = g_nvrtc.CreateProgram(&prog, src.c_str(), "shader.cu", 3, hdr, hdr_names);
    if (rc != 0) { err = std::string("nvrtcCreateProgram: ") + g_nvrtc.GetErrorString(rc); return false; }
    for (const char *t : kShaderTables) g_nvrtc.AddNameExpression(prog, t);
    // the numeric contract of kernels.cu: only explicit fmaf() is fused, IEEE division and square root, no flush to zero.
    // -default-device: kernels.h's host declarations, and unannotated helpers of the shader, are device code here
    const char *opts[] = {"--gpu-architecture=sm_90a", "-std=c++17", "--fmad=false", "--prec-div=true", "--prec-sqrt=true",
                          "--ftz=false", "-default-device"};
    rc = g_nvrtc.CompileProgram(prog, 7, opts);
    if (rc != 0) {
        size_t n = 0;
        g_nvrtc.GetProgramLogSize(prog, &n);
        std::string log(n, '\0');
        if (n) g_nvrtc.GetProgramLog(prog, &log[0]);
        err = std::string("shader does not compile (") + g_nvrtc.GetErrorString(rc) + "):\n" + log.c_str();
        g_nvrtc.DestroyProgram(&prog);
        return false;
    }
    size_t n = 0;
    g_nvrtc.GetCUBINSize(prog, &n);
    cubin.resize(n);
    if (n) g_nvrtc.GetCUBIN(prog, cubin.data());
    names.clear();
    for (const char *t : kShaderTables) {
        const char *lowered = nullptr;
        g_nvrtc.GetLoweredName(prog, t, &lowered);
        names.push_back(lowered ? lowered : "");
    }
    g_nvrtc.DestroyProgram(&prog);
    return true;
}

// smr_shader_param_type -> ShaderParamType; false with the reason on a malformed type
static bool param_type_from_c(const smr_shader_param_type *t, ShaderParamType &out, std::string &err, int depth) {
    if (depth > 64) { err = "shader parameter type too deep"; return false; }
    out.kind = t->kind;
    if (t->name) out.name = t->name;
    if (t->kind >= SMR_SHADER_PARAM_F32 && t->kind <= SMR_SHADER_PARAM_I32) return true;
    if (t->kind != SMR_SHADER_PARAM_LIST && t->kind != SMR_SHADER_PARAM_STRUCT) { err = "unknown shader parameter kind"; return false; }
    if (!t->items || t->items_len == 0) { err = "a list or struct parameter type needs items"; return false; }
    if (t->kind == SMR_SHADER_PARAM_LIST && (t->items_len != 1 || t->length == 0)) {
        err = "a list parameter type has one item type and a length of at least 1";
        return false;
    }
    out.length = t->length;
    out.items.resize(t->items_len);
    for (uint32_t i = 0; i < t->items_len; i++) {
        if (t->kind == SMR_SHADER_PARAM_STRUCT && !t->items[i].name) { err = "a struct parameter type's field has no name"; return false; }
        if (!param_type_from_c(&t->items[i], out.items[i], err, depth + 1)) return false;
    }
    return true;
}

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
// row bytes and rows of plane `plane` of a width x height frame of format `fmt`; false: the format has no such plane
static bool plane_layout(int fmt, uint32_t w, uint32_t h, int plane, size_t &row_bytes, size_t &rows);

// ------------------------------------------------------------------------------------------------
class Renderer {
  public:
    explicit Renderer(const smr_options &o) : opts_(o) {}
    ~Renderer();
    smr_status init();

    smr_status register_input(const char *id);
    smr_status unregister_input(const char *id);
    smr_status set_input_deinterlace(const char *id, const smr_deinterlace *cfg);
    smr_status set_input_color(const char *id, const smr_input_color *c);
    smr_status debug_input_planes(const char *id, void *const planes[3], const uint32_t pitch[3], int32_t mem_kind);
    smr_status register_image(const char *id, const smr_image_spec *spec);
    smr_status register_svg_image(const char *id, const smr_svg_spec *spec);
    smr_status unregister_image(const char *id);
    smr_status register_web_renderer(const char *id, const smr_web_renderer_spec *spec);
    smr_status unregister_web_renderer(const char *id);
    smr_status web_set_frame(const char *id, const smr_web_frame *f);
    smr_status web_set_child_rects(const char *id, const smr_web_rect *rects, uint32_t n);
    smr_status register_shader(const char *id, const smr_shader_spec *spec);
    smr_status register_wgsl_shader(const char *id, const char *source);
    smr_status add_shader(const char *id, std::unique_ptr<ShaderProgram> program, const std::string &source);
    smr_status unregister_shader(const char *id);
    smr_status update_scene(const char *output_id, uint32_t w, uint32_t h, int32_t fmt, const smr_component *root);
    smr_status unregister_output(const char *id);
    smr_status set_layouts(const char *output_id, uint32_t w, uint32_t h, int32_t fmt, uint32_t root_w, uint32_t root_h,
                           const char *const *child_ids, uint32_t n_children, const smr_render_layout *layouts, uint32_t n);
    smr_status render_begin(uint64_t pts, const smr_input_frame *in, uint32_t n_in, smr_output_frame *out, uint32_t n_out);
    smr_status render_end();
    smr_status render_end_all();
    smr_status preprocess_frame(const smr_input_frame *f, uint32_t ow, uint32_t oh, void *rgba, uint32_t pitch, int32_t mem_kind,
                                bool premultiply = false);
    smr_status transcode_resize(const smr_input_frame *src, const smr_rendition *out, uint32_t n);
    smr_status video_nv12_to_rgba(const smr_video_color &converter, const smr_input_frame *src, const smr_video_color &frame,
                                  uint32_t ow, uint32_t oh, void *rgba, uint32_t pitch, int32_t mem_kind);
    smr_status video_rgba_to_nv12(const smr_video_color &converter, const smr_input_frame *src, uint32_t ow, uint32_t oh,
                                  void *const planes[2], const uint32_t pitch[2], int32_t mem_kind);
    smr_status render_text(uint32_t w, uint32_t h, smr_rgba bg, const smr_glyph *glyphs, uint32_t n, const smr_atlas *mask,
                           const smr_atlas *color, int32_t color_mode, void *rgba, uint32_t pitch, int32_t mem_kind);
    smr_status debug_set_inputs(uint64_t pts, const smr_input_frame *in, uint32_t n_in);
    smr_status debug_node_layouts(const char *output_id, std::optional<uint32_t> node, uint64_t pts, smr_render_layout *out,
                                  uint32_t cap, uint32_t *n, uint32_t *rw, uint32_t *rh);
    smr_status layouts_to_c(const std::vector<RenderLayout> &layouts, smr_render_layout *out, uint32_t cap, uint32_t *n);
    smr_status debug_image_nodes(const char *output_id, uint64_t pts, smr_image_node_info *out, uint32_t cap, uint32_t *n);
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
    // MOTION_ADAPTIVE's history: library copies of the input's last two frames of distinct pts, in hist[last] (the last
    // frame) and hist[last ^ 1] (the one before it)
    struct DeinterlaceHistory {
        int frames = 0;         // distinct frames held: 0, 1 or 2
        int last = 0;
        uint64_t pts = 0;       // the last frame's pts, format and size
        int32_t format = 0;
        uint32_t width = 0, height = 0;
    };
    struct Input {
        bool has_frame = false;
        dev::Tex tex;           // planes as they sit in HBM
        DevBuf planes[kTicksInFlight][3];    // owned copies of host frames, one set per tick in flight
        Resolution res;
        int node_tex = -1;      // index in the tick's texture table of the materialised RGBA8 node texture
        int raw_tex = -1;       // index of the virtual (fused K1/K2) texture
        int32_t format = -1;    // smr_frame_format of the last live frame (-1: none since registration)
        smr_deinterlace deint = {SMR_DEINTERLACE_OFF, SMR_FIELD_TOP_FIRST, 10};
        smr_input_color color = {SMR_MATRIX_DEFAULT, SMR_RANGE_DEFAULT};
        DeinterlaceHistory hist;
        DevBuf deint_out[kTicksInFlight][3];   // the deinterlaced planes `tex` points at, one set per tick in flight
        DevBuf hist_planes[2][3];
    };
    // A component node of an output's scene: its node texture as a layout child (premultiplied TEX_RGBA8, always live) and
    // the device memory behind it, allocated and freed in the order of stream_, so the ticks submitted before a scene update
    // finish reading it before it is released
    struct NodeTexture {
        Input in;
        std::shared_ptr<void> mem;
        size_t job_off = 0;     // its job in the parameter arena, when a tick draws it
    };
    // A Text component (TextRendererNode, transformations/text_renderer.rs): width x height (1 x 1 for 0 x 0), its glyphs
    // after the texture in `mem`
    struct TextNode : NodeTexture {
        dev::TextJob job = {};  // draws `in.tex`
        std::shared_ptr<void> atlas[2];   // the mask and colour atlases (shared within the scene)
        bool rendered = false;  // drawn since the last smr_update_scene of the output (`was_rendered`)
    };
    // An Image component (ImageNode, transformations/image.rs:137-187).  The node texture persists across ticks and is
    // rewritten, in the order of stream_, by the ticks whose frame differs from the one it holds.
    struct ImageNode : NodeTexture {
        ImageParams params;
        dev::ImageJob job = {}; // draws `in.tex` from the frame job.src
        int held = -1;          // the frame `in.tex` holds (-1: not drawn since the last smr_update_scene of the output)
        int held_before = -1;   // `held` when the current tick planned its draw
    };
    // A WebView component (WebRendererNode, transformations/web_renderer/node.rs), of the instance's size.  The node
    // texture is cleared when the node is made and redrawn, in the order of stream_, by every tick while the instance has a
    // frame.
    struct Output;
    struct WebNode : NodeTexture {
        WebParams params;
        Output *owner = nullptr;      // the output whose nodes its children are (set when a tick plans it)
        dev::WebJob job = {};   // draws `in.tex`; its planes are this tick's, packed into the parameter arena
        std::vector<dev::WebPlane> planes;
        std::vector<int> plane_child; // per plane: the child it shows (its texture is read when the tick is packed), -1 the page
        size_t planes_off = 0;
    };
    // A Shader component (ShaderNode, transformations/shader/node.rs).  The node texture persists and is redrawn, in the
    // order of stream_, by every tick.
    struct ShaderNode : NodeTexture {
        ShaderParams params;
        Output *owner = nullptr;   // the output whose nodes its children are (set when a tick plans it)
        dev::ShaderJob job = {};   // draws `in.tex`; its textures and parameter bytes are this tick's, in the parameter arena
        size_t tex_off = 0, params_off = SIZE_MAX;
    };
    struct Output {
        OutputNode node;
        std::vector<std::unique_ptr<TextNode>> texts;   // node.texts, in the same order
        std::vector<std::unique_ptr<ImageNode>> images; // node.images, in the same order
        std::vector<std::unique_ptr<WebNode>> webs;     // node.webs, in the same order
        std::vector<std::unique_ptr<ShaderNode>> shaders;   // node.shaders, in the same order
        // node.nested: each layout node's texture of the current tick, RGBA8 in the frame arena (has_frame false: it has no
        // pixels this tick, readers see the empty view)
        std::deque<Input> nested;
        uint64_t nodes_planned = 0;             // the tick whose texture table holds this output's node textures
        int32_t format = 0;
        Resolution res;
        DevBuf planes[kTicksInFlight][3];       // device staging for host outputs, one set per tick in flight: the read-back of
                                                // tick k runs on its own stream while tick k + 1 composes into the next set
        // tile plan of the composite (direct-tile owners + cost-sorted list of the tiles that are left), kept while the
        // flattened layers and the resamples feeding them stay the same (a static scene plans once)
        uint64_t tile_key = 0;
        bool tile_key_valid = false;
        std::vector<int> tile_owner_layer;       // per tile: index of the layer whose child is shown there 1:1 and alone, or -1
        std::vector<uint32_t> tile_list;         // tiles that are left for the composite, most expensive first
    };
    struct WeightKey {
        uint32_t scale_bits, offset_bits;
        int32_t n_out;
        bool operator<(const WeightKey &o) const {
            return std::tie(scale_bits, offset_bits, n_out) < std::tie(o.scale_bits, o.offset_bits, o.n_out);
        }
    };
    struct WeightEntry {         // one allocation: weights, inv and first, each from a 256-byte boundary
        DevMem<uint8_t> mem;
        float *weights = nullptr, *inv = nullptr;
        int32_t *first = nullptr;
        int taps = 0;
        uint64_t last_used = 0;
    };
    struct LaneTable { DevMem<uint8_t> perm; uint64_t last_used = 0; };

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
    // One launch of `kernel` after phase `phase` (-1: before the conversions) that draws the nodes of `nodes` that `in`
    // selects, in their order: their jobs and the prefix table of their 32 x 8 tile counts go to the parameter arena
    template <class Node, class Job, class In>
    void add_node_launch(const void *kernel, const char *name, int prof_class, int phase, const std::vector<Node *> &nodes,
                         Job Node::*job, In in) {
        NodeLaunch l{kernel, name, prof_class, phase, (int)std::count_if(nodes.begin(), nodes.end(), in)};
        if (l.n_jobs == 0) return;
        l.jobs_off = param_alloc(sizeof(Job) * l.n_jobs);
        l.begin_off = param_alloc(sizeof(int32_t) * (l.n_jobs + 1));
        int32_t *begin = reinterpret_cast<int32_t *>(param_host_.data() + l.begin_off);
        int k = 0;
        for (Node *n : nodes) {
            if (!in(n)) continue;
            const Job &j = n->*job;
            n->job_off = l.jobs_off + sizeof(Job) * k;
            memcpy(param_host_.data() + n->job_off, &j, sizeof(Job));
            begin[k++] = l.n_tiles;
            l.n_tiles += dev::node_tiles(j.dst.width, j.dst.height);
        }
        begin[k] = l.n_tiles;
        plan_.node_launches.push_back(l);
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
    smr_status plan_deinterlace(Input &I, const smr_input_frame &f, FrameView &v);
    struct LayoutEval {
        std::vector<Input *> child_in;                      // the Input behind each child; nullptr: the empty view
        std::vector<std::optional<Resolution>> child_res;
        Resolution res;                                     // the node's
        std::vector<RenderLayout> layouts;                  // flattened, untruncated
    };
    LayoutEval eval_layout(Output &o, LayoutParams &lp, uint64_t pts);
    smr_status plan_output(Output &o, smr_output_frame &of, uint64_t pts);
    Input *node_input(Output &o, const NodeRef &r);
    dev::Tex packed_node_tex(Output &o, const NodeRef &r);
    smr_status plan_layers(std::vector<RenderLayout> &layouts, const std::vector<Input *> &child_in, int W, int H,
                           std::vector<dev::LayerDev> &layers, std::vector<dev::MaskDev> &masks);
    smr_status plan_layout_node(Output &o, size_t k, uint64_t pts);
    smr_status child_texture(Input &in, RenderLayout &l, int &tex_index, int &tex_w, int &tex_h);
    smr_status get_weights(const KernelPass &p, const WeightEntry *&out);
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
    // Members are destroyed in reverse order, so these come first: each stream outlives the work and the stream-ordered
    // releases enqueued on it, web_pool_ outlives the web frames allocated from it, and retired_shaders_ outlives the
    // shader programs that retire their modules into it.
    Stream stream_;
    Stream copy_stream_, copy_stream2_;   // uploads alternate between two streams (two DMA engines)
    Stream d2h_stream_;                   // read-back of host outputs: overlaps the next tick's kernels
    // the tick's exchange step overlaps the previous tick's kernels: NCCL runs on its own stream, ordered after
    // everything submitted BEFORE the most recent tick and before the next one
    Stream comm_stream_;
    // Web frames: allocated on copy_stream_, released on stream_.  The pool never makes an allocation wait for a release
    // that is still pending on stream_ (no internal dependencies), so a copy does not wait for the ticks in flight.
    MemPool web_pool_;
    // Shader modules whose last user is gone: each is unloaded once the event recorded on stream_ at that time completes
    std::vector<std::pair<Library, Event>> retired_shaders_;
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
        dev::FusedVariant key;  // its kernel instantiation: the key of its launch
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
    struct FusedLaunch { dev::FusedVariant key; size_t pieces_off, begin_off; int nblocks; };
    // One launch of a node-texture kernel (launch_tile_jobs): launch_tick enqueues it after phase `phase`'s composite (-1:
    // before the conversions)
    struct NodeLaunch {
        const void *kernel;
        const char *name;                 // in a launch error
        int prof_class, phase;
        int n_jobs;                       // the nodes it draws, one job each
        size_t jobs_off, begin_off;       // in the parameter arena: their jobs, the prefix table of their tiles
        int n_tiles;
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
        std::vector<TextNode *> texts;        // text nodes drawn by this tick (one launch, before everything that reads them)
        std::vector<ImageNode *> images;      // image nodes drawn by this tick (likewise)
        std::vector<WebNode *> webs;          // web nodes drawn by this tick (after every node they may read, by depth)
        std::vector<ShaderNode *> shaders;    // shader nodes drawn by this tick (likewise)
        // the tick's phases: one per depth of its layout, shader and web nodes below the roots, then the roots'.  Phase p's
        // generic resample passes and composite jobs are those from phases[p] up to phases[p + 1] (the last entry: the end)
        struct Phase { size_t stages[3], composites; };
        std::vector<Phase> phases;
        std::map<std::tuple<int, uint32_t, uint32_t, uint32_t, uint32_t, int, int>, int> resample_cache;
        std::vector<FusedLaunch> fused_launches;
        std::vector<NodeLaunch> node_launches;   // the text, image, web and shader launches (pack_params)
        // k_deinterlace: one job per plane of the deinterlaced inputs, and each input's history before the tick planned it
        // (restored when the tick fails before its launches)
        std::vector<dev::DeinterlaceJob> deint;
        std::vector<std::pair<Input *, DeinterlaceHistory>> deint_history;
        size_t deint_off, deint_begin_off;
        int deint_tiles;
        size_t stage_off[3], weights_off, fused_off, composites_off;   // the packed job arrays in the parameter arena
        uint64_t launches, direct_tiles;
        bool nodes_enqueued;                  // the node launches before the conversions
        void clear() {   // keeps the vectors' capacity
            tex.clear();
            for (auto &s : stages) s.clear();
            fused.clear(); tmaps.clear(); weight_jobs.clear(); convert_jobs.clear();
            composites.clear(); outputs.clear(); fills.clear(); d2h.clear(); texts.clear(); images.clear(); webs.clear(); shaders.clear(); phases.clear();
            resample_cache.clear();
            fused_launches.clear(); node_launches.clear();
            deint.clear(); deint_history.clear();
            deint_tiles = 0;
            launches = direct_tiles = 0;
            nodes_enqueued = false;
        }
    } plan_;
    smr_status make_node_texture(int w, int h, bool clear, size_t extra_bytes, NodeTexture &n, dev::NodeTarget &t);
    using AtlasUploads = std::map<const TextAtlas *, std::shared_ptr<void>>;
    smr_status make_text_node(const std::shared_ptr<const TextPayload> &p, AtlasUploads &atlases, std::unique_ptr<TextNode> &out);
    smr_status make_image_node(const ImageParams &p, std::unique_ptr<ImageNode> &out);
    smr_status make_web_node(const WebParams &p, std::unique_ptr<WebNode> &out);
    void plan_web_node(Output &o, WebNode &n);
    smr_status make_shader_node(const ShaderParams &p, std::unique_ptr<ShaderNode> &out);
    void plan_shader_node(Output &o, ShaderNode &n, uint64_t pts);
    void reap_shaders(bool all);
    Event web_ev_;                             // the end of a web frame's copy: later launches on stream_ wait for it
    smr_status alloc_on_stream(size_t bytes, std::shared_ptr<void> &buf);
    Output &install_output(const char *output_id, OutputNode &&node, int32_t fmt, uint32_t w, uint32_t h);
    void plan_node_textures(Output &o, uint64_t pts);
    CompositeRec composite_rec(int W, int H, const std::vector<dev::LayerDev> &layers, const std::vector<dev::MaskDev> &masks);
    int composite_texture(CompositeRec pc);
    void plan_tiles(Output &o, CompositeRec &pc, const std::vector<dev::LayerDev> &layers, int W, int H);
    // the steps of render_begin, in order
    smr_status begin_tick();
    smr_status plan_tick(uint64_t pts, const smr_input_frame *in, uint32_t n_in, smr_output_frame *out, uint32_t n_out);
    smr_status resolve_frame_arena();
    void plan_fused_launches();
    smr_status pack_params();
    smr_status launch_tick();
    smr_status enqueue_readback(uint32_t n_out);
    std::vector<WeightKey> new_weight_keys_;   // cache entries whose k_weights launch is not enqueued yet
    void rollback_weights();                   // a tick that fails before that launch must not leave them behind
    // TMA kernels of the fused resample: descriptors of the source planes, cached per (pointer, pitch, size, kind)
    struct TmapKey {
        uintptr_t p; int pitch, w, h, kind;
        bool operator<(const TmapKey &o) const { return std::tie(p, pitch, w, h, kind) < std::tie(o.p, o.pitch, o.w, o.h, o.kind); }
    };
    std::map<TmapKey, CUtensorMap> tmap_cache_;
    // any-ratio TMA kernel: per (horizontal mapping, strip width) the lane <-> column-pair deal of every strip
    std::map<std::tuple<uint32_t, uint32_t, int32_t, int32_t>, LaneTable> lane_perms_;
    template <class Cache> void bound_cache(Cache &c);
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
    Event kernels_done_[kTicksInFlight];
    Event h2d_done2_[kTicksInFlight];
    int upload_rr_ = 0;
    Event h2d_done_[kTicksInFlight], tick_done_[kTicksInFlight];
    Event comm_done_, tick_start_;
    bool comm_pending_ = false, tick_started_ = false;
    std::deque<int> inflight_;
    int slot_ = 0;
    bool uploaded_ = false;
    int sm_count_ = 132;
    DevBuf text_job_;                  // smr_render_text: its one job and tile table
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
    // the steps of the blocking calls (smr_preprocess_frame, smr_premultiply_rgba8, smr_render_text, smr_transcode_resize,
    // the video converters)
    DevBuf pre_planes_[3], pre_out_;   // FramePreProcessor scratch (input_texture / rescale_texture / download_buffer)
    smr_status need_device();
    smr_status stage_in(DevBuf &scratch, const void *src, size_t src_pitch, size_t row_bytes, size_t rows);
    smr_status upload_pre_planes(const smr_input_frame &f, FrameView &v);
    struct TargetPlane {               // one plane a blocking call writes
        void *p; size_t pitch, row_bytes, rows; bool device;   // the caller's
        uint8_t *out; int out_pitch;                            // where its kernel writes it (place_targets)
    };
    smr_status place_targets(TargetPlane *t, size_t n);
    template <class Launch> smr_status launch_and_finish(const TargetPlane *t, size_t n, int kernel_class, Launch launch);
    Event call_ev_[2];                 // launch_and_finish's profiling events
    // smr_transcode_resize's per-axis tables, per (source length, output length); at most kTranscodeTapTables are kept, the
    // least recently used beyond that are released when a call needs room (no call uses more than 32)
    struct TapTable { DevBuf buf; uint64_t used = 0; };
    static constexpr size_t kTranscodeTapTables = 64;
    std::map<std::pair<uint32_t, uint32_t>, TapTable> transcode_taps_;
    uint64_t transcode_calls_ = 0;
    const dev::TranscodeTap *transcode_table(uint32_t in_len, uint32_t out_len);
    smr_status video_converter_ok(const smr_video_color &c);
    // optional per-kernel-class device timing (cudaEvents on the launching stream)
    void prof_mark(int kernel_class);
    bool profiling_ = false;
    std::vector<Event> prof_events_;
    size_t prof_next_event_ = 0;
    std::vector<std::pair<cudaEvent_t, int>> prof_marks_;
    smr_kernel_times prof_ = {};
    // NCCL communicator for shared-input replication (SURVEY 8e); libnccl is dlopen'ed on first use
    Owned<void *, nccl_comm_destroy> nccl_comm_;
    int comm_rank_ = 0, comm_size_ = 1;
    DevMem<int32_t> barrier_word_;               // 4 device bytes the per-tick all-reduce of the peer modes runs on
    // pools of smr_peer_pool_alloc / smr_peer_pool_open still alive
    std::vector<Owned<void *, cudaFree>> peer_own_;
    std::vector<IpcMapping> peer_opened_;
    template <class Pools> smr_status peer_pool_release(Pools &pools, void *dev_ptr);
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
    if (!stream_) return;   // host-only: nothing was made on a device
    cudaSetDevice(opts_.cuda_device);   // the members below are released on this device
    drain();   // no stream still runs work that reads what is released here
    // node textures, image assets and web frames free themselves on stream_ (web frames into web_pool_), and dropping a
    // shader program retires its module on stream_: all before the streams and the pool go
    outputs_.clear();
    scene_ = SceneState();
    cudaStreamSynchronize(stream_);   // those releases have run
    reap_shaders(true);   // every retired module's event has completed
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
    CUDA_OK(make(stream_, cudaStreamCreateWithFlags, cudaStreamNonBlocking));
    CUDA_OK(make(copy_stream_, cudaStreamCreateWithFlags, cudaStreamNonBlocking));
    CUDA_OK(make(copy_stream2_, cudaStreamCreateWithFlags, cudaStreamNonBlocking));
    CUDA_OK(make(d2h_stream_, cudaStreamCreateWithFlags, cudaStreamNonBlocking));
    for (int i = 0; i < kTicksInFlight; i++) CUDA_OK(make(kernels_done_[i], cudaEventCreateWithFlags, cudaEventDisableTiming));
    for (int i = 0; i < kTicksInFlight; i++) CUDA_OK(make(h2d_done2_[i], cudaEventCreateWithFlags, cudaEventDisableTiming));
    CUDA_OK(make(comm_stream_, cudaStreamCreateWithFlags, cudaStreamNonBlocking));
    CUDA_OK(make(comm_done_, cudaEventCreateWithFlags, cudaEventDisableTiming));
    CUDA_OK(make(tick_start_, cudaEventCreateWithFlags, cudaEventDisableTiming));
    CUDA_OK(make(web_ev_, cudaEventCreateWithFlags, cudaEventDisableTiming));
    {
        cudaMemPoolProps props = {};
        props.allocType = cudaMemAllocationTypePinned;
        props.location.type = cudaMemLocationTypeDevice;
        props.location.id = opts_.cuda_device;
        CUDA_OK(make(web_pool_, cudaMemPoolCreate, &props));
        int no = 0;
        CUDA_OK(cudaMemPoolSetAttribute(web_pool_, cudaMemPoolReuseAllowInternalDependencies, &no));
        uint64_t keep = UINT64_MAX;   // released frames stay in the pool for the next ones
        CUDA_OK(cudaMemPoolSetAttribute(web_pool_, cudaMemPoolAttrReleaseThreshold, &keep));
    }
    CUDA_OK(cudaDeviceGetAttribute(&sm_count_, cudaDevAttrMultiProcessorCount, opts_.cuda_device));
    for (int i = 0; i < kTicksInFlight; i++) {
        CUDA_OK(make(h2d_done_[i], cudaEventCreateWithFlags, cudaEventDisableTiming));
        CUDA_OK(make(tick_done_[i], cudaEventCreateWithFlags, cudaEventDisableTiming));
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

smr_status Renderer::set_input_deinterlace(const char *id, const smr_deinterlace *cfg) {
    if (!id || !cfg) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    auto it = inputs_.find(id);
    if (it == inputs_.end()) { set_error(std::string("input \"") + id + "\" is not registered"); return SMR_ERR_INVALID_ARGUMENT; }
    if (cfg->mode < SMR_DEINTERLACE_OFF || cfg->mode > SMR_DEINTERLACE_MOTION_ADAPTIVE) { set_error("unknown deinterlace mode"); return SMR_ERR_INVALID_ARGUMENT; }
    if (cfg->field_order != SMR_FIELD_TOP_FIRST && cfg->field_order != SMR_FIELD_BOTTOM_FIRST) { set_error("unknown field order"); return SMR_ERR_INVALID_ARGUMENT; }
    if (cfg->motion_threshold > 255) { set_error("motion threshold above 255"); return SMR_ERR_INVALID_ARGUMENT; }
    Input &I = it->second;
    if (cfg->mode != I.deint.mode || cfg->field_order != I.deint.field_order) I.hist = DeinterlaceHistory();
    I.deint = *cfg;
    return SMR_OK;
}

smr_status Renderer::set_input_color(const char *id, const smr_input_color *c) {
    if (!id || !c) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    auto it = inputs_.find(id);
    if (it == inputs_.end()) { set_error(std::string("input \"") + id + "\" is not registered"); return SMR_ERR_INVALID_ARGUMENT; }
    if (c->matrix < SMR_MATRIX_DEFAULT || c->matrix > SMR_MATRIX_BT601) { set_error("unknown colour matrix"); return SMR_ERR_INVALID_ARGUMENT; }
    if (c->range < SMR_RANGE_DEFAULT || c->range > SMR_RANGE_FULL) { set_error("unknown colour range"); return SMR_ERR_INVALID_ARGUMENT; }
    it->second.color = *c;
    return SMR_OK;
}

// inspection: the planes the last tick with a live frame of the input read for it, copied out on stream_ after that tick
smr_status Renderer::debug_input_planes(const char *id, void *const planes[3], const uint32_t pitch[3], int32_t mem_kind) {
    if (!id || !planes || !pitch || (mem_kind != SMR_MEM_HOST && mem_kind != SMR_MEM_DEVICE)) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    auto it = inputs_.find(id);
    if (it == inputs_.end() || it->second.format < 0) { set_error("no live frame of this input since it was registered"); return SMR_ERR_INVALID_ARGUMENT; }
    const Input &I = it->second;
    const uint8_t *src[3] = {I.tex.p0, I.tex.p1, I.tex.p2};
    const size_t spitch[3] = {(size_t)I.tex.pitch0, (size_t)I.tex.pitch1, (size_t)I.tex.pitch2};
    size_t row_bytes[3] = {}, rows[3] = {};
    for (int p = 0; p < 3; p++) {
        if (!plane_layout(I.format, (uint32_t)I.tex.width, (uint32_t)I.tex.height, p, row_bytes[p], rows[p])) continue;
        if (!planes[p] || (pitch[p] && pitch[p] < row_bytes[p])) { set_error("a target plane is null or its pitch is shorter than a row"); return SMR_ERR_INVALID_ARGUMENT; }
    }
    if (smr_status st = need_device(); st != SMR_OK) return st;
    for (int p = 0; p < 3; p++) {
        if (!rows[p]) continue;
        CUDA_OK(cudaMemcpy2DAsync(planes[p], pitch[p] ? pitch[p] : row_bytes[p], src[p], spitch[p], row_bytes[p], rows[p],
                                  cudaMemcpyDefault, stream_));
    }
    CUDA_OK(cudaStreamSynchronize(stream_));
    return SMR_OK;
}

// Memory allocated and released in the order of stream_: ticks submitted before the release finish reading it first
smr_status Renderer::alloc_on_stream(size_t bytes, std::shared_ptr<void> &buf) {
    cudaStream_t s = stream_;
    void *d = nullptr;
    CUDA_OK(cudaMallocAsync(&d, bytes, s));
    buf = std::shared_ptr<void>(d, [s](void *q) { cudaFreeAsync(q, s); });
    return SMR_OK;
}

smr_status Renderer::register_image(const char *id, const smr_image_spec *spec) {
    if (!id || !spec || !spec->frames) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    auto bad = [&](const char *why) { set_error(why); return SMR_ERR_INVALID_ARGUMENT; };
    if (spec->n_frames == 0) return bad("an image needs at least one frame");
    if (spec->n_frames > 1000) return bad("an animated image has at most 1000 frames");
    if (spec->width == 0 || spec->height == 0 || spec->width > 16384 || spec->height > 16384) return bad("image resolution out of range");
    const size_t row = (size_t)spec->width * 4, frame_bytes = row * spec->height;
    auto a = std::make_shared<ImageAsset>();
    a->width = spec->width; a->height = spec->height;
    uint64_t sum = 0;
    for (uint32_t i = 0; i < spec->n_frames; i++) {
        const smr_image_frame &f = spec->frames[i];
        if (!f.rgba) return bad("image frame pointer is null");
        if (f.pitch && f.pitch < row) return bad("image frame pitch smaller than a row");
        a->frame_pts.push_back(sum);
        if (spec->n_frames > 1 && __builtin_add_overflow(sum, f.delay_ns, &sum)) return bad("image frame delays overflow");
    }
    a->duration = sum ? sum : 1;
    if (!host_only_) {
        CUDA_OK(cudaSetDevice(opts_.cuda_device));
        std::shared_ptr<void> px;
        if (smr_status st = alloc_on_stream(frame_bytes * spec->n_frames, px); st != SMR_OK) return st;
        for (uint32_t i = 0; i < spec->n_frames; i++) {
            const smr_image_frame &f = spec->frames[i];
            CUDA_OK(cudaMemcpy2DAsync((uint8_t *)px.get() + frame_bytes * i, row, f.rgba, f.pitch ? f.pitch : row, row, spec->height,
                                      cudaMemcpyHostToDevice, stream_));
        }
        CUDA_OK(cudaStreamSynchronize(stream_));   // the caller's frames are free to change once this returns
        stats_.h2d_bytes += frame_bytes * spec->n_frames;
        a->pixels = std::move(px);
    }
    if (!scene_.register_image(id, std::move(a))) return bad("an image with this id is already registered");
    return SMR_OK;
}

// An SVG asset: its intrinsic size and the caller's rasteriser, in the registry bitmap assets use; nothing is drawn until
// a scene update resolves a node of it (make_image_node)
smr_status Renderer::register_svg_image(const char *id, const smr_svg_spec *spec) {
    if (!id || !spec || !spec->rasterize) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    if (spec->width == 0 || spec->height == 0 || spec->width > 16384 || spec->height > 16384) {
        set_error("SVG image resolution out of range");
        return SMR_ERR_INVALID_ARGUMENT;
    }
    auto a = std::make_shared<ImageAsset>();
    a->width = spec->width; a->height = spec->height;
    a->frame_pts.push_back(0);
    a->rasterize = spec->rasterize; a->user = spec->user;
    a->svg_id = id;
    if (!scene_.register_image(id, std::move(a))) { set_error("an image with this id is already registered"); return SMR_ERR_INVALID_ARGUMENT; }
    return SMR_OK;
}

smr_status Renderer::unregister_image(const char *id) {
    if (!id) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    if (!host_only_) CUDA_OK(cudaSetDevice(opts_.cuda_device));   // an asset no scene shows is released here, on stream_
    if (!scene_.unregister_image(id)) { set_error("image not registered"); return SMR_ERR_INVALID_ARGUMENT; }
    return SMR_OK;
}

smr_status Renderer::register_web_renderer(const char *id, const smr_web_renderer_spec *spec) {
    if (!id || !spec) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    auto bad = [&](const char *why) { set_error(why); return SMR_ERR_INVALID_ARGUMENT; };
    if (spec->width == 0 || spec->height == 0 || spec->width > 16384 || spec->height > 16384) return bad("web renderer resolution out of range");
    if (spec->embedding_method == SMR_WEB_CHROMIUM_EMBEDDING) {
        set_error("ChromiumEmbedding reads every child back to host memory each tick; only the native embedding methods are supported");
        return SMR_ERR_UNSUPPORTED;
    }
    if (spec->embedding_method != SMR_WEB_NATIVE_OVER_CONTENT && spec->embedding_method != SMR_WEB_NATIVE_UNDER_CONTENT)
        return bad("unknown web embedding method");
    auto w = std::make_shared<WebInstance>();
    w->width = spec->width; w->height = spec->height; w->embedding = spec->embedding_method;
    if (!scene_.register_web(id, std::move(w))) return bad("a web renderer with this id is already registered");
    return SMR_OK;
}

smr_status Renderer::unregister_web_renderer(const char *id) {
    if (!id) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    if (!host_only_) CUDA_OK(cudaSetDevice(opts_.cuda_device));   // a frame no scene shows is released here, on stream_
    if (!scene_.unregister_web(id)) { set_error("web renderer not registered"); return SMR_ERR_INVALID_ARGUMENT; }
    return SMR_OK;
}

// The page is copied once per call into a new buffer, on a copy stream: the call waits for that copy alone, not for the
// ticks in flight, and every launch enqueued on stream_ after it waits for the copy too.  The frame it replaces is released
// on stream_, so the ticks already submitted still read the frame they were planned with.
smr_status Renderer::web_set_frame(const char *id, const smr_web_frame *f) {
    if (!id || !f || !f->bgra) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    auto bad = [&](const char *why) { set_error(why); return SMR_ERR_INVALID_ARGUMENT; };
    WebInstance *w = scene_.web_instance(id);
    if (!w) return bad("web renderer not registered");
    if (f->width != w->width || f->height != w->height) return bad("web frame size differs from the web renderer's resolution");
    const size_t row = (size_t)w->width * 4, pitch = f->pitch ? f->pitch : row;
    if (pitch < row) return bad("web frame pitch smaller than a row");
    if (f->mem_kind != SMR_MEM_HOST && f->mem_kind != SMR_MEM_DEVICE) return bad("unknown mem_kind");
    if (host_only_) return SMR_OK;
    CUDA_OK(cudaSetDevice(opts_.cuda_device));
    void *d = nullptr;
    CUDA_OK(cudaMallocFromPoolAsync(&d, row * w->height, web_pool_, copy_stream_));
    cudaError_t e = cudaMemcpy2DAsync(d, row, f->bgra, pitch, row, w->height,
                                      f->mem_kind == SMR_MEM_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, copy_stream_);
    if (e == cudaSuccess) e = cudaEventRecord(web_ev_, copy_stream_);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(stream_, web_ev_, 0);
    if (e != cudaSuccess) {
        cudaFreeAsync(d, copy_stream_);
        set_error(std::string("web frame upload: ") + cudaGetErrorString(e));
        return SMR_ERR_CUDA;
    }
    cudaStream_t rs = stream_;
    // released on stream_, which has waited for the copy: every reader of the frame is a later launch on stream_
    std::shared_ptr<void> buf(d, [rs](void *q) { cudaFreeAsync(q, rs); });
    CUDA_OK(cudaEventSynchronize(web_ev_));   // the caller's plane is free to change once this returns
    if (f->mem_kind == SMR_MEM_HOST) stats_.h2d_bytes += row * w->height;
    w->frame = std::move(buf);
    return SMR_OK;
}

smr_status Renderer::web_set_child_rects(const char *id, const smr_web_rect *rects, uint32_t n) {
    if (!id || (n && !rects)) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    WebInstance *w = scene_.web_instance(id);
    if (!w) { set_error("web renderer not registered"); return SMR_ERR_INVALID_ARGUMENT; }
    if (n > 65536) { set_error("too many web child rects"); return SMR_ERR_INVALID_ARGUMENT; }
    std::vector<float> r(4 * (size_t)n);
    for (uint32_t i = 0; i < n; i++) {   // read_frame_position: `as f32`
        r[4 * i] = (float)rects[i].x; r[4 * i + 1] = (float)rects[i].y;
        r[4 * i + 2] = (float)rects[i].width; r[4 * i + 3] = (float)rects[i].height;
    }
    w->rects = std::move(r);
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

void Renderer::reap_shaders(bool all) {
    auto done = [all](const std::pair<Library, Event> &r) { return all || cudaEventQuery(r.second) == cudaSuccess; };
    retired_shaders_.erase(std::remove_if(retired_shaders_.begin(), retired_shaders_.end(), done), retired_shaders_.end());
}

smr_status Renderer::register_shader(const char *id, const smr_shader_spec *spec) {
    if (!id || !spec || !spec->source) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    if (scene_.has_shader(id)) { set_error("a shader with this id is already registered"); return SMR_ERR_INVALID_ARGUMENT; }
    std::string err;
    auto program = std::make_unique<ShaderProgram>();
    if (spec->param_type) {
        program->param_type.emplace();
        if (!param_type_from_c(spec->param_type, *program->param_type, err, 0)) { set_error(err); return SMR_ERR_INVALID_ARGUMENT; }
    }
    return add_shader(id, std::move(program), spec->source);
}

// WGSL: translated (wgsl.cpp), then compiled after wgsl_rt.cuh as a CUDA source is; the parameter type is the uniform's
smr_status Renderer::register_wgsl_shader(const char *id, const char *source) {
    if (!id || !source) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    if (scene_.has_shader(id)) { set_error("a shader with this id is already registered"); return SMR_ERR_INVALID_ARGUMENT; }
    wgsl::Translation t = wgsl::translate(source);
    if (t.status != SMR_OK) { set_error(t.error); return (smr_status)t.status; }
    auto program = std::make_unique<ShaderProgram>();
    program->param_type = std::move(t.param_type);
    program->wgsl = true;
    program->uniform_size = t.uniform_size;
    return add_shader(id, std::move(program), std::string(kSrc_wgsl_rt) + t.cuda);
}

// Compiles `source` into `program`, loads it on a device handle and registers it as `id` (the caller holds mu_)
smr_status Renderer::add_shader(const char *id, std::unique_ptr<ShaderProgram> program, const std::string &source) {
    std::string err;
    if (!nvrtc_load(err)) { set_error(err); return SMR_ERR_UNSUPPORTED; }
    std::vector<std::string> tables;
    if (!compile_shader(source, program->cubin, tables, err)) { set_error(err); return SMR_ERR_INVALID_ARGUMENT; }
    if (!host_only_) {
        CUDA_OK(cudaSetDevice(opts_.cuda_device));
        reap_shaders(false);
        cudaLibrary_t lib = nullptr;
        CUDA_OK(cudaLibraryLoadData(&lib, program->cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0));
        Library owned(lib);   // unloaded if what follows fails
        cudaKernel_t k = nullptr;
        const void *src[5];
        size_t bytes[5];
        cudaError_t e = cudaLibraryGetKernel(&k, lib, "smr_shader_main");
        if (e == cudaSuccess && !dev::table_symbols(src, bytes)) e = cudaErrorInvalidSymbol;
        for (int i = 0; i < 5 && e == cudaSuccess; i++) {   // the module's copies of the sampler and encode tables
            void *dst = nullptr;
            size_t n = 0;
            e = cudaLibraryGetGlobal(&dst, &n, lib, tables[i].c_str());
            if (e == cudaSuccess && n != bytes[i]) e = cudaErrorInvalidSymbol;
            if (e == cudaSuccess) e = cudaMemcpyAsync(dst, src[i], n, cudaMemcpyDeviceToDevice, stream_);
        }
        if (e == cudaSuccess) e = cudaStreamSynchronize(stream_);
        if (e != cudaSuccess) {
            set_error(std::string("loading the shader module: ") + cudaGetErrorString(e));
            return SMR_ERR_CUDA;
        }
        program->library = owned.release();
        program->kernel = (const void *)k;
    }
    // the module is unloaded after the ticks submitted before its last user let go of it
    std::shared_ptr<ShaderProgram> shared(program.release(), [this](ShaderProgram *p) {
        Library lib((cudaLibrary_t)p->library);
        delete p;
        if (!lib) return;
        cudaSetDevice(opts_.cuda_device);
        Event ev;
        if (make(ev, cudaEventCreateWithFlags, cudaEventDisableTiming) == cudaSuccess && cudaEventRecord(ev, stream_) == cudaSuccess)
            retired_shaders_.emplace_back(std::move(lib), std::move(ev));
        else   // no event: wait for the stream instead, then unload
            cudaStreamSynchronize(stream_);
    });
    if (!scene_.register_shader(id, std::move(shared))) { set_error("a shader with this id is already registered"); return SMR_ERR_INVALID_ARGUMENT; }
    return SMR_OK;
}

smr_status Renderer::unregister_shader(const char *id) {
    if (!id) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    if (!scene_.unregister_shader(id)) { set_error("shader not registered"); return SMR_ERR_INVALID_ARGUMENT; }
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
    // the text nodes are made (and uploaded) before the scene state changes, so that a failed upload leaves it as it was
    std::vector<std::shared_ptr<const TextPayload>> payloads;
    std::vector<const Component *> todo{&c};
    while (!todo.empty()) {
        const Component *k = todo.back();
        todo.pop_back();
        if (k->text) payloads.push_back(k->text);
        for (const Component &ch : k->children) todo.push_back(&ch);
    }
    std::map<const TextPayload *, std::unique_ptr<TextNode>> made;
    AtlasUploads atlases;
    if (!host_only_) CUDA_OK(cudaSetDevice(opts_.cuda_device));   // text memory is allocated and released on stream_
    for (const auto &p : payloads)
        if (smr_status st = make_text_node(p, atlases, made[p.get()]); st != SMR_OK) return st;
    OutputNode node;
    // image nodes have the resolution the scene state resolves; a node texture that cannot be allocated, or an SVG raster
    // the caller refuses, drops the update.  The image nodes come last, so that a rasteriser sees only scenes that passed
    // every other check.
    std::vector<std::unique_ptr<ImageNode>> images;
    std::vector<std::unique_ptr<WebNode>> webs;
    std::vector<std::unique_ptr<ShaderNode>> shaders;
    smr_status image_st = SMR_OK;
    auto make_all = [&](const auto &params, auto &nodes, auto make) {
        for (const auto &p : params) {
            nodes.emplace_back();
            if ((image_st = (this->*make)(p, nodes.back())) != SMR_OK) return false;
        }
        return true;
    };
    auto make_images = [&](OutputNode &n) {
        return make_all(n.webs, webs, &Renderer::make_web_node) && make_all(n.shaders, shaders, &Renderer::make_shader_node) &&
               make_all(n.images, images, &Renderer::make_image_node);
    };
    if (!scene_.update_scene(output_id, c, {w, h}, node, err, make_images)) {
        if (image_st != SMR_OK) return image_st;
        set_error(err);
        return SMR_ERR_SCENE;
    }
    Output &o = install_output(output_id, std::move(node), fmt, w, h);
    for (const auto &p : o.node.texts) o.texts.push_back(std::move(made[p.get()]));
    o.images = std::move(images);
    o.webs = std::move(webs);
    o.shaders = std::move(shaders);
    return SMR_OK;
}

// Output `output_id` (registered here if it is new) renders `node` from now on, in `fmt` at w x h, with no node textures
// until the caller moves in those it made for `node`.  The memory of the replaced ones is released on stream_, after the
// ticks that read it.
Renderer::Output &Renderer::install_output(const char *output_id, OutputNode &&node, int32_t fmt, uint32_t w, uint32_t h) {
    Output &o = outputs_[output_id];
    o.node = std::move(node);
    o.texts.clear(); o.images.clear(); o.webs.clear(); o.shaders.clear();
    o.nested.clear();
    o.nested.resize(o.node.nested.size());
    o.format = fmt;
    o.res = {w, h};
    return o;
}

// The bytes of a w x h node texture in its allocation, rounded up so that what follows it stays aligned
static size_t node_texture_bytes(int w, int h) { return ((size_t)w * h * 4 + 255) & ~(size_t)255; }

// A w x h node texture: `n.in` as a layout child and `t`, the target of the job that draws it.  On a device handle its
// memory, with `extra_bytes` more after the texture (at node_texture_bytes), is allocated on stream_, and with `clear` the
// texture is cleared to transparent there.
smr_status Renderer::make_node_texture(int w, int h, bool clear, size_t extra_bytes, NodeTexture &n, dev::NodeTarget &t) {
    Input &in = n.in;
    in.has_frame = true;
    in.res = {(size_t)w, (size_t)h};
    in.tex.kind = dev::TEX_RGBA8; in.tex.width = w; in.tex.height = h; in.tex.pitch0 = w * 4;
    t.width = w; t.height = h; t.mode = opts_.rendering_mode; t.out_pitch = w * 4;
    if (host_only_) return SMR_OK;
    if (smr_status st = alloc_on_stream(node_texture_bytes(w, h) + extra_bytes, n.mem); st != SMR_OK) return st;
    in.tex.p0 = t.out = (uint8_t *)n.mem.get();
    if (clear) CUDA_OK(cudaMemsetAsync(t.out, 0, (size_t)w * h * 4, stream_));
    return SMR_OK;
}

// A text node for `p`: the node texture (1 x 1 for 0 x 0), and on a device handle the glyph and atlas memory and the job
// that draws it.  Host memory is copied on stream_ (pageable sources: staged before the call returns).
smr_status Renderer::make_text_node(const std::shared_ptr<const TextPayload> &p, AtlasUploads &atlases,
                                    std::unique_ptr<TextNode> &out) {
    auto t = std::make_unique<TextNode>();
    const bool empty = p->width == 0 || p->height == 0;
    const int w = empty ? 1 : (int)p->width, h = empty ? 1 : (int)p->height;
    dev::TextJob &J = t->job;
    J.color_mode = p->color_mode;
    if (!empty) {   // 0 x 0: a transparent clear and no glyphs
        J.n_glyphs = (int)p->glyphs.size();
        shader_color(p->background, J.bg);
    }
    const size_t glyph_bytes = sizeof(smr_glyph) * (size_t)J.n_glyphs;
    if (smr_status st = make_node_texture(w, h, false, glyph_bytes, *t, J.dst); st != SMR_OK) return st;
    if (host_only_) { out = std::move(t); return SMR_OK; }
    cudaStream_t s = stream_;
    if (J.n_glyphs) {
        uint8_t *glyphs = J.dst.out + node_texture_bytes(w, h);
        CUDA_OK(cudaMemcpyAsync(glyphs, p->glyphs.data(), glyph_bytes, cudaMemcpyHostToDevice, s));
        stats_.h2d_bytes += glyph_bytes;
        J.glyphs = reinterpret_cast<const dev::GlyphDev *>(glyphs);
    }
    const TextAtlas *atl[2] = {p->mask.get(), p->color.get()};
    for (int k = 0; k < 2; k++) {
        if (!atl[k] || empty) continue;
        std::shared_ptr<void> &buf = atlases[atl[k]];   // one upload per atlas of the scene
        if (!buf) {
            if (smr_status st = alloc_on_stream(atl[k]->data.size(), buf); st != SMR_OK) return st;
            CUDA_OK(cudaMemcpyAsync(buf.get(), atl[k]->data.data(), atl[k]->data.size(), cudaMemcpyHostToDevice, s));
            stats_.h2d_bytes += atl[k]->data.size();
        }
        t->atlas[k] = buf;
        const uint8_t *d = (const uint8_t *)buf.get();
        if (k == 0) { J.mask = d; J.mask_w = (int)atl[k]->width; J.mask_h = (int)atl[k]->height; J.mask_pitch = (int)atl[k]->width; }
        else { J.color = d; J.color_w = (int)atl[k]->width; J.color_h = (int)atl[k]->height; J.color_pitch = (int)atl[k]->width * 4; }
    }
    out = std::move(t);
    return SMR_OK;
}

// An image node for `p`: its node texture, and the job that draws a frame of the asset into it.  An SVG asset is
// rasterised here by the caller at the node's resolution (SvgNodeState: one render per scene update) and the raster is
// copied after the node texture, in its memory (pageable source: staged before the call returns); a host-only handle
// drops it.  A rasteriser that refuses drops the update.
smr_status Renderer::make_image_node(const ImageParams &p, std::unique_ptr<ImageNode> &out) {
    auto n = std::make_unique<ImageNode>();
    n->params = p;
    dev::ImageJob &J = n->job;
    const ImageAsset &a = *p.asset;
    const int w = (int)p.resolution.width, h = (int)p.resolution.height;
    if (!a.svg()) {
        J.src.kind = dev::TEX_RGBA8; J.src.width = (int)a.width; J.src.height = (int)a.height; J.src.pitch0 = (int)a.width * 4;
        if (smr_status st = make_node_texture(w, h, false, 0, *n, J.dst); st != SMR_OK) return st;
        out = std::move(n);
        return SMR_OK;
    }
    const size_t bytes = (size_t)w * h * 4;
    std::vector<uint8_t> raster(bytes, 0);
    if (a.rasterize(a.user, (uint32_t)w, (uint32_t)h, raster.data(), (uint32_t)w * 4) != 0) {
        set_error("SVG image \"" + a.svg_id + "\": the rasteriser refused a raster of " + std::to_string(w) + " x " + std::to_string(h));
        return SMR_ERR_SCENE;
    }
    J.raster = 1;
    J.src.kind = dev::TEX_RGBA8; J.src.width = w; J.src.height = h; J.src.pitch0 = w * 4;
    if (smr_status st = make_node_texture(w, h, false, bytes, *n, J.dst); st != SMR_OK) return st;
    if (!host_only_) {
        uint8_t *dst = J.dst.out + node_texture_bytes(w, h);
        CUDA_OK(cudaMemcpyAsync(dst, raster.data(), bytes, cudaMemcpyHostToDevice, stream_));
        stats_.h2d_bytes += bytes;
        J.src.p0 = dst;
    }
    out = std::move(n);
    return SMR_OK;
}

// A web node for `p`: its node texture, cleared to transparent (new_web_renderer_node's ensure_size), and the job that draws it
smr_status Renderer::make_web_node(const WebParams &p, std::unique_ptr<WebNode> &out) {
    auto n = std::make_unique<WebNode>();
    n->params = p;
    if (smr_status st = make_node_texture((int)p.instance->width, (int)p.instance->height, true, 0, *n, n->job.dst); st != SMR_OK)
        return st;
    out = std::move(n);
    return SMR_OK;
}

// A shader node for `p`: its node texture (transparent until its first tick) and the job that draws it
smr_status Renderer::make_shader_node(const ShaderParams &p, std::unique_ptr<ShaderNode> &out) {
    auto n = std::make_unique<ShaderNode>();
    n->params = p;
    n->job.n_tex = (int)p.children.size();
    if (smr_status st = make_node_texture((int)p.resolution.width, (int)p.resolution.height, true, 0, *n, n->job.dst); st != SMR_OK)
        return st;
    out = std::move(n);
    return SMR_OK;
}

static inline long long snap256(float v);
static inline long long ceil_div256(long long a);

// One plane of WebRendererShader::render in a W x H target, from the entries of its vertex matrix that are not 0 or 1
// (vertices_transformation_matrix, transformation_matrices.rs:14-68; the website's is the identity).  The plane mesh's
// corners (+-1, +-1) map to clip x = m03 +- m00, y = m13 +- m11 (one rounding: the products by +-1 are exact) and to target
// pixels by the viewport transform x * W/2 + W/2, y * -H/2 + H/2 (fmaf); the texture coordinate runs from 0 at the corner
// (-1, +1) to 1 at (+1, -1).  NC-7 as in layer_geometry: corners snapped to 1/256 px, a pixel is covered when its centre
// lies in [x0, x1) x [y0, y1).  A quad mirrored on one axis faces back and is culled (cull_mode Back, common_pipeline.rs).
// False when the plane covers no pixel.
static bool web_plane(float m00, float m03, float m11, float m13, int W, int H, dev::WebPlane &p) {
    const float sx = (float)W / 2.0f, sy = (float)H / 2.0f;
    const float X0 = std::fma(m03 - m00, sx, sx), X1 = std::fma(m03 + m00, sx, sx);
    const float Y0 = std::fma(-(m13 + m11), sy, sy), Y1 = std::fma(-(m13 - m11), sy, sy);
    if (!(std::isfinite(X0) && std::isfinite(X1) && std::isfinite(Y0) && std::isfinite(Y1))) return false;
    if ((X1 < X0) != (Y1 < Y0)) return false;
    auto snap = [](float v) { return snap256(std::fmin(std::fmax(v, -1e7f), 1e7f)); };
    const long long x0 = snap(std::fmin(X0, X1)), x1 = snap(std::fmax(X0, X1));
    const long long y0 = snap(std::fmin(Y0, Y1)), y1 = snap(std::fmax(Y0, Y1));
    p.px0 = (int)std::max<long long>(ceil_div256(x0 - 128), 0); p.px1 = (int)std::min<long long>(ceil_div256(x1 - 128), W);
    p.py0 = (int)std::max<long long>(ceil_div256(y0 - 128), 0); p.py1 = (int)std::min<long long>(ceil_div256(y1 - 128), H);
    if (p.px0 >= p.px1 || p.py0 >= p.py1) return false;
    p.left = X0; p.width = X1 - X0; p.top = Y0; p.height = Y1 - Y0;
    return true;
}

// The planes a tick draws into web node `n` (WebRenderer::prepare_textures, renderer.rs:101-134), when its instance has a
// frame: the page, and each child zipped with the latest rect list, in the instance's embedding order.  The frame pointer
// and the rects are copied into this tick's parameters, so a later smr_web_set_frame / smr_web_set_child_rects does not
// change what the tick reads.  The children's textures are read when the tick is packed, once the layout nodes'
// frame-arena textures have addresses.
void Renderer::plan_web_node(Output &o, WebNode &n) {
    const WebInstance &w = *n.params.instance;
    if (!w.frame) return;   // no frame yet: the texture stays as it is (renderer.rs:89-96)
    n.owner = &o;
    const int W = (int)w.width, H = (int)w.height;
    dev::WebPlane site;
    site.tex.kind = dev::TEX_BGRA; site.tex.width = W; site.tex.height = H; site.tex.pitch0 = W * 4;
    site.tex.p0 = (const uint8_t *)w.frame.get();
    const bool site_ok = web_plane(1.0f, 0.0f, 1.0f, 0.0f, W, H, site);
    n.planes.clear();
    n.plane_child.clear();
    auto push = [&](const dev::WebPlane &pl, int child) { n.planes.push_back(pl); n.plane_child.push_back(child); };
    if (site_ok && w.embedding == SMR_WEB_NATIVE_OVER_CONTENT) push(site, -1);
    const size_t nc = std::min(n.params.children.size(), w.rects.size() / 4);
    const float sx = (float)W / 2.0f, sy = (float)H / 2.0f, a = 1.0f / sx, b = 1.0f / sy;
    for (size_t k = 0; k < nc; k++) {
        const float *r = &w.rects[4 * k];   // left, top, width, height
        const float tx = -((float)W / 2.0f) + (r[0] + r[2] / 2.0f), ty = (float)H / 2.0f - (r[1] + r[3] / 2.0f);
        dev::WebPlane pl;
        if (!web_plane(a * (sx * (r[2] / (float)W)), a * tx, b * (sy * (r[3] / (float)H)), b * ty, W, H, pl)) continue;
        push(pl, (int)k);
    }
    if (site_ok && w.embedding == SMR_WEB_NATIVE_UNDER_CONTENT) push(site, -1);
    n.job.n_planes = (int)n.planes.size();
    plan_.webs.push_back(&n);
}

// The textures a tick's draw of shader node `n` reads (its children, each its own node; an input without a live frame is the
// empty view) and BaseShaderParameters::time at `pts` (Duration::as_secs_f32: whole seconds plus nanoseconds / 1e9, in f32)
// The textures themselves are read when the tick is packed, once the layout nodes' frame-arena textures have addresses.
void Renderer::plan_shader_node(Output &o, ShaderNode &n, uint64_t pts) {
    n.owner = &o;
    n.job.time = (float)(pts / 1000000000ull) + (float)(uint32_t)(pts % 1000000000ull) / 1e9f;
    plan_.shaders.push_back(&n);
}

// A tick that renders output `o` at `pts`: each of its text, image, web and shader nodes enters the texture table.  The text nodes
// not drawn since the last smr_update_scene join the tick's text launch; the image nodes whose frame at `pts` (a Bitmap's
// or an SVG raster's only frame; AnimatedAsset::render's choice) is not the one their texture holds join its image
// launch; the web nodes whose instance has a frame join its web launch of their depth.
void Renderer::plan_node_textures(Output &o, uint64_t pts) {
    if (o.nodes_planned == tick_) return;
    o.nodes_planned = tick_;
    auto enter = [&](NodeTexture &n) {
        n.in.node_tex = -1;
        n.in.raw_tex = add_texture(n.in.tex, false);
    };
    for (auto &n : o.webs) {
        enter(*n);
        plan_web_node(o, *n);
    }
    for (auto &n : o.shaders) {   // every tick draws every shader node (ShaderNode::render has no cache)
        enter(*n);
        plan_shader_node(o, *n, pts);
    }
    for (auto &n : o.images) {
        enter(*n);
        const ImageAsset &a = *n->params.asset;
        const int frame = a.animated() ? (int)a.frame_at(pts, n->params.start_pts) : 0;
        if (frame == n->held) continue;
        n->held_before = n->held;
        n->held = frame;   // undone if the tick fails before its launch
        if (!a.svg()) n->job.src.p0 = (const uint8_t *)a.pixels.get() + (size_t)a.width * a.height * 4 * frame;
        plan_.images.push_back(n.get());
    }
    for (auto &t : o.texts) {
        enter(*t);
        if (t->rendered) continue;
        t->rendered = true;   // undone if the tick fails before its launch
        plan_.texts.push_back(t.get());
    }
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
    OutputNode node;   // the root is a layout: the given one
    node.resolution = {w, h};
    node.root_layout.given_layouts = std::move(ls);
    node.root_layout.given_resolution = {root_w, root_h};
    for (uint32_t i = 0; i < n_children; i++)
        node.root_layout.children.push_back({NodeRef::Input, -1, child_ids[i] ? child_ids[i] : ""});
    if (!host_only_) CUDA_OK(cudaSetDevice(opts_.cuda_device));   // the memory of the replaced nodes is released on stream_
    install_output(output_id, std::move(node), fmt, w, h);
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

static bool tex_is_yuv(const dev::Tex &t) {
    return t.kind == dev::TEX_YUV420 || t.kind == dev::TEX_NV12 || t.kind >= dev::TEX_YUV422;
}

// An input's smr_input_color over its frame's texture: DEFAULT keeps the format's rule (tex_kind_of_format: BT.709, full
// range for J420 only), an explicit value replaces it.  RGB kinds ignore the setting.
static void apply_input_color(const smr_input_color &c, dev::Tex &t) {
    if (!tex_is_yuv(t)) return;
    if (c.matrix != SMR_MATRIX_DEFAULT) t.matrix = c.matrix == SMR_MATRIX_BT601 ? 1 : 0;
    if (c.range != SMR_RANGE_DEFAULT) t.full_range = c.range == SMR_RANGE_FULL ? 1 : 0;
}

// Tex::matrix as smr_yuv_matrix, for inspection; 0 for a texture that is not YUV
static int32_t public_matrix(const dev::Tex &t) {
    return !tex_is_yuv(t) ? 0 : t.matrix == 1 ? SMR_MATRIX_BT601 : SMR_MATRIX_BT709;
}
static smr_fused_variant_info public_variant(const dev::FusedVariant &v) {
    smr_fused_variant_info o{};
    o.kernel = v.kind == dev::FusedVariant::TMA_INT ? SMR_FUSED_TMA_INT : v.kind == dev::FusedVariant::TMA_ANY ? SMR_FUSED_TMA_ANY : SMR_FUSED_LDG;
    o.ratio = v.ratio;
    o.window = v.kind == dev::FusedVariant::TMA_ANY ? dev::kTma0Window[v.window] : 0;
    o.box = v.box;
    o.src_class = v.src;
    o.range = v.range;
    o.matrix = v.matrix == 1 ? SMR_MATRIX_BT601 : SMR_MATRIX_BT709;
    return o;
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

static size_t align16(size_t n) { return (n + 15) & ~(size_t)15; }

// a live frame, checked and uploaded: host planes go to the slot's buffers on alternating copy streams.  A deinterlaced
// input's planes are staged at 16-byte aligned pitches, which k_deinterlace reads with 16-byte loads.
smr_status Renderer::upload_input(Input &I, const smr_input_frame &f) {
    FrameView v;
    if (smr_status st = read_frame(f, v); st != SMR_OK) return st;
    apply_input_color(I.color, v.tex);
    const bool deint = I.deint.mode != SMR_DEINTERLACE_OFF;
    for (int p = 0; p < 3 && f.mem_kind != SMR_MEM_DEVICE; p++) {
        FrameView::Plane &P = v.plane[p];
        if (!P.p) continue;
        const size_t pitch = deint ? align16(P.row_bytes) : P.row_bytes;
        DevBuf &buf = I.planes[slot_][p];
        CUDA_OK(buf.ensure(pitch * P.rows));
        cudaStream_t cs = (upload_rr_++ & 1) ? copy_stream2_ : copy_stream_;
        if (P.pitch == P.row_bytes && pitch == P.row_bytes)   // tightly packed (the reference's bytes::Bytes planes): one linear DMA
            CUDA_OK(cudaMemcpyAsync(buf.p, P.p, P.row_bytes * P.rows, cudaMemcpyHostToDevice, cs));
        else
            CUDA_OK(cudaMemcpy2DAsync(buf.p, pitch, P.p, P.pitch, P.row_bytes, P.rows, cudaMemcpyHostToDevice, cs));
        uploaded_ = true;
        stats_.h2d_bytes += P.row_bytes * P.rows;
        P.p = buf.p; P.pitch = pitch;
        set_tex_plane(v.tex, p, buf.p, pitch);
    }
    if (deint)
        if (smr_status st = plan_deinterlace(I, f, v); st != SMR_OK) return st;
    I.format = f.format;
    I.tex = v.tex;
    I.raw_tex = add_texture(v.tex, tex_is_yuv(v.tex));
    return SMR_OK;
}

// The tick's k_deinterlace jobs for a live frame of a deinterlaced input (NC-12), one per plane; `v` is pointed at the
// slot's deinterlaced planes.  MOTION_ADAPTIVE reads the previous frame from the history and, for a frame of a new pts,
// copies the current one into the other history set, which becomes the last.  Two sets suffice: the ticks run in order on
// stream_, and the set a tick writes is read only by later ticks.
smr_status Renderer::plan_deinterlace(Input &I, const smr_input_frame &f, FrameView &v) {
    DeinterlaceHistory &H = I.hist;
    plan_.deint_history.push_back({&I, H});
    int prev_set = -1;
    DevBuf *next = nullptr;
    if (I.deint.mode == SMR_DEINTERLACE_MOTION_ADAPTIVE) {
        if (H.frames && (H.format != f.format || H.width != f.width || H.height != f.height)) H = DeinterlaceHistory();
        const bool repeat = H.frames && H.pts == f.pts_ns;   // the same frame again: same bytes, history unchanged
        if (repeat) {
            prev_set = H.frames == 2 ? (H.last ^ 1) : -1;
        } else {
            prev_set = H.frames ? H.last : -1;
            next = I.hist_planes[H.last ^ 1];
            H.last ^= 1;
            H.frames = std::min(H.frames + 1, 2);
            H.pts = f.pts_ns; H.format = f.format; H.width = f.width; H.height = f.height;
        }
    }
    for (int p = 0; p < 3; p++) {
        const FrameView::Plane &P = v.plane[p];
        if (!P.p) continue;
        const size_t pitch = align16(P.row_bytes);
        DevBuf &out = I.deint_out[slot_][p];
        CUDA_OK(out.ensure(pitch * P.rows));
        dev::DeinterlaceJob j{};
        j.cur = P.p; j.cur_pitch = (int)P.pitch;
        if (prev_set >= 0) { j.prev = I.hist_planes[prev_set][p].p; j.prev_pitch = (int)pitch; }
        j.out = out.p; j.out_pitch = (int)pitch;
        if (next) {
            CUDA_OK(next[p].ensure(pitch * P.rows));
            j.hist = next[p].p; j.hist_pitch = (int)pitch;
        }
        j.row_bytes = (int)P.row_bytes; j.rows = (int)P.rows;
        j.rebuild = I.deint.field_order == SMR_FIELD_TOP_FIRST ? 1 : 0;
        j.threshold = I.deint.motion_threshold;
        j.tiles_x = dev::deinterlace_tiles_x(j.row_bytes);
        plan_.deint.push_back(j);
        set_tex_plane(v.tex, p, out.p, pitch);
    }
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
    dev::FusedVariant k;   // LDG, weights from smem
    int tmap_idx = -1, cols = 64;
    if (!box && hm.crop_offset == 0.0f && (sh == 2.0f || sh == 3.0f || sh == 4.0f)) k.ratio = (int)sh;   // LDG, int_weights.h
    if (tma && (k.ratio == 2 || k.ratio == 4) && rows8 <= (k.ratio == 4 ? dev::kTmaRing4 : dev::kTmaRing2) &&
        (tmap_idx = source_tmaps(t, src_class)) >= 0) {
        k.kind = dev::FusedVariant::TMA_INT;
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
            k = {dev::FusedVariant::TMA_ANY, 0, bucket, box ? 1 : 0};
    }
    if (box && k.kind != dev::FusedVariant::TMA_ANY) return -1;   // no other fused kernel reduces: generic passes
    k.src = src_class;
    k.range = dev::fused_launch_range(k, t.full_range);
    k.matrix = t.matrix;
    const WeightEntry *wh, *wv;
    if (get_weights(passes[0], wh) != SMR_OK || get_weights(passes[1], wv) != SMR_OK) return -2;
    size_t dst_off = frame_alloc((size_t)dw * dh * 4);
    dev::FusedJob j{};
    j.dst_w = dw; j.dst_h = dh; j.dst_pitch = dw * 4;
    j.taps_h = wh->taps; j.taps_v = wv->taps;
    j.w_h = wh->weights; j.inv_h = wh->inv; j.first_h = wh->first;
    j.w_v = wv->weights; j.inv_v = wv->inv; j.first_v = wv->first;
    if (k.kind == dev::FusedVariant::TMA_INT) j.v_same = vm.crop_offset == 0.0f && sv == sh && tv == th;
    if (k.kind == dev::FusedVariant::TMA_ANY) {
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
    if (it != lane_perms_.end()) {
        it->second.last_used = tick_;
        return it->second.perm;
    }
    bound_cache(lane_perms_);
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
    DevMem<uint8_t> owned(dev_perm);
    // pageable source: staged before the call returns
    if (cudaMemcpyAsync(dev_perm, perm.data(), perm.size(), cudaMemcpyHostToDevice, stream_) != cudaSuccess) {
        cudaGetLastError(); return nullptr;
    }
    cudaStreamSynchronize(stream_);   // once per geometry; keeps the pageable staging out of the steady state
    lane_perms_[key] = {std::move(owned), tick_};
    return dev_perm;
}

// Bounds a cache of device tables (weights_, lane_perms_): past 4096 entries, the entries this tick has not used are
// dropped once stream_ no longer reads them.  Jobs planned earlier in the tick keep theirs.
template <class Cache> void Renderer::bound_cache(Cache &c) {
    if (c.size() <= 4096) return;
    cudaStreamSynchronize(stream_);
    for (auto i = c.begin(); i != c.end();) i = i->second.last_used == tick_ ? std::next(i) : c.erase(i);
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
    for (const WeightKey &k : new_weight_keys_) weights_.erase(k);
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

// The blocking calls run one kernel each on stream_ and return once its result is complete, like the reference's
// device.poll (frame_pre_processor.rs:171-176); the caller's host buffers are borrowed for the call only.  Each checks its
// arguments, passes need_device, stages its host sources, places its targets, fills its job and calls launch_and_finish.
smr_status Renderer::need_device() {
    if (host_only_) { set_error("host-only handle (cuda_device = -1) has no device: no CPU fallback"); return SMR_ERR_CUDA; }
    CUDA_OK(cudaSetDevice(opts_.cuda_device));
    return SMR_OK;
}

// rows x row_bytes host bytes at src_pitch, copied packed into `scratch` on stream_ (pageable sources are staged before
// the copy returns).  Work still on stream_ may read `scratch`, so the stream drains before it is reallocated.
smr_status Renderer::stage_in(DevBuf &scratch, const void *src, size_t src_pitch, size_t row_bytes, size_t rows) {
    if (row_bytes * rows > scratch.cap) CUDA_OK(cudaStreamSynchronize(stream_));
    CUDA_OK(scratch.ensure(row_bytes * rows));
    CUDA_OK(cudaMemcpy2DAsync(scratch.p, row_bytes, src, src_pitch, row_bytes, rows, cudaMemcpyHostToDevice, stream_));
    stats_.h2d_bytes += row_bytes * rows;
    return SMR_OK;
}

// A frame read_frame has checked: host planes are staged into pre_planes_ and `v` is pointed at them; device planes stay
// where they are
smr_status Renderer::upload_pre_planes(const smr_input_frame &f, FrameView &v) {
    for (int p = 0; p < 3 && f.mem_kind != SMR_MEM_DEVICE; p++) {
        const FrameView::Plane &P = v.plane[p];
        if (!P.p) continue;
        if (smr_status st = stage_in(pre_planes_[p], P.p, P.pitch, P.row_bytes, P.rows); st != SMR_OK) return st;
        set_tex_plane(v.tex, p, pre_planes_[p].p, P.row_bytes);
    }
    return SMR_OK;
}

// Where the kernel writes each target plane: a device plane itself; host planes packed, in order, into pre_out_, which
// launch_and_finish copies back.  pre_out_ is sized for them all before a pointer into it is taken (ensure reallocates).
smr_status Renderer::place_targets(TargetPlane *t, size_t n) {
    size_t staged = 0;
    for (size_t i = 0; i < n; i++)
        if (!t[i].device) staged += t[i].row_bytes * t[i].rows;
    if (staged > pre_out_.cap) CUDA_OK(cudaStreamSynchronize(stream_));
    if (staged) CUDA_OK(pre_out_.ensure(staged));
    for (size_t i = 0, off = 0; i < n; i++) {
        if (t[i].device) { t[i].out = (uint8_t *)t[i].p; t[i].out_pitch = (int)t[i].pitch; continue; }
        t[i].out = pre_out_.p + off; t[i].out_pitch = (int)t[i].row_bytes;
        off += t[i].row_bytes * t[i].rows;
    }
    return SMR_OK;
}

// Enqueues the call's kernel (`launch` returns what a dev::launch_* does) and the copy-backs of its host targets, and waits
// for them.  The profiling events of `kernel_class` (-1: none) enclose the launch alone.
template <class Launch>
smr_status Renderer::launch_and_finish(const TargetPlane *t, size_t n, int kernel_class, Launch launch) {
    const bool prof = profiling_ && kernel_class >= 0;
    if (prof && !call_ev_[0]) {
        CUDA_OK(make(call_ev_[0], cudaEventCreateWithFlags, cudaEventDefault));
        CUDA_OK(make(call_ev_[1], cudaEventCreateWithFlags, cudaEventDefault));
    }
    if (prof) CUDA_OK(cudaEventRecord(call_ev_[0], stream_));
    if (launch() < 0) { set_error(dev::last_launch_error()); return SMR_ERR_CUDA; }
    stats_.kernel_launches++;
    if (prof) CUDA_OK(cudaEventRecord(call_ev_[1], stream_));
    for (size_t i = 0; i < n; i++) {
        if (t[i].device) continue;
        CUDA_OK(cudaMemcpy2DAsync(t[i].p, t[i].pitch, t[i].out, t[i].out_pitch, t[i].row_bytes, t[i].rows, cudaMemcpyDeviceToHost,
                                  stream_));
        stats_.d2h_bytes += t[i].row_bytes * t[i].rows;
    }
    CUDA_OK(cudaStreamSynchronize(stream_));
    if (prof) {
        float ms = 0.0f;
        CUDA_OK(cudaEventElapsedTime(&ms, call_ev_[0], call_ev_[1]));
        prof_.total_ms[kernel_class] += ms;
        prof_.launches[kernel_class] += 1;
    }
    return SMR_OK;
}

// One axis of gpu-video's transcoder resize (vulkan_transcoder/shader.wgsl, NC-10) for every output coordinate: what
// main and its samplers compute from (coordinate + 0.5) / size before they load a texel.  f32 throughout, each operation
// rounded on its own (-ffp-contract=off), sin in fp64 rounded to f32 (NC-8).
static float transcode_sinc(float x) {
    if (std::fabs(x) < 1e-6f) return 1.0f;
    const float px = 3.14159265358979323846f * x;
    return (float)std::sin((double)px) / px;
}
static float transcode_lanczos3(float x) { return std::fabs(x) >= 3.0f ? 0.0f : transcode_sinc(x) * transcode_sinc(x / 3.0f); }
static void transcode_axis(uint32_t in_len, uint32_t out_len, std::vector<dev::TranscodeTap> &taps) {
    taps.resize(out_len);
    const float fin = (float)in_len, fout = (float)out_len;
    for (uint32_t k = 0; k < out_len; k++) {
        dev::TranscodeTap &t = taps[k];
        const float coord = ((float)k + 0.5f) / fout;   // float_coords
        const float scaled = fin * coord;
        t.nearest = (int32_t)(uint32_t)scaled;            // u32(): truncation; scaled < in_len for in_len, out_len <= 16384
        const float fc = scaled - 0.5f;
        const float fl = std::floor(fc);
        t.lo = (int32_t)(uint32_t)std::fmax(fl, 0.0f);
        t.hi = std::min(t.lo + 1, (int32_t)in_len - 1);
        t.frac = fc - fl;
        t.center = (int32_t)fl;
        for (int d = 0; d < 6; d++) t.w[d] = transcode_lanczos3(fc - (fl + (float)(d - 2)));
    }
}

const dev::TranscodeTap *Renderer::transcode_table(uint32_t in_len, uint32_t out_len) {
    auto it = transcode_taps_.find({in_len, out_len});
    if (it == transcode_taps_.end()) {
        while (transcode_taps_.size() >= kTranscodeTapTables) {   // release the least recently used (not this call's)
            auto lru = transcode_taps_.begin();
            for (auto j = transcode_taps_.begin(); j != transcode_taps_.end(); ++j)
                if (j->second.used < lru->second.used) lru = j;
            if (lru->second.used == transcode_calls_) break;
            transcode_taps_.erase(lru);
        }
        std::vector<dev::TranscodeTap> host;
        transcode_axis(in_len, out_len, host);
        TapTable &t = transcode_taps_[{in_len, out_len}];
        const size_t bytes = sizeof(dev::TranscodeTap) * host.size();
        // pageable source: staged before cudaMemcpyAsync returns, and ordered before the launch on stream_
        if (t.buf.ensure(bytes) != cudaSuccess ||
            cudaMemcpyAsync(t.buf.p, host.data(), bytes, cudaMemcpyHostToDevice, stream_) != cudaSuccess) {
            transcode_taps_.erase({in_len, out_len});
            return nullptr;
        }
        it = transcode_taps_.find({in_len, out_len});
    }
    it->second.used = transcode_calls_;
    return reinterpret_cast<const dev::TranscodeTap *>(it->second.buf.p);
}

// VideoTranscoder's resize step (gpu-video vulkan_transcoder/pipeline.rs + shader.wgsl): every rendition in one launch
smr_status Renderer::transcode_resize(const smr_input_frame *src, const smr_rendition *out, uint32_t n) {
    if (!src || (n && !out)) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    if (n == 0 || n > (uint32_t)dev::kTranscodeMaxOutputs) {
        set_error("wrong output number: expected 1 to 8 renditions");
        return SMR_ERR_INVALID_ARGUMENT;
    }
    for (uint32_t i = 0; i < n; i++) {
        const smr_rendition &o = out[i];
        if (o.width == 0 || o.height == 0 || o.width > kMaxFrameDim || o.height > kMaxFrameDim || ((o.width | o.height) & 1)) {
            set_error("rendition " + std::to_string(i) + ": width and height must be even and in 2 .. 16384");
            return SMR_ERR_INVALID_ARGUMENT;
        }
        if (o.scaling != SMR_SCALE_NEAREST && o.scaling != SMR_SCALE_BILINEAR && o.scaling != SMR_SCALE_LANCZOS3) {
            set_error("rendition " + std::to_string(i) + ": unknown scaling algorithm");
            return SMR_ERR_INVALID_ARGUMENT;
        }
        if (o.mem_kind != SMR_MEM_HOST && o.mem_kind != SMR_MEM_DEVICE) {
            set_error("rendition " + std::to_string(i) + ": unknown mem_kind");
            return SMR_ERR_INVALID_ARGUMENT;
        }
        for (int p = 0; p < 2; p++) {   // an NV12 row is `width` bytes in both planes
            if (!o.planes[p]) { set_error("rendition " + std::to_string(i) + ": plane pointer is null"); return SMR_ERR_INVALID_ARGUMENT; }
            if (o.pitch[p] && o.pitch[p] < o.width) {
                set_error("rendition " + std::to_string(i) + ": pitch is smaller than a row");
                return SMR_ERR_INVALID_ARGUMENT;
            }
        }
    }
    FrameView v;
    if (smr_status st = read_frame(*src, v); st != SMR_OK) return st;
    if (src->format != SMR_FRAME_NV12) { set_error("the transcoder resize takes NV12 frames"); return SMR_ERR_UNSUPPORTED; }
    if ((src->width | src->height) & 1) { set_error("NV12 source width and height must be even"); return SMR_ERR_INVALID_ARGUMENT; }
    if (smr_status st = need_device(); st != SMR_OK) return st;
    if (smr_status st = upload_pre_planes(*src, v); st != SMR_OK) return st;
    TargetPlane t[2 * dev::kTranscodeMaxOutputs];   // Y and UV of each rendition
    for (uint32_t i = 0; i < n; i++) {   // an NV12 row is `width` bytes in both planes
        const smr_rendition &o = out[i];
        for (int p = 0; p < 2; p++)
            t[2 * i + p] = {o.planes[p], o.pitch[p] ? o.pitch[p] : o.width, o.width, p ? o.height / 2 : o.height,
                            o.mem_kind == SMR_MEM_DEVICE};
    }
    if (smr_status st = place_targets(t, 2 * n); st != SMR_OK) return st;

    dev::TranscodeLaunch L = {};
    L.src_y = v.tex.p0; L.src_uv = v.tex.p1;
    L.pitch_y = v.tex.pitch0; L.pitch_uv = v.tex.pitch1;
    L.width = (int)src->width; L.height = (int)src->height;
    L.n = (int)n;
    transcode_calls_++;
    int blocks = 0;
    for (uint32_t i = 0; i < n; i++) {
        const smr_rendition &o = out[i];
        dev::TranscodeOut &J = L.out[i];
        J.width = (int)o.width; J.height = (int)o.height; J.scaling = o.scaling;
        J.y = t[2 * i].out; J.pitch_y = t[2 * i].out_pitch;
        J.uv = t[2 * i + 1].out; J.pitch_uv = t[2 * i + 1].out_pitch;
        J.tx = transcode_table(src->width, o.width);
        J.ty = transcode_table(src->height, o.height);
        J.cx = transcode_table(src->width / 2, o.width / 2);
        J.cy = transcode_table(src->height / 2, o.height / 2);
        if (!J.tx || !J.ty || !J.cx || !J.cy) { set_error("out of device memory for the transcoder tables"); return SMR_ERR_OUT_OF_MEMORY; }
        J.tiles_x = (int)((o.width / 2 + dev::kTranscodeTileX - 1) / dev::kTranscodeTileX);
        J.tile_begin = blocks;
        blocks += J.tiles_x * (int)((o.height / 2 + dev::kTranscodeTileY - 1) / dev::kTranscodeTileY);
    }
    return launch_and_finish(t, 2 * n, SMR_KERNEL_TRANSCODE, [&] { return dev::launch_transcode(L, blocks, stream_); });
}

// gpu-video's converters (wgpu_helpers/): WgpuConverterParameters as `new` checks them (OnlyLimitedBT709Supported)
static bool video_color_known(const smr_video_color &c) {
    return c.color_space >= SMR_COLOR_SPACE_UNSPECIFIED && c.color_space <= SMR_COLOR_SPACE_BT601_PAL &&
           (c.color_range == SMR_COLOR_RANGE_FULL || c.color_range == SMR_COLOR_RANGE_LIMITED);
}
smr_status Renderer::video_converter_ok(const smr_video_color &c) {
    if (!video_color_known(c)) { set_error("unknown color space or color range"); return SMR_ERR_INVALID_ARGUMENT; }
    if (c.color_space != SMR_COLOR_SPACE_BT709 || c.color_range != SMR_COLOR_RANGE_LIMITED) {
        set_error("only limited-range BT.709 converters are supported");
        return SMR_ERR_UNSUPPORTED;
    }
    return SMR_OK;
}

// WgpuNv12ToRgbaConverter: create_input_bind_group + convert (gpu-video wgpu_helpers/nv12_to_rgba.rs)
smr_status Renderer::video_nv12_to_rgba(const smr_video_color &converter, const smr_input_frame *src, const smr_video_color &frame,
                                        uint32_t ow, uint32_t oh, void *rgba, uint32_t pitch, int32_t mem_kind) {
    if (!src || !rgba) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    if (smr_status st = video_converter_ok(converter); st != SMR_OK) return st;
    if (!video_color_known(frame)) { set_error("unknown frame color space or color range"); return SMR_ERR_INVALID_ARGUMENT; }
    if ((frame.color_space != SMR_COLOR_SPACE_UNSPECIFIED && frame.color_space != converter.color_space) ||
        frame.color_range != converter.color_range) {
        set_error("incompatible frame: its color space and range do not match the converter's");
        return SMR_ERR_INVALID_ARGUMENT;
    }
    if ((ow == 0) != (oh == 0) || ow > kMaxFrameDim || oh > kMaxFrameDim) {
        set_error("output resolution out of range");
        return SMR_ERR_INVALID_ARGUMENT;
    }
    if (mem_kind != SMR_MEM_HOST && mem_kind != SMR_MEM_DEVICE) { set_error("unknown mem_kind"); return SMR_ERR_INVALID_ARGUMENT; }
    FrameView v;
    if (smr_status st = read_frame(*src, v); st != SMR_OK) return st;
    if (src->format != SMR_FRAME_NV12) { set_error("the NV12 to RGBA converter takes NV12 frames"); return SMR_ERR_UNSUPPORTED; }
    if ((src->width | src->height) & 1) { set_error("NV12 source width and height must be even"); return SMR_ERR_INVALID_ARGUMENT; }
    if (ow == 0) { ow = src->width; oh = src->height; }
    const size_t row = (size_t)ow * 4;
    if (pitch && pitch < row) { set_error("output pitch smaller than a row"); return SMR_ERR_INVALID_ARGUMENT; }
    if (mem_kind == SMR_MEM_DEVICE && (((uintptr_t)rgba | (pitch ? pitch : row)) & 3)) {
        set_error("device RGBA8 planes are 4-byte aligned");
        return SMR_ERR_INVALID_ARGUMENT;
    }
    if (smr_status st = need_device(); st != SMR_OK) return st;
    if (smr_status st = upload_pre_planes(*src, v); st != SMR_OK) return st;
    TargetPlane t = {rgba, pitch ? pitch : row, row, oh, mem_kind == SMR_MEM_DEVICE};
    if (smr_status st = place_targets(&t, 1); st != SMR_OK) return st;
    dev::VideoConvertJob J = {};
    J.src = v.tex;
    J.out_w = (int)ow; J.out_h = (int)oh;
    J.out = t.out; J.out_pitch = t.out_pitch;
    return launch_and_finish(&t, 1, SMR_KERNEL_VIDEO_CONVERT, [&] { return dev::launch_video_nv12_to_rgba(J, stream_); });
}

// WgpuRgbaToNv12Converter::convert (gpu-video wgpu_helpers/rgba_to_nv12.rs): rgba_to_nv12.wgsl is K11, so the kernel is
// k_output's NV12 target
smr_status Renderer::video_rgba_to_nv12(const smr_video_color &converter, const smr_input_frame *src, uint32_t ow, uint32_t oh,
                                        void *const planes[2], const uint32_t pitch[2], int32_t mem_kind) {
    if (!src || !planes) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    if (smr_status st = video_converter_ok(converter); st != SMR_OK) return st;
    if (ow == 0 || oh == 0 || ow > kMaxFrameDim || oh > kMaxFrameDim || ((ow | oh) & 1)) {
        set_error("NV12 target width and height must be even and in 2 .. 16384");
        return SMR_ERR_INVALID_ARGUMENT;
    }
    if (mem_kind != SMR_MEM_HOST && mem_kind != SMR_MEM_DEVICE) { set_error("unknown mem_kind"); return SMR_ERR_INVALID_ARGUMENT; }
    uint32_t tp[2];
    for (int p = 0; p < 2; p++) {   // an NV12 row is `ow` bytes in both planes
        tp[p] = pitch && pitch[p] ? pitch[p] : ow;
        if (!planes[p]) { set_error("target plane pointer is null"); return SMR_ERR_INVALID_ARGUMENT; }
        if (tp[p] < ow) { set_error("target pitch is smaller than a row"); return SMR_ERR_INVALID_ARGUMENT; }
    }
    FrameView v;
    if (smr_status st = read_frame(*src, v); st != SMR_OK) return st;
    if (src->format != SMR_FRAME_RGBA8) { set_error("the RGBA to NV12 converter takes RGBA8 frames"); return SMR_ERR_UNSUPPORTED; }
    if (smr_status st = need_device(); st != SMR_OK) return st;
    if (smr_status st = upload_pre_planes(*src, v); st != SMR_OK) return st;
    const bool device = mem_kind == SMR_MEM_DEVICE;
    TargetPlane t[2] = {{planes[0], tp[0], ow, oh, device}, {planes[1], tp[1], ow, oh / 2, device}};
    if (smr_status st = place_targets(t, 2); st != SMR_OK) return st;
    dev::OutputJob J = {};
    J.src = v.tex;
    J.out_w = (int)ow; J.out_h = (int)oh;
    J.out_format = SMR_OUT_NV12;
    J.out0 = t[0].out; J.out1 = t[1].out;
    J.out_pitch0 = t[0].out_pitch; J.out_pitch1 = t[1].out_pitch;
    return launch_and_finish(t, 2, SMR_KERNEL_OUTPUT, [&] { return dev::launch_output(J, stream_); });
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
    if (smr_status st = need_device(); st != SMR_OK) return st;
    const bool rescale = ow != 0 || oh != 0;
    // the output size is checked after the input size and before the rest of the frame
    if (rescale && frame_size_ok(*f) && (ow == 0 || oh == 0 || ow > 16384 || oh > 16384)) {
        set_error("output resolution out of range");
        return SMR_ERR_INVALID_ARGUMENT;
    }
    FrameView v;
    if (smr_status st = read_frame(*f, v); st != SMR_OK) return st;
    if (!rescale) { ow = f->width; oh = f->height; }
    TargetPlane t = {rgba, pitch ? pitch : (size_t)ow * 4, (size_t)ow * 4, oh, mem_kind == SMR_MEM_DEVICE};
    if (t.pitch < t.row_bytes) { set_error("output pitch smaller than a row"); return SMR_ERR_BUFFER_TOO_SMALL; }
    if (t.device && ((t.pitch | (uintptr_t)t.p) & 3)) { set_error("device RGBA8 planes are 4-byte aligned"); return SMR_ERR_INVALID_ARGUMENT; }
    if (smr_status st = upload_pre_planes(*f, v); st != SMR_OK) return st;
    if (smr_status st = place_targets(&t, 1); st != SMR_OK) return st;
    const int kind = premultiply ? 2 : (rescale ? 1 : 0);
    return launch_and_finish(&t, 1, -1, [&] {
        return dev::launch_preprocess(v.tex, opts_.rendering_mode, kind, t.out, t.out_pitch, (int)ow, (int)oh, stream_);
    });
}

// TextRendererNode::render (transformations/text_renderer.rs:72-167): clear + glyphon's glyph quads
smr_status Renderer::render_text(uint32_t w, uint32_t h, smr_rgba bg, const smr_glyph *glyphs, uint32_t n, const smr_atlas *mask,
                                 const smr_atlas *color, int32_t color_mode, void *rgba, uint32_t pitch, int32_t mem_kind) {
    static_assert(sizeof(smr_glyph) == sizeof(dev::GlyphDev), "smr_glyph is copied to the device as it is");
    if (!rgba || (n && !glyphs) || (color_mode != 0 && color_mode != 1)) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    if (smr_status st = need_device(); st != SMR_OK) return st;
    // a zero-sized text texture is a transparent 1x1 one in the reference (text_renderer.rs:77-85); here the caller skips it
    if (w == 0 || h == 0 || w > 16384 || h > 16384) { set_error("text texture resolution out of range"); return SMR_ERR_INVALID_ARGUMENT; }
    if (n > (1u << 22)) { set_error("too many glyphs"); return SMR_ERR_INVALID_ARGUMENT; }
    bool need[2] = {false, false};   // the mask atlas, the colour atlas
    for (uint32_t i = 0; i < n; i++) {
        if (glyphs[i].content == SMR_GLYPH_MASK) need[0] = true;
        else if (glyphs[i].content == SMR_GLYPH_COLOR) need[1] = true;
        else { set_error("glyph content type must be SMR_GLYPH_COLOR or SMR_GLYPH_MASK"); return SMR_ERR_INVALID_ARGUMENT; }
    }
    const smr_atlas *atl[2] = {mask, color};
    size_t atl_row[2] = {};
    for (int k = 0; k < 2; k++) {
        const smr_atlas *a = atl[k];
        if (!need[k]) continue;
        if (!a || !a->data || a->width == 0 || a->height == 0 || a->width > 16384 || a->height > 16384) {
            set_error(k == 0 ? "mask glyphs need a mask atlas" : "colour glyphs need a colour atlas");
            return SMR_ERR_INVALID_ARGUMENT;
        }
        atl_row[k] = (size_t)a->width * (k == 0 ? 1 : 4);
        if (a->pitch && a->pitch < atl_row[k]) { set_error("atlas pitch smaller than a row"); return SMR_ERR_INVALID_ARGUMENT; }
    }
    TargetPlane t = {rgba, pitch ? pitch : (size_t)w * 4, (size_t)w * 4, h, mem_kind == SMR_MEM_DEVICE};
    if (t.pitch < t.row_bytes) { set_error("output pitch smaller than a row"); return SMR_ERR_BUFFER_TOO_SMALL; }
    if (t.device && ((t.pitch | (uintptr_t)t.p) & 3)) { set_error("device RGBA8 planes are 4-byte aligned"); return SMR_ERR_INVALID_ARGUMENT; }

    for (int k = 0; k < 2; k++) {
        const smr_atlas *a = atl[k];
        if (!need[k]) continue;
        if (smr_status st = stage_in(pre_planes_[k], a->data, a->pitch ? a->pitch : atl_row[k], atl_row[k], a->height); st != SMR_OK)
            return st;
    }
    if (n) {
        if (smr_status st = stage_in(pre_planes_[2], glyphs, sizeof(smr_glyph) * n, sizeof(smr_glyph) * n, 1); st != SMR_OK)
            return st;
    }
    if (smr_status st = place_targets(&t, 1); st != SMR_OK) return st;
    dev::TextJob J = {};
    J.dst.width = (int)w; J.dst.height = (int)h; J.dst.mode = opts_.rendering_mode; J.color_mode = color_mode; J.n_glyphs = (int)n;
    J.dst.out = t.out; J.dst.out_pitch = t.out_pitch;
    shader_color(RGBA{bg.r, bg.g, bg.b, bg.a}, J.bg);
    if (need[0]) { J.mask = pre_planes_[0].p; J.mask_w = (int)mask->width; J.mask_h = (int)mask->height; J.mask_pitch = (int)atl_row[0]; }
    if (need[1]) { J.color = pre_planes_[1].p; J.color_w = (int)color->width; J.color_h = (int)color->height; J.color_pitch = (int)atl_row[1]; }
    if (n) J.glyphs = reinterpret_cast<const dev::GlyphDev *>(pre_planes_[2].p);
    // the job and its tile table, as the tick's text launch reads them from the parameter arena (pageable sources: staged
    // before the copies return)
    const size_t begin_off = (sizeof(dev::TextJob) + 15) & ~(size_t)15;
    const int32_t begin[2] = {0, dev::node_tiles((int)w, (int)h)};
    CUDA_OK(text_job_.ensure(begin_off + sizeof(begin)));
    CUDA_OK(cudaMemcpyAsync(text_job_.p, &J, sizeof(J), cudaMemcpyHostToDevice, stream_));
    CUDA_OK(cudaMemcpyAsync(text_job_.p + begin_off, begin, sizeof(begin), cudaMemcpyHostToDevice, stream_));
    return launch_and_finish(&t, 1, -1, [&] {
        return dev::launch_tile_jobs(dev::node_kernel(dev::NODE_TEXT), text_job_.p, (const int32_t *)(text_job_.p + begin_off), 1,
                                     begin[1], "k_text", stream_);
    });
}

smr_status Renderer::get_weights(const KernelPass &p, const WeightEntry *&out) {
    WeightKey key;
    float scale = p.mapping.scale(), offset = p.mapping.crop_offset;
    memcpy(&key.scale_bits, &scale, 4);
    memcpy(&key.offset_bits, &offset, 4);
    key.n_out = p.mapping.dst_len;
    auto it = weights_.find(key);
    if (it != weights_.end()) {
        it->second.last_used = tick_;
        out = &it->second;
        return SMR_OK;
    }
    bound_cache(weights_);
    const int taps = resample_taps(scale);
    if (taps < 1 || taps > 4096) { set_error("resampler tap count out of range"); return SMR_ERR_INVALID_ARGUMENT; }
    auto up256 = [](size_t n) { return (n + 255) & ~(size_t)255; };
    const size_t w_bytes = up256(sizeof(float) * (size_t)taps * key.n_out), inv_bytes = up256(sizeof(float) * key.n_out);
    uint8_t *d = nullptr;
    if (cudaMalloc(&d, w_bytes + inv_bytes + sizeof(int32_t) * key.n_out) != cudaSuccess) {
        cudaGetLastError();
        set_error("out of device memory for resampler weight tables");
        return SMR_ERR_CUDA;
    }
    WeightEntry &e = weights_[key];
    e.mem.reset(d);
    e.weights = (float *)d; e.inv = (float *)(d + w_bytes); e.first = (int32_t *)(d + w_bytes + inv_bytes);
    e.taps = taps; e.last_used = tick_;
    new_weight_keys_.push_back(key);
    dev::WeightJob j;
    j.scale = scale; j.offset = offset; j.n_out = key.n_out; j.taps = e.taps;
    j.weights = e.weights; j.inv_wsum = e.inv; j.first = e.first;
    plan_.weight_jobs.push_back(j);
    out = &e;
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
            if (f.key.kind != dev::FusedVariant::TMA_INT || f.key.ratio != 4 || !fj.v_same || ((fj.dst_w | fj.dst_h) & 1)) continue;
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

// Layout node `lp` of output `o` at `pts` (LayoutNode::render, layout.rs:170-181): its children (sources[i].resolution(),
// layout.rs:176-179), its resolution and its flattened layouts.  Evaluating them advances the state of `lp`: o.node's when
// rendering, a copy's for inspection.
Renderer::LayoutEval Renderer::eval_layout(Output &o, LayoutParams &lp, uint64_t pts) {
    LayoutEval e;
    for (const NodeRef &r : lp.children) {
        Input *in = node_input(o, r);
        e.child_in.push_back(in);
        e.child_res.push_back(in ? std::optional<Resolution>(in->res) : std::nullopt);
    }
    e.res = lp.resolution(pts);
    e.layouts = lp.layouts(pts, e.child_res);
    return e;
}

// The Input behind a render node: a text, image, web, shader or layout node's texture, or a caller's input; nullptr when it
// has no pixels this tick (an input without a live frame, a layout node of no size), which reads as the empty view
Renderer::Input *Renderer::node_input(Output &o, const NodeRef &r) {
    switch (r.kind) {
        case NodeRef::Text: return &o.texts[r.index]->in;
        case NodeRef::Image: return &o.images[r.index]->in;
        case NodeRef::Web: return &o.webs[r.index]->in;
        case NodeRef::Shader: return &o.shaders[r.index]->in;
        case NodeRef::Layout: return (size_t)r.index < o.nested.size() && o.nested[r.index].has_frame ? &o.nested[r.index] : nullptr;
        case NodeRef::Input: break;
    }
    auto it = inputs_.find(r.input_id);
    return it != inputs_.end() && it->second.has_frame ? &it->second : nullptr;
}

// The texture a shader or web node's draw reads for child `r` once the tick's frame-arena addresses are resolved: a layout
// node's composite from the texture table, any other node's own texture; the empty view when it has no pixels this tick
dev::Tex Renderer::packed_node_tex(Output &o, const NodeRef &r) {
    Input *in = node_input(o, r);
    if (!in) return dev::Tex();
    return r.kind == NodeRef::Layout ? plan_.tex[in->raw_tex].tex : in->tex;
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
            const WeightEntry *we;
            smr_status st = get_weights(kp, we);
            if (st != SMR_OK) return st;
            dev::ResampleJob j{};
            j.axis = kp.mapping.axis; j.perp_offset = kp.perp_offset; j.taps = we->taps;
            j.weights = we->weights; j.inv_wsum = we->inv; j.first = we->first;
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

// The composite layers of a W x H layout node: each child's texture (resampled where the layout scales it) and its masks
smr_status Renderer::plan_layers(std::vector<RenderLayout> &layouts, const std::vector<Input *> &child_in, int W, int H,
                                 std::vector<dev::LayerDev> &layers, std::vector<dev::MaskDev> &masks) {
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
    return SMR_OK;
}

// Layout node k of output `o` below its root (LayoutNode::render): its layouts are evaluated every tick (update_state and
// Tiles::last_layout advance as in the reference whether or not anything shows the node), then composited into an RGBA8
// frame-arena texture of the tick's resolution (no tile plan, no direct tiles), which its readers take as a child texture
smr_status Renderer::plan_layout_node(Output &o, size_t k, uint64_t pts) {
    Input &nn = o.nested[k];
    nn.has_frame = false;
    nn.node_tex = nn.raw_tex = -1;
    LayoutEval e = eval_layout(o, o.node.nested[k], pts);
    if (e.res.width == 0 || e.res.height == 0 || e.res.width > 16384 || e.res.height > 16384) return SMR_OK;
    if (e.layouts.size() > opts_.max_layouts_count) e.layouts.resize(opts_.max_layouts_count);
    const int W = (int)e.res.width, H = (int)e.res.height;
    std::vector<dev::LayerDev> layers;
    std::vector<dev::MaskDev> masks;
    if (smr_status st = plan_layers(e.layouts, e.child_in, W, H, layers, masks); st != SMR_OK) return st;
    nn.raw_tex = composite_texture(composite_rec(W, H, layers, masks));
    nn.tex = plan_.tex[nn.raw_tex].tex;
    nn.res = e.res;
    nn.has_frame = true;
    return SMR_OK;
}

// A composite of `layers` (and their `masks`) into a W x H target, which the caller sets
Renderer::CompositeRec Renderer::composite_rec(int W, int H, const std::vector<dev::LayerDev> &layers,
                                               const std::vector<dev::MaskDev> &masks) {
    CompositeRec pc;
    memset(&pc.job, 0, sizeof(pc.job));
    pc.job.width = W; pc.job.height = H; pc.job.mode = opts_.rendering_mode;
    pc.job.n_layers = (int)layers.size();
    pc.layers_off = param_put(layers.data(), sizeof(dev::LayerDev) * layers.size());
    pc.masks_off = param_put(masks.data(), sizeof(dev::MaskDev) * masks.size());
    return pc;
}

// Plans composite `pc` into an RGBA8 frame-arena texture of its size; returns that texture's index in the table
int Renderer::composite_texture(CompositeRec pc) {
    const int W = pc.job.width, H = pc.job.height;
    pc.out_frame_off = frame_alloc((size_t)W * H * 4);
    pc.job.out_format = -1;
    pc.job.out_pitch0 = W * 4;
    plan_.composites.push_back(pc);
    dev::Tex t;
    t.kind = dev::TEX_RGBA8; t.width = W; t.height = H; t.pitch0 = W * 4;
    return add_texture(t, false, pc.out_frame_off);
}

smr_status Renderer::plan_output(Output &o, smr_output_frame &of, uint64_t pts) {
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
    auto to_planes = [&](CompositeRec &pc) {   // the composite writes the output's planes (K10/K11 fused)
        pc.job.out_format = o.format;
        pc.job.out0 = dst[0]; pc.job.out1 = dst[1]; pc.job.out2 = dst[2];
        pc.job.out_pitch0 = pitch[0]; pc.job.out_pitch1 = pitch[1]; pc.job.out_pitch2 = pitch[2];
    };

    plan_node_textures(o, pts);
    if (o.node.root) {  // pass-through: the root texture IS the node texture
        Input *root_in = node_input(o, *o.node.root);
        if (!root_in) { push_fill(); return SMR_OK; }
        Input &in = *root_in;
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
            std::vector<dev::LayerDev> layers(1);
            bool skip;
            prepare_layer(l, (int)of.width, (int)of.height, in.raw_tex, (int)of.width, (int)of.height, layers[0], skip);
            if (skip) layers.clear();
            CompositeRec pc = composite_rec((int)of.width, (int)of.height, layers, {});
            to_planes(pc);
            plan_.composites.push_back(pc);
            return SMR_OK;
        }
        push_output_job(in.raw_tex);
        return SMR_OK;
    }

    LayoutEval e = eval_layout(o, o.node.root_layout, pts);
    if (e.res.width == 0 || e.res.height == 0 || e.res.width > 16384 || e.res.height > 16384) { push_fill(); return SMR_OK; }
    if (e.layouts.size() > opts_.max_layouts_count) e.layouts.resize(opts_.max_layouts_count);  // params.rs:176-182

    const int W = (int)e.res.width, H = (int)e.res.height;
    std::vector<dev::LayerDev> layers;
    std::vector<dev::MaskDev> masks;
    if (smr_status st = plan_layers(e.layouts, e.child_in, W, H, layers, masks); st != SMR_OK) return st;
    CompositeRec pc = composite_rec(W, H, layers, masks);

    bool same_size = (size_t)W == o.res.width && (size_t)H == o.res.height;
    bool fused_fmt = o.format == SMR_OUT_PLANAR_YUV420 || o.format == SMR_OUT_NV12;
    bool fusable = same_size && (o.format == SMR_OUT_RGBA8 || (fused_fmt && (W % 2 == 0) && (H % 2 == 0)));
    if (fusable) {
        to_planes(pc);
        if (fused_fmt) plan_tiles(o, pc, layers, W, H);
        plan_.composites.push_back(pc);
    } else {
        if (o.format == SMR_OUT_RGBA8) { set_error("RGBA output must match the root layout resolution"); return SMR_ERR_UNSUPPORTED; }
        push_output_job(composite_texture(pc));
    }
    return SMR_OK;
}

smr_status Renderer::render_begin(uint64_t pts, const smr_input_frame *in, uint32_t n_in, smr_output_frame *out,
                                  uint32_t n_out) {
    if ((n_in && !in) || (n_out && !out)) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    if (host_only_) { set_error("host-only handle (cuda_device = -1) cannot render: no CPU fallback"); return SMR_ERR_CUDA; }
    CUDA_OK(cudaSetDevice(opts_.cuda_device));
    if (smr_status st = begin_tick(); st != SMR_OK) return st;
    // any return from here (a status or an exception) before a launch is enqueued undoes what the tick planned for it: the
    // new weight-cache entries are dropped, the text and image nodes are left to the next tick
    struct TickGuard {
        Renderer &r;
        ~TickGuard() {
            if (!r.new_weight_keys_.empty()) r.rollback_weights();   // emptied once the k_weights launch is enqueued
            if (r.plan_.nodes_enqueued) return;
            for (TextNode *t : r.plan_.texts) t->rendered = false;
            for (ImageNode *n : r.plan_.images) n->held = n->held_before;
            for (auto &h : r.plan_.deint_history) h.first->hist = h.second;
        }
    } guard{*this};
    smr_status st = plan_tick(pts, in, n_in, out, n_out);
    if (st == SMR_OK) st = resolve_frame_arena();
    if (st == SMR_OK) plan_fused_launches();
    if (st == SMR_OK) st = pack_params();
    if (st == SMR_OK) st = launch_tick();
    if (st == SMR_OK) st = enqueue_readback(n_out);
    return st;
}

// A new tick: its slot, free for it, an empty plan and empty arenas
smr_status Renderer::begin_tick() {
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
    return SMR_OK;
}

// The tick's inputs and its plan, phase by phase; plan_.phases gets each phase's start and the end of the last
smr_status Renderer::plan_tick(uint64_t pts, const smr_input_frame *in, uint32_t n_in, smr_output_frame *out, uint32_t n_out) {
    smr_status st = select_inputs(pts, in, n_in, [&](Input &I, const smr_input_frame *f) {
        I.node_tex = I.raw_tex = -1;
        return f ? upload_input(I, *f) : SMR_OK;
    });
    if (st != SMR_OK) return st;
    // the outputs up to the first that is not registered: those before it are planned, as they always were, before the
    // tick fails on it
    std::vector<Output *> outs;
    int max_depth = 0;   // of the layout, shader and web nodes below the roots
    for (uint32_t i = 0; i < n_out; i++) {
        auto it = out[i].output_id ? outputs_.find(out[i].output_id) : outputs_.end();
        if (it == outputs_.end()) break;
        Output &o = it->second;
        outs.push_back(&o);
        for (const LayoutParams &lp : o.node.nested) max_depth = std::max(max_depth, lp.depth);
        for (const ShaderParams &sp : o.node.shaders) max_depth = std::max(max_depth, sp.depth);
        for (const WebParams &wp : o.node.webs) max_depth = std::max(max_depth, wp.depth);
    }
    auto mark = [&]() {
        plan_.phases.push_back({{plan_.stages[0].size(), plan_.stages[1].size(), plan_.stages[2].size()}, plan_.composites.size()});
    };
    for (int d = 1; d <= max_depth; d++) {   // the layout nodes below the roots, shallow first (a tick without any: no phase)
        mark();
        for (Output *o : outs) {
            for (size_t k = 0; k < o->node.nested.size(); k++) {
                if (o->node.nested[k].depth != d) continue;
                plan_node_textures(*o, pts);
                if ((st = plan_layout_node(*o, k, pts)) != SMR_OK) return st;
            }
        }
    }
    mark();   // the roots
    for (uint32_t i = 0; i < n_out; i++) {
        if (i == outs.size()) {
            if (!out[i].output_id) return SMR_ERR_INVALID_ARGUMENT;
            set_error(std::string("Output \"") + out[i].output_id + "\" does not exist, register it first");
            return SMR_ERR_OUTPUT_NOT_REGISTERED;
        }
        st = plan_output(*outs[i], out[i], pts);
        if (st != SMR_OK) return st;
    }
    mark();   // the end of the roots' phase
    return SMR_OK;
}

// Orders the tick's kernels after its inputs, sizes the frame arena and resolves the plan's frame-arena addresses
smr_status Renderer::resolve_frame_arena() {
    // everything already on the stream belongs to earlier ticks: a broadcast issued after this call may overwrite any
    // buffer those ticks read once this event has fired
    CUDA_OK(cudaEventRecord(tick_start_, stream_));
    tick_started_ = true;
    if (comm_pending_) {   // this tick's shared inputs arrive on the communication stream
        CUDA_OK(cudaStreamWaitEvent(stream_, comm_done_, 0));
        comm_pending_ = false;
    }
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
    return SMR_OK;
}

// The tick's fused resamples over a persistent grid, one launch per kernel variant; runs before the composites' tile lists
// are packed, as a job cut at an odd row gives its direct tiles back to its composite
void Renderer::plan_fused_launches() {
    for (size_t i = 0; i < plan_.fused.size(); i++) {
        const dev::FusedVariant &v = plan_.fused[i].key;
        if (std::any_of(plan_.fused.begin(), plan_.fused.begin() + i, [&](const FusedRec &f) { return f.key == v; })) continue;
        std::vector<int> idx, widths, heights, cols;
        dev::FusedShape shape{};
        for (size_t ji = i; ji < plan_.fused.size(); ji++) {
            const FusedRec &f = plan_.fused[ji];
            if (!(f.key == v)) continue;
            shape = dev::fused_shape(f.key, f.job);
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
        plan_.fused_launches.push_back({v, param_put(pieces.data(), sizeof(dev::FusedPiece) * pieces.size()),
                                        param_put(begin.data(), sizeof(int) * begin.size()), (int)begin.size() - 1});
    }
}

// Packs the parameter arena, turns its offsets into device pointers in the packed jobs and ships it in one copy
smr_status Renderer::pack_params() {
    const size_t tex_off = param_put_all(plan_.tex, &TexRec::tex);
    for (int s = 0; s < 3; s++) plan_.stage_off[s] = param_put_all(plan_.stages[s], &StageRec::job);
    plan_.weights_off = param_put(plan_.weight_jobs.data(), sizeof(dev::WeightJob) * plan_.weight_jobs.size());
    const size_t tm_off = param_put(plan_.tmaps.data(), sizeof(CUtensorMap) * plan_.tmaps.size());
    for (CompositeRec &pc : plan_.composites) {   // direct-tile maps (one byte per tile: the owner's id) and tile lists
        if (pc.direct_off != SIZE_MAX) {
            bool any = false;
            for (size_t t = 0; t < pc.direct_owner.size(); t++) {
                param_host_[pc.direct_off + t] = pc.direct_owner[t] >= 0 ? (uint8_t)(pc.direct_owner[t] + 1) : 0;
                any = any || pc.direct_owner[t] >= 0;
                plan_.direct_tiles += pc.direct_owner[t] >= 0 ? 1 : 0;
            }
            if (!any) pc.direct_off = SIZE_MAX;
        }
        if (pc.use_list) {
            pc.list_off = param_put(pc.list.data(), sizeof(uint32_t) * pc.list.size());
            pc.job.n_tiles = (int)pc.list.size();
        }
    }
    plan_.fused_off = param_put_all(plan_.fused, &FusedRec::job);
    plan_.composites_off = param_put_all(plan_.composites, &CompositeRec::job);   // read by k_composite_multi
    if (!plan_.deint.empty()) {   // the deinterlace jobs and the prefix table of their blocks
        plan_.deint_off = param_put(plan_.deint.data(), sizeof(dev::DeinterlaceJob) * plan_.deint.size());
        std::vector<int32_t> begin(plan_.deint.size() + 1, 0);
        for (size_t i = 0; i < plan_.deint.size(); i++)
            begin[i + 1] = begin[i] + dev::deinterlace_tiles(plan_.deint[i].row_bytes, plan_.deint[i].rows);
        plan_.deint_tiles = begin.back();
        plan_.deint_begin_off = param_put(begin.data(), sizeof(int32_t) * begin.size());
    }
    for (WebNode *n : plan_.webs) {   // the children's textures, frame-arena addresses resolved
        for (size_t i = 0; i < n->planes.size(); i++)
            if (n->plane_child[i] >= 0) n->planes[i].tex = packed_node_tex(*n->owner, n->params.children[n->plane_child[i]]);
        n->planes_off = param_put(n->planes.data(), sizeof(dev::WebPlane) * n->planes.size());
    }
    for (ShaderNode *n : plan_.shaders) {   // likewise
        n->tex_off = param_alloc(sizeof(dev::Tex) * n->params.children.size());
        for (size_t k = 0; k < n->params.children.size(); k++)
            reinterpret_cast<dev::Tex *>(param_host_.data() + n->tex_off)[k] = packed_node_tex(*n->owner, n->params.children[k]);
        const std::vector<uint8_t> &b = n->params.param_bytes;
        n->params_off = b.empty() ? SIZE_MAX : param_put(b.data(), b.size());
    }
    // the node-texture launches, in the order launch_tick enqueues those of one phase
    auto all = [](const NodeTexture *) { return true; };
    add_node_launch(dev::node_kernel(dev::NODE_TEXT), "k_text", SMR_KERNEL_CONVERT, -1, plan_.texts, &TextNode::job, all);
    add_node_launch(dev::node_kernel(dev::NODE_IMAGE), "k_image", SMR_KERNEL_IMAGE, -1, plan_.images, &ImageNode::job, all);
    for (int d = 1; d + 1 < (int)plan_.phases.size(); d++) {   // each depth below the roots
        for (size_t i = 0; i < plan_.shaders.size(); i++) {   // one launch per shader, in the order of its first node
            auto same = [&](const ShaderNode *n) { return n->params.depth == d && n->params.shader == plan_.shaders[i]->params.shader; };
            if (same(plan_.shaders[i]) && std::none_of(plan_.shaders.begin(), plan_.shaders.begin() + i, same))
                add_node_launch(plan_.shaders[i]->params.shader->kernel, "smr_shader_main", SMR_KERNEL_SHADER, d - 1, plan_.shaders,
                                &ShaderNode::job, same);
        }
        add_node_launch(dev::node_kernel(dev::NODE_WEB), "k_web", SMR_KERNEL_WEB, d == 1 ? -1 : d - 1, plan_.webs, &WebNode::job,
                        [&](const WebNode *n) { return n->params.depth == d; });
    }
    // the arena is sized: its offsets become device pointers in the packed jobs
    CUDA_OK(param_pinned_[slot_].ensure(param_used_));
    CUDA_OK(param_dev_[slot_].ensure(param_used_));
    uint8_t *pd = param_dev_[slot_].p;
    auto dev_ptr = [&](size_t off) -> uint8_t * { return off != SIZE_MAX ? pd + off : nullptr; };
    for (WebNode *n : plan_.webs)   // the nodes' own arena data in their packed jobs
        reinterpret_cast<dev::WebJob *>(param_host_.data() + n->job_off)->planes = (const dev::WebPlane *)(pd + n->planes_off);
    for (ShaderNode *n : plan_.shaders) {
        dev::ShaderJob *j = reinterpret_cast<dev::ShaderJob *>(param_host_.data() + n->job_off);
        j->tex = (const dev::Tex *)(pd + n->tex_off);
        j->params = dev_ptr(n->params_off);
    }
    dev::FusedJob *fj = reinterpret_cast<dev::FusedJob *>(param_host_.data() + plan_.fused_off);
    for (size_t i = 0; i < plan_.fused.size(); i++) {
        const FusedRec &f = plan_.fused[i];
        if (f.tmap_idx >= 0) {
            const uint8_t *m = pd + tm_off + sizeof(CUtensorMap) * (size_t)f.tmap_idx;
            fj[i].tm0 = m; fj[i].tm1 = m + sizeof(CUtensorMap); fj[i].tm2 = m + 2 * sizeof(CUtensorMap);
        }
        fj[i].direct_map = dev_ptr(f.direct_off);
    }
    dev::CompositeJob *cj = reinterpret_cast<dev::CompositeJob *>(param_host_.data() + plan_.composites_off);
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
    return SMR_OK;
}

// Enqueues the tick's kernels on stream_, in this order: k_deinterlace (it rewrites inputs before anything reads them); the
// text nodes, the image nodes and the web nodes of depth 1 (they
// read inputs, text and image nodes only); k_convert, k_weights, the fused resamples; per phase p, its generic resample
// passes, its composite (the last phase's: ONE launch for every output) and then, after its layout nodes of depth p + 1, the
// shader nodes of that depth (one launch per shader) and its web nodes; the output jobs; the fills.
smr_status Renderer::launch_tick() {
    const uint8_t *pd = param_dev_[slot_].p, *ph = param_host_.data();
    auto launched = [&](int n, int kernel_class) {   // n: the kernels a launcher enqueued, -1: it failed and the tick ends
        if (n < 0) {
            set_error(dev::last_launch_error());
            cudaStreamSynchronize(stream_);
            return false;
        }
        plan_.launches += (uint64_t)n;
        prof_mark(kernel_class);
        return true;
    };
    auto launch_nodes = [&](int phase) {   // the node launches after `phase`, in list order
        for (const NodeLaunch &l : plan_.node_launches)
            if (l.phase == phase && !launched(dev::launch_tile_jobs(l.kernel, pd + l.jobs_off, (const int32_t *)(pd + l.begin_off),
                                                                    l.n_jobs, l.n_tiles, l.name, stream_), l.prof_class)) return false;
        return true;
    };
    prof_mark(-1);
    if (!plan_.deint.empty() &&
        !launched(dev::launch_deinterlace((const dev::DeinterlaceJob *)(pd + plan_.deint_off), (const int32_t *)(pd + plan_.deint_begin_off),
                                          (int)plan_.deint.size(), plan_.deint_tiles, stream_), SMR_KERNEL_DEINTERLACE)) return SMR_ERR_CUDA;
    if (!launch_nodes(-1)) return SMR_ERR_CUDA;
    plan_.nodes_enqueued = true;
    for (auto &cv : plan_.convert_jobs) {
        const dev::Tex &src = plan_.tex[cv.first].tex;
        if (!launched(dev::launch_convert_to_rgba(src, frame_dev_.p + cv.second, src.width * 4, stream_), SMR_KERNEL_CONVERT))
            return SMR_ERR_CUDA;
    }
    if (!plan_.weight_jobs.empty() &&
        !launched(dev::launch_weights((const dev::WeightJob *)(pd + plan_.weights_off), plan_.weight_jobs.data(),
                                      (int)plan_.weight_jobs.size(), stream_), SMR_KERNEL_WEIGHTS)) return SMR_ERR_CUDA;
    new_weight_keys_.clear();   // the tables are being computed on the stream: the cache entries are good
    for (const FusedLaunch &fl : plan_.fused_launches)
        if (!launched(dev::launch_resample_fused(fl.key, (const dev::FusedJob *)(pd + plan_.fused_off), (const dev::FusedPiece *)(pd + fl.pieces_off),
                                                 (const int *)(pd + fl.begin_off), fl.nblocks, stream_), SMR_KERNEL_RESAMPLE_FUSED))
            return SMR_ERR_CUDA;
    for (size_t p = 0; p + 1 < plan_.phases.size(); p++) {
        const TickPlan::Phase &b = plan_.phases[p], &e = plan_.phases[p + 1];
        for (int s = 0; s < 3; s++) {
            const size_t off = plan_.stage_off[s] + sizeof(dev::ResampleJob) * b.stages[s];
            const int count = (int)(e.stages[s] - b.stages[s]);
            if (count && !launched(dev::launch_resample((const dev::ResampleJob *)(pd + off), (const dev::ResampleJob *)(ph + off), count,
                                                        stream_), SMR_KERNEL_RESAMPLE_BOX + s)) return SMR_ERR_CUDA;
        }
        if (e.composites > b.composites &&
            !launched(dev::launch_composite((const dev::CompositeJob *)(pd + plan_.composites_off) + b.composites,
                                            (const dev::CompositeJob *)(ph + plan_.composites_off) + b.composites,
                                            (const dev::LayerDev *)(ph + plan_.composites[b.composites].layers_off),
                                            (int)(e.composites - b.composites), stream_), SMR_KERNEL_COMPOSITE)) return SMR_ERR_CUDA;
        if (!launch_nodes((int)p)) return SMR_ERR_CUDA;
    }
    for (OutputRec &o : plan_.outputs)
        if (!launched(dev::launch_output(o.job, stream_), SMR_KERNEL_OUTPUT)) return SMR_ERR_CUDA;
    for (Fill &f : plan_.fills)
        if (!launched(dev::launch_fill_yuv(f.p[0], f.p[1], f.p[2], f.pitch[0], f.pitch[1], f.pitch[2], f.w, f.h, f.fmt,
                                           f.yuv[0], f.yuv[1], f.yuv[2], stream_), SMR_KERNEL_FILL)) return SMR_ERR_CUDA;
    return SMR_OK;
}

// The read-back of the host outputs, on its own stream: the staging planes are per slot, so the next tick's kernels need
// not wait for it
smr_status Renderer::enqueue_readback(uint32_t n_out) {
    cudaStream_t done_on = stream_;   // the stream the tick's last operation goes to
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
    stats_.kernel_launches += plan_.launches;
    stats_.last_render_kernel_launches = plan_.launches;
    stats_.last_render_direct_tiles = plan_.direct_tiles;
    stats_.frames_rendered += n_out;
    CUDA_OK(cudaEventRecord(tick_done_[slot_], done_on));
    inflight_.push_back(slot_);
    return SMR_OK;
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
        const smr_fused_variant_info v = public_variant(f.key);
        o.kernel = v.kernel; o.ratio = v.ratio; o.window = v.window; o.box = v.box; o.src_class = v.src_class;
        o.full_range = j.src.full_range;
        o.v_same = j.v_same;
        o.strip_cols = dev::fused_shape(f.key, j).strip_cols;
        o.src_width = (uint32_t)j.src.width; o.src_height = (uint32_t)j.src.height;
        o.dst_width = (uint32_t)j.dst_w; o.dst_height = (uint32_t)j.dst_h;
        o.taps_h = j.taps_h; o.taps_v = j.taps_v;
        o.direct = f.direct_off != SIZE_MAX ? 1 : 0;
        o.matrix = public_matrix(j.src);
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
                o.tex_matrix = public_matrix(t);
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
    reap_shaders(false);
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
        Event e;
        if (make(e, cudaEventCreateWithFlags, cudaEventDefault) != cudaSuccess) return;
        prof_events_.push_back(std::move(e));
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
    void *comm = nullptr;
    int rc = g_nccl.CommInitRank(&comm, nranks, nid, rank);
    if (rc != 0) { set_error(std::string("ncclCommInitRank: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error")); return SMR_ERR_CUDA; }
    if (nccl_comm_) { cudaStreamSynchronize(comm_stream_); cudaStreamSynchronize(stream_); }   // as comm_destroy, for the one replaced
    nccl_comm_.reset(comm);
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
        int32_t *word = nullptr;
        CUDA_OK(cudaMalloc(&word, 256));
        barrier_word_.reset(word);
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
    Owned<void *, cudaFree> owned(p);
    cudaIpcMemHandle_t h;
    if (cudaIpcGetMemHandle(&h, p) != cudaSuccess) { cudaGetLastError(); set_error("cudaIpcGetMemHandle failed"); return SMR_ERR_CUDA; }
    memcpy(handle, &h, 64);
    peer_own_.push_back(std::move(owned));
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
    peer_opened_.emplace_back(p);
    *dev_ptr = p;
    return SMR_OK;
}

smr_status Renderer::peer_pool_close(void *dev_ptr) { return peer_pool_release(peer_opened_, dev_ptr); }
smr_status Renderer::peer_pool_free(void *dev_ptr) { return peer_pool_release(peer_own_, dev_ptr); }

// Closes or frees a peer pool once no stream reads it
template <class Pools> smr_status Renderer::peer_pool_release(Pools &pools, void *dev_ptr) {
    std::lock_guard<std::mutex> g(mu_);
    auto it = std::find_if(pools.begin(), pools.end(), [dev_ptr](const auto &p) { return (void *)p == dev_ptr; });
    if (it == pools.end()) return SMR_ERR_INVALID_ARGUMENT;
    CUDA_OK(cudaSetDevice(opts_.cuda_device));
    cudaStreamSynchronize(stream_);
    if (comm_stream_) cudaStreamSynchronize(comm_stream_);
    tmap_cache_.clear();   // descriptors of planes inside the pool
    pools.erase(it);
    return SMR_OK;
}

smr_status Renderer::comm_destroy() {
    std::lock_guard<std::mutex> g(mu_);
    if (nccl_comm_) {
        cudaSetDevice(opts_.cuda_device);
        cudaStreamSynchronize(comm_stream_);   // the collectives run here
        cudaStreamSynchronize(stream_);
        nccl_comm_.reset();
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

smr_status Renderer::debug_image_nodes(const char *output_id, uint64_t pts, smr_image_node_info *out, uint32_t cap, uint32_t *n) {
    if (!output_id || !n) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    auto it = outputs_.find(output_id);
    if (it == outputs_.end()) { set_error("output not registered"); return SMR_ERR_OUTPUT_NOT_REGISTERED; }
    const std::vector<ImageParams> &images = it->second.node.images;
    *n = (uint32_t)images.size();
    if (!out) return SMR_OK;
    if (cap < *n) return SMR_ERR_BUFFER_TOO_SMALL;
    for (uint32_t i = 0; i < *n; i++) {
        const ImageParams &p = images[i];
        out[i] = {(uint32_t)p.resolution.width, (uint32_t)p.resolution.height, p.start_pts,
                  p.asset->animated() ? (uint32_t)p.asset->frame_at(pts, p.start_pts) : 0u};
    }
    return SMR_OK;
}

// Layout node `node` of an output: 0 is the root when the root is a layout, the nodes below it follow in DFS order.  No
// `node` (smr_debug_layouts): the root, which has no layouts at 0 x 0 when it is not a layout.
smr_status Renderer::debug_node_layouts(const char *output_id, std::optional<uint32_t> node, uint64_t pts, smr_render_layout *out,
                                        uint32_t cap, uint32_t *n, uint32_t *rw, uint32_t *rh) {
    if (!output_id || !n) return SMR_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> g(mu_);
    auto it = outputs_.find(output_id);
    if (it == outputs_.end()) { set_error("output not registered"); return SMR_ERR_OUTPUT_NOT_REGISTERED; }
    Output &o = it->second;
    const bool root_layout = !o.node.root;
    const LayoutParams *lp = nullptr;
    if (root_layout && node.value_or(0) == 0) {
        lp = &o.node.root_layout;
    } else if (node) {
        const size_t k = *node - (root_layout ? 1 : 0);
        if (k >= o.node.nested.size()) { set_error("no such layout node"); return SMR_ERR_INVALID_ARGUMENT; }
        lp = &o.node.nested[k];
    }
    if (!lp) {
        *n = 0;
        if (rw) *rw = 0;
        if (rh) *rh = 0;
        return SMR_OK;
    }
    LayoutParams copy = *lp;   // inspection does not advance the node's state
    const LayoutEval e = eval_layout(o, copy, pts);
    if (rw) *rw = (uint32_t)e.res.width;
    if (rh) *rh = (uint32_t)e.res.height;
    return layouts_to_c(e.layouts, out, cap, n);
}

smr_status Renderer::layouts_to_c(const std::vector<RenderLayout> &layouts, smr_render_layout *out, uint32_t cap, uint32_t *n) {
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
smr_status smr_set_input_deinterlace(smr_renderer *r, const char *id, const smr_deinterlace *cfg) {
    SMR_GUARD(r->impl.set_input_deinterlace(id, cfg))
}
smr_status smr_set_input_color(smr_renderer *r, const char *id, const smr_input_color *c) {
    SMR_GUARD(r->impl.set_input_color(id, c))
}
smr_status smr_debug_input_planes(smr_renderer *r, const char *id, void *const planes[3], const uint32_t pitch[3], int32_t mem_kind) {
    SMR_GUARD(r->impl.debug_input_planes(id, planes, pitch, mem_kind))
}
smr_status smr_register_image(smr_renderer *r, const char *id, const smr_image_spec *spec) { SMR_GUARD(r->impl.register_image(id, spec)) }
smr_status smr_register_svg_image(smr_renderer *r, const char *id, const smr_svg_spec *spec) { SMR_GUARD(r->impl.register_svg_image(id, spec)) }
smr_status smr_unregister_image(smr_renderer *r, const char *id) { SMR_GUARD(r->impl.unregister_image(id)) }
smr_status smr_register_web_renderer(smr_renderer *r, const char *id, const smr_web_renderer_spec *spec) {
    SMR_GUARD(r->impl.register_web_renderer(id, spec))
}
smr_status smr_unregister_web_renderer(smr_renderer *r, const char *id) { SMR_GUARD(r->impl.unregister_web_renderer(id)) }
smr_status smr_web_set_frame(smr_renderer *r, const char *id, const smr_web_frame *frame) { SMR_GUARD(r->impl.web_set_frame(id, frame)) }
smr_status smr_web_set_child_rects(smr_renderer *r, const char *id, const smr_web_rect *rects, uint32_t n) {
    SMR_GUARD(r->impl.web_set_child_rects(id, rects, n))
}
smr_status smr_register_shader(smr_renderer *r, const char *id, const smr_shader_spec *spec) { SMR_GUARD(r->impl.register_shader(id, spec)) }
smr_status smr_register_wgsl_shader(smr_renderer *r, const char *id, const char *wgsl_source) {
    SMR_GUARD(r->impl.register_wgsl_shader(id, wgsl_source))
}
smr_status smr_unregister_shader(smr_renderer *r, const char *id) { SMR_GUARD(r->impl.unregister_shader(id)) }
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
smr_status smr_debug_transcode_taps(uint32_t in_len, uint32_t out_len, int32_t *nearest, int32_t *bilinear, float *frac,
                                    int32_t *center, float *lanczos) {
    if (!nearest || !bilinear || !frac || !center || !lanczos || in_len == 0 || out_len == 0 || in_len > 16384 || out_len > 16384)
        return SMR_ERR_INVALID_ARGUMENT;
    std::vector<smr::dev::TranscodeTap> taps;
    smr::transcode_axis(in_len, out_len, taps);
    for (uint32_t k = 0; k < out_len; k++) {
        const smr::dev::TranscodeTap &t = taps[k];
        nearest[k] = t.nearest;
        bilinear[2 * k] = t.lo; bilinear[2 * k + 1] = t.hi;
        frac[k] = t.frac;
        center[k] = t.center;
        for (int d = 0; d < 6; d++) lanczos[6 * k + d] = t.w[d];
    }
    return SMR_OK;
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
smr_status smr_transcode_resize(smr_renderer *r, const smr_input_frame *src, const smr_rendition *out, uint32_t n) {
    SMR_GUARD(r->impl.transcode_resize(src, out, n))
}
smr_status smr_video_nv12_to_rgba(smr_renderer *r, smr_video_color converter, const smr_input_frame *src, smr_video_color frame,
                                  uint32_t out_width, uint32_t out_height, void *rgba, uint32_t pitch, int32_t mem_kind) {
    SMR_GUARD(r->impl.video_nv12_to_rgba(converter, src, frame, out_width, out_height, rgba, pitch, mem_kind))
}
smr_status smr_video_rgba_to_nv12(smr_renderer *r, smr_video_color converter, const smr_input_frame *src, uint32_t out_width,
                                  uint32_t out_height, void *const planes[2], const uint32_t pitch[2], int32_t mem_kind) {
    SMR_GUARD(r->impl.video_rgba_to_nv12(converter, src, out_width, out_height, planes, pitch, mem_kind))
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
                             uint32_t *n, uint32_t *rw, uint32_t *rh) { SMR_GUARD(r->impl.debug_node_layouts(output_id, std::nullopt, pts, out, cap, n, rw, rh)) }
smr_status smr_debug_image_nodes(smr_renderer *r, const char *output_id, uint64_t pts, smr_image_node_info *out, uint32_t cap,
                                 uint32_t *n) { SMR_GUARD(r->impl.debug_image_nodes(output_id, pts, out, cap, n)) }
smr_status smr_debug_set_inputs(smr_renderer *r, uint64_t pts, const smr_input_frame *in, uint32_t n_in) { SMR_GUARD(r->impl.debug_set_inputs(pts, in, n_in)) }
smr_status smr_debug_fused_jobs(smr_renderer *r, smr_fused_job_info *out, uint32_t cap, uint32_t *n) { SMR_GUARD(r->impl.debug_fused_jobs(out, cap, n)) }
smr_status smr_debug_fused_variants(smr_fused_variant_info *out, uint32_t cap, uint32_t *n) {
    if (!n) return SMR_ERR_INVALID_ARGUMENT;
    std::vector<smr::dev::FusedVariant> v(smr::dev::fused_variants(nullptr, 0));
    smr::dev::fused_variants(v.data(), (int)v.size());
    *n = (uint32_t)v.size();
    if (!out) return SMR_OK;
    if (cap < v.size()) return SMR_ERR_BUFFER_TOO_SMALL;
    for (size_t i = 0; i < v.size(); i++) out[i] = smr::public_variant(v[i]);
    return SMR_OK;
}
smr_status smr_debug_composite_layers(smr_renderer *r, smr_composite_layer_info *out, uint32_t cap, uint32_t *n) {
    SMR_GUARD(r->impl.debug_composite_layers(out, cap, n))
}
smr_status smr_debug_node_layouts(smr_renderer *r, const char *output_id, uint32_t node, uint64_t pts_ns, smr_render_layout *out,
                                  uint32_t capacity, uint32_t *n_out, uint32_t *root_width, uint32_t *root_height) {
    SMR_GUARD(r->impl.debug_node_layouts(output_id, node, pts_ns, out, capacity, n_out, root_width, root_height))
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
