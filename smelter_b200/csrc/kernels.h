// kernels.h -- device-side job descriptors + launchers of the sm_90a compositor kernels.
// Host code (renderer.cpp, g++) and kernels.cu (nvcc) share this header; it is plain C++.
#pragma once

#include <cstddef>
#include <cstdint>

namespace smr {
namespace dev {

// A texture a kernel can read.  Everything the reference keeps in wgpu textures lives in plain
// pitched device buffers: input planes as uploaded, RGBA8 node textures, f16 resampler scratch.
enum TexKind : int32_t {
    TEX_NONE = 0,
    TEX_RGBA8 = 1,   // premultiplied RGBA8; `srgb` says whether fetches decode (srgb view) or not
    TEX_YUV420 = 2,  // planes y,u,v (K1 fused into the consumer)
    TEX_NV12 = 3,    // planes y,uv  (K2 fused into the consumer)
    TEX_F16 = 4,     // Rgba16Float scratch
    TEX_BGRA = 5,
    TEX_ARGB = 6,
    TEX_YUV422 = 7,  // planar, chroma (w/2) x h
    TEX_YUV444 = 8,  // planar, chroma w x h
    TEX_UYVY = 9,    // interleaved 4:2:2, one plane of (w/2) x h texels {U,Y0,V,Y1} (K3)
    TEX_YUYV = 10,   // ... {Y0,U,Y1,V}
};
// output formats follow smr_output_format: 0 = planar 4:2:0, 1 = planar 4:2:2, 2 = planar 4:4:4, 3 = RGBA8, 4 = NV12.
// Size of one chroma plane (texture/planar_yuv.rs:64-83)
inline
#ifdef __CUDACC__
__host__ __device__
#endif
void chroma_dims(int out_format, int w, int h, int &cw, int &ch) {
    cw = out_format == 2 ? w : w / 2;
    ch = (out_format == 1 || out_format == 2) ? h : h / 2;
}

struct Tex {
    int32_t kind = TEX_NONE;
    int32_t width = 0, height = 0;
    int32_t full_range = 0;
    const uint8_t *p0 = nullptr, *p1 = nullptr, *p2 = nullptr;
    int32_t pitch0 = 0, pitch1 = 0, pitch2 = 0;  // bytes per row
};

struct MaskDev {
    float radius[4];
    float top, left, width, height;
    float edge, corner;              // its interior (interior.h); edge = +inf: none
};

// One flattened RenderLayout, prepared on the host for the composite kernel
// (uniform blocks of layout/params.rs:199-317 + the vertex stage of apply_layouts.wgsl:174-243).
struct alignas(16) LayerDev {
    int32_t type;       // 0 texture, 1 color, 2 box shadow
    int32_t rotated;
    float left, top, width, height;  // the quad (box shadow: grown by blur_radius)
    float content_w, content_h;      // size passed to roundedRectSDF
    float cx, cy, cs, sn;            // quad centre (fb coords), cos/sin of rotation
    int32_t px0, px1, py0, py1;      // unrotated: exactly covered pixels [px0,px1)x[py0,py1); rotated: bbox
    long long vx[4], vy[4];          // rotated: vertices snapped to 1/256 px, clockwise on screen
    float border_radius[4];
    float color[4];                  // premultiplied shader colour (wgpu/utils.rs:51-71)
    float border_color[4];
    float border_width, blur_radius;
    int32_t tex;                     // index into the texture table; -1 = empty 1x1 texture
    float crop_sx, crop_ox, crop_sy, crop_oy;  // crop_w/dim, crop_left/dim, crop_h/dim, crop_top/dim
    int32_t mask_begin, mask_count;
    // host-proved fast region: for pixels in [ix0,ix1)x[iy0,iy1) the rounded-rect / border / mask factors are
    // all exactly 1 (>= 2 px inside every edge and radius), so the fragment is the bare colour or sample
    int32_t ix0, ix1, iy0, iy1;   // the full-height bar: core x range, y up to the straight edges
    int32_t jx0, jx1, jy0, jy1;   // the full-width bar (the two bars form a plus that leaves out the corner squares)
    int32_t fast;                    // FAST_* bits
    int32_t tx_off, ty_off;          // FAST_IDENT: texel = (px + tx_off, py + ty_off)
    uint32_t const_bytes;            // FAST_CONST: bytes an opaque colour leaves in the target (RGBA little endian)
    float int_edge, int_corner;      // the layer rect's interior (interior.h); int_edge = +inf: none
};
// FAST_LUT: translucent bare colour -- inside the bars the blend is a per-channel function of the target byte
// FAST_OPAQUE: inside the bars the layer REPLACES the target bytes (opaque constant, or 1:1 texels of a texture
// whose alpha is 255 everywhere) -- earlier layers cannot show through there
// FAST_SAMPLE: axis-aligned opaque RGBA8 child that is NOT 1:1 -- inside the bars each pixel is the filtered,
// re-encoded sample alone (source alpha exactly 1)
// FAST_HALF (with FAST_SAMPLE): CpuOptimized, planar 4:2:0 / NV12 child shown at exactly half its size on whole pixels
// -- every output pixel is the weight-1/2 bilinear tap of one aligned 2x2 texel quad: texel = (2 (px + tx_off), 2 (py + ty_off))
enum : int32_t { FAST_IDENT = 1, FAST_CONST = 2, FAST_LUT = 4, FAST_OPAQUE = 8, FAST_SAMPLE = 16, FAST_HALF = 32 };

// field order matters for speed: k_composite_multi's instruction schedule follows the offsets of its shared copy of the job
struct CompositeJob {
    int32_t width, height;           // render target (root node texture) size
    int32_t mode;                    // 0 GpuOptimized (sRGB target, linear blend), 1 CpuOptimized
    int32_t n_layers;
    const LayerDev *layers;          // device copy
    // with direct tiles in the tick the launch covers only the tiles that are left: block b works on tile
    // (tile_list[b] & 0xffff, tile_list[b] >> 16), row-major order; nullptr: block (x, y) = tile (x, y)
    const uint32_t *tile_list;
    const MaskDev *masks;
    const Tex *textures;
    // outputs: RGBA8 target and/or fused YUV planes (K10/K11)
    int32_t out_format;              // smr_output_format, or -1: RGBA8 node texture only
    uint8_t *out0, *out1, *out2;
    int32_t out_pitch0, out_pitch1, out_pitch2;
    // direct tiles (fused K10/K11 outputs only): direct_map[ty * map_w + tx] != 0 (the owner's FusedJob.direct_id) says that tile (128 x 16 pixels) lies
    // wholly inside the exact 1:1 interior of ONE opaque resampled child with nothing painted over it -- the fused
    // resample kernel has already written its Y / chroma bytes (FusedJob.direct_map), the composite skips the tile
    const uint8_t *direct_map;
    int32_t map_w;
    int32_t n_tiles;                 // entries of tile_list
};
constexpr int kDirectTileW = 128, kDirectTileH = 16;   // = the composite's block tile (CB_X * CT_W x CB_Y * CT_H)
// launch_composite runs k_composite_p (job and layers in the parameter block) for one job of at most this many layers,
// k_composite_multi otherwise
constexpr int kCompositeParamLayers = 96;

// Most source texels one box-pass texel averages: a crop inside a 16384 x 16384 source shrunk to one pixel needs
// 2^12 x 2^12.  Planning refuses a layout that would need more (the box loop's trip count, which must fit 32 bits).
constexpr uint64_t kMaxBoxTexels = 1ull << 24;

// one Lanczos pass (resample.wgsl) or box pass (downsample.wgsl)
struct ResampleJob {
    Tex src;                // TEX_RGBA8 (decoded through the srgb view), TEX_F16, or a YUV kind (fused K1/K2)
    int32_t axis;           // 0 horizontal, 1 vertical
    int32_t perp_offset;
    int32_t taps;
    int32_t dst_w, dst_h;
    int32_t dst_f16;        // 1: Rgba16Float target, 0: sRGB8 target
    uint8_t *dst;
    int32_t dst_pitch;      // bytes
    const float *weights;   // [n_out][taps]
    const float *inv_wsum;  // [n_out]
    const int32_t *first;   // [n_out]
    int32_t box_fx, box_fy; // box pass when box_fx*box_fy > 1 (then weights unused); the host keeps the product <= kMaxBoxTexels
};

// K1/K2 + both Lanczos passes fused (YUV source, horizontal pass first): see k_resample_fused
struct FusedJob {
    Tex src;                // TEX_YUV420 / TEX_NV12, even width and height
    int32_t dst_w, dst_h;
    uint8_t *dst;           // sRGB8 RGBA8
    int32_t dst_pitch;
    int32_t taps_h, taps_v;
    const float *w_h, *inv_h;
    const int32_t *first_h;
    const float *w_v, *inv_v;
    const int32_t *first_v;
    // TMA kernels: device copies of the CUtensorMap of each source plane (luma; NV12 chroma as u16 texels, or U; V)
    const void *tm0, *tm1, *tm2;
    int32_t v_same;         // TMA kernels: the vertical mapping is the same integer ratio with zero offset (weights = int_weight<S>)
    int32_t strip_cols;     // any-ratio TMA kernel: output columns per strip of THIS job (<= 64, even)
    const uint8_t *lane_perm;   // any-ratio TMA kernel: [strip][32] which pair of the strip's columns each lane owns (nullptr: lane l owns pair l)
    // integer-ratio TMA kernel with v_same: K10 / K11 straight out of the vertical pass.  Where the child is shown 1:1, opaque and
    // uncovered (the composite's direct tiles, CompositeJob.direct_map), a resampled pixel IS the output frame's pixel:
    // its Y and the chroma of its 2 x 2 block are written here, from the registers that hold the encoded bytes, and
    // the composite never reads them back.  (fx, fy): frame position of dst (0, 0), both even; dst_w, dst_h even.
    const uint8_t *direct_map;  // nullptr: no direct output for this job; else tile (tx, ty) is this job's iff the byte == direct_id
    int32_t direct_id;          // 1 .. 255 (children may overlap in the frame: a tile belongs to the topmost one only)
    int32_t map_w;
    int32_t fx, fy;
    int32_t out_format;         // 0 planar 4:2:0 (out0 / out1 / out2), 4 NV12 (out0 / out1)
    uint8_t *out0, *out1, *out2;
    int32_t out_pitch0, out_pitch1, out_pitch2;
};
// a contiguous run of output rows of one 64-column strip of one job; each block of the persistent grid gets an
// equal share of the launch's rows as a short list of pieces (renderer.cpp: partition_fused)
struct FusedPiece {
    int32_t job, strip, oy_begin, oy_end;
};
// LDG-staged kernel: output columns per strip, warps per block, and the taps per axis the host admits to any fused kernel
// (kernels.cu asserts that the LDG kernel's row and ring hold every ratio <= 4 within them)
constexpr int kFusedStripCols = 64, kFusedWarps = 8, kFusedMaxTaps = 25;
// TMA-staged kernels: output columns per strip, ring rows (>= taps_v + ceil(7 * vertical scale)), box sizes of the
// tensor maps the host encodes (bytes x rows; NV12 chroma in u16 texels)
constexpr int kTmaStripCols4 = 58, kTmaStripCols2 = 122, kTmaRing4 = 54, kTmaRing2 = 28;
// luma and NV12 chroma are addressed in 2-byte elements (a box may be at most 256 elements wide), planar chroma in bytes
constexpr int kTmaLumaBoxW = 136, kTmaLumaBoxH = 32, kTmaNv12BoxW = 144, kTmaPlanarBoxW = 160, kTmaChromaBoxH = 18;
constexpr int kTma0Groups = 2, kTma0MaxSpan = 256, kTma0MaxTaps = 25;
constexpr int kTma0Window[4] = {20, 25, 29, 33};

// Which kernel resamples a FusedJob (host side only; every job of one launch has the same kernel, source class and
// launch range)
struct FusedKernel {
    enum Kind : int32_t {
        LDG,      // k_resample_fused_int: LDG-staged, weights from smem (ratio 0) or from int_weights.h (integer ratio 2 / 3 / 4)
        TMA_INT,  // k_resample_tma3 (resample_tma3.cuh): integer ratio 2 / 4, TMA-staged, weights from int_weights.h
        TMA_ANY,  // k_resample_tma0 (resample_tma0.cuh): any ratio <= 4, TMA-staged, a tap loop of kTma0Window[window] slots;
                  // with `box` on a source box-reduced 2:1
    } kind = LDG;
    int32_t ratio = 0, window = 0, box = 0;
    bool operator==(const FusedKernel &o) const { return kind == o.kind && ratio == o.ratio && window == o.window && box == o.box; }
};
// What a launch of a fused kernel needs to know: output columns per strip of job `j`, blocks (eight-warp groups) per SM
// of the persistent grid, and the rows a block's share of the partition is a multiple of
struct FusedShape { int strip_cols, groups_per_sm, row_gran; };
// The source range a launch of kernel k is specialised for: the integer-ratio TMA kernel builds a luma table for one
// range (1 full, 0 limited), so its launches are single-range; every other kernel reads the range per job (0)
inline int fused_launch_range(const FusedKernel &k, const FusedJob &j) {
    return k.kind == FusedKernel::TMA_INT && j.src.full_range ? 1 : 0;
}
inline FusedShape fused_shape(const FusedKernel &k, const FusedJob &j) {
    switch (k.kind) {
        case FusedKernel::TMA_INT: return {k.ratio == 4 ? kTmaStripCols4 : kTmaStripCols2, 3, 2};
        case FusedKernel::TMA_ANY: return {j.strip_cols, kTma0Groups, 8};
        default: return {kFusedStripCols, 3, 8};
    }
}

struct WeightJob {          // resample.wgsl:42-86 evaluated once per output coordinate
    float scale, offset;
    int32_t n_out, taps;
    float *weights;
    float *inv_wsum;
    int32_t *first;
};

struct OutputJob {          // K10/K11 stand-alone (root size != output size, or odd sizes)
    Tex src;                // TEX_RGBA8 raw bytes, or a YUV kind when the root is an InputStream
    int32_t out_w, out_h;
    int32_t out_format;
    uint8_t *out0, *out1, *out2;
    int32_t out_pitch0, out_pitch1, out_pitch2;
};

// TextRendererNode::render (text_renderer.rs:72-167): glyphon's prepared glyph quads, same layout as smr_glyph
struct GlyphDev {
    int32_t x, y;                 // quad origin in the text texture (may be negative / beyond the edge: clipped per pixel)
    uint16_t w, h, ax, ay;        // quad size; origin in the atlas its `content` names
    uint8_t color[4];             // straight-alpha sRGB colour
    int32_t content;              // 0 colour atlas (RGBA8), 1 mask atlas (R8)
};
// The node texture a node job draws: width x height RGBA8 at `out`, written through the mode's view
struct NodeTarget {
    int32_t width, height;
    int32_t mode;                 // 0 GpuOptimized (sRGB views), 1 CpuOptimized
    uint8_t *out; int32_t out_pitch;
};
struct TextJob {
    NodeTarget dst;
    int32_t color_mode;           // glyphon ColorMode: 0 Accurate (colours -> linear, colour atlas sRGB), 1 Web
    int32_t n_glyphs;
    float bg[4];                  // premultiplied shader colour of the clear (wgpu/utils.rs:51-71)
    const GlyphDev *glyphs;
    const uint8_t *mask; int32_t mask_w, mask_h, mask_pitch;
    const uint8_t *color; int32_t color_w, color_h, color_pitch;
};

// ImageNode::render (transformations/image.rs:178-187): one asset frame drawn into a node texture of the node's resolution
struct ImageJob {
    NodeTarget dst;               // the node's resolution
    Tex src;                      // the frame: TEX_RGBA8, straight alpha; with `raster`, premultiplied and of dst's size
    int32_t raster;               // 1: src is an SVG raster (svg_image.rs:144-167), 0: an asset frame
};

// One plane of WebRendererShader::render (web_renderer/shader.rs:53-114): a quad of the plane mesh through its vertex
// matrix, rasterised by NC-7 on the host (renderer.cpp: web_plane), and the bare linear sample of `tex` at the
// interpolated texture coordinate (u, v) = ((x + .5 - left) / width, (y + .5 - top) / height)
struct WebPlane {
    Tex tex;                      // the page (TEX_BGRA: the fragment's b <-> r swap), a child's node texture, or TEX_NONE
    int32_t px0, px1, py0, py1;   // exactly the covered pixels [px0, px1) x [py0, py1), inside the target
    float left, top, width, height;   // the quad's corners in target pixels (width / height may be negative: mirrored)
};
// WebRenderer::render (web_renderer/renderer.rs:78-99) for a node with a frame: clear to transparent, then each plane in
// order, blended with PREMULTIPLIED_ALPHA_BLENDING through the node texture's view and stored as 8 bits
struct WebJob {
    NodeTarget dst;               // the instance's resolution
    int32_t n_planes;
    const WebPlane *planes;
};

// ShaderNode::render (transformations/shader/node.rs, pipeline.rs:81-140) for one node: clear to transparent, then
// max(1, n_tex) full-target planes, each pixel's smr_fragment at its centre blended with PREMULTIPLIED_ALPHA_BLENDING
// through the node texture's view and stored as 8 bits.  The kernel is the shader module's own (shader_rt.cuh).
struct ShaderJob {
    NodeTarget dst;               // the node's resolution
    int32_t n_tex;                // texture_count: the children, in order
    float time;                   // BaseShaderParameters::time, pts as Duration::as_secs_f32
    const Tex *tex;               // n_tex child textures (TEX_NONE: the empty view), in the parameter arena
    const uint8_t *params;        // ShaderParam::to_bytes, in the parameter arena (null: no parameter)
};

// gpu-video's transcoder resize (vulkan_transcoder/shader.wgsl, NC-10): one output coordinate of one axis, computed on the
// host (renderer.cpp: transcode_axis) so that the kernel evaluates no transcendental
struct TranscodeTap {
    int32_t nearest;              // u32(in * float_coords)
    int32_t lo, hi;               // bilinear: u32(max(floor(fc), 0)), min(lo + 1, in - 1)
    float frac;                   // bilinear: fc - floor(fc), from the unclamped fc
    int32_t center;               // Lanczos3: floor(fc)
    float w[6];                   // Lanczos3: lanczos3_weight(fc - (center + d)), d = -2 .. 3
};
constexpr int kTranscodeMaxOutputs = 8;                  // the reference's binding arrays hold eight renditions
constexpr int kTranscodeTileX = 32, kTranscodeTileY = 8; // chroma samples per block (a thread: one sample, its 2 x 2 luma quad)
struct TranscodeOut {             // one NV12 rendition
    uint8_t *y, *uv;
    int32_t pitch_y, pitch_uv;
    int32_t width, height;        // even
    int32_t scaling;              // 0 nearest, 1 bilinear, 2 Lanczos3 (ScalingAlgorithm)
    const TranscodeTap *tx, *ty;  // luma: in -> out per axis
    const TranscodeTap *cx, *cy;  // chroma: in / 2 -> out / 2 per axis
    int32_t tiles_x;              // blocks per row of tiles
    int32_t tile_begin;           // first block of this rendition
};
struct TranscodeLaunch {          // every rendition of one call: one launch
    const uint8_t *src_y, *src_uv;   // NV12 crop, origin (0, 0); uv 2-byte aligned
    int32_t pitch_y, pitch_uv;
    int32_t width, height;        // even
    int32_t n;
    TranscodeOut out[kTranscodeMaxOutputs];
};

// host tables pushed once per device (numeric contract NC-1/3/4)
void upload_tables(const float *u8n, const float *srgb_dec, const float *srgb_enc_thr);
// the device tables of node_sample.cuh in this module (c_u8n, c_dec, c_thr, c_yl, c_enc1): addresses and bytes, for the
// copies a shader module receives when it is loaded.  false on a CUDA error
bool table_symbols(const void *ptr[5], size_t bytes[5]);

typedef void *Stream;  // cudaStream_t

// each returns the number of kernels it launched (for smr_stats / bench gpu_launches)
int launch_convert_to_rgba(const Tex &src, uint8_t *dst, int dst_pitch, Stream s);
int launch_weights(const WeightJob *jobs_dev, const WeightJob *jobs_host, int n_jobs, Stream s);
// k_weights for one mapping on the current device, synchronously: the n_out x *taps weights (when they fit in cap), and
// 1 / weight_sum and the first tap of every output coordinate.  1 done, 0 cap too small, -1 CUDA error
int debug_weights(float scale, float offset, int n_out, float *w_host, size_t cap, int *taps, float *inv_host, int32_t *first_host);
// NC-8's sin_cr / cos_cr (the functions k_weights calls) on n host values, synchronously.  1 done, -1 CUDA error
int debug_sincos(const float *x_host, int n, float *s_host, float *c_host);
int launch_resample(const ResampleJob *jobs_dev, const ResampleJob *jobs_host, int n_jobs, Stream s);
// source class of the fused kernel's template: 0 planar 4:2:0, 1 NV12, 2 UYVY, 3 YUYV; -1 not supported
inline int fused_source_class(int tex_kind) {
    return tex_kind == TEX_YUV420 ? 0 : tex_kind == TEX_NV12 ? 1 : tex_kind == TEX_UYVY ? 2 : tex_kind == TEX_YUYV ? 3 : -1;
}
// FramePreProcessor: node texture of `src` (rescale = 0) or its linear-filtered rescale to out_w x out_h
int launch_preprocess(const Tex &src, int mode, int rescale, uint8_t *out, int out_pitch, int out_w, int out_h, Stream s);
// text node textures: clear + glyph quads alpha-blended in list order, every job of jobs_dev in one launch.  Job i owns the
// 32 x 8 tiles [tile_begin_dev[i], tile_begin_dev[i + 1]) of the grid (node_tiles of each job, prefix sums); n_tiles =
// tile_begin[n_jobs]
inline int node_tiles(int width, int height) { return ((width + 31) / 32) * ((height + 7) / 8); }
int launch_text(const TextJob *jobs_dev, const int32_t *tile_begin_dev, int n_jobs, int n_tiles, Stream s);
// image node textures: the frame of each job sampled, premultiplied and stored; jobs and tiles as for launch_text
int launch_image(const ImageJob *jobs_dev, const int32_t *tile_begin_dev, int n_jobs, int n_tiles, Stream s);
// web view node textures: each job's planes drawn over a transparent clear; jobs and tiles as for launch_text
int launch_web(const WebJob *jobs_dev, const int32_t *tile_begin_dev, int n_jobs, int n_tiles, Stream s);
// shader node textures of one shader module: `kernel` is its smr_shader_main (a cudaKernel_t); jobs and tiles as for
// launch_text
int launch_shader(const void *kernel, const ShaderJob *jobs_dev, const int32_t *tile_begin_dev, int n_jobs, int n_tiles, Stream s);
// full_range: fused_launch_range of every job of the launch
int launch_resample_fused(const FusedKernel &k, int src, int full_range, const FusedJob *jobs_dev, const FusedPiece *pieces_dev,
                          const int *piece_begin_dev, int nblocks, Stream s);
// every output of a tick in one launch; jobs_dev[i] == jobs_host[i], layers / masks / textures device pointers.  One output
// with a short layer list (layers0_host: host copy of jobs_host[0].layers) passes job and layers in the parameter block
int launch_composite(const CompositeJob *jobs_dev, const CompositeJob *jobs_host, const LayerDev *layers0_host, int n, Stream s);
int launch_output(const OutputJob &job, Stream s);
// every rendition of L in one launch of n_blocks blocks (the last rendition's tile_begin + its tiles)
int launch_transcode(const TranscodeLaunch &L, int n_blocks, Stream s);
int launch_fill_yuv(uint8_t *p0, uint8_t *p1, uint8_t *p2, int pitch0, int pitch1, int pitch2, int w, int h,
                    int out_format, uint8_t y, uint8_t u, uint8_t v, Stream s);
const char *last_launch_error();

}  // namespace dev
}  // namespace smr
