/*
 * smelter_b200.h -- C ABI of the H100-native per-output-frame compositor.
 *
 * Drop-in boundary: this library replaces `smelter_render::Renderer`
 * (reference: smelter-render/src/state.rs:95-193).  There is no C ABI in the reference (it is a Rust
 * crate on wgpu); each entry point below names the Rust method it stands in for, so a Rust shim can
 * re-implement `Renderer` 1:1 over these symbols (see INTEGRATION.md).
 *
 * Conventions: plain C types only; every function returns smr_status (0 = ok) and never throws or
 * aborts across the boundary; ids are NUL-terminated UTF-8 (the reference's `InputId`/`OutputId`
 * are `Arc<str>`); all pointers are borrowed for the duration of the call only -- with ONE exception: the HOST planes
 * (inputs and outputs) handed to smr_render_begin are read / written by asynchronous copies and must stay valid and
 * untouched until the smr_render_end that retires that tick (smr_render has no such window: it returns when the tick
 * it submitted is complete); a handle is
 * internally synchronised exactly like the reference's `Arc<Mutex<InnerRenderer>>` (state.rs:54-55).
 * The product path has NO CPU fallback: every pixel is produced by sm_90a CUDA kernels.
 */
#ifndef SMELTER_B200_H
#define SMELTER_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct smr_renderer smr_renderer;

/* error.rs:10-66 variants that exist on this path, flattened to status codes */
typedef enum {
    SMR_OK = 0,
    SMR_ERR_INVALID_ARGUMENT = 1,
    SMR_ERR_CUDA = 2,                 /* RenderSceneError::WgpuError / InitRendererEngineError analogue */
    SMR_ERR_OUTPUT_NOT_REGISTERED = 3,/* UpdateSceneError::OutputNotRegistered / unknown output in render */
    SMR_ERR_SCENE = 4,                /* UpdateSceneError::SceneError (duplicate ids, unknown root size) */
    SMR_ERR_UNSUPPORTED = 5,          /* component / format outside the compositor hot path (SURVEY 8f) */
    SMR_ERR_OUT_OF_MEMORY = 6,
    SMR_ERR_BUFFER_TOO_SMALL = 7
} smr_status;

/* RenderingMode, types.rs:9-18 (WebGl is out of scope) */
typedef enum { SMR_MODE_GPU_OPTIMIZED = 0, SMR_MODE_CPU_OPTIMIZED = 1 } smr_rendering_mode;

/* RendererOptions, state.rs:43-52.  device/queue become a CUDA device ordinal. */
typedef struct {
    int32_t cuda_device;               /* SMELTER_GPU_DEVICE_ID analogue (src/config.rs:142); -1 = host-only
                                          handle for scene/layout inspection (cannot render) */
    int32_t rendering_mode;            /* smr_rendering_mode */
    uint32_t max_layouts_count;        /* DEFAULT_MAX_LAYOUTS_COUNT = 100 (layout.rs:23); 0 = default */
    uint64_t stream_fallback_timeout_ns;
    uint32_t framerate_num, framerate_den;
} smr_options;

/* ------------------------------- scene::Component (scene/components.rs) ---------------------- */
typedef enum {
    SMR_COMPONENT_INPUT_STREAM = 0,
    SMR_COMPONENT_VIEW = 1,
    SMR_COMPONENT_TILES = 2,
    SMR_COMPONENT_RESCALER = 3,
    /* declared so a shim can forward them; smr_update_scene answers SMR_ERR_UNSUPPORTED */
    SMR_COMPONENT_SHADER = 4,
    SMR_COMPONENT_WEB_VIEW = 5,
    SMR_COMPONENT_IMAGE = 6,
    SMR_COMPONENT_TEXT = 7
} smr_component_type;

typedef struct { uint8_t r, g, b, a; } smr_rgba;                                  /* RGBAColor */
typedef struct { float top_left, top_right, bottom_right, bottom_left; } smr_border_radius;
typedef struct { float offset_x, offset_y, blur_radius; smr_rgba color; } smr_box_shadow;
typedef struct { float top, right, bottom, left; } smr_padding;
typedef struct { int32_t has_value; float value; } smr_opt_f32;                    /* Option<f32> */

typedef enum { SMR_INTERP_LINEAR = 0, SMR_INTERP_BOUNCE = 1, SMR_INTERP_CUBIC_BEZIER = 2 } smr_interpolation_kind;
typedef struct {                                                                   /* Option<Transition> */
    int32_t present;
    uint64_t duration_ns;
    int32_t interpolation_kind;
    double x1, y1, x2, y2;       /* CubicBezier control points */
    int32_t should_interrupt;
} smr_transition;

typedef struct {                                                                   /* Position */
    int32_t is_absolute;         /* 0: Static{width,height}; 1: Absolute(AbsolutePosition) */
    smr_opt_f32 width, height;
    int32_t horizontal_from_right; float horizontal_offset; /* LeftOffset / RightOffset */
    int32_t vertical_from_bottom; float vertical_offset;    /* TopOffset / BottomOffset */
    float rotation_degrees;
} smr_position;

typedef enum { SMR_DIRECTION_ROW = 0, SMR_DIRECTION_COLUMN = 1 } smr_direction;
typedef enum { SMR_OVERFLOW_VISIBLE = 0, SMR_OVERFLOW_HIDDEN = 1, SMR_OVERFLOW_FIT = 2 } smr_overflow;
typedef enum { SMR_RESCALE_FIT = 0, SMR_RESCALE_FILL = 1 } smr_rescale_mode;
typedef enum { SMR_HALIGN_LEFT = 0, SMR_HALIGN_RIGHT = 1, SMR_HALIGN_JUSTIFIED = 2, SMR_HALIGN_CENTER = 3 } smr_horizontal_align;
typedef enum { SMR_VALIGN_TOP = 0, SMR_VALIGN_CENTER = 1, SMR_VALIGN_BOTTOM = 2, SMR_VALIGN_JUSTIFIED = 3 } smr_vertical_align;

/* One node of the Component tree.  Fields that do not apply to `type` are ignored.
 * Use smr_component_default() to get the reference's `Default` values (components.rs:289-347). */
typedef struct smr_component {
    int32_t type;                          /* smr_component_type */
    const char *id;                        /* Option<ComponentId>; NULL = None */
    const struct smr_component *children;  /* View/Tiles: children; Rescaler: exactly one child */
    uint32_t children_len;
    const char *input_id;                  /* InputStream */

    smr_position position;                 /* View, Rescaler */
    smr_transition transition;             /* View, Rescaler, Tiles */
    smr_border_radius border_radius;       /* View, Rescaler */
    float border_width;
    smr_rgba border_color;
    const smr_box_shadow *box_shadow;
    uint32_t box_shadow_len;

    int32_t direction;                     /* View */
    int32_t overflow;
    smr_rgba background_color;             /* View, Tiles */
    smr_padding padding;                   /* View */

    int32_t rescale_mode;                  /* Rescaler */
    int32_t horizontal_align;              /* Rescaler, Tiles */
    int32_t vertical_align;

    smr_opt_f32 tiles_width, tiles_height; /* Tiles */
    uint32_t tile_aspect_ratio_w, tile_aspect_ratio_h;
    float tiles_margin, tiles_padding;
} smr_component;

/* ------------------------------------ frames (types.rs:21-119) ------------------------------- */
typedef enum {
    SMR_FRAME_PLANAR_YUV420 = 0,   /* FrameData::PlanarYuv420: planes y,u,v */
    SMR_FRAME_PLANAR_YUVJ420 = 1,  /* FrameData::PlanarYuvJ420 (full range) */
    SMR_FRAME_NV12 = 2,            /* FrameData::Nv12: planes y, uv */
    SMR_FRAME_BGRA = 3,            /* FrameData::Bgra */
    SMR_FRAME_ARGB = 4,            /* FrameData::Argb */
    SMR_FRAME_RGBA8 = 5,           /* FrameData::Rgba8UnormWgpuTexture analogue: premultiplied RGBA8 */
    SMR_FRAME_PLANAR_YUV422 = 6,   /* FrameData::PlanarYuv422: planes y (w x h), u, v (w/2 x h) */
    SMR_FRAME_PLANAR_YUV444 = 7,   /* FrameData::PlanarYuv444: planes y, u, v (w x h) */
    SMR_FRAME_UYVY422 = 8,         /* FrameData::InterleavedUyvy422: one plane, rows of (w/2) x {U,Y0,V,Y1} */
    SMR_FRAME_YUYV422 = 9          /* FrameData::InterleavedYuyv422: one plane, rows of (w/2) x {Y0,U,Y1,V} */
} smr_frame_format;

typedef enum { SMR_MEM_HOST = 0, SMR_MEM_DEVICE = 1 } smr_mem_kind;

typedef struct {                   /* one entry of FrameSet<InputId> */
    const char *input_id;
    int32_t format;                /* smr_frame_format */
    uint32_t width, height;        /* Frame::resolution */
    uint64_t pts_ns;               /* Frame::pts */
    const void *planes[3];         /* tightly packed when pitch == 0 */
    uint32_t pitch[3];             /* bytes per row */
    int32_t mem_kind;              /* smr_mem_kind; DEVICE = zero-copy (Nv12WgpuTexture analogue) */
} smr_input_frame;
/* Alignment of SMR_MEM_DEVICE planes (pointer and pitch alike; SMR_ERR_INVALID_ARGUMENT otherwise):
 *  - 4-byte texel formats (RGBA8, BGRA, ARGB, UYVY, YUYV): 4-byte aligned.
 *  - Planar 4:2:0 (YUV420, YUVJ420) and NV12: the luma plane, and the NV12 chroma plane, 2-byte aligned (the kernels
 *    read pixel pairs and {u, v} pairs); planar U and V planes may start at any byte.
 * Host planes are copied into aligned buffers and have no such rule.
 * The same holds for SMR_MEM_DEVICE planes of smr_output_frame: an RGBA8 output plane is 4-byte aligned, pointer and
 * pitch (SMR_ERR_INVALID_ARGUMENT before any kernel is launched otherwise); YUV output planes may start at any byte.
 * Crops of texture layouts (smr_set_layouts): every crop field must be finite (SMR_ERR_INVALID_ARGUMENT otherwise).  A crop
 * shrunk by more than 4:1 is first box-averaged by a power of two per axis; smr_render refuses, with
 * SMR_ERR_INVALID_ARGUMENT before any kernel is launched, a layout whose box pass would average more than 2^24 source
 * texels per reduced texel -- the most a crop inside a 16384 x 16384 frame needs to reach one pixel. */

typedef enum {                     /* OutputFrameFormat, types.rs:187-194 */
    SMR_OUT_PLANAR_YUV420 = 0,     /* PlanarYuv420Bytes */
    SMR_OUT_PLANAR_YUV422 = 1,     /* PlanarYuv422Bytes: u, v planes (w/2) x h */
    SMR_OUT_PLANAR_YUV444 = 2,     /* PlanarYuv444Bytes: u, v planes w x h */
    SMR_OUT_RGBA8 = 3,             /* RgbaWgpuTexture analogue */
    SMR_OUT_NV12 = 4               /* Nv12WgpuTexture analogue */
} smr_output_format;

typedef struct {                   /* one entry of FrameSet<OutputId>; caller owns the buffers */
    const char *output_id;
    void *planes[3];               /* capacity: see smr_output_plane_sizes() */
    uint32_t pitch[3];             /* 0 = tightly packed */
    int32_t mem_kind;              /* where the planes live */
    /* filled by smr_render */
    uint32_t width, height;
    int32_t format;
    uint64_t pts_ns;
} smr_output_frame;

/* Flattened layout (RenderLayout, transformations/layout.rs:59-98) -- debug/inspection channel
 * used by the parity tests to feed the CPU oracle the very layouts the kernels drew. */
#define SMR_MAX_MASKS 20           /* params.rs:15 */
typedef struct { float radius[4]; float top, left, width, height; } smr_mask;
typedef struct {
    int32_t type;                  /* 0 texture, 1 color, 2 box shadow (apply_layouts.wgsl:66-71) */
    float top, left, width, height, rotation_degrees;
    float border_radius[4];        /* tl, tr, br, bl */
    smr_rgba color, border_color;
    float border_width, blur_radius;
    int32_t child_index;
    float crop_top, crop_left, crop_width, crop_height;
    int32_t masks_len;
    smr_mask masks[SMR_MAX_MASKS];
} smr_render_layout;

typedef struct {
    uint64_t frames_rendered;       /* output frames produced */
    uint64_t kernel_launches;       /* CUDA kernels launched by this handle */
    uint64_t h2d_bytes, d2h_bytes;  /* bytes copied across PCIe by smr_render */
    uint64_t last_render_kernel_launches;
    uint64_t last_render_direct_tiles;   /* 128 x 16 output tiles of the last tick whose Y / chroma bytes the fused resample
                                            kernel wrote itself (1:1 opaque child interiors), skipped by the composite */
} smr_stats;

/* per-kernel-class device time, measured with cudaEvents on the launching stream when profiling is on
 * (the reference has no GPU timestamps: `timestamp_writes: None`, e.g. rgba_to_yuv.rs:104) */
typedef enum {
    SMR_KERNEL_CONVERT = 0,        /* K1/K2/K4 materialised node texture */
    SMR_KERNEL_WEIGHTS = 1,        /* Lanczos weight tables for new mappings */
    SMR_KERNEL_RESAMPLE_BOX = 2,   /* K7 */
    SMR_KERNEL_RESAMPLE_FIRST = 3, /* K8 first pass -> f16 */
    SMR_KERNEL_RESAMPLE_LAST = 4,  /* K8 last pass -> sRGB8 */
    SMR_KERNEL_COMPOSITE = 5,      /* K9 (+K10/K11 fused) */
    SMR_KERNEL_OUTPUT = 6,         /* K10/K11 stand-alone */
    SMR_KERNEL_FILL = 7,           /* K6 */
    SMR_KERNEL_RESAMPLE_FUSED = 8, /* K1/K2 + both K8 passes in one kernel */
    SMR_KERNEL_CLASSES = 9
} smr_kernel_class;
typedef struct {
    double total_ms[SMR_KERNEL_CLASSES];
    uint64_t launches[SMR_KERNEL_CLASSES];
} smr_kernel_times;

/* ------------------------------------------ entry points ------------------------------------ */
/* Renderer::new(RendererOptions)                                    state.rs:96-100,196-211 */
smr_status smr_create(const smr_options *opts, smr_renderer **out);
void smr_destroy(smr_renderer *r);

/* Renderer::register_input / unregister_input                       state.rs:102-113 */
smr_status smr_register_input(smr_renderer *r, const char *input_id);
smr_status smr_unregister_input(smr_renderer *r, const char *input_id);

/* Renderer::update_scene(output_id, resolution, output_format, scene_root)   state.rs:177-188 */
smr_status smr_update_scene(smr_renderer *r, const char *output_id, uint32_t width, uint32_t height,
                            int32_t output_format, const smr_component *scene_root);
/* Renderer::unregister_output                                       state.rs:115-123 */
smr_status smr_unregister_output(smr_renderer *r, const char *output_id);

/* Renderer::render(FrameSet<InputId>) -> FrameSet<OutputId>         state.rs:173-175,220-252
 * Renders every output listed in `outputs` at `pts_ns` (FrameSet::pts).  Blocks until the output
 * planes are complete (the reference blocks in device.poll, render_loop.rs:177-183). */
smr_status smr_render(smr_renderer *r, uint64_t pts_ns, const smr_input_frame *inputs, uint32_t n_inputs,
                      smr_output_frame *outputs, uint32_t n_outputs);

/* The same with the waits split off, so a caller can overlap ticks (at most SMR_TICKS_IN_FLIGHT in flight; one more
 * smr_render_begin first waits for the oldest and retires it):
 * smr_render_begin enqueues uploads + kernels + downloads and returns; smr_render_end retires the OLDEST tick in
 * flight.  The ticks execute in submission order on one stream; running the host a few ticks ahead keeps the GPU fed
 * across host-side hiccups (the ticks of the benchmark configurations last 0.25 - 0.5 ms).  Host planes of a tick belong to the library from its smr_render_begin until the smr_render_end that
 * retires it.  A plane's pitch must be >= its row bytes (SMR_ERR_INVALID_ARGUMENT otherwise). */
#define SMR_TICKS_IN_FLIGHT 4
smr_status smr_render_begin(smr_renderer *r, uint64_t pts_ns, const smr_input_frame *inputs, uint32_t n_inputs,
                            smr_output_frame *outputs, uint32_t n_outputs);
smr_status smr_render_end(smr_renderer *r);

/* FramePreProcessor::process_to_bytes (state/frame_pre_processor.rs:81-100): one frame in any input format ->
 * RGBA8 bytes of its node texture (sRGB-encoded in GpuOptimized), optionally rescaled with the linear sampler
 * (rgba_rescale.wgsl) to out_width x out_height; 0 x 0 keeps the source resolution.  Blocking, like the reference.
 * `rgba` has out_height rows of `pitch` bytes (0 = tightly packed), host or device memory per `mem_kind`. */
smr_status smr_preprocess_frame(smr_renderer *r, const smr_input_frame *frame, uint32_t out_width, uint32_t out_height,
                                void *rgba, uint32_t pitch, int32_t mem_kind);

/* PremultiplyAlphaPipeline (wgpu/utils/add_premultiplied_alpha.rs + .wgsl:24-35), the last pass of the reference's
 * image-asset upload (transformations/image/svg_image.rs:155-167): a STRAIGHT-alpha RGBA8 frame (format
 * SMR_FRAME_RGBA8) -> premultiplied RGBA8 through the renderer's texture views (sRGB decode / encode around the
 * multiplication in GpuOptimized, plain bytes in CpuOptimized).  The result is what SMR_FRAME_RGBA8 inputs of
 * smr_render are expected to hold.  Blocking; `rgba` has height rows of `pitch` bytes (0 = tightly packed). */
smr_status smr_premultiply_rgba8(smr_renderer *r, const smr_input_frame *frame, void *rgba, uint32_t pitch, int32_t mem_kind);

/* Text nodes (SURVEY 8f-2): TextRendererNode::render (transformations/text_renderer.rs:72-167).  Shaping and glyph
 * rasterisation (cosmic-text / swash inside glyphon, CPU code in the reference too) stay on the caller's side; what the
 * reference does on the GPU -- clear the node texture to the component's background colour (:141-150) and draw glyphon's
 * prepared glyph quads over it (`text_renderer.render`, :163) -- happens here: `glyphs` is glyphon's GlyphToRender list
 * after its clipping to TextBounds (quad origin, size, atlas origin, colour, content type), the atlases are its mask
 * (R8) and colour (RGBA8) atlas pages.  Quads are alpha-blended in list order (wgpu::BlendState::ALPHA_BLENDING) through
 * the node texture's view.  color_mode: glyphon ColorMode, 0 = Accurate (TextAtlas::new, :95-100), 1 = Web.  The
 * result (width x height RGBA8, premultiplied by construction) is the text node's texture: hand it to smr_render as a
 * SMR_FRAME_RGBA8 input (device memory: zero copy) -- like the reference, render it once per scene update
 * (`was_rendered`, :73-75), not per frame.  glyphs and atlases are HOST memory; `rgba` per mem_kind.  Blocking. */
typedef enum { SMR_GLYPH_COLOR = 0, SMR_GLYPH_MASK = 1 } smr_glyph_content;      /* glyphon ContentType */
typedef struct {
    int32_t x, y;                  /* top-left pixel of the quad in the text texture */
    uint16_t width, height;
    uint16_t atlas_x, atlas_y;     /* top-left texel in the atlas `content` names */
    smr_rgba color;                /* glyphon::Color: straight alpha, sRGB */
    int32_t content;               /* smr_glyph_content */
} smr_glyph;
typedef struct { const void *data; uint32_t width, height, pitch; } smr_atlas;   /* pitch 0 = tightly packed */
smr_status smr_render_text(smr_renderer *r, uint32_t width, uint32_t height, smr_rgba background, const smr_glyph *glyphs,
                           uint32_t n_glyphs, const smr_atlas *mask_atlas, const smr_atlas *color_atlas, int32_t color_mode,
                           void *rgba, uint32_t pitch, int32_t mem_kind);

/* inspection (no device needed): the balanced row partition the fused resample launch uses for jobs of
 * dst_w[i] x dst_h[i] output pixels on `max_blocks` resident blocks.  pieces: 4 ints each {job, strip, row_begin,
 * row_end}; block b owns pieces [begin[b], begin[b + 1]). */
smr_status smr_debug_partition(const int32_t *dst_w, const int32_t *dst_h, uint32_t n_jobs, uint32_t max_blocks,
                               int32_t *pieces, uint32_t pieces_cap, uint32_t *n_pieces, int32_t *begin,
                               uint32_t begin_cap, uint32_t *n_blocks);

/* inspection (no device needed): the tile plan of a composite with fused K10 / K11 output (Renderer::plan_tiles).  The
 * width x height frame is cut into 128 x 16 tiles (row-major, tiles_x = ceil(width / 128)).  boxes: 14 ints per layer in
 * painter's order {px0, px1, py0, py1 (pixel bounding box), ix0, ix1, iy0, iy1, jx0, jx1, jy0, jy1 (the two exact-interior
 * bars), opaque (the interior replaces the target), job (fused resample job that could write the layer's tiles itself, -1:
 * none)}.  owner_layer[t]: the layer whose job finishes tile t directly, or -1; tiles[]: the tiles left for the composite
 * ((ty << 16) | tx), most expensive first when `sorted` != 0, row-major otherwise. */
/* inspection (needs a device): the Lanczos3 weight table the weight kernel computes for output coordinates 0 .. n_out - 1
 * (1 <= n_out <= 16384) of the mapping (scale, offset), 0 < scale <= 1024, read back.  *taps is the tap count; weights
 * receives n_out x *taps floats, row by row (SMR_ERR_BUFFER_TOO_SMALL when that exceeds cap); inv and first receive, per
 * output coordinate, 1 / weight_sum and the index of the first tap. */
smr_status smr_debug_weights(float scale, float offset, uint32_t n_out, float *weights, size_t cap, uint32_t *taps, float *inv,
                             int32_t *first);
/* inspection (needs a device): the weight kernel's sin and cos (f32 argument, evaluated in fp64, rounded to f32) of n
 * host values x into host arrays s and c. */
smr_status smr_debug_sincos(const float *x, uint32_t n, float *s, float *c);

smr_status smr_debug_tile_plan(const int32_t *boxes, uint32_t n_layers, uint32_t width, uint32_t height, int32_t sorted,
                               int32_t *owner_layer, uint32_t owner_cap, uint32_t *tiles, uint32_t tiles_cap, uint32_t *n_tiles);

/* inspection (no device access): the fused resample jobs of the handle's most recently planned tick, one record per job in
 * plan order, as they were launched -- after the partition, so `direct` already reflects a job sent back to the
 * composite because its piece of the launch was cut at an odd row.  *n is the job count; records go to `out` when they
 * fit in cap (SMR_ERR_BUFFER_TOO_SMALL otherwise; out = NULL asks for the count). */
typedef enum {
    SMR_FUSED_LDG = 0,             /* k_resample_fused_int<ratio, src_class> */
    SMR_FUSED_TMA_INT = 1,         /* k_resample_tma3<ratio, src_class> */
    SMR_FUSED_TMA_ANY = 2          /* k_resample_tma0<src_class, window, box> */
} smr_fused_kernel;
typedef struct {
    int32_t kernel;                /* smr_fused_kernel */
    int32_t ratio;                 /* template ratio: 2 / 3 / 4, or 0 (any ratio; always 0 for SMR_FUSED_TMA_ANY) */
    int32_t window;                /* SMR_FUSED_TMA_ANY: slots of a lane's tap window (20, 25, 29 or 33); else 0 */
    int32_t box;                   /* SMR_FUSED_TMA_ANY: 1 when the source is box-reduced 2:1 on the fly */
    int32_t src_class;             /* 0 planar 4:2:0, 1 NV12, 2 UYVY, 3 YUYV */
    int32_t full_range;            /* the source's range (1 full, 0 limited) */
    int32_t v_same;                /* SMR_FUSED_TMA_INT: the vertical mapping is the horizontal one (compiled-in weights) */
    int32_t strip_cols;            /* output columns per strip of the launch's partition */
    uint32_t src_width, src_height, dst_width, dst_height;
    int32_t taps_h, taps_v;
    int32_t direct;                /* the job writes the output bytes of its direct tiles itself */
} smr_fused_job_info;
smr_status smr_debug_fused_jobs(smr_renderer *r, smr_fused_job_info *out, uint32_t cap, uint32_t *n);

/* inspection (no device access): the generic resample passes of the handle's most recently planned tick -- every
 * resampled child the fused kernels do not take -- one record per pass: box passes, then first passes, then last passes,
 * each in plan order.  *n is the record count; records go to `out` when it is not NULL.  *n_convert is the number of
 * k_convert jobs (input -> RGBA8 node texture) of the tick; convert_kinds, when not NULL, receives the texture kind each
 * reads.  SMR_ERR_BUFFER_TOO_SMALL when a list does not fit its cap. */
typedef enum { SMR_STAGE_BOX = 0, SMR_STAGE_FIRST = 1, SMR_STAGE_LAST = 2 } smr_resample_stage;
typedef enum {
    SMR_STAGE_SRC_RAW = 0,         /* the input's own texture (an RGBA8 input) */
    SMR_STAGE_SRC_CONVERTED = 1,   /* the RGBA8 node texture k_convert wrote from an input of kind src_kind */
    SMR_STAGE_SRC_F16 = 2          /* the half-precision result of the previous pass (src_kind 4) */
} smr_stage_source;
typedef struct {
    int32_t stage;                 /* smr_resample_stage */
    int32_t axis;                  /* Lanczos pass: 0 horizontal, 1 vertical; box pass: -1 */
    int32_t box_fx, box_fy;        /* box pass: source texels averaged per axis; 1 x 1 for a Lanczos pass */
    int32_t taps;                  /* Lanczos taps per output texel (0 for a box pass) */
    int32_t perp_offset;           /* one-pass plan: integer offset along the other axis */
    int32_t source;                /* smr_stage_source */
    int32_t src_kind;              /* texture kind, as smr_composite_layer_info.tex_kind (4: half-precision RGBA) */
    uint32_t src_width, src_height, dst_width, dst_height;
    int32_t dst_f16;               /* 1: writes half-precision RGBA for the next pass, 0: the sRGB RGBA8 result */
} smr_resample_stage_info;
smr_status smr_debug_resample_stages(smr_renderer *r, smr_resample_stage_info *out, uint32_t cap, uint32_t *n,
                                     int32_t *convert_kinds, uint32_t convert_cap, uint32_t *n_convert);

/* inspection (no device needed): the composite's interior proof for one layout drawn into a width x height target.
 * Inside it every alpha factor of the fragment shader is exactly 1, so the layer paints its bare colour or sample there.
 * box: 12 ints {px0, px1, py0, py1 (pixel bounding box), ix0, ix1, iy0, iy1, jx0, jx1, jy0, jy1 (the two interior bars,
 * which pick the layer's fast class and its direct tiles)}, all 0 when the layer covers no pixel.  shortcut (width *
 * height bytes, row-major; may be NULL): 1 where the composite's general path skips the fragment shader. */
smr_status smr_debug_interior(const smr_render_layout *layout, uint32_t width, uint32_t height, int32_t box[12],
                              uint8_t *shortcut);

/* inspection (no device access): the layers of every composite job of the handle's most recently planned tick, as they
 * were launched, one record per layer in job order, then painter's order (layers that cover no pixel are left out).  *n is
 * the record count; records go to `out` when they fit in cap (SMR_ERR_BUFFER_TOO_SMALL otherwise; out = NULL asks for
 * the count). */
typedef enum {
    SMR_COMPOSITE_PARAM = 0,       /* k_composite_p: one job, its layers in the kernel's parameter block */
    SMR_COMPOSITE_MULTI = 1        /* k_composite_multi: several jobs, or more layers than the parameter block holds */
} smr_composite_kernel;
typedef struct {
    int32_t job;                   /* composite job (outputs of the tick in smr_render order, those that composite) */
    int32_t kernel;                /* smr_composite_kernel */
    int32_t layer;                 /* index in the job's layer list */
    int32_t type;                  /* 0 texture, 1 colour, 2 box shadow */
    int32_t rotated;
    int32_t fast;                  /* fast-class bits: 1 IDENT, 2 CONST, 4 LUT, 8 OPAQUE (occludes), 16 SAMPLE, 32 HALF */
    int32_t box[12];               /* as smr_debug_interior */
    int32_t tx_off, ty_off;        /* IDENT / HALF: texel offset of pixel (0, 0) */
    int32_t mask_count;
    int32_t tex_kind;              /* the texture the kernel reads: 0 none, 1 RGBA8, 2 planar 4:2:0, 3 NV12, 5 BGRA, 6 ARGB,
                                      7 planar 4:2:2, 8 planar 4:4:4, 9 UYVY, 10 YUYV */
    int32_t tex_width, tex_height;
    int32_t tex_pitch[3];          /* bytes per row of each plane (0: unused) */
    int32_t tex_align[3];          /* each plane's address mod 16 */
    int32_t width, height;         /* the job's target */
    int32_t out_format;            /* smr_output_format of the fused K10 / K11 stores, or -1: an RGBA8 frame for k_output */
} smr_composite_layer_info;
smr_status smr_debug_composite_layers(smr_renderer *r, smr_composite_layer_info *out, uint32_t cap, uint32_t *n);

/* byte sizes of the planes smr_render writes for an output (0 for unused planes) */
smr_status smr_output_plane_sizes(uint32_t width, uint32_t height, int32_t output_format, size_t sizes[3]);

/* reference `Default` impls for each component type                 components.rs:289-347 */
void smr_component_default(int32_t type, smr_component *out);

/* inspection: flattened layouts of an output at pts (the input resolutions are those of the last
 * smr_render).  Does not advance any scene state. */
smr_status smr_debug_layouts(smr_renderer *r, const char *output_id, uint64_t pts_ns,
                             smr_render_layout *out, uint32_t capacity, uint32_t *n_out,
                             uint32_t *root_width, uint32_t *root_height);

/* The FLATTENED form of the boundary (SURVEY 8b): a host that keeps the reference's scene/ tree (Component tree,
 * transitions, NestedLayout::flatten -- all Rust) hands over, per output and whenever they change, the RenderLayout[]
 * that transformations/layout/params.rs:169-333 would pack into uniform blocks: same fields, same units (pixels of
 * the root_width x root_height layout node texture), painter's order.  child_ids[k] is the input id of the node's
 * k-th child (scene/layout.rs:84-93), which `child_index` of a texture layout refers to.  Registers the output like
 * smr_update_scene does; stays in force until the next smr_set_layouts / smr_update_scene of that output.  The
 * resampler planning (layout.rs:238-278) and everything below it still happen here, per tick. */
smr_status smr_set_layouts(smr_renderer *r, const char *output_id, uint32_t width, uint32_t height, int32_t format,
                           uint32_t root_width, uint32_t root_height, const char *const *child_ids, uint32_t n_children,
                           const smr_render_layout *layouts, uint32_t n_layouts);

/* inspection: record the pts / input resolutions of a FrameSet exactly as smr_render would
 * (scene.register_render_event + populate_inputs bookkeeping) without touching any plane.  Together
 * with smr_options.cuda_device = -1 (host-only handle: scene + layout engine, smr_render refuses) this
 * lets the host logic be tested on a box without a GPU. */
smr_status smr_debug_set_inputs(smr_renderer *r, uint64_t pts_ns, const smr_input_frame *inputs, uint32_t n_inputs);

/* ---- multi-GPU (new: the reference is single-device, render_loop.rs:232-236 loops outputs serially) -------
 * Outputs shard across GPUs (one handle per GPU, no data-path collective).  The single exchange step is
 * replicating an input frame to every GPU that hosts an output referencing it: ncclBroadcast over NVLink,
 * all shared inputs of a tick in one ncclGroup, enqueued on the handle's stream (the next smr_render on that
 * handle is ordered after it).  The unique id travels over whatever transport the host already has. */
smr_status smr_comm_get_unique_id(uint8_t id[128]);
smr_status smr_comm_init(smr_renderer *r, const uint8_t id[128], int32_t rank, int32_t nranks);
/* frames[i]: device-resident planes, identical geometry on every rank; root_ranks[i] holds the data.
 * Asynchronous: the NCCL group runs on the handle's communication stream, after every tick submitted BEFORE the most
 * recent smr_render_begin has finished and before the next smr_render_begin's kernels -- i.e. it overlaps the tick in
 * flight.  The planes must therefore not be the ones the most recently submitted tick reads (alternate two sets).
 * smr_comm_broadcast_inputs replicates every frame to every rank, one ncclBroadcast per plane.
 * smr_comm_exchange_inputs is the selective form: consumer_masks[i] has bit k set when rank k hosts an output that
 * reads frame i (NULL = every rank); a frame all ranks need is broadcast, any other is sent point to point
 * (ncclSend / ncclRecv in the same group) to exactly its consumers.  flags: SMR_COMM_POOLED declares that the planes
 * are laid out identically on every rank (one frame pool per ingest GPU); only then are consecutive planes that share
 * root and consumers and are contiguous in memory merged into one message.  All ranks must pass the same list. */
#define SMR_COMM_POOLED 1u
smr_status smr_comm_broadcast_inputs(smr_renderer *r, const smr_input_frame *frames, uint32_t n,
                                     const int32_t *root_ranks);
smr_status smr_comm_exchange_inputs(smr_renderer *r, const smr_input_frame *frames, uint32_t n, const int32_t *root_ranks,
                                    const uint64_t *consumer_masks, uint32_t flags);
/* Peer memory over NVLink / NVSwitch (one process per GPU, one node).  A frame pool allocated with smr_peer_pool_alloc can
 * be mapped by the handles of the other GPUs: pass the 64-byte CUDA IPC handle over the host transport and open it there.
 * A pointer into an opened pool is an ordinary SMR_MEM_DEVICE plane pointer for smr_render: the kernels read it over
 * NVLink (the fused resample kernel by TMA tile loads -- the transfer overlaps the arithmetic tile by tile, nothing is
 * staged in local HBM).  Two ways to use it for the shared inputs of a tick:
 *   SMR_COMM_PEER_DIRECT (flag of smr_comm_exchange_inputs): no data moves; the call is only the cross-rank ordering (a
 *     4-byte all-reduce on the communication stream).  The caller passes, in smr_render, plane pointers into the ROOT's
 *     pool for frames rooted elsewhere.  A pool set may be rewritten three ticks later at the earliest (three sets).
 *   smr_comm_pull_inputs: after the same ordering step, frames rooted elsewhere are copied from peer_frames[i] (planes in
 *     the root's opened pool) to frames[i] (local planes) by the copy engines -- no SM time, unlike the NCCL kernels of
 *     smr_comm_exchange_inputs.  Two sets suffice.
 * The reference has no counterpart (single device). */
#define SMR_COMM_PEER_DIRECT 2u
smr_status smr_peer_pool_alloc(smr_renderer *r, size_t bytes, void **dev_ptr, uint8_t handle[64]);
smr_status smr_peer_pool_open(smr_renderer *r, const uint8_t handle[64], void **dev_ptr);
smr_status smr_peer_pool_close(smr_renderer *r, void *dev_ptr);
smr_status smr_peer_pool_free(smr_renderer *r, void *dev_ptr);
smr_status smr_comm_pull_inputs(smr_renderer *r, const smr_input_frame *frames, const smr_input_frame *peer_frames, uint32_t n,
                                const int32_t *root_ranks, const uint64_t *consumer_masks);
smr_status smr_comm_destroy(smr_renderer *r);

/* Texture upload / read-back glue of smelter-core (pipeline/decoder/ffmpeg_utils.rs:67-79 copy_plane_from_av,
 * pipeline/encoder/ffmpeg_utils.rs:77-84 write_plane_to_av_frame): a frame pool the caller keeps across ticks is
 * page-locked ONCE; SMR_MEM_HOST planes inside a registered range are then moved by direct DMA (no staging copy in
 * the driver), uploads of a tick are spread over two copy streams.  Already registered memory is not an error. */
smr_status smr_host_register(void *ptr, size_t bytes);
smr_status smr_host_unregister(void *ptr);

smr_status smr_get_stats(smr_renderer *r, smr_stats *out);
smr_status smr_set_profiling(smr_renderer *r, int32_t enabled);   /* also resets the accumulated times */
smr_status smr_get_kernel_times(smr_renderer *r, smr_kernel_times *out);
void *smr_cuda_stream(smr_renderer *r);          /* cudaStream_t the handle launches on */
const char *smr_last_error(smr_renderer *r);     /* ErrorStack::into_string analogue; valid until next call */
const char *smr_version(void);

#ifdef __cplusplus
}
#endif
#endif /* SMELTER_B200_H */
