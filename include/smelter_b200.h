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
    SMR_COMPONENT_SHADER = 4,      /* accepted when smr_component.shader_id is set, see there */
    SMR_COMPONENT_WEB_VIEW = 5,    /* accepted when smr_component.web_renderer_id is set, see there */
    SMR_COMPONENT_IMAGE = 6,       /* accepted when smr_component.image_id is set, see there */
    SMR_COMPONENT_TEXT = 7         /* payload in smr_component.text */
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

struct smr_text;

/* ShaderParam (scene/components.rs:40-55) and the type a shader declares for it (smr_shader_spec.param_type) */
typedef enum {
    SMR_SHADER_PARAM_F32 = 0, SMR_SHADER_PARAM_U32 = 1, SMR_SHADER_PARAM_I32 = 2,
    SMR_SHADER_PARAM_LIST = 3, SMR_SHADER_PARAM_STRUCT = 4
} smr_shader_param_kind;
typedef struct smr_shader_param {
    int32_t kind;                          /* smr_shader_param_kind */
    const char *field_name;                /* a Struct's field: its name (ShaderParamStructField::field_name) */
    float f32; uint32_t u32; int32_t i32;  /* the scalar of its kind */
    const struct smr_shader_param *items;  /* List: the elements; Struct: the fields */
    uint32_t items_len;
} smr_shader_param;

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

    const struct smr_text *text;           /* Text (smr_text below) */

    /* Image (ImageComponent, scene/components.rs:63-80): an asset registered with smr_register_image, shown at
     * image_width x image_height (a missing side follows from the asset's aspect ratio, both missing: the asset's size).
     * NULL image_id: SMR_ERR_UNSUPPORTED, which is what a caller built before these fields existed sends (the tag and
     * nothing else).  An id that is not registered, the empty string (the reference's Default) included, is
     * SceneError::ImageNotFound: SMR_ERR_SCENE. */
    const char *image_id;
    smr_opt_f32 image_width, image_height;

    /* WebView (WebViewComponent, scene/components.rs:55-61): the instance registered with smr_register_web_renderer, and
     * in `children` the components embedded in the page, zipped in order with the instance's child rects
     * (smr_web_set_child_rects).  A child has an id and is an InputStream, Image or Text component, or a View, Tiles or
     * Rescaler that declares both width and height (a layout node of its own, holding any component).  A WebView or
     * Shader child, and a View, Tiles or Rescaler child without both sides, are SMR_ERR_UNSUPPORTED (see
     * smr_update_scene).  NULL web_renderer_id: SMR_ERR_UNSUPPORTED, which is what a caller built before this field
     * existed sends. */
    const char *web_renderer_id;

    /* Shader (ShaderComponent, scene/components.rs:29-38): the shader registered with smr_register_shader, its parameter
     * (NULL: None), the node's size (Size; the node texture is (size_t)shader_width x (size_t)shader_height), and in
     * `children` its textures, in order.  NULL shader_id: SMR_ERR_UNSUPPORTED, which is what a caller built before these
     * fields existed sends.  See smr_update_scene for the rules. */
    const char *shader_id;
    const smr_shader_param *shader_param;
    float shader_width, shader_height;
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
    SMR_KERNEL_IMAGE = 9,          /* image node textures (k_image) */
    SMR_KERNEL_WEB = 10,           /* web view node textures (k_web) */
    SMR_KERNEL_SHADER = 11,        /* shader node textures (each shader module's smr_shader_main) */
    SMR_KERNEL_TRANSCODE = 12,     /* transcoder renditions (k_transcode, smr_transcode_resize) */
    SMR_KERNEL_VIDEO_CONVERT = 13, /* NV12 -> RGBA frame converter (k_video_nv12_to_rgba, smr_video_nv12_to_rgba); the
                                      reverse converter is k_output and counts as SMR_KERNEL_OUTPUT */
    SMR_KERNEL_DEINTERLACE = 14,   /* deinterlaced input planes (k_deinterlace, smr_set_input_deinterlace) */
    SMR_KERNEL_CLASSES = 15
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

/* Deinterlacing of an interlaced input (new: the reference has no deinterlacer).  Interlaced sources (1080i SDI capture,
 * PAFF / MBAFF broadcast H.264) deliver woven frames: two fields, captured half a frame period apart, on alternate rows.
 * Converted and resampled as they are, moving content combs, and a downscale aliases the combs.  With a mode set, every
 * frame of the input is deinterlaced on the GPU before anything reads it (the rest of the tick is unchanged).
 * The rule, byte for byte (DESIGN.md NC-12): each plane of the frame (the three planes of planar formats, NV12's luma and
 * interleaved chroma planes, the one plane of UYVY / YUYV / BGRA / ARGB / RGBA8) is processed on its own, byte by byte
 * along its row bytes; row parity within the plane decides the field, the half-height chroma planes of 4:2:0 included.
 * SMR_FIELD_TOP_FIRST keeps the even rows and rebuilds the odd ones, SMR_FIELD_BOTTOM_FIRST keeps the odd rows and
 * rebuilds the even ones.  For a rebuilt row y: a = row y - 1 (row y + 1 when y - 1 is outside the plane), b = row y + 1
 * (row y - 1 when y + 1 is outside the plane); a plane of one row is copied unchanged.
 *   SMR_DEINTERLACE_FIELD: out = (a + b + 1) >> 1.
 *   SMR_DEINTERLACE_MOTION_ADAPTIVE: c = the current row y, p, pa, pb = rows y, a and b of the previous frame;
 *     m = max(|c - p|, |a - pa|, |b - pb|), out = m <= motion_threshold ? c : (a + b + 1) >> 1.  Without a previous frame
 *     the rebuilt rows follow FIELD.
 * The previous frame is the last frame of the input with another pts_ns, kept by the library as a copy (the caller may
 * rewrite its planes once the tick that read them has retired).  A frame with the same pts_ns, format and size as the last
 * one is the same frame (the queue repeats frames when an input is slower than the output): it gives the same bytes and
 * does not advance the history.  A change of format or size clears the history, and so does a call here that changes
 * the mode or the field order (a call that only changes the threshold keeps it); a tick in which the input has no live
 * frame leaves it alone.  The setting lasts until it is changed, or until smr_unregister_input, which drops it and the
 * history.  SMR_DEINTERLACE_OFF (the default) leaves the input exactly as without this call.
 * A shim maps DeckLink's detected field dominance (bmdUpperFieldFirst: TOP_FIRST, bmdLowerFieldFirst: BOTTOM_FIRST) and
 * turns the mode off for progressive display modes (see INTEGRATION.md).
 * SMR_ERR_INVALID_ARGUMENT: a NULL id or cfg, an id that is not registered, an unknown mode or field order,
 * motion_threshold above 255.  A host-only handle stores the setting. */
typedef enum { SMR_DEINTERLACE_OFF = 0, SMR_DEINTERLACE_FIELD = 1, SMR_DEINTERLACE_MOTION_ADAPTIVE = 2 } smr_deinterlace_mode;
typedef enum { SMR_FIELD_TOP_FIRST = 0, SMR_FIELD_BOTTOM_FIRST = 1 } smr_field_order;
typedef struct {
    int32_t mode;                  /* smr_deinterlace_mode */
    int32_t field_order;           /* smr_field_order */
    uint32_t motion_threshold;     /* MOTION_ADAPTIVE: T, 0 .. 255 */
} smr_deinterlace;
smr_status smr_set_input_deinterlace(smr_renderer *r, const char *input_id, const smr_deinterlace *cfg);
/* The colour matrix and range of a YUV input (new: the reference reads every YUV input as BT.709, limited range except
 * PlanarYuvJ420).  SD capture (NTSC / PAL), V4L2 webcams and MJPEG / JFIF sources are BT.601; screen capture and some
 * cameras send full range.  The caller knows which from the source's metadata (ffmpeg's AVFrame colorspace / color_range,
 * the DeckLink display mode, V4L2's ycbcr_enc / quantization; see INTEGRATION.md).
 *   matrix: SMR_MATRIX_DEFAULT is BT.709; SMR_MATRIX_BT601 converts with r = y + 1.402 (v - .5),
 *     g = y - 0.3441 (u - .5) - 0.7141 (v - .5), b = y + 1.772 (u - .5) (DESIGN.md NC-13): the matrix only, no change of
 *     primaries.
 *   range: SMR_RANGE_DEFAULT is full for SMR_FRAME_PLANAR_YUVJ420 and limited for every other YUV format; an explicit
 *     value overrides that for every YUV format (planar 4:2:0, J420, NV12, 4:2:2, 4:4:4, UYVY, YUYV).
 * RGB formats (BGRA, ARGB, RGBA8) store the setting and ignore it.  {DEFAULT, DEFAULT} leaves the input exactly as without
 * this call.  The setting lasts until it is changed, or until smr_unregister_input, which drops it; a tick converts with
 * the setting in force at its smr_render_begin (ticks in flight keep theirs).  The blocking calls take a frame, not an
 * input, and keep their own rules (smr_preprocess_frame, the transcoder, the video converters).
 * SMR_ERR_INVALID_ARGUMENT: a NULL id or c, an id that is not registered, an unknown matrix or range.  A host-only handle
 * stores the setting. */
typedef enum { SMR_MATRIX_DEFAULT = 0, SMR_MATRIX_BT709 = 1, SMR_MATRIX_BT601 = 2 } smr_yuv_matrix;
typedef enum { SMR_RANGE_DEFAULT = 0, SMR_RANGE_LIMITED = 1, SMR_RANGE_FULL = 2 } smr_yuv_range;
typedef struct {
    int32_t matrix;                /* smr_yuv_matrix */
    int32_t range;                 /* smr_yuv_range */
} smr_input_color;
smr_status smr_set_input_color(smr_renderer *r, const char *input_id, const smr_input_color *c);
/* inspection (needs a device; blocking): the planes the kernels of the most recent tick that had a live frame of the input
 * read for it, after deinterlacing, copied into planes[p] (rows of the frame's row bytes, at pitch[p], 0 = tightly packed;
 * host or device memory per mem_kind).  The plane sizes are those of the frame (smr_input_frame).  Valid once that tick
 * has retired.  For an input without deinterlacing these are the library's copy of a host frame, or the caller's device
 * planes as they are now.  SMR_ERR_INVALID_ARGUMENT: a NULL id, planes or pitch, a NULL plane the format has, an id that
 * is not registered or has had no live frame since it was registered, an unknown mem_kind. */
smr_status smr_debug_input_planes(smr_renderer *r, const char *input_id, void *const planes[3], const uint32_t pitch[3],
                                  int32_t mem_kind);

/* Renderer::register_renderer / unregister_renderer for RendererSpec::Image   state.rs:123-166, registry.rs:57-68
 * An image asset arrives decoded, as straight-alpha RGBA8 frames of width x height in HOST memory (PNG / JPEG / GIF
 * decoding stays with the caller, as text shaping does).  n_frames == 1 is a Bitmap asset (delay ignored), n_frames >= 2
 * an Animated one (image.rs:69-79): frame k's pts is the sum of the delays before it, the animation's duration the sum
 * of all delays, and a zero sum counts as 1 ns (animated_image.rs:52-112).  SMR_ERR_INVALID_ARGUMENT: a NULL id, spec
 * or frame pointer, n_frames == 0 (NoFrames) or above 1000 (TooManyFrames), a side of 0 or above 16384, a pitch below
 * 4 * width, delays whose sum does not fit 64 bits, an id already registered (RegisterError::KeyTaken), unregistering an
 * unknown id; a failed call registers nothing.  The pixels are copied before the call returns (to the device, on the
 * handle's stream); a host-only handle keeps sizes and timing only.  An asset is shared by the registry and every scene
 * node that resolved it: unregistering removes the registry entry only, scenes already showing the asset keep drawing it,
 * and its device memory is released on the handle's stream after the last tick that reads it.  Registering the same id
 * again makes a new asset: a scene updated afterwards restarts its animation (Arc::ptr_eq, image_component.rs:100-111).
 * SVG assets register through smr_register_svg_image below, into the same registry; smr_unregister_image removes
 * either kind.  Not supported: URL / file sources (ImageSource). */
typedef struct { const void *rgba; uint32_t pitch; uint64_t delay_ns; } smr_image_frame;   /* pitch 0 = packed */
typedef struct { uint32_t width, height; const smr_image_frame *frames; uint32_t n_frames; } smr_image_spec;
smr_status smr_register_image(smr_renderer *r, const char *image_id, const smr_image_spec *spec);
smr_status smr_unregister_image(smr_renderer *r, const char *image_id);

/* Renderer::register_renderer for RendererSpec::Image with ImageType::Svg (transformations/image/svg_image.rs).  SVG
 * parsing and rasterisation stay with the caller, as text shaping and image decoding do: the library asks for a raster
 * when the reference would draw one, at the resolution the reference would use.
 * width x height is the asset's intrinsic size, the parsed tree's size truncated to integers (SvgAsset::resolution); the
 * node resolution follows from it exactly as for a bitmap asset (see smr_update_scene).
 * rasterize fills `rgba` (height rows of `pitch` bytes, pitch == 4 * width, zeroed on entry, valid only during the call)
 * with the asset drawn at width x height, premultiplied RGBA8 as tiny-skia's Pixmap holds it (svg_image.rs:262-292: the
 * tree scaled by resolution / tree.size in f32), and returns 0; anything else refuses the scene update.  It is called
 * during smr_update_scene, once per SVG image node of the updated output (the root, layout children, and children of
 * Shaders, WebViews and layout nodes), with that node's resolution, after the scene has passed every other check: a
 * refused scene never calls it.  It runs on the calling thread under the handle's lock, so it must not call into the
 * same handle.  `user` must stay valid until smr_unregister_image of the id, or smr_destroy, returns; after an unregister
 * the rasteriser is never called again.  A host-only handle calls it too and drops the pixels.
 * SMR_ERR_INVALID_ARGUMENT: a NULL id, spec or rasterize, a side of 0 or above 16384, an id already registered as any
 * kind of image (KeyTaken); a failed call registers nothing.  Registering the same id again after an unregister makes a
 * new asset. */
typedef int32_t (*smr_svg_rasterize_fn)(void *user, uint32_t width, uint32_t height, uint8_t *rgba, uint32_t pitch);
typedef struct { uint32_t width, height; smr_svg_rasterize_fn rasterize; void *user; } smr_svg_spec;
smr_status smr_register_svg_image(smr_renderer *r, const char *image_id, const smr_svg_spec *spec);

/* Renderer::register_renderer / unregister_renderer for RendererSpec::WebRenderer   state.rs:137-143
 * The browser (CEF) stays with the caller, and so does the URL: the library receives what CEF's on_paint delivers (one
 * BGRA plane of width x height, smr_web_set_frame) and the child rectangles of the GET_FRAME_POSITIONS reply
 * (smr_web_set_child_rects), and draws the node texture on the GPU (web_renderer/renderer.rs:78-134).  Embedding:
 * SMR_WEB_NATIVE_OVER_CONTENT draws the page, then each child over it; SMR_WEB_NATIVE_UNDER_CONTENT each child, then the
 * page over them; SMR_WEB_CHROMIUM_EMBEDDING (the page draws the children itself, from textures read back every tick) is
 * SMR_ERR_UNSUPPORTED.  SMR_ERR_INVALID_ARGUMENT: a NULL id or spec, a side of 0 or above 16384, an unknown embedding
 * method, an id already registered, unregistering an unknown id.  An instance is shared by the registry and the scene that
 * shows it: unregistering removes the registry entry only, and a scene still showing it keeps drawing its last frame. */
typedef enum { SMR_WEB_CHROMIUM_EMBEDDING = 0, SMR_WEB_NATIVE_OVER_CONTENT = 1, SMR_WEB_NATIVE_UNDER_CONTENT = 2 } smr_web_embedding;
typedef struct { uint32_t width, height; int32_t embedding_method; } smr_web_renderer_spec;
smr_status smr_register_web_renderer(smr_renderer *r, const char *instance_id, const smr_web_renderer_spec *spec);
smr_status smr_unregister_web_renderer(smr_renderer *r, const char *instance_id);
/* The page as CEF's on_paint hands it over: BGRA8, premultiplied, exactly the instance's width x height, pitch bytes per
 * row (0 = packed, at least 4 * width), in host or device memory (mem_kind).  The plane is copied before the call returns,
 * on a copy stream: the call waits for that copy, not for the renders in flight, which keep drawing the frame they were
 * submitted with.  The renders after it draw this frame until the next one arrives (renderer.rs:136-142).  Before the first frame the node
 * texture is transparent.  SMR_ERR_INVALID_ARGUMENT: a NULL id, frame or pointer, a size other than the instance's, a pitch
 * below 4 * width, an unknown instance. */
typedef struct { const void *bgra; uint32_t width, height, pitch; int32_t mem_kind; } smr_web_frame;
smr_status smr_web_set_frame(smr_renderer *r, const char *instance_id, const smr_web_frame *frame);
/* The GET_FRAME_POSITIONS reply (browser_client.rs:28-93): child k is drawn at rects[k] (page pixels, narrowed to f32,
 * rotation 0).  The latest list wins; children and rects are zipped, so extra children or extra rects are not drawn.
 * n = 0 (rects may then be NULL) draws no child.  SMR_ERR_INVALID_ARGUMENT: a NULL id, NULL rects with n > 0, more than
 * 65536 rects, an unknown instance. */
typedef struct { double x, y, width, height; } smr_web_rect;
smr_status smr_web_set_child_rects(smr_renderer *r, const char *instance_id, const smr_web_rect *rects, uint32_t n);

/* Renderer::register_renderer / unregister_renderer for RendererSpec::Shader   state.rs:123-166, registry.rs:57-68
 * The reference compiles WGSL through naga and wgpu; here a shader is CUDA C++, compiled for sm_90a by NVRTC when it is
 * registered.  `source` (NUL-terminated) defines one device function, smr_fragment, of the signature
 *   float4 (smr_fragment_in in, const smr_base_params &base, const void *params, const smr_textures &tex)
 * in.tex_coords runs from (0, 0) at the node texture's top-left corner to (1, 1); in.position is the pixel centre in
 * texture pixels (x + .5, y + .5, 0, 1).  base has BaseShaderParameters' fields and values (base_params.rs): plane_id,
 * time (the pts in seconds, Duration::as_secs_f32), output_resolution (the node's size) and texture_count.  params points
 * at the parameter's bytes (ShaderParam::to_bytes: the scalars, little-endian, tightly concatenated; NULL without a
 * parameter).  tex.sample(i, uv) samples child i with the reference's sampler (linear, clamp to edge) through the node
 * texture's view: sRGB-decoded in GpuOptimized mode, raw in CpuOptimized mode, premultiplied; an index at or above
 * texture_count samples the empty view.  The returned colour is premultiplied.  The library prepends the header that
 * declares these types (smelter_b200/csrc/shader_rt.cuh).  A CUDA shader has no user vertex stage: every plane is the
 * full-target quad under the identity transform.  smr_register_wgsl_shader below takes the reference's WGSL instead,
 * vertex stage included; both share this registry.
 * The source is compiled with --fmad=false and without fast math, so its arithmetic is reproducible.  NVRTC is loaded at
 * run time (libnvrtc.so.12); when it cannot be, registration answers SMR_ERR_UNSUPPORTED with the reason in
 * smr_last_error.  A compile error is SMR_ERR_INVALID_ARGUMENT (CreateShaderError) with NVRTC's log in smr_last_error.
 * A host-only handle compiles too (the source is validated) but loads nothing.
 * param_type: the parameter's type (the WGSL uniform of the reference), a tree of F32 / U32 / I32 scalars, LISTs (one
 * item: the element type, `length` elements) and STRUCTs (items: the fields, each with its `name`); NULL: no parameter.
 * SMR_ERR_INVALID_ARGUMENT also for a NULL id, spec or source, a malformed type, an id already registered (KeyTaken),
 * unregistering an unknown id.  A shader is shared by the registry and the scenes that show it: unregistering removes the
 * registry entry only, a scene still showing it keeps drawing it, and its module is unloaded after the last tick that
 * launched it. */
typedef struct smr_shader_param_type {
    int32_t kind;                                  /* smr_shader_param_kind */
    const char *name;                              /* a struct field's name (ignored elsewhere) */
    const struct smr_shader_param_type *items;     /* LIST: exactly one, the element type; STRUCT: the fields */
    uint32_t items_len;
    uint32_t length;                               /* LIST: the element count (at least 1) */
} smr_shader_param_type;
typedef struct { const char *source; const smr_shader_param_type *param_type; } smr_shader_spec;
smr_status smr_register_shader(smr_renderer *r, const char *shader_id, const smr_shader_spec *spec);
smr_status smr_unregister_shader(smr_renderer *r, const char *shader_id);

/* RendererSpec::Shader(ShaderSpec { source }) as the reference takes it: `wgsl_source` is WGSL that contains the shader
 * header (shader_header.wgsl: textures, sampler_ and base_params: BaseShaderParameters as var<immediate>) and defines
 * @vertex vs_main(VertexInput) and @fragment fs_main returning @location(0) vec4<f32>.  It is translated to CUDA C++
 * (smelter_b200/csrc/wgsl.cpp, against wgsl_rt.cuh) and compiled as smr_register_shader compiles, host-only handles
 * included; it shares that registry (KeyTaken, unregistering, scenes keeping an unregistered shader).
 * Statuses: SMR_ERR_INVALID_ARGUMENT (CreateShaderError) for WGSL that does not parse or type-check, or that fails the
 * reference's header validation (a missing header global or one of another type, var<push_constant> for base_params,
 * vs_main without exactly one VertexInput, a group(1) binding(0) that is not var<uniform>); smr_last_error names the
 * line and column.  SMR_ERR_UNSUPPORTED for valid WGSL outside the subset, named in smr_last_error: derivatives
 * (dpdx, fwidth, ...), storage buffers, atomics, override, pointers, textures and bindings other than the header's and
 * the uniform, f16, and builtins not in the list of accepted builtins in DESIGN.md ("WGSL builtins"), which states each
 * one's exact rule.  textureSampleBias is fragment-only: vs_main, or a function it calls, using it is
 * SMR_ERR_INVALID_ARGUMENT; textureSample, textureSampleLevel, textureSampleGrad and textureSampleBaseClampToEdge may
 * also be used in vs_main.  textureGather's component must be a const-expression in 0..3 (SMR_ERR_INVALID_ARGUMENT).
 * The module language DESIGN.md states ("WGSL module language") is accepted: var<private> (per-invocation state: every
 * vs_main vertex and every fs_main fragment, each plane's and each triangle's included, starts from the initial value;
 * an initializer must be a const-expression), texture_2d<f32> and sampler values in helper parameters and lets, alias,
 * const_assert, hexadecimal float literals (exactly representable), @size / @align on struct members (they move the
 * uniform's fields), an fs_main result struct whose only member is @location(0) vec4<f32>, and diagnostic directives and
 * attributes (checked, then ignored).  Their misuse is SMR_ERR_INVALID_ARGUMENT with line and column: a var<private>
 * initializer that is not a const-expression or a var<private> of a texture or sampler type; a var or const of a texture
 * or sampler, a function returning one or an entry point taking one; an alias cycle, redeclaration or unknown target; a
 * const_assert that is false or not a const-expression; a hexadecimal float that is not exactly representable; an
 * @align that is not a positive power of two or is below the member type's alignment, or an @size below its SizeOf;
 * two diagnostic filters giving one rule two severities, a diagnostic directive after a declaration, or @diagnostic
 * anywhere but on a function or a control-flow statement.  requires directives stay SMR_ERR_UNSUPPORTED.
 * In a module with var<private>, operands are evaluated left to right, as WGSL orders them.
 * The parameter type is the uniform's WGSL type: scalars, vectors (a LIST of exactly N scalars), matrices (a LIST of
 * exactly R rows of C scalars), arrays (a LIST of at most N) and structs, validated as validation.rs does.  The bytes
 * stay ShaderParam::to_bytes (tight); the shader reads them at WGSL uniform-address-space offsets (AlignOf, SizeOf,
 * array stride), as the reference's GPU reads that buffer, and bytes beyond those supplied (a short list, or no
 * parameter) read as zero.
 * Drawing (ShaderPipeline::render): the node texture is cleared to transparent, then max(1, texture_count) planes are
 * drawn, plane_id -1 without children; each is the plane mesh (4 vertices, indices 0,1,2 and 2,3,0) through vs_main, a
 * triangle list with front face counter-clockwise and back faces culled (the plane as the mesh gives it is front-facing).
 * The rasteriser's arithmetic is the contract, stated in full at the WGSL section of smelter_b200/csrc/shader_rt.cuh:
 * window coordinates snapped to 1/256 px; integer edge functions and the top-left rule (a pixel on an edge two triangles
 * share is drawn once); f32 barycentrics E_i / A; perspective-correct varyings by default, @interpolate(linear) and
 * @interpolate(flat) (the provoking vertex is the triangle's first) honoured; @builtin(position) is (x + .5, y + .5,
 * depth, 1/w).  A fragment whose depth z/w is outside [0, 1] is not drawn.  A plane with a vertex whose clip w is not
 * above 0, or whose window coordinate is beyond 2^20 px, is not drawn at all (there is no homogeneous clipping).
 * `discard` leaves the pixel as it was; every other fragment is blended with PREMULTIPLIED_ALPHA_BLENDING and stored as
 * 8 bits, through the sRGB view in GpuOptimized mode, with the same sampler and blend as a CUDA shader. */
smr_status smr_register_wgsl_shader(smr_renderer *r, const char *shader_id, const char *wgsl_source);

/* Renderer::update_scene(output_id, resolution, output_format, scene_root)   state.rs:177-188
 * Components: InputStream, View, Tiles, Rescaler, Text, Image, WebView and Shader (anywhere, the root included).  A
 * Text, Image, WebView or Shader root follows the rules of an InputStream root (an RGBA output has the node's size).
 * Shader (scene/shader_component.rs, transformations/shader/node.rs): SMR_ERR_SCENE, the scene staying as it was: a shader
 * that is not registered (ShaderNotFound), a parameter that does not match the shader's type
 * (ShaderNodeParametersValidationError, validation.rs:314-520: the same kind; a list no longer than the type's length,
 * each element matching; a struct with the same number of fields, the same names in order, each value matching; a
 * parameter for a shader without a parameter type is NoBindingInShader), a node size that resolves to 0 or above 16384,
 * a View, Tiles or Rescaler child without width and height (UnknownDimensionsForLayoutNodeRoot, scene_state.rs:198-228).
 * Its children are render nodes of their own: InputStream, Image, Text, WebView, Shader, View, Tiles or Rescaler
 * components.  A View, Tiles or Rescaler child is a layout node of its own (scene_state.rs:154-196): its size is its width
 * and height at the last render's pts, its resolution at each render SizedLayoutComponent::resolution, and its layout
 * state (transitions, Tiles' last layout) carries over scene updates as the root's does; every render evaluates its
 * layouts and composites them into a texture of that resolution, which the shader samples (a resolution of 0 or above
 * 16384 samples the empty view).  More than 16 children is SMR_ERR_UNSUPPORTED (the reference fails in wgpu validation,
 * SHADER_INPUT_TEXTURES_AMOUNT).  Every render
 * clears the node texture and draws max(1, texture_count) planes (plane_id -1 without children), each pixel's
 * smr_fragment blended with premultiplied alpha and stored as 8 bits (pipeline.rs:81-140).  A child input without a live
 * frame samples the empty view.  A tick draws the nodes below the roots in order of depth (1 + the deepest child's; an
 * input, text or image 0): the web nodes of depth 1 first, then per depth the resample passes and one composite launch
 * for its layout nodes, one launch per shader for its shader nodes and one launch for its web nodes; the roots'
 * composite comes last.
 * WebView (scene/web_view_component.rs): its size is the instance's resolution.  SMR_ERR_SCENE, the scene staying as it
 * was: an instance that is not registered (WebRendererNotFound), a child without an id (WebViewChildWithoutId), an
 * instance shown by two WebViews of any outputs, at any depth of nesting (WebRendererUsageNotExclusive).  The node texture
 * is transparent when the scene is set; each render with a frame clears it and draws the planes in the embedding order,
 * each child through its rect with the linear sampler and every plane blended with premultiplied alpha and stored as 8
 * bits (shader.rs:53-114).  A child input without a live frame draws nothing.  A View, Tiles or Rescaler child is a layout
 * node of its own, as under a Shader: its size is its width and height at the last render's pts, its layout state carries
 * over scene updates, every render evaluates and composites it whether or not the instance has a frame, and a
 * resolution of 0 or above 16384 draws nothing.  Below it any component may appear, Shaders and WebViews included (a
 * sizeless layout root there is UnknownDimensionsForLayoutNodeRoot).  SMR_ERR_UNSUPPORTED: a WebView or Shader child of a
 * WebView, and a View, Tiles or Rescaler child of a WebView without both width and height (Tiles: tiles_width and
 * tiles_height; View and Rescaler: the position's).  The reference answers UnknownDimensionsForLayoutNodeRoot for the
 * sizeless layout child and accepts the WebView and Shader children; these shapes keep the status they had before
 * layout children were accepted, so that callers that relied on it see no change.
 * Image (scene/image_component.rs): the node's resolution is round(image_width) x round(image_height); with one side
 * missing the other follows from the asset's aspect ratio, which the reference takes as the integer division
 * width / height (640 x 360 gives 1, a portrait asset 0); with both missing it is the asset's size.  A resolved side of 0
 * or above 16384 is SMR_ERR_SCENE and leaves the scene as it was.  A component with an id whose previous state is an Image
 * with the same id, image_id, width and height and the same asset keeps its start pts; anything else starts at the pts
 * of the last render.  The node texture is the asset frame sampled with the linear sampler at the node's resolution and
 * premultiplied (add_premultiplied_alpha.wgsl).  A Bitmap node is drawn by the first smr_render of the output after each
 * smr_update_scene of it.  An Animated node shows, at every tick, the frame whose pts is closest to
 * (pts - start_pts) % duration (the first such frame on a tie); pts - start_pts saturates at 0 where the reference's
 * subtraction would underflow.  A tick whose frame is the one the node texture already holds launches nothing for it.
 * An SVG node (smr_register_svg_image) is rasterised by the caller during smr_update_scene at the node's resolution and
 * drawn once, by the first smr_render of the output after the update, with its start pts and frame 0.  GpuOptimized
 * converts the raster as the reference's two passes do (remove_premultiplied_alpha.wgsl through UNORM views, then
 * add_premultiplied_alpha.wgsl through sRGB views); CpuOptimized stores its bytes unchanged.  A rasteriser that returns
 * non-zero is SMR_ERR_SCENE, smr_last_error naming the image id and the resolution, and leaves the scene as it was. */
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

/* gpu-video's transcoder resize (VideoTranscoder, vulkan_transcoder/shader.wgsl + pipeline.rs): one NV12 frame -> n NV12
 * renditions, each at its own size with its own ScalingAlgorithm, in ONE kernel launch ("decode once, encode a ladder").
 * `src` is an SMR_FRAME_NV12 frame, host or device; its width x height is the decoder's cropped extent with origin (0, 0),
 * so a 1920 x 1088 surface with a 1080-row crop is passed as height 1080 with the surface's pointers and pitch.  Nothing
 * outside the crop is read.  Each rendition's y plane has height rows of `width` bytes, its uv plane height / 2 rows of
 * width / 2 {u, v} pairs, each at its pitch (0 = tightly packed) in host or device memory per mem_kind; bytes past a
 * row's width are not written.  Arithmetic: DESIGN.md NC-10.  Blocking, like smr_preprocess_frame.
 * SMR_ERR_INVALID_ARGUMENT (checked before anything needs a device, so a host-only handle answers it too): n = 0 or
 * n > 8 (WrongOutputNumber), a rendition side that is 0, odd or above 16384, an unknown scaling, a null plane, a pitch
 * shorter than a row, an unknown mem_kind, an odd source side, and smr_render's checks of the source frame (size,
 * planes, pitch, device-plane alignment).  SMR_ERR_UNSUPPORTED: a source format other than NV12. */
typedef enum { SMR_SCALE_NEAREST = 0, SMR_SCALE_BILINEAR = 1, SMR_SCALE_LANCZOS3 = 2 } smr_scaling_algorithm;  /* ScalingAlgorithm as u32 */
typedef struct {
    uint32_t width, height;        /* TranscoderOutputParameters::output_width / output_height */
    int32_t scaling;               /* smr_scaling_algorithm */
    void *planes[2];               /* NV12: y, uv */
    uint32_t pitch[2];             /* 0 = tightly packed */
    int32_t mem_kind;              /* smr_mem_kind */
} smr_rendition;
#define SMR_MAX_RENDITIONS 8
smr_status smr_transcode_resize(smr_renderer *r, const smr_input_frame *src, const smr_rendition *out, uint32_t n);

/* gpu-video's frame converters (wgpu_helpers/: WgpuNv12ToRgbaConverter, WgpuRgbaToNv12Converter): one conversion per
 * call, on the renderer's stream, blocking like smr_preprocess_frame.  Both are full-target draws sampled with a linear,
 * clamp-to-edge sampler at the target's pixel centres, so a target of another size than the source is a bilinear
 * rescale.  The result does not depend on the renderer's rendering mode.
 * `converter` is the converter's WgpuConverterParameters; only (BT709, Limited) exists (OnlyLimitedBT709Supported:
 * SMR_ERR_UNSUPPORTED for every other pair).
 *
 * smr_video_nv12_to_rgba: `src` is an SMR_FRAME_NV12 frame, host or device, whose width x height is the decoder's crop
 * with origin (0, 0), as smr_transcode_resize takes it; nothing outside the crop is read.  `frame` is the decoded frame's
 * metadata: its color_space must be Unspecified or the converter's and its color_range the converter's
 * (IncompatibleFrame: SMR_ERR_INVALID_ARGUMENT).  `rgba` has out_height rows of `pitch` bytes (0 = tightly packed) in
 * host or device memory per mem_kind; bytes past a row's out_width x 4 are not written.  0 x 0 is the source size.
 * Arithmetic: DESIGN.md NC-11.
 * smr_video_rgba_to_nv12: `src` is an SMR_FRAME_RGBA8 frame of any size, read as raw bytes (an Rgba8Unorm view); alpha is
 * not used.  The target's y plane has out_height rows of out_width bytes, its uv plane out_height / 2 rows of
 * out_width / 2 {u, v} pairs, each at its pitch (0, or a NULL `pitch`: tightly packed); bytes past a row are not written.  The arithmetic is
 * K11's (rgba_to_nv12.wgsl), the kernel k_output's.
 * Checked before anything needs a device, so a host-only handle answers them too: SMR_ERR_UNSUPPORTED for the converter
 * pair and for a source format other than NV12 (nv12_to_rgba) or RGBA8 (rgba_to_nv12); SMR_ERR_INVALID_ARGUMENT for
 * an unknown enum value, an odd NV12 side, a target side of 0 (except 0 x 0 for nv12_to_rgba) or above 16384, an odd
 * NV12 target side, a null plane, a pitch shorter than a row, an unknown mem_kind, a device RGBA target whose pointer or
 * pitch is not 4-byte aligned, and smr_render's checks of the source frame (size, planes, pitch, device-plane alignment). */
typedef enum { SMR_COLOR_SPACE_UNSPECIFIED = 0, SMR_COLOR_SPACE_BT709 = 1, SMR_COLOR_SPACE_BT601_NTSC = 2,
               SMR_COLOR_SPACE_BT601_PAL = 3 } smr_color_space;                     /* gpu-video device.rs ColorSpace */
typedef enum { SMR_COLOR_RANGE_FULL = 0, SMR_COLOR_RANGE_LIMITED = 1 } smr_color_range;   /* device.rs ColorRange */
typedef struct { int32_t color_space, color_range; } smr_video_color;   /* WgpuConverterParameters / a frame's metadata */
smr_status smr_video_nv12_to_rgba(smr_renderer *r, smr_video_color converter, const smr_input_frame *src, smr_video_color frame,
                                  uint32_t out_width, uint32_t out_height, void *rgba, uint32_t pitch, int32_t mem_kind);
smr_status smr_video_rgba_to_nv12(smr_renderer *r, smr_video_color converter, const smr_input_frame *src, uint32_t out_width,
                                  uint32_t out_height, void *const planes[2], const uint32_t pitch[2], int32_t mem_kind);

/* Text nodes (SURVEY 8f-2): TextRendererNode::render (transformations/text_renderer.rs:72-167).  Shaping and glyph
 * rasterisation (cosmic-text / swash inside glyphon, CPU code in the reference too) stay on the caller's side; what the
 * reference does on the GPU -- clear the node texture to the component's background colour (:141-150) and draw glyphon's
 * prepared glyph quads over it (`text_renderer.render`, :163) -- happens here: `glyphs` is glyphon's GlyphToRender list
 * after its clipping to TextBounds (quad origin, size, atlas origin, colour, content type), the atlases are its mask
 * (R8) and colour (RGBA8) atlas pages.  Quads are alpha-blended in list order (wgpu::BlendState::ALPHA_BLENDING) through
 * the node texture's view.  color_mode: glyphon ColorMode, 0 = Accurate (TextAtlas::new, :95-100), 1 = Web.  The
 * result (width x height RGBA8, premultiplied by construction) is the text node's texture.  glyphs and atlases are HOST
 * memory; `rgba` per mem_kind.  Blocking.  A scene draws text through SMR_COMPONENT_TEXT (smr_text below) instead. */
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

/* The payload of a Text component (smr_component.text): StatefulTextComponent's laid-out buffer (scene/text_component.rs).
 * The caller shapes the text (cosmic-text) and prepares its glyphs (glyphon) as for smr_render_text; width x height is the
 * resolution its layout produced, which is the component's size in the scene (scene.rs:101-127).  smr_update_scene checks
 * it with smr_render_text's rules (SMR_ERR_INVALID_ARGUMENT: NULL payload, a glyph content other than COLOR / MASK, a
 * missing atlas, a side above 16384, more than 2^22 glyphs), except that 0 x 0 is legal: like the reference
 * (text_renderer.rs:77-85) its node texture is one transparent pixel.  Everything is copied before smr_update_scene
 * returns; an atlas several components pass by the same pointer is uploaded once.  The node texture is drawn by the first
 * smr_render of the output after each smr_update_scene of it (`was_rendered`, text_renderer.rs:73-75), then composited
 * like any premultiplied RGBA8 child. */
typedef struct smr_text {
    uint32_t width, height;
    smr_rgba background;
    const smr_glyph *glyphs;
    uint32_t n_glyphs;
    const smr_atlas *mask_atlas, *color_atlas;
    int32_t color_mode;
} smr_text;

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
/* inspection (no device needed): the host tables smr_transcode_resize's kernel reads for one axis of in_len source
 * texels and out_len output texels (each 1 .. 16384; a luma axis is (in, out), a chroma axis (in / 2, out / 2)).  Per
 * output coordinate k: nearest[k]; bilinear[2 k], bilinear[2 k + 1] = x0, x1 and frac[k]; center[k] and
 * lanczos[6 k .. 6 k + 5], the Lanczos3 weights of taps center - 2 .. center + 3 (DESIGN.md NC-10). */
smr_status smr_debug_transcode_taps(uint32_t in_len, uint32_t out_len, int32_t *nearest, int32_t *bilinear, float *frac,
                                    int32_t *center, float *lanczos);

smr_status smr_debug_tile_plan(const int32_t *boxes, uint32_t n_layers, uint32_t width, uint32_t height, int32_t sorted,
                               int32_t *owner_layer, uint32_t owner_cap, uint32_t *tiles, uint32_t tiles_cap, uint32_t *n_tiles);

/* inspection (no device access): the fused resample jobs of the handle's most recently planned tick, one record per job in
 * plan order, as they were launched -- after the partition, so `direct` already reflects a job sent back to the
 * composite because its piece of the launch was cut at an odd row.  *n is the job count; records go to `out` when they
 * fit in cap (SMR_ERR_BUFFER_TOO_SMALL otherwise; out = NULL asks for the count). */
typedef enum {
    SMR_FUSED_LDG = 0,             /* k_resample_fused_int<ratio, src_class, matrix, full_range of UYVY / YUYV> */
    SMR_FUSED_TMA_INT = 1,         /* k_resample_tma3<ratio, src_class, full_range, matrix> */
    SMR_FUSED_TMA_ANY = 2          /* k_resample_tma0<src_class, window, box, matrix> */
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
    int32_t matrix;                /* the source's matrix: SMR_MATRIX_BT709 or SMR_MATRIX_BT601 */
} smr_fused_job_info;
smr_status smr_debug_fused_jobs(smr_renderer *r, smr_fused_job_info *out, uint32_t cap, uint32_t *n);
/* inspection (no handle, no device access): the fused resample kernel instantiations the library is compiled with, one
 * record per instantiation.  A fused launch runs the jobs of one record, and a job whose record is missing fails its tick
 * with SMR_ERR_CUDA.  *n is the record count; records go to `out` when they fit in cap (SMR_ERR_BUFFER_TOO_SMALL
 * otherwise; out = NULL asks for the count). */
typedef struct {
    int32_t kernel;                /* smr_fused_kernel */
    int32_t ratio;                 /* as in smr_fused_job_info */
    int32_t window;                /* as in smr_fused_job_info: 20, 25, 29 or 33 slots for SMR_FUSED_TMA_ANY, else 0 */
    int32_t box;                   /* as in smr_fused_job_info */
    int32_t src_class;             /* 0 planar 4:2:0, 1 NV12, 2 UYVY, 3 YUYV */
    int32_t range;                 /* the range the kernel is specialised for: 1 full; 0 limited, or read per job */
    int32_t matrix;                /* smr_yuv_matrix: SMR_MATRIX_BT709 or SMR_MATRIX_BT601 */
} smr_fused_variant_info;
smr_status smr_debug_fused_variants(smr_fused_variant_info *out, uint32_t cap, uint32_t *n);

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
    int32_t tex_matrix;            /* a YUV texture's matrix: SMR_MATRIX_BT709 or SMR_MATRIX_BT601; 0 for other kinds */
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
/* inspection (no device needed): the same for any layout node of an output's render graph.  node 0 is the root when the
 * root is a layout (for an output of smr_set_layouts, the root layout it was given); the layout nodes below it (a View,
 * Tiles or Rescaler child of a Shader) follow in DFS order, children before parents.  root_width x root_height is the node's resolution at pts.  SMR_ERR_INVALID_ARGUMENT: no such node. */
smr_status smr_debug_node_layouts(smr_renderer *r, const char *output_id, uint32_t node, uint64_t pts_ns,
                                  smr_render_layout *out, uint32_t capacity, uint32_t *n_out,
                                  uint32_t *root_width, uint32_t *root_height);
/* inspection (no device needed): the image nodes of an output's scene, the root or the node children in DFS order: the
 * node's resolution, its start pts, and the asset frame a render at pts_ns shows.  SMR_ERR_BUFFER_TOO_SMALL when they do
 * not fit in capacity (out = NULL asks for the count). */
typedef struct { uint32_t width, height; uint64_t start_pts_ns; uint32_t frame; } smr_image_node_info;
smr_status smr_debug_image_nodes(smr_renderer *r, const char *output_id, uint64_t pts_ns, smr_image_node_info *out,
                                 uint32_t capacity, uint32_t *n_out);

/* The FLATTENED form of the boundary (SURVEY 8b): a host that keeps the reference's scene/ tree (Component tree,
 * transitions, NestedLayout::flatten -- all Rust) hands over, per output and whenever they change, the RenderLayout[]
 * that transformations/layout/params.rs:169-333 would pack into uniform blocks: same fields, same units (pixels of
 * the root_width x root_height layout node texture), painter's order.  child_ids[k] is the input id of the node's
 * k-th child (scene/layout.rs:84-93), which `child_index` of a texture layout refers to; children here are inputs only
 * (a Text child needs smr_update_scene, or its texture from smr_render_text passed as an input).  Registers the output like
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
