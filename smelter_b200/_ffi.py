"""ctypes view of include/smelter_b200.h.  Loading fails loudly when the CUDA library is missing:
there is no CPU fallback behind this package."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# SMR_LIB_PATH: a differently built copy of the same library (e.g. another revision's build, for an A/B comparison)
LIB_PATH = os.environ.get("SMR_LIB_PATH") or os.path.join(_HERE, "libsmelter_b200.so")

SMR_OK = 0
STATUS_NAMES = {0: "SMR_OK", 1: "SMR_ERR_INVALID_ARGUMENT", 2: "SMR_ERR_CUDA", 3: "SMR_ERR_OUTPUT_NOT_REGISTERED",
                4: "SMR_ERR_SCENE", 5: "SMR_ERR_UNSUPPORTED", 6: "SMR_ERR_OUT_OF_MEMORY", 7: "SMR_ERR_BUFFER_TOO_SMALL"}

MODE_GPU_OPTIMIZED, MODE_CPU_OPTIMIZED = 0, 1
COMPONENT_INPUT_STREAM, COMPONENT_VIEW, COMPONENT_TILES, COMPONENT_RESCALER = 0, 1, 2, 3
COMPONENT_SHADER, COMPONENT_WEB_VIEW, COMPONENT_IMAGE, COMPONENT_TEXT = 4, 5, 6, 7
FRAME_PLANAR_YUV420, FRAME_PLANAR_YUVJ420, FRAME_NV12, FRAME_BGRA, FRAME_ARGB, FRAME_RGBA8 = 0, 1, 2, 3, 4, 5
FRAME_PLANAR_YUV422, FRAME_PLANAR_YUV444, FRAME_UYVY422, FRAME_YUYV422 = 6, 7, 8, 9
MEM_HOST, MEM_DEVICE = 0, 1
OUT_PLANAR_YUV420, OUT_PLANAR_YUV422, OUT_PLANAR_YUV444, OUT_RGBA8, OUT_NV12 = 0, 1, 2, 3, 4
MAX_MASKS = 20


class Options(C.Structure):
    _fields_ = [("cuda_device", C.c_int32), ("rendering_mode", C.c_int32), ("max_layouts_count", C.c_uint32),
                ("stream_fallback_timeout_ns", C.c_uint64), ("framerate_num", C.c_uint32), ("framerate_den", C.c_uint32)]


class Rgba(C.Structure):
    _fields_ = [("r", C.c_uint8), ("g", C.c_uint8), ("b", C.c_uint8), ("a", C.c_uint8)]


class BorderRadius(C.Structure):
    _fields_ = [("top_left", C.c_float), ("top_right", C.c_float), ("bottom_right", C.c_float), ("bottom_left", C.c_float)]


class BoxShadow(C.Structure):
    _fields_ = [("offset_x", C.c_float), ("offset_y", C.c_float), ("blur_radius", C.c_float), ("color", Rgba)]


class Padding(C.Structure):
    _fields_ = [("top", C.c_float), ("right", C.c_float), ("bottom", C.c_float), ("left", C.c_float)]


class OptF32(C.Structure):
    _fields_ = [("has_value", C.c_int32), ("value", C.c_float)]


class Transition(C.Structure):
    _fields_ = [("present", C.c_int32), ("duration_ns", C.c_uint64), ("interpolation_kind", C.c_int32),
                ("x1", C.c_double), ("y1", C.c_double), ("x2", C.c_double), ("y2", C.c_double),
                ("should_interrupt", C.c_int32)]


class Position(C.Structure):
    _fields_ = [("is_absolute", C.c_int32), ("width", OptF32), ("height", OptF32),
                ("horizontal_from_right", C.c_int32), ("horizontal_offset", C.c_float),
                ("vertical_from_bottom", C.c_int32), ("vertical_offset", C.c_float),
                ("rotation_degrees", C.c_float)]


class Component(C.Structure):
    pass


Component._fields_ = [
    ("type", C.c_int32), ("id", C.c_char_p), ("children", C.POINTER(Component)), ("children_len", C.c_uint32),
    ("input_id", C.c_char_p),
    ("position", Position), ("transition", Transition), ("border_radius", BorderRadius),
    ("border_width", C.c_float), ("border_color", Rgba), ("box_shadow", C.POINTER(BoxShadow)),
    ("box_shadow_len", C.c_uint32),
    ("direction", C.c_int32), ("overflow", C.c_int32), ("background_color", Rgba), ("padding", Padding),
    ("rescale_mode", C.c_int32), ("horizontal_align", C.c_int32), ("vertical_align", C.c_int32),
    ("tiles_width", OptF32), ("tiles_height", OptF32),
    ("tile_aspect_ratio_w", C.c_uint32), ("tile_aspect_ratio_h", C.c_uint32),
    ("tiles_margin", C.c_float), ("tiles_padding", C.c_float),
]


class InputFrame(C.Structure):
    _fields_ = [("input_id", C.c_char_p), ("format", C.c_int32), ("width", C.c_uint32), ("height", C.c_uint32),
                ("pts_ns", C.c_uint64), ("planes", C.c_void_p * 3), ("pitch", C.c_uint32 * 3), ("mem_kind", C.c_int32)]


class OutputFrame(C.Structure):
    _fields_ = [("output_id", C.c_char_p), ("planes", C.c_void_p * 3), ("pitch", C.c_uint32 * 3),
                ("mem_kind", C.c_int32), ("width", C.c_uint32), ("height", C.c_uint32), ("format", C.c_int32),
                ("pts_ns", C.c_uint64)]


class Mask(C.Structure):
    _fields_ = [("radius", C.c_float * 4), ("top", C.c_float), ("left", C.c_float), ("width", C.c_float),
                ("height", C.c_float)]


class RenderLayout(C.Structure):
    _fields_ = [("type", C.c_int32), ("top", C.c_float), ("left", C.c_float), ("width", C.c_float),
                ("height", C.c_float), ("rotation_degrees", C.c_float), ("border_radius", C.c_float * 4),
                ("color", Rgba), ("border_color", Rgba), ("border_width", C.c_float), ("blur_radius", C.c_float),
                ("child_index", C.c_int32), ("crop_top", C.c_float), ("crop_left", C.c_float),
                ("crop_width", C.c_float), ("crop_height", C.c_float), ("masks_len", C.c_int32),
                ("masks", Mask * MAX_MASKS)]


class Atlas(C.Structure):       # smr_atlas
    _fields_ = [("data", C.c_void_p), ("width", C.c_uint32), ("height", C.c_uint32), ("pitch", C.c_uint32)]


GLYPH_COLOR, GLYPH_MASK = 0, 1
# smr_glyph as a numpy record (24 bytes, the C layout): glyphon's GlyphToRender after clipping
GLYPH_DTYPE = [("x", "<i4"), ("y", "<i4"), ("width", "<u2"), ("height", "<u2"), ("atlas_x", "<u2"), ("atlas_y", "<u2"),
               ("color", "u1", (4,)), ("content", "<i4")]


class Stats(C.Structure):
    _fields_ = [("frames_rendered", C.c_uint64), ("kernel_launches", C.c_uint64), ("h2d_bytes", C.c_uint64),
                ("d2h_bytes", C.c_uint64), ("last_render_kernel_launches", C.c_uint64), ("last_render_direct_tiles", C.c_uint64)]


FUSED_LDG, FUSED_TMA_INT, FUSED_TMA_ANY = 0, 1, 2


class FusedJobInfo(C.Structure):   # smr_fused_job_info
    _fields_ = [("kernel", C.c_int32), ("ratio", C.c_int32), ("window", C.c_int32), ("box", C.c_int32),
                ("src_class", C.c_int32), ("full_range", C.c_int32), ("v_same", C.c_int32), ("strip_cols", C.c_int32),
                ("src_width", C.c_uint32), ("src_height", C.c_uint32), ("dst_width", C.c_uint32), ("dst_height", C.c_uint32),
                ("taps_h", C.c_int32), ("taps_v", C.c_int32), ("direct", C.c_int32)]


STAGE_BOX, STAGE_FIRST, STAGE_LAST = 0, 1, 2
STAGE_SRC_RAW, STAGE_SRC_CONVERTED, STAGE_SRC_F16 = 0, 1, 2


class ResampleStageInfo(C.Structure):   # smr_resample_stage_info
    _fields_ = [("stage", C.c_int32), ("axis", C.c_int32), ("box_fx", C.c_int32), ("box_fy", C.c_int32), ("taps", C.c_int32),
                ("perp_offset", C.c_int32), ("source", C.c_int32), ("src_kind", C.c_int32), ("src_width", C.c_uint32),
                ("src_height", C.c_uint32), ("dst_width", C.c_uint32), ("dst_height", C.c_uint32), ("dst_f16", C.c_int32)]


COMPOSITE_PARAM, COMPOSITE_MULTI = 0, 1


class CompositeLayerInfo(C.Structure):   # smr_composite_layer_info
    _fields_ = [("job", C.c_int32), ("kernel", C.c_int32), ("layer", C.c_int32), ("type", C.c_int32), ("rotated", C.c_int32),
                ("fast", C.c_int32), ("box", C.c_int32 * 12), ("tx_off", C.c_int32), ("ty_off", C.c_int32),
                ("mask_count", C.c_int32), ("tex_kind", C.c_int32), ("tex_width", C.c_int32), ("tex_height", C.c_int32),
                ("tex_pitch", C.c_int32 * 3), ("tex_align", C.c_int32 * 3), ("width", C.c_int32), ("height", C.c_int32),
                ("out_format", C.c_int32)]


KERNEL_CLASSES = ["convert", "weights", "resample_box", "resample_first", "resample_last", "composite", "output",
                  "fill", "resample_fused"]


class KernelTimes(C.Structure):
    _fields_ = [("total_ms", C.c_double * 9), ("launches", C.c_uint64 * 9)]


EXPORTS = [
    "smr_create", "smr_destroy", "smr_register_input", "smr_unregister_input", "smr_update_scene",
    "smr_unregister_output", "smr_set_layouts", "smr_render", "smr_render_begin", "smr_render_end", "smr_preprocess_frame", "smr_premultiply_rgba8", "smr_render_text", "smr_debug_partition", "smr_debug_tile_plan", "smr_debug_weights", "smr_debug_sincos", "smr_debug_fused_jobs", "smr_debug_resample_stages", "smr_debug_composite_layers", "smr_debug_interior", "smr_output_plane_sizes",
    "smr_component_default", "smr_debug_layouts", "smr_debug_set_inputs", "smr_get_stats", "smr_set_profiling", "smr_get_kernel_times",
    "smr_comm_get_unique_id", "smr_comm_init", "smr_comm_broadcast_inputs", "smr_comm_exchange_inputs", "smr_comm_pull_inputs", "smr_peer_pool_alloc", "smr_peer_pool_open", "smr_peer_pool_close", "smr_peer_pool_free", "smr_comm_destroy", "smr_host_register", "smr_host_unregister", "smr_cuda_stream", "smr_last_error",
    "smr_version",
]

_lib = None


def lib():
    """The C-ABI library.  Raises (never falls back) if it was not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -m smelter_b200.build` "
            "(the H100 compositor has no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    L.smr_create.argtypes = [C.POINTER(Options), C.POINTER(vp)]
    L.smr_destroy.argtypes = [vp]
    L.smr_destroy.restype = None
    L.smr_register_input.argtypes = [vp, C.c_char_p]
    L.smr_unregister_input.argtypes = [vp, C.c_char_p]
    L.smr_update_scene.argtypes = [vp, C.c_char_p, C.c_uint32, C.c_uint32, C.c_int32, C.POINTER(Component)]
    L.smr_unregister_output.argtypes = [vp, C.c_char_p]
    for f in (L.smr_render, L.smr_render_begin):
        f.argtypes = [vp, C.c_uint64, C.POINTER(InputFrame), C.c_uint32, C.POINTER(OutputFrame), C.c_uint32]
    L.smr_render_end.argtypes = [vp]
    L.smr_preprocess_frame.argtypes = [vp, C.POINTER(InputFrame), C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_int32]
    L.smr_preprocess_frame.restype = C.c_int32
    L.smr_premultiply_rgba8.argtypes = [vp, C.POINTER(InputFrame), C.c_void_p, C.c_uint32, C.c_int32]
    L.smr_premultiply_rgba8.restype = C.c_int32
    L.smr_render_text.argtypes = [vp, C.c_uint32, C.c_uint32, Rgba, C.c_void_p, C.c_uint32, C.POINTER(Atlas), C.POINTER(Atlas),
                                  C.c_int32, C.c_void_p, C.c_uint32, C.c_int32]
    L.smr_render_text.restype = C.c_int32
    L.smr_debug_partition.argtypes = [C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_uint32, C.c_uint32, C.POINTER(C.c_int32),
                                      C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_int32), C.c_uint32, C.POINTER(C.c_uint32)]
    L.smr_debug_partition.restype = C.c_int32
    L.smr_debug_tile_plan.argtypes = [C.POINTER(C.c_int32), C.c_uint32, C.c_uint32, C.c_uint32, C.c_int32, C.POINTER(C.c_int32), C.c_uint32,
                                      C.POINTER(C.c_uint32), C.c_uint32, C.POINTER(C.c_uint32)]
    L.smr_debug_tile_plan.restype = C.c_int32
    L.smr_debug_weights.argtypes = [C.c_float, C.c_float, C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(C.c_uint32), C.c_void_p,
                                    C.c_void_p]
    L.smr_debug_weights.restype = C.c_int32
    L.smr_debug_sincos.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    L.smr_debug_sincos.restype = C.c_int32
    L.smr_debug_fused_jobs.argtypes = [vp, C.POINTER(FusedJobInfo), C.c_uint32, C.POINTER(C.c_uint32)]
    L.smr_debug_fused_jobs.restype = C.c_int32
    L.smr_debug_resample_stages.argtypes = [vp, C.POINTER(ResampleStageInfo), C.c_uint32, C.POINTER(C.c_uint32),
                                            C.POINTER(C.c_int32), C.c_uint32, C.POINTER(C.c_uint32)]
    L.smr_debug_resample_stages.restype = C.c_int32
    L.smr_debug_composite_layers.argtypes = [vp, C.POINTER(CompositeLayerInfo), C.c_uint32, C.POINTER(C.c_uint32)]
    L.smr_debug_composite_layers.restype = C.c_int32
    L.smr_debug_interior.argtypes = [C.POINTER(RenderLayout), C.c_uint32, C.c_uint32, C.POINTER(C.c_int32 * 12), C.c_void_p]
    L.smr_debug_interior.restype = C.c_int32
    L.smr_output_plane_sizes.argtypes = [C.c_uint32, C.c_uint32, C.c_int32, C.POINTER(C.c_size_t * 3)]
    L.smr_component_default.argtypes = [C.c_int32, C.POINTER(Component)]
    L.smr_component_default.restype = None
    L.smr_debug_layouts.argtypes = [vp, C.c_char_p, C.c_uint64, C.POINTER(RenderLayout), C.c_uint32,
                                    C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    L.smr_debug_set_inputs.argtypes = [vp, C.c_uint64, C.POINTER(InputFrame), C.c_uint32]
    L.smr_get_stats.argtypes = [vp, C.POINTER(Stats)]
    L.smr_comm_get_unique_id.argtypes = [C.POINTER(C.c_uint8 * 128)]
    L.smr_comm_init.argtypes = [vp, C.POINTER(C.c_uint8 * 128), C.c_int32, C.c_int32]
    L.smr_comm_broadcast_inputs.argtypes = [vp, C.POINTER(InputFrame), C.c_uint32, C.POINTER(C.c_int32)]
    L.smr_set_layouts.argtypes = [vp, C.c_char_p, C.c_uint32, C.c_uint32, C.c_int32, C.c_uint32, C.c_uint32,
                                  C.POINTER(C.c_char_p), C.c_uint32, C.POINTER(RenderLayout), C.c_uint32]
    L.smr_host_register.argtypes = [C.c_void_p, C.c_size_t]
    L.smr_host_unregister.argtypes = [C.c_void_p]
    L.smr_comm_exchange_inputs.argtypes = [vp, C.POINTER(InputFrame), C.c_uint32, C.POINTER(C.c_int32), C.POINTER(C.c_uint64),
                                           C.c_uint32]
    L.smr_comm_pull_inputs.argtypes = [vp, C.POINTER(InputFrame), C.POINTER(InputFrame), C.c_uint32, C.POINTER(C.c_int32),
                                       C.POINTER(C.c_uint64)]
    L.smr_peer_pool_alloc.argtypes = [vp, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_uint8 * 64)]
    L.smr_peer_pool_open.argtypes = [vp, C.POINTER(C.c_uint8 * 64), C.POINTER(C.c_void_p)]
    L.smr_peer_pool_close.argtypes = [vp, C.c_void_p]
    L.smr_peer_pool_free.argtypes = [vp, C.c_void_p]
    L.smr_comm_destroy.argtypes = [vp]
    L.smr_set_profiling.argtypes = [vp, C.c_int32]
    L.smr_get_kernel_times.argtypes = [vp, C.POINTER(KernelTimes)]
    L.smr_cuda_stream.argtypes = [vp]
    L.smr_cuda_stream.restype = vp
    L.smr_last_error.argtypes = [vp]
    L.smr_last_error.restype = C.c_char_p
    L.smr_version.restype = C.c_char_p
    _lib = L
    return L
