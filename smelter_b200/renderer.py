"""Python mirror of the reference's renderer interface over the C ABI.

Names, argument meaning and error behaviour follow `smelter_render::Renderer`
(smelter-render/src/state.rs:95-193), `scene::Component` (scene/components.rs) and
`Frame/FrameData/FrameSet` (types.rs:21-119) so the parity tests read like the reference's render tests
(integration-tests/src/render_tests/harness/test_case.rs).  Nothing here computes pixels: every call
goes to libsmelter_b200.so (hand-written sm_90a kernels).
"""
import ctypes as C
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple, Union

import numpy as np

from . import _ffi as F


class RendererError(RuntimeError):
    def __init__(self, status, message):
        super().__init__(f"{F.STATUS_NAMES.get(status, status)}: {message}")
        self.status = status


class UpdateSceneError(RendererError):
    pass


class RenderSceneError(RendererError):
    pass


# ------------------------------------------------------------------------------------------------
# types.rs
# ------------------------------------------------------------------------------------------------
class RenderingMode:
    GpuOptimized = F.MODE_GPU_OPTIMIZED
    CpuOptimized = F.MODE_CPU_OPTIMIZED


class OutputFrameFormat:
    PlanarYuv420Bytes = F.OUT_PLANAR_YUV420
    PlanarYuv422Bytes = F.OUT_PLANAR_YUV422
    PlanarYuv444Bytes = F.OUT_PLANAR_YUV444
    RgbaWgpuTexture = F.OUT_RGBA8   # RGBA8 premultiplied texture (device or host buffer here)
    Nv12WgpuTexture = F.OUT_NV12


@dataclass(frozen=True)
class Resolution:
    width: int
    height: int


@dataclass
class YuvPlanes:
    y_plane: np.ndarray
    u_plane: np.ndarray
    v_plane: np.ndarray


@dataclass
class NvPlanes:
    y_plane: np.ndarray
    uv_planes: np.ndarray


@dataclass
class FrameData:
    """FrameData enum: kind in {PlanarYuv420, PlanarYuv422, PlanarYuv444, PlanarYuvJ420, InterleavedUyvy422,
    InterleavedYuyv422, Nv12, Bgra, Argb, Rgba8}.
    `planes` are numpy arrays (host) or integer device pointers (device=True)."""
    kind: str
    planes: tuple
    device: bool = False

    @staticmethod
    def PlanarYuv420(p: YuvPlanes):
        return FrameData("PlanarYuv420", (p.y_plane, p.u_plane, p.v_plane))

    @staticmethod
    def PlanarYuv422(p: YuvPlanes):
        return FrameData("PlanarYuv422", (p.y_plane, p.u_plane, p.v_plane))

    @staticmethod
    def PlanarYuv444(p: YuvPlanes):
        return FrameData("PlanarYuv444", (p.y_plane, p.u_plane, p.v_plane))

    @staticmethod
    def InterleavedUyvy422(data):
        return FrameData("InterleavedUyvy422", (data,))

    @staticmethod
    def InterleavedYuyv422(data):
        return FrameData("InterleavedYuyv422", (data,))

    @staticmethod
    def PlanarYuvJ420(p: YuvPlanes):
        return FrameData("PlanarYuvJ420", (p.y_plane, p.u_plane, p.v_plane))

    @staticmethod
    def Nv12(p: NvPlanes):
        return FrameData("Nv12", (p.y_plane, p.uv_planes))

    @staticmethod
    def Bgra(data):
        return FrameData("Bgra", (data,))

    @staticmethod
    def Argb(data):
        return FrameData("Argb", (data,))

    @staticmethod
    def Rgba8(data):
        return FrameData("Rgba8", (data,))


_FRAME_KIND = {"PlanarYuv420": F.FRAME_PLANAR_YUV420, "PlanarYuvJ420": F.FRAME_PLANAR_YUVJ420,
               "Nv12": F.FRAME_NV12, "Bgra": F.FRAME_BGRA, "Argb": F.FRAME_ARGB, "Rgba8": F.FRAME_RGBA8,
               "PlanarYuv422": F.FRAME_PLANAR_YUV422, "PlanarYuv444": F.FRAME_PLANAR_YUV444,
               "InterleavedUyvy422": F.FRAME_UYVY422, "InterleavedYuyv422": F.FRAME_YUYV422}


def plane_shapes(fmt: int, width: int, height: int) -> List[Tuple[int, int]]:
    """(rows, row bytes) of each plane of a width x height frame of smr_frame_format `fmt`, as the library reads it"""
    cw, ch = width // 2, height // 2
    if fmt in (F.FRAME_PLANAR_YUV420, F.FRAME_PLANAR_YUVJ420):
        return [(height, width), (ch, cw), (ch, cw)]
    if fmt == F.FRAME_NV12:
        return [(height, width), (ch, 2 * cw)]
    if fmt == F.FRAME_PLANAR_YUV422:
        return [(height, width), (height, cw), (height, cw)]
    if fmt == F.FRAME_PLANAR_YUV444:
        return [(height, width)] * 3
    if fmt in (F.FRAME_UYVY422, F.FRAME_YUYV422):
        return [(height, 4 * cw)]
    if fmt in (F.FRAME_BGRA, F.FRAME_ARGB, F.FRAME_RGBA8):
        return [(height, 4 * width)]
    raise ValueError(f"unknown frame format {fmt}")


class DeinterlaceMode:   # smr_deinterlace_mode
    Off = F.DEINTERLACE_OFF
    Field = F.DEINTERLACE_FIELD
    MotionAdaptive = F.DEINTERLACE_MOTION_ADAPTIVE


class FieldOrder:        # smr_field_order
    TopFirst = F.FIELD_TOP_FIRST
    BottomFirst = F.FIELD_BOTTOM_FIRST


class YuvMatrix:         # smr_yuv_matrix
    Default = F.MATRIX_DEFAULT   # BT.709
    BT709 = F.MATRIX_BT709
    BT601 = F.MATRIX_BT601


class YuvRange:          # smr_yuv_range
    Default = F.RANGE_DEFAULT    # full for PLANAR_YUVJ420, limited for every other YUV format
    Limited = F.RANGE_LIMITED
    Full = F.RANGE_FULL


@dataclass
class Frame:
    data: FrameData
    resolution: Resolution
    pts: float = 0.0   # seconds (Duration)


@dataclass
class FrameSet:
    frames: Dict[str, Frame] = field(default_factory=dict)
    pts: float = 0.0


class ScalingAlgorithm:
    """gpu-video's ScalingAlgorithm (parameters.rs), the filter of one transcoder rendition"""
    NearestNeighbor = F.SCALE_NEAREST
    Bilinear = F.SCALE_BILINEAR
    Lanczos3 = F.SCALE_LANCZOS3


class ColorSpace:
    """gpu-video's ColorSpace (device.rs), a decoded frame's or a converter's colour space"""
    Unspecified = F.COLOR_SPACE_UNSPECIFIED
    BT709 = F.COLOR_SPACE_BT709
    BT601Ntsc = F.COLOR_SPACE_BT601_NTSC
    BT601Pal = F.COLOR_SPACE_BT601_PAL


class ColorRange:
    """gpu-video's ColorRange (device.rs)"""
    Full = F.COLOR_RANGE_FULL
    Limited = F.COLOR_RANGE_LIMITED


class FramePreProcessor:
    """smelter_render::FramePreProcessor (state/frame_pre_processor.rs:33-116) over a Renderer handle."""

    def __init__(self, renderer):
        self._r = renderer

    def process_to_bytes(self, frame: "Frame", resolution: Optional["Resolution"] = None) -> np.ndarray:
        return self._r.preprocess_frame(frame, resolution)


# ------------------------------------------------------------------------------------------------
# scene types (scene/types.rs, scene/components.rs) -- same field names and defaults
# ------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class RGBAColor:
    r: int = 0
    g: int = 0
    b: int = 0
    a: int = 0


@dataclass(frozen=True)
class BorderRadius:
    top_left: float = 0.0
    top_right: float = 0.0
    bottom_right: float = 0.0
    bottom_left: float = 0.0

    @staticmethod
    def new_with_radius(r):
        return BorderRadius(r, r, r, r)


BorderRadius.ZERO = BorderRadius()


@dataclass(frozen=True)
class BoxShadow:
    offset_x: float = 0.0
    offset_y: float = 0.0
    blur_radius: float = 0.0
    color: RGBAColor = RGBAColor()


@dataclass(frozen=True)
class Padding:
    top: float = 0.0
    right: float = 0.0
    bottom: float = 0.0
    left: float = 0.0


class HorizontalAlign:
    Left, Right, Justified, Center = 0, 1, 2, 3


class VerticalAlign:
    Top, Center, Bottom, Justified = 0, 1, 2, 3


class Overflow:
    Visible, Hidden, Fit = 0, 1, 2


class ViewChildrenDirection:
    Row, Column = 0, 1


class RescaleMode:
    Fit, Fill = 0, 1


@dataclass(frozen=True)
class InterpolationKind:
    kind: int = 0  # 0 Linear, 1 Bounce, 2 CubicBezier
    x1: float = 0.0
    y1: float = 0.0
    x2: float = 0.0
    y2: float = 0.0


InterpolationKind.Linear = InterpolationKind(0)
InterpolationKind.Bounce = InterpolationKind(1)
InterpolationKind.CubicBezier = staticmethod(lambda x1, y1, x2, y2: InterpolationKind(2, x1, y1, x2, y2))


@dataclass(frozen=True)
class Transition:
    duration: float = 0.0  # seconds
    interpolation_kind: InterpolationKind = InterpolationKind()
    should_interrupt: bool = False


@dataclass(frozen=True)
class Position:
    """Position::Static{width,height} or Position::Absolute(AbsolutePosition)."""
    absolute: bool = False
    width: Optional[float] = None
    height: Optional[float] = None
    left: Optional[float] = None     # HorizontalPosition::LeftOffset
    right: Optional[float] = None    # HorizontalPosition::RightOffset
    top: Optional[float] = None      # VerticalPosition::TopOffset
    bottom: Optional[float] = None   # VerticalPosition::BottomOffset
    rotation_degrees: float = 0.0

    @staticmethod
    def Static(width=None, height=None):
        return Position(False, width, height)

    @staticmethod
    def Absolute(width=None, height=None, left=None, right=None, top=None, bottom=None, rotation_degrees=0.0):
        return Position(True, width, height, left, right, top, bottom, rotation_degrees)


@dataclass
class InputStreamComponent:
    input_id: str = ""
    id: Optional[str] = None


@dataclass
class ViewComponent:
    id: Optional[str] = None
    children: list = field(default_factory=list)
    direction: int = ViewChildrenDirection.Row
    position: Position = Position()
    transition: Optional[Transition] = None
    overflow: int = Overflow.Hidden
    background_color: RGBAColor = RGBAColor(0, 0, 0, 0)
    border_radius: BorderRadius = BorderRadius()
    border_width: float = 0.0
    border_color: RGBAColor = RGBAColor(0, 0, 0, 0)
    box_shadow: list = field(default_factory=list)
    padding: Padding = Padding()


@dataclass
class RescalerComponent:
    child: object = None
    id: Optional[str] = None
    position: Position = Position()
    transition: Optional[Transition] = None
    mode: int = RescaleMode.Fit
    horizontal_align: int = HorizontalAlign.Center
    vertical_align: int = VerticalAlign.Center
    border_radius: BorderRadius = BorderRadius()
    border_width: float = 0.0
    border_color: RGBAColor = RGBAColor(0, 0, 0, 0)
    box_shadow: list = field(default_factory=list)


@dataclass
class TilesComponent:
    id: Optional[str] = None
    children: list = field(default_factory=list)
    width: Optional[float] = None
    height: Optional[float] = None
    background_color: RGBAColor = RGBAColor(0, 0, 0, 0)
    tile_aspect_ratio: Tuple[int, int] = (16, 9)
    margin: float = 0.0
    padding: float = 0.0
    horizontal_align: int = HorizontalAlign.Center
    vertical_align: int = VerticalAlign.Center
    transition: Optional[Transition] = None


@dataclass
class TextComponent:
    """A Text component as the caller laid it out (smr_text): cosmic-text's resolution (width x height) and glyphon's
    prepared glyph quads (records of _ffi.GLYPH_DTYPE, painter's order) over its mask atlas ((h, w) uint8) and colour
    atlas ((h, w, 4) uint8).  color_mode: glyphon ColorMode, 0 Accurate, 1 Web."""
    id: Optional[str] = None
    width: int = 0
    height: int = 0
    background_color: RGBAColor = RGBAColor(0, 0, 0, 0)
    glyphs: Optional[np.ndarray] = None
    mask_atlas: Optional[np.ndarray] = None
    color_atlas: Optional[np.ndarray] = None
    color_mode: int = 0


@dataclass
class ImageComponent:
    """An Image component (scene/components.rs:63-80): the asset registered as `image_id` (Renderer.register_image), shown at
    width x height; a missing side follows from the asset's aspect ratio, both missing: the asset's size."""
    id: Optional[str] = None
    image_id: str = ""
    width: Optional[float] = None
    height: Optional[float] = None


@dataclass
class WebViewComponent:
    """A WebView component (scene/components.rs:55-61): the web renderer instance registered as `instance_id`
    (Renderer.register_web_renderer) at its resolution, with `children` (each with an id) drawn at the instance's child
    rects (Renderer.set_web_child_rects).  A child is an InputStream, Image or Text component, or a View, Tiles or Rescaler
    with both width and height (Tiles: width and height; View and Rescaler: the position's), which is a layout node of its
    own and may hold any component, Shaders and WebViews included.  A WebView or Shader child, and a View, Tiles or
    Rescaler child without both sides, raise RendererError with status SMR_ERR_UNSUPPORTED."""
    id: Optional[str] = None
    instance_id: str = ""
    children: List["Component"] = field(default_factory=list)


@dataclass
class ShaderParam:
    """A ShaderParam value (scene/components.rs:40-55): kind one of "f32", "u32", "i32" (value: the scalar), "list" (value:
    a list of ShaderParam) or "struct" (value: a list of (field name, ShaderParam) pairs)."""
    kind: str
    value: object

    @staticmethod
    def f32(v):
        return ShaderParam("f32", float(v))

    @staticmethod
    def u32(v):
        return ShaderParam("u32", int(v))

    @staticmethod
    def i32(v):
        return ShaderParam("i32", int(v))

    @staticmethod
    def list(items):
        return ShaderParam("list", list(items))

    @staticmethod
    def struct(fields):
        return ShaderParam("struct", [(str(n), v) for n, v in fields])


@dataclass
class ShaderParamType:
    """The type of a shader's parameter (smr_shader_param_type): kind "f32", "u32", "i32", "list" (item: the element type,
    length: the element count) or "struct" (fields: (name, ShaderParamType) pairs)."""
    kind: str
    item: Optional["ShaderParamType"] = None
    length: int = 0
    fields: List[Tuple[str, "ShaderParamType"]] = field(default_factory=list)


@dataclass
class ShaderComponent:
    """A Shader component (scene/components.rs:29-38): the shader registered as `shader_id` (Renderer.register_shader) drawn
    into a node of width x height, with `children` as its textures and `shader_param` as its parameter (None: none)."""
    id: Optional[str] = None
    shader_id: str = ""
    shader_param: Optional[ShaderParam] = None
    width: float = 0.0
    height: float = 0.0
    children: List["Component"] = field(default_factory=list)


Component = Union[InputStreamComponent, ViewComponent, RescalerComponent, TilesComponent, TextComponent, ImageComponent,
                  WebViewComponent, ShaderComponent]

_PARAM_KINDS = {"f32": F.SHADER_PARAM_F32, "u32": F.SHADER_PARAM_U32, "i32": F.SHADER_PARAM_I32, "list": F.SHADER_PARAM_LIST,
                "struct": F.SHADER_PARAM_STRUCT}


def _param_to_c(p, keep, name=None):
    """ShaderParam -> smr_shader_param (buffers kept alive in `keep`)"""
    c = F.ShaderParam()
    c.kind = _PARAM_KINDS[p.kind]
    if name is not None:
        nb = name.encode()
        keep.append(nb)
        c.field_name = nb
    if p.kind == "f32":
        c.f32 = float(p.value)
    elif p.kind == "u32":
        c.u32 = int(p.value)
    elif p.kind == "i32":
        c.i32 = int(p.value)
    else:
        items = [_param_to_c(v, keep) for v in p.value] if p.kind == "list" else [_param_to_c(v, keep, n) for n, v in p.value]
        if items:
            arr = (F.ShaderParam * len(items))(*items)
            keep.append(arr)
            c.items, c.items_len = arr, len(items)
    return c


def _param_type_to_c(t, keep, name=None):
    """ShaderParamType -> smr_shader_param_type"""
    c = F.ShaderParamType()
    c.kind = _PARAM_KINDS[t.kind]
    if name is not None:
        nb = name.encode()
        keep.append(nb)
        c.name = nb
    items = ([_param_type_to_c(t.item, keep)] if t.kind == "list" and t.item is not None else
             [_param_type_to_c(v, keep, n) for n, v in t.fields] if t.kind == "struct" else [])
    if items:
        arr = (F.ShaderParamType * len(items))(*items)
        keep.append(arr)
        c.items, c.items_len = arr, len(items)
    c.length = int(t.length)
    return c


def _opt(v):
    return F.OptF32(1, float(v)) if v is not None else F.OptF32(0, 0.0)


def _rgba(c):
    return F.Rgba(c.r, c.g, c.b, c.a)


def _secs_to_ns(s):
    return int(round(float(s) * 1e9))


def _fill_common(c, comp, keep):
    p = comp.position
    cp = F.Position()
    cp.is_absolute = int(p.absolute)
    cp.width, cp.height = _opt(p.width), _opt(p.height)
    if p.absolute:
        if p.right is not None:
            cp.horizontal_from_right, cp.horizontal_offset = 1, float(p.right)
        else:
            cp.horizontal_from_right, cp.horizontal_offset = 0, float(p.left or 0.0)
        if p.bottom is not None:
            cp.vertical_from_bottom, cp.vertical_offset = 1, float(p.bottom)
        else:
            cp.vertical_from_bottom, cp.vertical_offset = 0, float(p.top or 0.0)
        cp.rotation_degrees = float(p.rotation_degrees)
    c.position = cp
    _fill_transition(c, comp.transition)
    r = comp.border_radius
    c.border_radius = F.BorderRadius(r.top_left, r.top_right, r.bottom_right, r.bottom_left)
    c.border_width = float(comp.border_width)
    c.border_color = _rgba(comp.border_color)
    if comp.box_shadow:
        arr = (F.BoxShadow * len(comp.box_shadow))(*[
            F.BoxShadow(s.offset_x, s.offset_y, s.blur_radius, _rgba(s.color)) for s in comp.box_shadow])
        keep.append(arr)
        c.box_shadow = arr
        c.box_shadow_len = len(comp.box_shadow)


def _fill_transition(c, t):
    if t is None:
        return
    k = t.interpolation_kind
    c.transition = F.Transition(1, _secs_to_ns(t.duration), k.kind, k.x1, k.y1, k.x2, k.y2, int(t.should_interrupt))


def _to_c(comp, keep):
    """Component -> smr_component (keeps referenced buffers alive in `keep`)."""
    c = F.Component()
    if isinstance(comp, InputStreamComponent):
        F.lib().smr_component_default(F.COMPONENT_INPUT_STREAM, C.byref(c))
        iid = comp.input_id.encode()
        keep.append(iid)
        c.input_id = iid
    elif isinstance(comp, ViewComponent):
        F.lib().smr_component_default(F.COMPONENT_VIEW, C.byref(c))
        _fill_common(c, comp, keep)
        c.direction, c.overflow = comp.direction, comp.overflow
        c.background_color = _rgba(comp.background_color)
        pd = comp.padding
        c.padding = F.Padding(pd.top, pd.right, pd.bottom, pd.left)
        _children(c, comp.children, keep)
    elif isinstance(comp, RescalerComponent):
        F.lib().smr_component_default(F.COMPONENT_RESCALER, C.byref(c))
        _fill_common(c, comp, keep)
        c.rescale_mode = comp.mode
        c.horizontal_align, c.vertical_align = comp.horizontal_align, comp.vertical_align
        child = comp.child if comp.child is not None else ViewComponent()
        _children(c, [child], keep)
    elif isinstance(comp, TextComponent):
        F.lib().smr_component_default(F.COMPONENT_TEXT, C.byref(c))
        g = _glyphs(comp.glyphs)
        keep.append(g)
        t = F.Text(comp.width, comp.height, _rgba(comp.background_color), g.ctypes.data if len(g) else None, len(g),
                   _atlas(comp.mask_atlas, 1, keep), _atlas(comp.color_atlas, 4, keep), int(comp.color_mode))
        keep.append(t)
        c.text = C.pointer(t)
    elif isinstance(comp, ImageComponent):
        F.lib().smr_component_default(F.COMPONENT_IMAGE, C.byref(c))
        c.image_id = comp.image_id.encode()
        c.image_width, c.image_height = _opt(comp.width), _opt(comp.height)
    elif isinstance(comp, WebViewComponent):
        F.lib().smr_component_default(F.COMPONENT_WEB_VIEW, C.byref(c))
        c.web_renderer_id = comp.instance_id.encode()
        _children(c, comp.children, keep)
    elif isinstance(comp, TilesComponent):
        F.lib().smr_component_default(F.COMPONENT_TILES, C.byref(c))
        _fill_transition(c, comp.transition)
        c.tiles_width, c.tiles_height = _opt(comp.width), _opt(comp.height)
        c.background_color = _rgba(comp.background_color)
        c.tile_aspect_ratio_w, c.tile_aspect_ratio_h = comp.tile_aspect_ratio
        c.tiles_margin, c.tiles_padding = float(comp.margin), float(comp.padding)
        c.horizontal_align, c.vertical_align = comp.horizontal_align, comp.vertical_align
        _children(c, comp.children, keep)
    elif isinstance(comp, ShaderComponent):
        F.lib().smr_component_default(F.COMPONENT_SHADER, C.byref(c))
        sid = comp.shader_id.encode()
        keep.append(sid)
        c.shader_id = sid
        if comp.shader_param is not None:
            pc = _param_to_c(comp.shader_param, keep)
            keep.append(pc)
            c.shader_param = C.pointer(pc)
        c.shader_width, c.shader_height = float(comp.width), float(comp.height)
        _children(c, comp.children, keep)
    else:
        # any other object: forward its tag with shader_id left NULL, which is what a caller built before the Shader
        # fields existed sends, so the library answers SMR_ERR_UNSUPPORTED
        c.type = getattr(comp, "component_type", F.COMPONENT_SHADER)
    if getattr(comp, "id", None) is not None:
        cid = comp.id.encode()
        keep.append(cid)
        c.id = cid
    return c


def _glyphs(glyphs):
    return np.ascontiguousarray(glyphs if glyphs is not None else np.zeros(0, F.GLYPH_DTYPE), dtype=np.dtype(F.GLYPH_DTYPE))


def _atlas(a, channels, keep):
    """an (h, w) R8 (channels 1) or (h, w, 4) RGBA8 atlas -> pointer to smr_atlas, or None"""
    if a is None:
        return None
    a = np.ascontiguousarray(a, np.uint8)
    assert a.ndim == (2 if channels == 1 else 3) and (channels == 1 or a.shape[2] == 4)
    s = F.Atlas(a.ctypes.data, a.shape[1], a.shape[0], 0)
    keep += [a, s]
    return C.pointer(s)


def _children(c, children, keep):
    if not children:
        return
    arr = (F.Component * len(children))(*[_to_c(ch, keep) for ch in children])
    keep.append(arr)
    c.children = arr
    c.children_len = len(children)


# ------------------------------------------------------------------------------------------------
# Renderer (state.rs:43-193)
# ------------------------------------------------------------------------------------------------
@dataclass
class RendererOptions:
    rendering_mode: int = RenderingMode.GpuOptimized
    max_layouts_count: int = 100                 # DEFAULT_MAX_LAYOUTS_COUNT
    stream_fallback_timeout: float = 3.0         # seconds (harness/utils.rs:86)
    framerate: Tuple[int, int] = (30, 1)
    cuda_device: int = 0                         # stands in for device/queue


class Renderer:
    def __init__(self, opts: RendererOptions = None):
        opts = opts or RendererOptions()
        self._lib = F.lib()
        self._h = C.c_void_p()
        o = F.Options(opts.cuda_device, opts.rendering_mode, opts.max_layouts_count,
                      _secs_to_ns(opts.stream_fallback_timeout), opts.framerate[0], opts.framerate[1])
        st = self._lib.smr_create(C.byref(o), C.byref(self._h))
        if st != F.SMR_OK:
            raise RendererError(st, (self._lib.smr_last_error(None) or b"").decode())
        self._outputs: Dict[str, Tuple[Resolution, int]] = {}
        self._input_geometry: Dict[str, Tuple[int, int, int]] = {}   # the last rendered frame's (format, width, height)
        self._svg_rasterizers = {}
        self.opts = opts

    def close(self):
        if getattr(self, "_h", None):
            self._lib.smr_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _err(self):
        return (self._lib.smr_last_error(self._h) or b"").decode()

    def _check(self, st, exc=RendererError):
        if st != F.SMR_OK:
            raise exc(st, self._err())

    def register_input(self, input_id: str):
        self._check(self._lib.smr_register_input(self._h, input_id.encode()))

    def unregister_input(self, input_id: str):
        self._check(self._lib.smr_unregister_input(self._h, input_id.encode()))
        self._input_geometry.pop(input_id, None)

    def set_input_deinterlace(self, input_id: str, mode: int, field_order: int = FieldOrder.TopFirst, motion_threshold: int = 10):
        """deinterlace every frame of a registered interlaced input before the scene reads it (smr_set_input_deinterlace):
        `mode` a DeinterlaceMode, `field_order` the FieldOrder of the source, `motion_threshold` MotionAdaptive's T (0 .. 255)"""
        cfg = F.Deinterlace(int(mode), int(field_order), int(motion_threshold))
        self._check(self._lib.smr_set_input_deinterlace(self._h, input_id.encode(), C.byref(cfg)))

    def set_input_color(self, input_id: str, matrix: int = YuvMatrix.Default, range: int = YuvRange.Default):
        """the colour matrix (YuvMatrix) and range (YuvRange) a registered YUV input is converted with (smr_set_input_color);
        Default keeps the format's rule, RGB inputs ignore the setting"""
        c = F.InputColor(int(matrix), int(range))
        self._check(self._lib.smr_set_input_color(self._h, input_id.encode(), C.byref(c)))

    def debug_input_planes(self, input_id: str) -> List[np.ndarray]:
        """the planes the kernels of the last render with a live frame of the input read for it, after deinterlacing: one
        (rows, row bytes) uint8 array per plane of the input's last frame passed to render / render_raw"""
        if input_id not in self._input_geometry:
            raise RendererError(1, f"no frame of input \"{input_id}\" was rendered")   # SMR_ERR_INVALID_ARGUMENT
        planes = [np.empty(shape, np.uint8) for shape in plane_shapes(*self._input_geometry[input_id])]
        ptrs = (C.c_void_p * 3)(*[p.ctypes.data for p in planes])
        self._check(self._lib.smr_debug_input_planes(self._h, input_id.encode(), C.byref(ptrs), C.byref((C.c_uint32 * 3)()),
                                                     F.MEM_HOST))
        return planes

    def _note_inputs(self, in_arr, n_in):
        for i in range(n_in):
            f = in_arr[i]
            if f.input_id:
                self._input_geometry[f.input_id.decode()] = (f.format, f.width, f.height)

    def register_image(self, image_id: str, frames, delays=None):
        """Renderer::register_renderer for an image that arrives decoded: `frames` is one (h, w, 4) uint8 straight-alpha
        array (a Bitmap asset) or a sequence of them, all of one size (two or more: an Animated asset, with `delays`, one
        per frame, in nanoseconds)."""
        if isinstance(frames, np.ndarray) and frames.ndim == 3:
            frames = [frames]
        frames = [np.ascontiguousarray(f, np.uint8) for f in frames]
        delays = [0] * len(frames) if delays is None else [int(d) for d in delays]
        assert len(delays) == len(frames) and all(f.ndim == 3 and f.shape == frames[0].shape and f.shape[2] == 4 for f in frames)
        arr = (F.ImageFrame * max(1, len(frames)))(*[F.ImageFrame(f.ctypes.data, 0, d) for f, d in zip(frames, delays)])
        h, w = frames[0].shape[:2] if frames else (0, 0)
        spec = F.ImageSpec(w, h, arr, len(frames))
        self._check(self._lib.smr_register_image(self._h, image_id.encode(), C.byref(spec)))

    def register_svg_image(self, image_id: str, width: int, height: int, rasterize):
        """Renderer::register_renderer for ImageType::Svg: the caller parses the SVG.  (width, height) is its intrinsic
        size (the tree's size truncated); `rasterize(w, h)` returns the asset drawn at w x h as an (h, w, 4) uint8
        premultiplied array.  It is called during update_scene, once per SVG node, with the node's resolution; an exception
        or an array of another shape or dtype refuses the update (RendererError, SMR_ERR_SCENE)."""
        def trampoline(user, w, h, rgba, pitch):
            try:
                px = np.asarray(rasterize(int(w), int(h)))
                if px.dtype != np.uint8 or px.shape != (h, w, 4):
                    return 1
                dst = np.ctypeslib.as_array(rgba, shape=(h, pitch))
                dst[:, :w * 4] = px.reshape(h, w * 4)
                return 0
            except Exception:
                return 1
        fn = F.SVG_RASTERIZE_FN(trampoline)
        spec = F.SvgSpec(int(width), int(height), fn, None)
        self._check(self._lib.smr_register_svg_image(self._h, image_id.encode(), C.byref(spec)))
        self._svg_rasterizers[image_id] = fn     # called back until the id is unregistered

    def unregister_image(self, image_id: str):
        self._check(self._lib.smr_unregister_image(self._h, image_id.encode()))
        self._svg_rasterizers.pop(image_id, None)

    def register_web_renderer(self, instance_id: str, width: int, height: int, embedding_method=F.WEB_NATIVE_OVER_CONTENT):
        """Renderer::register_renderer for RendererSpec::WebRenderer: the browser and its URL stay with the caller, which
        hands over the painted frames (set_web_frame) and the child rects (set_web_child_rects)"""
        spec = F.WebRendererSpec(int(width), int(height), int(embedding_method))
        self._check(self._lib.smr_register_web_renderer(self._h, instance_id.encode(), C.byref(spec)))

    def register_shader(self, shader_id: str, source: str, param_type: Optional[ShaderParamType] = None):
        """Renderer::register_renderer for RendererSpec::Shader: `source` is CUDA C++ defining smr_fragment (see
        include/smelter_b200.h), compiled here for sm_90a; `param_type` the type of its parameter (None: none)"""
        keep = []
        src = source.encode()
        pt = _param_type_to_c(param_type, keep) if param_type is not None else None
        spec = F.ShaderSpec(src, C.pointer(pt) if pt is not None else None)
        self._check(self._lib.smr_register_shader(self._h, shader_id.encode(), C.byref(spec)))

    def register_wgsl_shader(self, shader_id: str, source: str):
        """Renderer::register_renderer for RendererSpec::Shader(ShaderSpec { source }) as the reference takes it: WGSL with
        the shader header, vs_main and fs_main (see smr_register_wgsl_shader); its parameter type is its uniform's"""
        self._check(self._lib.smr_register_wgsl_shader(self._h, shader_id.encode(), source.encode()))

    def unregister_shader(self, shader_id: str):
        self._check(self._lib.smr_unregister_shader(self._h, shader_id.encode()))

    def unregister_web_renderer(self, instance_id: str):
        self._check(self._lib.smr_unregister_web_renderer(self._h, instance_id.encode()))

    def set_web_frame(self, instance_id: str, bgra, mem_kind=F.MEM_HOST):
        """the page as CEF's on_paint delivers it: an (h, w, 4) uint8 premultiplied BGRA array of the instance's size, or with
        mem_kind MEM_DEVICE a CUDA tensor of that shape; copied before this returns"""
        h, w = bgra.shape[:2]
        if mem_kind == F.MEM_HOST:
            bgra = np.ascontiguousarray(bgra, np.uint8)
            ptr, pitch = bgra.ctypes.data, w * 4
        else:
            ptr, pitch = bgra.data_ptr(), bgra.stride(0)
        frame = F.WebFrame(ptr, w, h, pitch, mem_kind)
        self._check(self._lib.smr_web_set_frame(self._h, instance_id.encode(), C.byref(frame)))

    def set_web_child_rects(self, instance_id: str, rects):
        """the GET_FRAME_POSITIONS reply: one (x, y, width, height) per child, in page pixels"""
        arr = (F.WebRect * max(1, len(rects)))(*[F.WebRect(*map(float, r)) for r in rects])
        self._check(self._lib.smr_web_set_child_rects(self._h, instance_id.encode(), arr if rects else None, len(rects)))

    def unregister_output(self, output_id: str):
        self._check(self._lib.smr_unregister_output(self._h, output_id.encode()))
        self._outputs.pop(output_id, None)

    def update_scene(self, output_id: str, resolution: Resolution, output_format: int, scene_root):
        keep = []
        root = _to_c(scene_root, keep)
        st = self._lib.smr_update_scene(self._h, output_id.encode(), resolution.width, resolution.height,
                                        output_format, C.byref(root))
        self._check(st, UpdateSceneError)
        self._outputs[output_id] = (resolution, output_format)

    # -- frames --------------------------------------------------------------------------------
    @staticmethod
    def _plane_ptr(p, device):
        if device:
            return int(p), None
        a = np.ascontiguousarray(p, dtype=np.uint8)
        return a.ctypes.data, a

    def _input_frames(self, frame_set: FrameSet, keep):
        arr = (F.InputFrame * max(1, len(frame_set.frames)))()
        for i, (iid, fr) in enumerate(frame_set.frames.items()):
            f = arr[i]
            bid = iid.encode()
            keep.append(bid)
            f.input_id = bid
            f.format = _FRAME_KIND[fr.data.kind]
            f.width, f.height = fr.resolution.width, fr.resolution.height
            f.pts_ns = _secs_to_ns(fr.pts)
            f.mem_kind = F.MEM_DEVICE if fr.data.device else F.MEM_HOST
            for pi, pl in enumerate(fr.data.planes):
                ptr, a = self._plane_ptr(pl, fr.data.device)
                keep.append(a)
                f.planes[pi] = ptr
        return arr

    def _one_frame(self, frame: Frame):
        """the one source frame of a blocking call: (smr_input_frame array, the buffers it points into)"""
        keep = []
        return self._input_frames(FrameSet(frames={"_": frame}), keep), keep

    def render(self, input: FrameSet, outputs: Optional[List[str]] = None) -> FrameSet:
        """Renderer::render(FrameSet<InputId>) -> FrameSet<OutputId>.  Output planes are host numpy arrays."""
        keep = []
        in_arr = self._input_frames(input, keep)
        ids = list(self._outputs.keys()) if outputs is None else list(outputs)
        out_arr = (F.OutputFrame * max(1, len(ids)))()
        bufs = {}
        for i, oid in enumerate(ids):
            if oid not in self._outputs:
                raise RenderSceneError(3, f"Output \"{oid}\" does not exist")
            res, fmt = self._outputs[oid]
            sizes = (C.c_size_t * 3)()
            self._check(self._lib.smr_output_plane_sizes(res.width, res.height, fmt, C.byref(sizes)))
            planes = [np.empty(sizes[p], np.uint8) if sizes[p] else None for p in range(3)]
            bufs[oid] = planes
            bid = oid.encode()
            keep.append(bid)
            out_arr[i].output_id = bid
            out_arr[i].mem_kind = F.MEM_HOST
            for p in range(3):
                if planes[p] is not None:
                    out_arr[i].planes[p] = planes[p].ctypes.data
        st = self._lib.smr_render(self._h, _secs_to_ns(input.pts), in_arr, len(input.frames), out_arr, len(ids))
        self._check(st, RenderSceneError)
        self._note_inputs(in_arr, len(input.frames))
        result = FrameSet(pts=input.pts)
        for i, oid in enumerate(ids):
            w, h, fmt = out_arr[i].width, out_arr[i].height, out_arr[i].format
            pl = bufs[oid]
            if fmt == F.OUT_PLANAR_YUV420:
                data = FrameData.PlanarYuv420(YuvPlanes(pl[0].reshape(h, w), pl[1].reshape(h // 2, w // 2),
                                                        pl[2].reshape(h // 2, w // 2)))
            elif fmt == F.OUT_PLANAR_YUV422:
                data = FrameData.PlanarYuv422(YuvPlanes(pl[0].reshape(h, w), pl[1].reshape(h, w // 2),
                                                        pl[2].reshape(h, w // 2)))
            elif fmt == F.OUT_PLANAR_YUV444:
                data = FrameData.PlanarYuv444(YuvPlanes(pl[0].reshape(h, w), pl[1].reshape(h, w), pl[2].reshape(h, w)))
            elif fmt == F.OUT_NV12:
                data = FrameData.Nv12(NvPlanes(pl[0].reshape(h, w), pl[1].reshape(h // 2, w // 2, 2)))
            else:
                data = FrameData.Rgba8(pl[0].reshape(h, w, 4))
            result.frames[oid] = Frame(data, Resolution(w, h), input.pts)
        return result

    def preprocess_frame(self, frame: Frame, resolution: Optional[Resolution] = None) -> np.ndarray:
        """FramePreProcessor::process_to_bytes (state/frame_pre_processor.rs:81-100): one frame -> RGBA8 bytes of
        its node texture, optionally rescaled (linear sampler) to `resolution`.  Returns an (h, w, 4) uint8 array."""
        arr, keep = self._one_frame(frame)
        ow, oh = (resolution.width, resolution.height) if resolution else (0, 0)
        w, h = (ow, oh) if resolution else (frame.resolution.width, frame.resolution.height)
        out = np.empty((h, w, 4), np.uint8)
        self._check(self._lib.smr_preprocess_frame(self._h, arr, ow, oh, out.ctypes.data, 0, F.MEM_HOST), RenderSceneError)
        return out

    def transcode_resize(self, frame: Frame, renditions) -> List[Tuple[np.ndarray, np.ndarray]]:
        """VideoTranscoder's resize step (gpu-video vulkan_transcoder): one NV12 frame -> up to eight NV12 renditions in one
        launch.  `renditions` is a sequence of (width, height, ScalingAlgorithm); returns, per rendition, its (h, w) Y plane
        and its (h / 2, w / 2, 2) UV plane as host arrays."""
        arr, keep = self._one_frame(frame)
        outs = (F.Rendition * max(1, len(renditions)))()
        planes = []
        for i, (w, h, scaling) in enumerate(renditions):
            y, uv = np.empty((h, w), np.uint8), np.empty((h // 2, w // 2, 2), np.uint8)
            planes.append((y, uv))
            outs[i].width, outs[i].height, outs[i].scaling, outs[i].mem_kind = w, h, scaling, F.MEM_HOST
            outs[i].planes[0], outs[i].planes[1] = y.ctypes.data, uv.ctypes.data
        self._check(self._lib.smr_transcode_resize(self._h, arr, outs, len(renditions)), RenderSceneError)
        return planes

    def video_nv12_to_rgba(self, frame: Frame, resolution: Optional[Resolution] = None,
                           converter=(ColorSpace.BT709, ColorRange.Limited),
                           frame_color=(ColorSpace.Unspecified, ColorRange.Limited)) -> np.ndarray:
        """gpu-video's WgpuNv12ToRgbaConverter: one NV12 frame (its crop, origin (0, 0)) -> Rgba8Unorm bytes, bilinearly
        rescaled to `resolution` when it is given.  `converter` is the converter's (ColorSpace, ColorRange), `frame_color`
        the decoded frame's metadata.  Returns an (h, w, 4) uint8 array."""
        arr, keep = self._one_frame(frame)
        ow, oh = (resolution.width, resolution.height) if resolution else (0, 0)
        w, h = (ow, oh) if resolution else (frame.resolution.width, frame.resolution.height)
        out = np.empty((h, w, 4), np.uint8)
        self._check(self._lib.smr_video_nv12_to_rgba(self._h, F.VideoColor(*converter), arr, F.VideoColor(*frame_color), ow, oh,
                                                     out.ctypes.data, 0, F.MEM_HOST), RenderSceneError)
        return out

    def video_rgba_to_nv12(self, frame: Frame, resolution: Optional[Resolution] = None,
                           converter=(ColorSpace.BT709, ColorRange.Limited)) -> Tuple[np.ndarray, np.ndarray]:
        """gpu-video's WgpuRgbaToNv12Converter: one RGBA8 frame (raw bytes, alpha unused) -> NV12 planes, bilinearly
        rescaled to `resolution` (even sides; default: the frame's size).  Returns the (h, w) Y plane and the
        (h / 2, w / 2, 2) UV plane."""
        arr, keep = self._one_frame(frame)
        w, h = (resolution.width, resolution.height) if resolution else (frame.resolution.width, frame.resolution.height)
        y, uv = np.empty((h, w), np.uint8), np.empty((h // 2, w // 2, 2), np.uint8)
        planes = (C.c_void_p * 2)(y.ctypes.data, uv.ctypes.data)
        self._check(self._lib.smr_video_rgba_to_nv12(self._h, F.VideoColor(*converter), arr, w, h, planes, None, F.MEM_HOST),
                    RenderSceneError)
        return y, uv

    def set_layouts(self, output_id: str, resolution: Resolution, output_format: int, root: Tuple[int, int],
                    child_input_ids: List[str], layouts):
        """the flattened boundary (smr_set_layouts): `layouts` are _ffi.RenderLayout structs (e.g. from debug_layouts
        of another handle, or built by a host that runs the reference's scene/** itself)"""
        ids = (C.c_char_p * max(1, len(child_input_ids)))(*[i.encode() for i in child_input_ids])
        arr = (F.RenderLayout * max(1, len(layouts)))(*layouts)
        self._check(self._lib.smr_set_layouts(self._h, output_id.encode(), resolution.width, resolution.height, output_format,
                                              root[0], root[1], ids, len(child_input_ids), arr, len(layouts)), UpdateSceneError)
        self._outputs[output_id] = (resolution, output_format)

    def premultiply_rgba8(self, rgba: np.ndarray) -> np.ndarray:
        """PremultiplyAlphaPipeline (wgpu/utils/add_premultiplied_alpha.wgsl): straight-alpha (h, w, 4) uint8 ->
        premultiplied RGBA8 through the renderer's views; the result is a valid FrameData.Rgba8 input."""
        rgba = np.ascontiguousarray(rgba, np.uint8)
        h, w = rgba.shape[:2]
        arr, keep = self._one_frame(Frame(FrameData.Rgba8(rgba), Resolution(w, h), 0.0))
        out = np.empty((h, w, 4), np.uint8)
        self._check(self._lib.smr_premultiply_rgba8(self._h, arr, out.ctypes.data, 0, F.MEM_HOST), RenderSceneError)
        return out

    def render_text(self, width: int, height: int, background: "RGBAColor", glyphs: np.ndarray,
                    mask_atlas: Optional[np.ndarray] = None, color_atlas: Optional[np.ndarray] = None,
                    color_mode: int = 0) -> np.ndarray:
        """TextRendererNode::render (transformations/text_renderer.rs:72-167): clear to the text component's background
        colour, then glyphon's prepared glyph quads (records of _ffi.GLYPH_DTYPE, painter's order) alpha-blended from
        the mask atlas ((h, w) uint8) / colour atlas ((h, w, 4) uint8).  Returns the (height, width, 4) node texture --
        a valid FrameData.Rgba8 input.  A zero-sized text texture is one transparent pixel (text_renderer.rs:77-85)."""
        if width == 0 or height == 0:
            return np.zeros((1, 1, 4), np.uint8)
        g = _glyphs(glyphs)
        keep = []
        out = np.empty((height, width, 4), np.uint8)
        self._check(self._lib.smr_render_text(self._h, width, height, _rgba(background), g.ctypes.data if len(g) else None, len(g),
                                              _atlas(mask_atlas, 1, keep), _atlas(color_atlas, 4, keep), int(color_mode),
                                              out.ctypes.data, 0, F.MEM_HOST), RenderSceneError)
        return out

    # -- zero-copy path (device pointers in and out; used by bench.py's `value` leg) ---------------
    def render_raw(self, pts_ns, in_arr, n_in, out_arr, n_out, wait=True):
        st = self._lib.smr_render_begin(self._h, pts_ns, in_arr, n_in, out_arr, n_out)
        self._check(st, RenderSceneError)
        self._note_inputs(in_arr, n_in)
        if wait:
            self._check(self._lib.smr_render_end(self._h), RenderSceneError)

    def wait(self):
        self._check(self._lib.smr_render_end(self._h), RenderSceneError)

    # -- inspection ----------------------------------------------------------------------------
    def debug_set_inputs(self, pts: float, resolutions: Dict[str, Resolution], frame_pts: Optional[float] = None):
        """Record pts + input resolutions as `render` would, without any frame data (host-only testing)."""
        keep = []
        arr = (F.InputFrame * max(1, len(resolutions)))()
        for i, (iid, res) in enumerate(resolutions.items()):
            b = iid.encode()
            keep.append(b)
            arr[i].input_id = b
            arr[i].width, arr[i].height = res.width, res.height
            arr[i].pts_ns = _secs_to_ns(pts if frame_pts is None else frame_pts)
        self._check(self._lib.smr_debug_set_inputs(self._h, _secs_to_ns(pts), arr, len(resolutions)))

    def debug_layouts(self, output_id: str, pts: float = 0.0):
        n = C.c_uint32()
        rw, rh = C.c_uint32(), C.c_uint32()
        pts_ns = _secs_to_ns(pts)
        self._check(self._lib.smr_debug_layouts(self._h, output_id.encode(), pts_ns, None, 0, C.byref(n),
                                                C.byref(rw), C.byref(rh)))
        arr = (F.RenderLayout * max(1, n.value))()
        self._check(self._lib.smr_debug_layouts(self._h, output_id.encode(), pts_ns, arr, n.value, C.byref(n),
                                                C.byref(rw), C.byref(rh)))
        return [arr[i] for i in range(n.value)], (rw.value, rh.value)

    def debug_node_layouts(self, output_id: str, node: int, pts: float = 0.0):
        """smr_debug_node_layouts: the flattened layouts of layout node `node` of an output's render graph (0: the root when
        it is a layout; the layout nodes below it follow in DFS order) and its resolution at `pts`"""
        n = C.c_uint32()
        rw, rh = C.c_uint32(), C.c_uint32()
        pts_ns = _secs_to_ns(pts)
        self._check(self._lib.smr_debug_node_layouts(self._h, output_id.encode(), int(node), pts_ns, None, 0, C.byref(n),
                                                     C.byref(rw), C.byref(rh)))
        arr = (F.RenderLayout * max(1, n.value))()
        self._check(self._lib.smr_debug_node_layouts(self._h, output_id.encode(), int(node), pts_ns, arr, n.value, C.byref(n),
                                                     C.byref(rw), C.byref(rh)))
        return [arr[i] for i in range(n.value)], (rw.value, rh.value)

    def debug_image_nodes(self, output_id: str, pts: float = 0.0):
        """The image nodes of an output's scene (smr_debug_image_nodes): [((width, height), start pts in ns, the frame a
        render at `pts` shows)], the root or the node children in DFS order."""
        n = C.c_uint32()
        self._check(self._lib.smr_debug_image_nodes(self._h, output_id.encode(), _secs_to_ns(pts), None, 0, C.byref(n)))
        arr = (F.ImageNodeInfo * max(1, n.value))()
        self._check(self._lib.smr_debug_image_nodes(self._h, output_id.encode(), _secs_to_ns(pts), arr, n.value, C.byref(n)))
        return [((a.width, a.height), int(a.start_pts_ns), int(a.frame)) for a in arr[:n.value]]

    def debug_fused_jobs(self):
        """The fused resample jobs of the last planned tick (smr_debug_fused_jobs), one dict per job in plan order:
        kernel ("ldg" / "tma_int" / "tma_any"), ratio, window, box, src_class, full_range, v_same, strip_cols,
        src (w, h), dst (w, h), taps_h, taps_v, direct, matrix (YuvMatrix.BT709 / BT601)."""
        n = C.c_uint32()
        self._check(self._lib.smr_debug_fused_jobs(self._h, None, 0, C.byref(n)))
        arr = (F.FusedJobInfo * max(1, n.value))()
        self._check(self._lib.smr_debug_fused_jobs(self._h, arr, n.value, C.byref(n)))
        kinds = {F.FUSED_LDG: "ldg", F.FUSED_TMA_INT: "tma_int", F.FUSED_TMA_ANY: "tma_any"}
        out = []
        for j in arr[:n.value]:
            d = {k: getattr(j, k) for k, _ in F.FusedJobInfo._fields_}
            d["kernel"] = kinds[j.kernel]
            d["src"] = (d.pop("src_width"), d.pop("src_height"))
            d["dst"] = (d.pop("dst_width"), d.pop("dst_height"))
            out.append(d)
        return out

    def debug_resample_stages(self):
        """The generic resample passes and k_convert jobs of the last planned tick (smr_debug_resample_stages):
        (stages, convert_kinds).  stages: one dict per pass -- box passes, first passes, last passes, each in plan order --
        with stage ("box" / "first" / "last"), axis (-1 for a box pass), box_fx, box_fy, taps, perp_offset, source ("raw" /
        "converted" / "f16"), src_kind, src (w, h), dst (w, h), dst_f16.  convert_kinds: the texture kind each k_convert
        job reads."""
        n, nc = C.c_uint32(), C.c_uint32()
        self._check(self._lib.smr_debug_resample_stages(self._h, None, 0, C.byref(n), None, 0, C.byref(nc)))
        arr = (F.ResampleStageInfo * max(1, n.value))()
        kinds = (C.c_int32 * max(1, nc.value))()
        self._check(self._lib.smr_debug_resample_stages(self._h, arr, n.value, C.byref(n), kinds, nc.value, C.byref(nc)))
        stage_names = {F.STAGE_BOX: "box", F.STAGE_FIRST: "first", F.STAGE_LAST: "last"}
        source_names = {F.STAGE_SRC_RAW: "raw", F.STAGE_SRC_CONVERTED: "converted", F.STAGE_SRC_F16: "f16"}
        out = []
        for j in arr[:n.value]:
            d = {k: getattr(j, k) for k, _ in F.ResampleStageInfo._fields_}
            d["stage"] = stage_names[j.stage]
            d["source"] = source_names[j.source]
            d["src"] = (d.pop("src_width"), d.pop("src_height"))
            d["dst"] = (d.pop("dst_width"), d.pop("dst_height"))
            out.append(d)
        return out, list(kinds[:nc.value])

    def debug_composite_layers(self):
        """The layers of the last planned tick's composite jobs (smr_debug_composite_layers), one dict per layer in job
        order, then painter's order: job, kernel ("p" / "multi"), layer, type, rotated, fast, box (12 ints: pixel box and
        both interior bars), tx_off, ty_off, mask_count, tex_kind, tex_width, tex_height, tex_pitch, tex_align, width,
        height, out_format, tex_matrix (YuvMatrix.BT709 / BT601 for a YUV texture, else 0)."""
        n = C.c_uint32()
        self._check(self._lib.smr_debug_composite_layers(self._h, None, 0, C.byref(n)))
        arr = (F.CompositeLayerInfo * max(1, n.value))()
        self._check(self._lib.smr_debug_composite_layers(self._h, arr, n.value, C.byref(n)))
        out = []
        for j in arr[:n.value]:
            d = {k: getattr(j, k) for k, _ in F.CompositeLayerInfo._fields_}
            for k in ("box", "tex_pitch", "tex_align"):
                d[k] = tuple(d[k])
            d["kernel"] = "p" if j.kernel == F.COMPOSITE_PARAM else "multi"
            out.append(d)
        return out

    def stats(self):
        s = F.Stats()
        self._check(self._lib.smr_get_stats(self._h, C.byref(s)))
        return {k: getattr(s, k) for k, _ in F.Stats._fields_}

    # -- multi-GPU: shared-input replication over NCCL (include/smelter_b200.h smr_comm_*) ------------------
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = (C.c_uint8 * 128)()
        st = F.lib().smr_comm_get_unique_id(C.byref(buf))
        if st != F.SMR_OK:
            raise RendererError(st, (F.lib().smr_last_error(None) or b"").decode())
        return bytes(buf)

    def comm_init(self, unique_id: bytes, rank: int, nranks: int):
        buf = (C.c_uint8 * 128)(*unique_id)
        self._check(self._lib.smr_comm_init(self._h, C.byref(buf), rank, nranks))

    def comm_broadcast_inputs(self, in_arr, n, roots):
        arr = (C.c_int32 * max(1, n))(*roots)
        self._check(self._lib.smr_comm_broadcast_inputs(self._h, in_arr, n, arr))

    COMM_POOLED = 1

    COMM_PEER_DIRECT = 2

    def comm_exchange_inputs(self, in_arr, n, roots, consumer_masks=None, pooled=False, peer_direct=False):
        """selective replication: frame i goes from rank roots[i] to the ranks whose bit is set in consumer_masks[i]
        (None: to every rank); pooled=True declares an identical plane layout on every rank (contiguous runs merge);
        peer_direct=True moves nothing (the tick's kernels read the roots' pools over NVLink): ordering step only"""
        arr = (C.c_int32 * max(1, n))(*roots)
        masks = None if consumer_masks is None else (C.c_uint64 * max(1, n))(*consumer_masks)
        flags = (self.COMM_POOLED if pooled else 0) | (self.COMM_PEER_DIRECT if peer_direct else 0)
        self._check(self._lib.smr_comm_exchange_inputs(self._h, in_arr, n, arr, masks, flags))

    def comm_pull_inputs(self, in_arr, peer_arr, n, roots, consumer_masks=None):
        """copy-engine form: frames rooted elsewhere are copied from peer_arr[i] (planes in the root's opened pool)
        to in_arr[i] (local planes) after the cross-rank ordering step"""
        arr = (C.c_int32 * max(1, n))(*roots)
        masks = None if consumer_masks is None else (C.c_uint64 * max(1, n))(*consumer_masks)
        self._check(self._lib.smr_comm_pull_inputs(self._h, in_arr, peer_arr, n, arr, masks))

    def peer_pool_alloc(self, nbytes: int):
        """(device pointer, 64-byte IPC handle) of a frame pool other GPUs' handles can open"""
        ptr = C.c_void_p()
        h = (C.c_uint8 * 64)()
        self._check(self._lib.smr_peer_pool_alloc(self._h, nbytes, C.byref(ptr), C.byref(h)))
        return ptr.value, bytes(h)

    def peer_pool_open(self, handle: bytes) -> int:
        h = (C.c_uint8 * 64).from_buffer_copy(handle)
        ptr = C.c_void_p()
        self._check(self._lib.smr_peer_pool_open(self._h, C.byref(h), C.byref(ptr)))
        return ptr.value

    def peer_pool_close(self, ptr: int):
        self._check(self._lib.smr_peer_pool_close(self._h, ptr))

    def peer_pool_free(self, ptr: int):
        self._check(self._lib.smr_peer_pool_free(self._h, ptr))

    def comm_destroy(self):
        self._check(self._lib.smr_comm_destroy(self._h))

    def set_profiling(self, enabled: bool):
        self._check(self._lib.smr_set_profiling(self._h, int(enabled)))

    def kernel_times(self):
        """{kernel class: (total device ms, launches)} since set_profiling(True)."""
        t = F.KernelTimes()
        self._check(self._lib.smr_get_kernel_times(self._h, C.byref(t)))
        return {name: (t.total_ms[i], int(t.launches[i])) for i, name in enumerate(F.KERNEL_CLASSES)}

    def cuda_stream(self):
        return self._lib.smr_cuda_stream(self._h)
