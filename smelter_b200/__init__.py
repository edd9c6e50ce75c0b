"""smelter_b200 -- H100-native per-output-frame video compositor, drop-in for smelter-render's
`Renderer` (see include/smelter_b200.h for the C ABI, INTEGRATION.md for the Rust-side binding).

The package is a thin ctypes mirror of the reference interface; all pixels come from
libsmelter_b200.so (hand-written sm_90a CUDA).  There is no CPU fallback."""
from .renderer import (  # noqa: F401
    BorderRadius, BoxShadow, ColorRange, ColorSpace, Component, DeinterlaceMode, FieldOrder, Frame, FrameData, FramePreProcessor, FrameSet, HorizontalAlign, ImageComponent, InputStreamComponent,
    InterpolationKind, NvPlanes, OutputFrameFormat, Overflow, Padding, Position, Renderer, RendererError,
    RendererOptions, RenderingMode, RenderSceneError, RescaleMode, RescalerComponent, Resolution, RGBAColor, ScalingAlgorithm, ShaderComponent,
    ShaderParam, ShaderParamType,
    TextComponent, TilesComponent, Transition, UpdateSceneError, VerticalAlign, ViewChildrenDirection, ViewComponent, WebViewComponent,
    YuvMatrix, YuvPlanes, YuvRange,
)
