// scene.h -- host-side scene model of the compositor (C++ restatement of smelter-render/src/scene/*).
//
// The reference keeps this math on the CPU too (SURVEY 8a-7/a-8): Component tree -> stateful tree
// (transitions) -> NestedLayout -> flatten -> RenderLayout[].  Only the resulting RenderLayout list
// reaches the GPU.  All arithmetic is f32 (f64 for easing) in the reference's order of operations.
#pragma once

#include <cstddef>
#include <cstdint>
#include <functional>
#include <map>
#include <memory>
#include <optional>
#include <string>
#include <utility>
#include <vector>

#include "../../include/smelter_b200.h"

namespace smr {

struct Size {
    float width = 0.0f, height = 0.0f;
};

struct Resolution {
    size_t width = 0, height = 0;
    bool operator==(const Resolution &o) const { return width == o.width && height == o.height; }
};

struct RGBA {
    uint8_t r = 0, g = 0, b = 0, a = 0;
    bool operator==(const RGBA &o) const { return r == o.r && g == o.g && b == o.b && a == o.a; }
};

// scene/types.rs:91-160
struct BorderRadius {
    float top_left = 0, top_right = 0, bottom_right = 0, bottom_left = 0;
    BorderRadius clip_to_size(Size size) const;
    BorderRadius operator*(float rhs) const;
    BorderRadius operator/(float rhs) const { return *this * (1.0f / rhs); }
    BorderRadius operator+(float rhs) const;
    BorderRadius operator-(float rhs) const { return *this + (-rhs); }
    bool operator==(const BorderRadius &o) const {
        return top_left == o.top_left && top_right == o.top_right && bottom_right == o.bottom_right &&
               bottom_left == o.bottom_left;
    }
};

struct BoxShadow {
    float offset_x = 0, offset_y = 0, blur_radius = 0;
    RGBA color;
    bool operator==(const BoxShadow &o) const {
        return offset_x == o.offset_x && offset_y == o.offset_y && blur_radius == o.blur_radius && color == o.color;
    }
};

struct Padding {
    float top = 0, right = 0, bottom = 0, left = 0;
    float horizontal() const { return left + right; }
    float vertical() const { return top + bottom; }
    bool operator==(const Padding &o) const {
        return top == o.top && right == o.right && bottom == o.bottom && left == o.left;
    }
};

using OptF = std::optional<float>;

// components.rs:199-206 + types.rs:66-86
struct Position {
    bool absolute = false;
    OptF width, height;
    bool from_right = false;
    float horizontal_offset = 0;
    bool from_bottom = false;
    float vertical_offset = 0;
    float rotation_degrees = 0;
    Position with_border(float border_width) const;   // components/position.rs:6-29
    Position with_padding(const Padding &p) const;    // components/position.rs:31-54
    bool operator==(const Position &o) const;
};

struct InterpolationKind {
    int kind = SMR_INTERP_LINEAR;
    double x1 = 0, y1 = 0, x2 = 0, y2 = 0;
    double state(double t) const;  // transition.rs:108-118
};

struct Transition {
    uint64_t duration_ns = 0;
    InterpolationKind interpolation;
    bool should_interrupt = false;
};

// A Text component's laid-out payload (smr_text), copied out of the caller's memory.  Atlases are tightly packed and shared
// by the components of one smr_update_scene that passed the same smr_atlas data pointer.
struct TextAtlas {
    std::vector<uint8_t> data;
    uint32_t width = 0, height = 0;
};
struct TextPayload {
    uint32_t width = 0, height = 0;   // the caller's layout resolution; 0 x 0 draws one transparent pixel
    RGBA background;
    std::vector<smr_glyph> glyphs;
    std::shared_ptr<const TextAtlas> mask, color;   // null when no glyph reads it
    int32_t color_mode = 0;
};

// A registered image (transformations/image.rs: Image::Bitmap for one frame, Image::Animated for more, Image::Svg with a
// rasteriser).  Scene nodes hold it by shared_ptr, and the identity of the object is what state inheritance compares
// (Arc::ptr_eq).
struct ImageAsset {
    uint32_t width = 0, height = 0;    // Svg: the intrinsic size
    std::vector<uint64_t> frame_pts;   // AnimationFrame::pts, the sum of the delays before each frame; one entry for a Bitmap
                                       // or an Svg
    uint64_t duration = 1;             // animation_duration (animated_image.rs:101-104)
    std::shared_ptr<void> pixels;      // device memory: the frames, straight-alpha RGBA8, packed, one after the other (host-only
                                       // or Svg: null)
    smr_svg_rasterize_fn rasterize = nullptr;   // Svg: the caller's rasteriser and its `user`, called per node at scene update
    void *user = nullptr;
    std::string svg_id;                // Svg: the id it was registered under, named when its rasteriser refuses
    bool svg() const { return rasterize != nullptr; }
    bool animated() const { return frame_pts.size() > 1; }
    // AnimatedAsset::render's frame choice (animated_image.rs:120-136); pts - start_pts saturates at 0
    size_t frame_at(uint64_t pts, uint64_t start_pts) const;
};

// ImageRenderParams (scene/image_component.rs:10-15)
struct ImageParams {
    std::shared_ptr<const ImageAsset> asset;
    uint64_t start_pts = 0;
    Resolution resolution;
};

// A registered web renderer instance (transformations/web_renderer/renderer.rs: WebRenderer).  The registry and the scene
// nodes that show it hold it by shared_ptr.  The renderer owns the latest frame and child rects; a scene only reads the size.
struct WebInstance {
    uint32_t width = 0, height = 0;
    int32_t embedding = 1;                // smr_web_embedding (never SMR_WEB_CHROMIUM_EMBEDDING)
    std::shared_ptr<void> frame;          // device memory: the latest page, BGRA8 packed (null: no frame yet)
    std::vector<float> rects;             // the latest child rects: x, y, width, height per child, narrowed to f32
};

// The type of a shader's parameter (smr_shader_param_type): the tree of scalars, fixed-length lists and structs that stands
// in for the WGSL uniform type the reference reads out of the shader module (pipeline.rs:143-160)
// A WGSL shader's uniform type (smr_register_wgsl_shader) adds vectors and matrices, which only the module can declare.
constexpr int32_t kShaderParamVector = 5;   // vecN: length N, items[0] the scalar
constexpr int32_t kShaderParamMatrix = 6;   // matCxR: length R (rows), items[0] the row, a vector of C scalars
struct ShaderParamType {
    int32_t kind = SMR_SHADER_PARAM_F32;  // smr_shader_param_kind, kShaderParamVector or kShaderParamMatrix
    std::string name;                     // a struct field's name
    std::vector<ShaderParamType> items;   // List / Vector / Matrix: the element type (one); Struct: the fields, in order
    uint32_t length = 0;                  // List: the element count; Vector: N; Matrix: rows
};
// A ShaderParam value (scene/components.rs:40-55)
struct ShaderParamValue {
    int32_t kind = SMR_SHADER_PARAM_F32;
    std::string field_name;               // a Struct's field
    float f32 = 0;
    uint32_t u32 = 0;
    int32_t i32 = 0;
    std::vector<ShaderParamValue> items;  // List: the elements; Struct: the fields
    void to_bytes(std::vector<uint8_t> &out) const;   // ShaderParamExt::to_bytes (node.rs:92-115)
};
// A registered shader (transformations/shader.rs: Shader): its parameter type and its compiled module.  The registry and
// the scene nodes hold it by shared_ptr; the renderer unloads the module after the last tick that launched it.
struct ShaderProgram {
    std::optional<ShaderParamType> param_type;
    bool wgsl = false;                    // built by smr_register_wgsl_shader: drawn through its vertex stage
    uint32_t uniform_size = 0;            // WGSL: SizeOf of the uniform; the parameter bytes are zero-padded to it
    std::vector<char> cubin;              // NVRTC's image for sm_90a
    void *library = nullptr;              // cudaLibrary_t (device handles only)
    const void *kernel = nullptr;         // its smr_shader_main, a cudaKernel_t
};

// scene::Component (scene.rs:50-60); only the variants on the compositor path
struct Component {
    int type = SMR_COMPONENT_VIEW;
    std::optional<std::string> id;
    std::vector<Component> children;
    std::string input_id;
    Position position;
    std::optional<Transition> transition;
    BorderRadius border_radius;
    float border_width = 0;
    RGBA border_color;
    std::vector<BoxShadow> box_shadow;
    int direction = SMR_DIRECTION_ROW;
    int overflow = SMR_OVERFLOW_HIDDEN;
    RGBA background_color;
    Padding padding;
    int rescale_mode = SMR_RESCALE_FIT;
    int horizontal_align = SMR_HALIGN_CENTER;
    int vertical_align = SMR_VALIGN_CENTER;
    OptF tiles_width, tiles_height;
    uint32_t tile_aspect_w = 16, tile_aspect_h = 9;
    float tiles_margin = 0, tiles_padding = 0;
    std::shared_ptr<const TextPayload> text;
    std::string image_id;                  // Image
    OptF image_width, image_height;
    std::string web_renderer_id;           // WebView (children: the embedded components)
    std::string shader_id;                 // Shader (children: its textures)
    std::optional<ShaderParamValue> shader_param;
    float shader_width = 0, shader_height = 0;
};

// Converts the C tree; returns false + message for variants outside the hot path.
bool component_from_c(const smr_component *c, Component &out, std::string &err, int depth = 0);

// ----- transformations/layout.rs:40-165 -------------------------------------------------------
struct Crop {
    float top = 0, left = 0, width = 0, height = 0;
};

struct Mask {
    BorderRadius radius;
    float top = 0, left = 0, width = 0, height = 0;
};

struct LayoutContent {
    enum Kind { Color, ChildNode, None } kind = None;
    RGBA color;
    size_t index = 0;
    Size size;
};

struct RenderLayout {
    enum Kind { Color = 1, ChildNode = 0, BoxShadow = 2 };  // numeric = layout_type of the shader
    float top = 0, left = 0, width = 0, height = 0, rotation_degrees = 0;
    BorderRadius border_radius;
    std::vector<Mask> masks;
    Kind kind = Color;
    RGBA color;         // Color / BoxShadow
    RGBA border_color;  // Color / ChildNode
    float border_width = 0;
    size_t index = 0;   // ChildNode
    Crop crop;          // ChildNode
    float blur_radius = 0;
};

struct NestedLayout {
    float top = 0, left = 0, width = 0, height = 0, rotation_degrees = 0;
    float scale_x = 1.0f, scale_y = 1.0f;
    std::optional<Crop> crop;
    std::optional<Mask> mask;
    LayoutContent content;
    float border_width = 0;
    RGBA border_color;
    BorderRadius border_radius;
    std::vector<BoxShadow> box_shadow;
    std::vector<NestedLayout> children;
    size_t child_nodes_count = 0;

    static NestedLayout child_nodes_placeholder(size_t child_nodes_count);  // layout.rs:280-304
    // layout/flatten.rs:10-22
    std::vector<RenderLayout> flatten(const std::vector<std::optional<Resolution>> &input_resolutions,
                                      Resolution resolution) const;
};

// ----- stateful components (scene/{view,rescaler,tiles}_component.rs) --------------------------
struct ViewParam {
    std::optional<std::string> id;
    int direction = SMR_DIRECTION_ROW;
    Position position;
    int overflow = SMR_OVERFLOW_HIDDEN;
    RGBA background_color;
    BorderRadius border_radius;
    float border_width = 0;
    RGBA border_color;
    std::vector<BoxShadow> box_shadow;
    Padding padding;
    bool operator==(const ViewParam &o) const;
};

struct RescalerParam {
    std::optional<std::string> id;
    Position position;
    int mode = SMR_RESCALE_FIT;
    int horizontal_align = SMR_HALIGN_CENTER;
    int vertical_align = SMR_VALIGN_CENTER;
    BorderRadius border_radius;
    float border_width = 0;
    RGBA border_color;
    std::vector<BoxShadow> box_shadow;
    bool operator==(const RescalerParam &o) const;
};

struct TilesParam {
    std::optional<std::string> id;
    OptF width, height;
    RGBA background_color;
    uint32_t aspect_w = 16, aspect_h = 9;
    float margin = 0, padding = 0;
    int horizontal_align = SMR_HALIGN_CENTER;
    int vertical_align = SMR_VALIGN_CENTER;
    bool operator==(const TilesParam &o) const;
};

struct TileId {
    bool is_component = false;
    std::string component_id;
    size_t index = 0;
    bool operator==(const TileId &o) const {
        return is_component == o.is_component && component_id == o.component_id && index == o.index;
    }
};

struct Tile {
    TileId id;
    float top = 0, left = 0, width = 0, height = 0;
};
using OptTile = std::optional<Tile>;
using TilesSnapshot = std::pair<std::vector<OptTile>, Size>;

// scene/transition.rs:20-106
struct TransitionState {
    double offset_progress = 0.0, offset_state = 0.0;
    uint64_t start_pts_ns = 0;
    uint64_t duration_ns = 0;
    InterpolationKind interpolation;

    static std::optional<TransitionState> create(const std::optional<Transition> &current,
                                                 const std::optional<TransitionState> &previous,
                                                 bool props_changed, bool interrupt_previous,
                                                 uint64_t last_pts_ns);
    double state(uint64_t pts_ns) const;
    bool is_finished(uint64_t pts_ns) const { return start_pts_ns + duration_ns <= pts_ns; }
};

struct Stateful {
    enum Kind { InputStream, View, Tiles, Rescaler, Text, Image, WebView, Shader } kind = View;
    // InputStream (scene/input_stream_component.rs), Text (scene/text_component.rs), Image (scene/image_component.rs),
    // WebView (scene/web_view_component.rs): the node children of a layout
    std::string input_id;
    std::optional<std::string> leaf_component_id;
    Size size;                                // InputStream: its last frame's resolution; Text: the layout resolution; Image: the
                                              // node's; WebView: the instance's
    std::shared_ptr<const TextPayload> text;
    std::string image_id;                     // Image: the component (with leaf_component_id) ...
    OptF image_width, image_height;
    ImageParams image;                        // ... and what it resolved to
    std::shared_ptr<WebInstance> web;         // WebView: the instance; `children` are its embedded components (render
                                              // nodes of their own, not laid out by the WebView's parent)
    std::shared_ptr<const ShaderProgram> shader;   // Shader: the program; `children` are its textures (render nodes)
    std::optional<ShaderParamValue> shader_param;
    // View
    std::optional<ViewParam> view_start;
    ViewParam view_end;
    // Rescaler
    std::optional<RescalerParam> rescaler_start;
    RescalerParam rescaler_end;
    // Tiles
    TilesParam tiles;
    std::optional<TilesSnapshot> tiles_start, tiles_last_layout;

    std::optional<TransitionState> transition;
    std::vector<Stateful> children;  // Rescaler: exactly one

    bool is_layout() const { return kind == View || kind == Tiles || kind == Rescaler; }
    const std::optional<std::string> &component_id() const;
    OptF width(uint64_t pts) const;   // scene.rs:105-117
    OptF height(uint64_t pts) const;  // scene.rs:119-131
    Position position(uint64_t pts) const;
    NestedLayout layout(Size size, uint64_t pts);  // scene/layout.rs:44-50
    void node_children(std::vector<const Stateful *> &out) const;  // scene/layout.rs:95-103
    size_t node_children_count() const;
    void update_state(const std::optional<Resolution> *inputs, size_t n);  // scene/layout.rs:105-137
};

// A render node of an output (scene/layout.rs:95-103): the caller's input `input_id`, or entry `index` of the output's
// list of that kind (OutputNode::texts, images, webs, shaders or nested)
struct NodeRef {
    enum Kind { Input, Text, Image, Web, Shader, Layout } kind = Input;
    int index = -1;
    std::string input_id;
};

// A layout node (scene_state.rs:154-228, NodeParams::Layout): an output's root that is a layout, or a View, Tiles or
// Rescaler whose parent is a Shader or a WebView.  Its own clone of the stateful component, its size (the output's resolution for the
// root; node_size at the last render's pts, the component's width and height, otherwise), its node children in DFS order,
// and its depth (1 + its deepest child's; unused for the root).  A node below the root is composited into its own texture
// every tick.  smr_set_layouts gives the root's flattened layouts and resolution instead, used as they are.
struct LayoutParams {
    Stateful root;
    Size size;
    std::vector<NodeRef> children;
    int depth = 1;
    std::optional<std::vector<RenderLayout>> given_layouts;   // smr_set_layouts: `root` and `size` are unused
    Resolution given_resolution;
    Resolution resolution(uint64_t pts) const;   // SizedLayoutComponent::resolution (scene/layout.rs:245-257)
    // The flattened layouts at `pts` (layout.rs:176-181), untruncated; laying them out advances the state of `root`
    std::vector<RenderLayout> layouts(uint64_t pts, const std::vector<std::optional<Resolution>> &inputs);
};

// A WebView render node (state/node.rs:127-141, NodeParams::Web): the instance and its children, each its own node.
// depth: 1 + the deepest child's, as for ShaderParams.
struct WebParams {
    std::shared_ptr<WebInstance> instance;
    std::vector<NodeRef> children;            // Input, Text, Image or Layout nodes
    int depth = 1;
};

// A Shader render node (state/node.rs, NodeParams::Shader): the program, the parameter bytes, the node's resolution
// (Size as Resolution: `as usize`) and its children, each its own node.  depth: 1 + the deepest child's (an input, text or
// image 0; a web, shader or layout node its own), so that a tick draws every child before the node that reads it.
struct ShaderParams {
    std::shared_ptr<const ShaderProgram> shader;
    std::vector<uint8_t> param_bytes;
    Resolution resolution;
    std::vector<NodeRef> children;
    int depth = 1;
};

// scene/scene_state.rs
struct OutputNode {
    std::optional<NodeRef> root;              // the root render node; empty: the root is a layout, `root_layout`
    LayoutParams root_layout;
    std::vector<std::shared_ptr<const TextPayload>> texts;   // the output's text nodes (the root, or children in DFS order)
    std::vector<ImageParams> images;          // the output's image nodes, likewise (web view children included)
    std::vector<WebParams> webs;              // the output's web nodes, likewise
    std::vector<ShaderParams> shaders;        // the output's shader nodes, children before parents
    std::vector<LayoutParams> nested;         // the output's layout nodes below the root, DFS order, children before parents
    Resolution resolution;
};

class SceneState {
  public:
    void register_render_event(uint64_t pts_ns, std::map<std::string, Resolution> input_resolutions);
    void unregister_output(const std::string &output_id);
    // returns false and fills err on SceneError.  `accept` sees the new node before any state changes; when it returns
    // false the update is dropped and the scene stays as it was.
    bool update_scene(const std::string &output_id, const Component &root, Resolution resolution,
                      OutputNode &out, std::string &err, const std::function<bool(OutputNode &)> &accept = nullptr);
    // the image registry (registry.rs:57-68): false when the id is taken / unknown
    bool register_image(const std::string &image_id, std::shared_ptr<const ImageAsset> asset);
    bool unregister_image(const std::string &image_id);
    // the web renderer registry (registry.rs:57-68), likewise; web_instance: nullptr when the id is unknown
    bool register_web(const std::string &instance_id, std::shared_ptr<WebInstance> instance);
    bool unregister_web(const std::string &instance_id);
    WebInstance *web_instance(const std::string &instance_id) const;
    // the shader registry (registry.rs:57-68), likewise
    bool register_shader(const std::string &shader_id, std::shared_ptr<const ShaderProgram> shader);
    bool unregister_shader(const std::string &shader_id);
    bool has_shader(const std::string &shader_id) const { return shaders_.count(shader_id) != 0; }
    uint64_t last_pts() const { return last_pts_ns_; }

  private:
    struct OutputSceneState {
        Stateful root;
        Resolution resolution;
    };
    std::map<std::string, Component> output_scenes_;
    std::map<std::string, OutputSceneState> output_states_;
    uint64_t last_pts_ns_ = 0;
    std::map<std::string, Resolution> input_resolutions_;
    std::map<std::string, std::shared_ptr<const ImageAsset>> images_;
    std::map<std::string, std::shared_ptr<WebInstance>> webs_;
    std::map<std::string, std::shared_ptr<const ShaderProgram>> shaders_;
};

double cubic_bezier_easing(double progress, double x1, double y1, double x2, double y2);
double bounce_easing(double t);

}  // namespace smr
