// scene.cpp -- host layout engine: Component tree -> NestedLayout (see scene.h).
// Restates smelter-render/src/scene/** ; each block cites the file:line it follows.
#include "scene.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <set>
#include <tuple>

namespace smr {

// ------------------------------------------------------------------------------------------------
// value types (scene/types.rs)
// ------------------------------------------------------------------------------------------------
static inline float fclamp(float v, float lo, float hi) { return std::fmin(std::fmax(v, lo), hi); }

BorderRadius BorderRadius::clip_to_size(Size size) const {  // types.rs:109-117
    float max_radius = std::fmax(0.0f, std::fmin(size.width, size.height) / 2.0f);
    return {fclamp(top_left, 0.0f, max_radius), fclamp(top_right, 0.0f, max_radius),
            fclamp(bottom_right, 0.0f, max_radius), fclamp(bottom_left, 0.0f, max_radius)};
}
BorderRadius BorderRadius::operator*(float rhs) const {
    return {top_left * rhs, top_right * rhs, bottom_right * rhs, bottom_left * rhs};
}
BorderRadius BorderRadius::operator+(float rhs) const {  // types.rs:141-152: floors at 0
    return {std::fmax(top_left + rhs, 0.0f), std::fmax(top_right + rhs, 0.0f),
            std::fmax(bottom_right + rhs, 0.0f), std::fmax(bottom_left + rhs, 0.0f)};
}

static OptF map_add(const OptF &v, float d) { return v ? OptF(*v + d) : OptF(); }

Position Position::with_border(float bw) const {
    Position p = *this;
    p.width = map_add(width, 2.0f * bw);
    p.height = map_add(height, 2.0f * bw);
    return p;
}
Position Position::with_padding(const Padding &pad) const {
    Position p = *this;
    p.width = map_add(width, pad.horizontal());
    p.height = map_add(height, pad.vertical());
    return p;
}
bool Position::operator==(const Position &o) const {
    if (absolute != o.absolute || width != o.width || height != o.height) return false;
    if (!absolute) return true;
    return from_right == o.from_right && horizontal_offset == o.horizontal_offset &&
           from_bottom == o.from_bottom && vertical_offset == o.vertical_offset &&
           rotation_degrees == o.rotation_degrees;
}

bool ViewParam::operator==(const ViewParam &o) const {
    return id == o.id && direction == o.direction && position == o.position && overflow == o.overflow &&
           background_color == o.background_color && border_radius == o.border_radius &&
           border_width == o.border_width && border_color == o.border_color && box_shadow == o.box_shadow &&
           padding == o.padding;
}
bool RescalerParam::operator==(const RescalerParam &o) const {
    return id == o.id && position == o.position && mode == o.mode && horizontal_align == o.horizontal_align &&
           vertical_align == o.vertical_align && border_radius == o.border_radius &&
           border_width == o.border_width && border_color == o.border_color && box_shadow == o.box_shadow;
}
bool TilesParam::operator==(const TilesParam &o) const {
    return id == o.id && width == o.width && height == o.height && background_color == o.background_color &&
           aspect_w == o.aspect_w && aspect_h == o.aspect_h && margin == o.margin && padding == o.padding &&
           horizontal_align == o.horizontal_align && vertical_align == o.vertical_align;
}

// ------------------------------------------------------------------------------------------------
// C struct -> Component
// ------------------------------------------------------------------------------------------------
static RGBA rgba_from_c(const smr_rgba &c) { return {c.r, c.g, c.b, c.a}; }
static OptF optf_from_c(const smr_opt_f32 &o) { return o.has_value ? OptF(o.value) : OptF(); }

// The atlases of one tree, by the caller's data pointer and geometry (pointer, width, height, pitch, row bytes): each is
// copied once
using AtlasKey = std::tuple<const void *, uint32_t, uint32_t, size_t, size_t>;
using AtlasCopies = std::map<AtlasKey, std::shared_ptr<const TextAtlas>>;

// smr_text -> TextPayload with smr_render_text's checks (0 x 0 allowed: the reference's 1 x 1 transparent node texture)
static bool text_from_c(const smr_text *t, AtlasCopies &atlases, std::shared_ptr<const TextPayload> &out, std::string &err) {
    if (!t) { err = "Text component without a payload"; return false; }
    if (t->width > 16384 || t->height > 16384) { err = "text texture resolution out of range"; return false; }
    if (t->n_glyphs > (1u << 22)) { err = "too many glyphs"; return false; }
    if (t->n_glyphs && !t->glyphs) { err = "glyph pointer is null"; return false; }
    if (t->color_mode != 0 && t->color_mode != 1) { err = "text color_mode must be 0 (Accurate) or 1 (Web)"; return false; }
    auto p = std::make_shared<TextPayload>();
    p->width = t->width; p->height = t->height;
    p->background = rgba_from_c(t->background);
    p->color_mode = t->color_mode;
    p->glyphs.assign(t->glyphs, t->glyphs + t->n_glyphs);
    bool need[2] = {false, false};   // mask, colour
    for (const smr_glyph &g : p->glyphs) {
        if (g.content == SMR_GLYPH_MASK) need[0] = true;
        else if (g.content == SMR_GLYPH_COLOR) need[1] = true;
        else { err = "glyph content type must be SMR_GLYPH_COLOR or SMR_GLYPH_MASK"; return false; }
    }
    const smr_atlas *atl[2] = {t->mask_atlas, t->color_atlas};
    std::shared_ptr<const TextAtlas> *dst[2] = {&p->mask, &p->color};
    for (int k = 0; k < 2; k++) {
        if (!need[k]) continue;
        const smr_atlas *a = atl[k];
        if (!a || !a->data || a->width == 0 || a->height == 0 || a->width > 16384 || a->height > 16384) {
            err = k == 0 ? "mask glyphs need a mask atlas" : "colour glyphs need a colour atlas";
            return false;
        }
        const size_t row = (size_t)a->width * (k == 0 ? 1 : 4), sp = a->pitch ? a->pitch : row;
        if (sp < row) { err = "atlas pitch smaller than a row"; return false; }
        const AtlasKey key{a->data, a->width, a->height, sp, row};
        auto hit = atlases.find(key);
        if (hit != atlases.end()) { *dst[k] = hit->second; continue; }
        auto copy = std::make_shared<TextAtlas>();
        copy->width = a->width; copy->height = a->height;
        copy->data.resize(row * a->height);
        for (uint32_t y = 0; y < a->height; y++)
            memcpy(copy->data.data() + row * y, (const uint8_t *)a->data + sp * y, row);
        atlases[key] = copy;
        *dst[k] = copy;
    }
    out = std::move(p);
    return true;
}

static bool shader_param_from_c(const smr_shader_param *p, ShaderParamValue &out, std::string &err, int depth) {
    if (depth > 64) { err = "shader parameter too deep"; return false; }
    out.kind = p->kind;
    if (p->field_name) out.field_name = p->field_name;
    switch (p->kind) {
        case SMR_SHADER_PARAM_F32: out.f32 = p->f32; return true;
        case SMR_SHADER_PARAM_U32: out.u32 = p->u32; return true;
        case SMR_SHADER_PARAM_I32: out.i32 = p->i32; return true;
        case SMR_SHADER_PARAM_LIST:
        case SMR_SHADER_PARAM_STRUCT:
            if (p->items_len && !p->items) { err = "shader parameter items pointer is null"; return false; }
            if (p->items_len > (1u << 20)) { err = "shader parameter has too many items"; return false; }
            out.items.resize(p->items_len);
            for (uint32_t i = 0; i < p->items_len; i++) {
                if (p->kind == SMR_SHADER_PARAM_STRUCT && !p->items[i].field_name) { err = "shader parameter field without a name"; return false; }
                if (!shader_param_from_c(&p->items[i], out.items[i], err, depth + 1)) return false;
            }
            return true;
        default: err = "unknown shader parameter kind"; return false;
    }
}

void ShaderParamValue::to_bytes(std::vector<uint8_t> &out) const {   // little-endian, like the host
    const void *v = kind == SMR_SHADER_PARAM_F32 ? (const void *)&f32 : kind == SMR_SHADER_PARAM_U32 ? (const void *)&u32 : (const void *)&i32;
    if (kind <= SMR_SHADER_PARAM_I32) { out.insert(out.end(), (const uint8_t *)v, (const uint8_t *)v + 4); return; }
    for (const ShaderParamValue &i : items) i.to_bytes(out);
}

static bool component_from_c(const smr_component *c, Component &out, std::string &err, int depth, AtlasCopies &atlases) {
    if (!c) { err = "null component"; return false; }
    if (depth > 256) { err = "component tree too deep"; return false; }
    out = Component();
    out.type = c->type;
    if (c->id) out.id = std::string(c->id);
    switch (c->type) {
        case SMR_COMPONENT_INPUT_STREAM:
            if (!c->input_id) { err = "InputStream without input_id"; return false; }
            out.input_id = c->input_id;
            return true;
        case SMR_COMPONENT_TEXT:
            return text_from_c(c->text, atlases, out.text, err);
        case SMR_COMPONENT_IMAGE:
            if (!c->image_id) { err = "component type outside the compositor hot path (Image without image_id)"; return false; }
            out.image_id = c->image_id;
            out.image_width = optf_from_c(c->image_width);
            out.image_height = optf_from_c(c->image_height);
            return true;
        case SMR_COMPONENT_WEB_VIEW:
            if (!c->web_renderer_id) { err = "component type outside the compositor hot path (WebView without web_renderer_id)"; return false; }
            out.web_renderer_id = c->web_renderer_id;
            if (c->children_len && !c->children) { err = "children pointer is null"; return false; }
            out.children.resize(c->children_len);
            for (uint32_t i = 0; i < c->children_len; i++) {
                // a direct WebView or Shader child, and a layout child without both sides, stay refused with the status
                // they had before layout children were accepted (the reference would answer
                // UnknownDimensionsForLayoutNodeRoot for the sizeless layout child)
                const smr_component &k = c->children[i];
                const bool sized = k.type == SMR_COMPONENT_TILES ? k.tiles_width.has_value && k.tiles_height.has_value
                                                                 : k.position.width.has_value && k.position.height.has_value;
                if (k.type == SMR_COMPONENT_WEB_VIEW || k.type == SMR_COMPONENT_SHADER ||
                    ((k.type == SMR_COMPONENT_VIEW || k.type == SMR_COMPONENT_TILES || k.type == SMR_COMPONENT_RESCALER) && !sized)) {
                    err = "a WebView or Shader child of a WebView, or a View, Tiles or Rescaler child without width and height, "
                          "is outside the compositor hot path";
                    return false;
                }
                if (!component_from_c(&k, out.children[i], err, depth + 1, atlases)) return false;
            }
            return true;
        case SMR_COMPONENT_SHADER:
            if (!c->shader_id) { err = "component type outside the compositor hot path (Shader without shader_id)"; return false; }
            out.shader_id = c->shader_id;
            out.shader_width = c->shader_width;
            out.shader_height = c->shader_height;
            if (c->shader_param) {
                out.shader_param.emplace();
                if (!shader_param_from_c(c->shader_param, *out.shader_param, err, 0)) return false;
            }
            if (c->children_len && !c->children) { err = "children pointer is null"; return false; }
            if (c->children_len > 16) { err = "a Shader with more than 16 children is outside the compositor hot path (16 textures)"; return false; }
            out.children.resize(c->children_len);
            for (uint32_t i = 0; i < c->children_len; i++)
                if (!component_from_c(&c->children[i], out.children[i], err, depth + 1, atlases)) return false;
            return true;
        case SMR_COMPONENT_VIEW:
        case SMR_COMPONENT_TILES:
        case SMR_COMPONENT_RESCALER:
            break;
        default:
            err = "component type outside the compositor hot path";
            return false;
    }
    if (c->type == SMR_COMPONENT_RESCALER && c->children_len != 1) {
        err = "Rescaler needs exactly one child";
        return false;
    }
    if (c->children_len && !c->children) { err = "children pointer is null"; return false; }
    out.children.resize(c->children_len);
    for (uint32_t i = 0; i < c->children_len; i++)
        if (!component_from_c(&c->children[i], out.children[i], err, depth + 1, atlases)) return false;

    const smr_position &p = c->position;
    out.position.absolute = p.is_absolute != 0;
    out.position.width = optf_from_c(p.width);
    out.position.height = optf_from_c(p.height);
    out.position.from_right = p.horizontal_from_right != 0;
    out.position.horizontal_offset = p.horizontal_offset;
    out.position.from_bottom = p.vertical_from_bottom != 0;
    out.position.vertical_offset = p.vertical_offset;
    out.position.rotation_degrees = p.rotation_degrees;
    if (c->transition.present) {
        Transition t;
        t.duration_ns = c->transition.duration_ns;
        t.interpolation.kind = c->transition.interpolation_kind;
        t.interpolation.x1 = c->transition.x1; t.interpolation.y1 = c->transition.y1;
        t.interpolation.x2 = c->transition.x2; t.interpolation.y2 = c->transition.y2;
        t.should_interrupt = c->transition.should_interrupt != 0;
        out.transition = t;
    }
    out.border_radius = {c->border_radius.top_left, c->border_radius.top_right, c->border_radius.bottom_right,
                         c->border_radius.bottom_left};
    out.border_width = c->border_width;
    out.border_color = rgba_from_c(c->border_color);
    if (c->box_shadow_len && !c->box_shadow) { err = "box_shadow pointer is null"; return false; }
    for (uint32_t i = 0; i < c->box_shadow_len; i++) {
        const smr_box_shadow &s = c->box_shadow[i];
        out.box_shadow.push_back({s.offset_x, s.offset_y, s.blur_radius, rgba_from_c(s.color)});
    }
    out.direction = c->direction;
    out.overflow = c->overflow;
    out.background_color = rgba_from_c(c->background_color);
    out.padding = {c->padding.top, c->padding.right, c->padding.bottom, c->padding.left};
    out.rescale_mode = c->rescale_mode;
    out.horizontal_align = c->horizontal_align;
    out.vertical_align = c->vertical_align;
    out.tiles_width = optf_from_c(c->tiles_width);
    out.tiles_height = optf_from_c(c->tiles_height);
    out.tile_aspect_w = c->tile_aspect_ratio_w;
    out.tile_aspect_h = c->tile_aspect_ratio_h;
    out.tiles_margin = c->tiles_margin;
    out.tiles_padding = c->tiles_padding;
    if (c->type == SMR_COMPONENT_TILES && (out.tile_aspect_w == 0 || out.tile_aspect_h == 0)) {
        err = "Tiles tile_aspect_ratio must be non-zero";
        return false;
    }
    return true;
}

bool component_from_c(const smr_component *c, Component &out, std::string &err, int depth) {
    AtlasCopies atlases;
    return component_from_c(c, out, err, depth, atlases);
}

// ------------------------------------------------------------------------------------------------
// easing (scene/transition/{bounce,cubic_bezier}.rs) -- f64
// ------------------------------------------------------------------------------------------------
double bounce_easing(double t) {  // bounce.rs:1-14
    const double n1 = 7.5625, d1 = 2.75;
    if (t < (1.0 / d1)) return n1 * t * t;
    if (t < (2.0 / d1)) return n1 * (t - 1.5 / d1) * (t - 1.5 / d1) + 0.75;
    if (t < (2.5 / d1)) return n1 * (t - 2.25 / d1) * (t - 2.25 / d1) + 0.9375;
    return n1 * (t - 2.625 / d1) * (t - 2.625 / d1) + 0.984375;
}

static const double kAllowedError = 1e-7;  // cubic_bezier.rs:3
static bool close_to(double a, double b) { return std::fabs(a - b) < kAllowedError; }
static double clamp_root(double v) {  // cubic_bezier.rs:120-137
    if (v < 0.0) return v >= -kAllowedError ? 0.0 : NAN;
    if (v > 1.0) return v <= 1.0 + kAllowedError ? 1.0 : NAN;
    return v;  // NaN passes through as NaN
}

static double find_first_cubic_root(double p0, double p1, double p2, double p3) {  // cubic_bezier.rs:32-112
    double a = 3.0 * (p0 - 2.0 * p1 + p2);
    double b = 3.0 * (p1 - p0);
    double c = p0;
    double d = -p0 + 3.0 * (p1 - p2) + p3;
    if (close_to(d, 0.0)) {
        if (close_to(a, 0.0)) {
            if (close_to(b, 0.0)) return NAN;
            return clamp_root(-c / b);
        }
        double q = std::sqrt(b * b - 4.0 * a * c);
        double a2 = 2.0 * a;
        double root = clamp_root((q - b) / a2);
        if (!std::isnan(root)) return root;
        return clamp_root((-b - q) / a2);
    }
    a = a / d; b = b / d; c = c / d;
    double o3 = (3.0 * b - a * a) / 9.0;
    double q2 = (2.0 * (a * a * a) - 9.0 * a * b + 27.0 * c) / 54.0;
    double a3 = a / 3.0;
    double discriminant = q2 * q2 + o3 * o3 * o3;
    const double PI = 3.14159265358979323846264338327950288;
    if (discriminant < 0.0) {
        double mp33 = -(o3 * o3 * o3);
        double r = std::sqrt(mp33);
        double cos_phi = std::fmin(std::fmax(-q2 / r, -1.0), 1.0);
        double phi = std::acos(cos_phi);
        double t1 = 2.0 * std::cbrt(r);
        double root = clamp_root(t1 * std::cos(phi / 3.0) - a3);
        if (!std::isnan(root)) return root;
        root = clamp_root(t1 * std::cos((phi + 2.0 * PI) / 3.0) - a3);
        if (!std::isnan(root)) return root;
        return clamp_root(t1 * std::cos((phi + 4.0 * PI) / 3.0) - a3);
    }
    if (discriminant == 0.0) {
        double u1 = -std::cbrt(q2);
        double root = clamp_root(2.0 * u1 - a3);
        if (!std::isnan(root)) return root;
        return clamp_root(-u1 - a3);
    }
    double sd = std::sqrt(discriminant);
    double u1 = std::cbrt(-q2 + sd);
    double v1 = std::cbrt(q2 + sd);
    return clamp_root(u1 - v1 - a3);
}

double cubic_bezier_easing(double progress, double x1, double y1, double x2, double y2) {  // cubic_bezier.rs:5-20
    if (close_to(progress, 0.0)) return 0.0;
    if (close_to(progress, 1.0)) return 1.0;
    double t = find_first_cubic_root(-progress, x1 - progress, x2 - progress, 1.0 - progress);
    if (std::isnan(t)) return 1.0;
    double a = 1.0 / 3.0 + (y1 - y2);
    double b = y2 - 2.0 * y1;
    double c = y1;
    double v = 3.0 * ((a * t + b) * t + c) * t;
    return std::fmin(std::fmax(v, 0.0), 1.0);
}

double InterpolationKind::state(double t) const {
    switch (kind) {
        case SMR_INTERP_BOUNCE: return bounce_easing(t);
        case SMR_INTERP_CUBIC_BEZIER: return cubic_bezier_easing(t, x1, y1, x2, y2);
        default: return t;
    }
}

// Duration::as_secs_f64
static double secs_f64(uint64_t ns) {
    return (double)(ns / 1000000000ull) + (double)(ns % 1000000000ull) / 1000000000.0;
}

std::optional<TransitionState> TransitionState::create(const std::optional<Transition> &current,
                                                       const std::optional<TransitionState> &previous,
                                                       bool props_changed, bool interrupt_previous,
                                                       uint64_t last_pts) {  // transition.rs:39-79
    auto from_options = [&](const Transition &t) {
        TransitionState s;
        s.start_pts_ns = last_pts;
        s.duration_ns = t.duration_ns;
        s.interpolation = t.interpolation;
        return s;
    };
    if (previous && !previous->is_finished(last_pts)) {
        if (props_changed && interrupt_previous) {
            if (current) return from_options(*current);
            return std::nullopt;
        }
        uint64_t end = previous->start_pts_ns + previous->duration_ns;
        uint64_t remaining = end > last_pts ? end - last_pts : 0;
        TransitionState s;
        s.offset_progress = 1.0 - (secs_f64(remaining) / secs_f64(previous->duration_ns));
        s.offset_state = previous->interpolation.state(s.offset_progress);
        s.start_pts_ns = last_pts;
        s.duration_ns = remaining;
        s.interpolation = current ? current->interpolation : previous->interpolation;
        return s;
    }
    if (props_changed && current) return from_options(*current);
    return std::nullopt;
}

double TransitionState::state(uint64_t pts) const {  // transition.rs:91-102
    double progress = (secs_f64(pts) - secs_f64(start_pts_ns)) / secs_f64(duration_ns);
    progress = offset_progress + progress * (1.0 - offset_progress);
    if (progress < 0.0) progress = 0.0;  // f64::clamp: NaN stays NaN
    if (progress > 1.0) progress = 1.0;
    double st = interpolation.state(progress);
    return (st - offset_state) / (1.0 - offset_state);
}

// ------------------------------------------------------------------------------------------------
// ContinuousValue (scene/types/interpolation.rs, components/interpolation.rs)
// ------------------------------------------------------------------------------------------------
static float lerp_f32(float a, float b, double s) { return (float)((double)a + (((double)b - (double)a) * s)); }
static OptF lerp_opt(const OptF &a, const OptF &b, double s) {
    if (a && b) return OptF(lerp_f32(*a, *b, s));
    return b;
}
static Position lerp_position(const Position &a, const Position &b, double s) {  // components/interpolation.rs:8-52
    if (a.absolute != b.absolute) return b;
    Position r = b;
    r.width = lerp_opt(a.width, b.width, s);
    r.height = lerp_opt(a.height, b.height, s);
    if (!b.absolute) return r;
    if (a.from_right == b.from_right) r.horizontal_offset = lerp_f32(a.horizontal_offset, b.horizontal_offset, s);
    if (a.from_bottom == b.from_bottom) r.vertical_offset = lerp_f32(a.vertical_offset, b.vertical_offset, s);
    r.rotation_degrees = lerp_f32(a.rotation_degrees, b.rotation_degrees, s);
    return r;
}
static BorderRadius lerp_radius(const BorderRadius &a, const BorderRadius &b, double s) {
    return {lerp_f32(a.top_left, b.top_left, s), lerp_f32(a.top_right, b.top_right, s),
            lerp_f32(a.bottom_right, b.bottom_right, s), lerp_f32(a.bottom_left, b.bottom_left, s)};
}
static std::vector<BoxShadow> lerp_shadows(const std::vector<BoxShadow> &a, const std::vector<BoxShadow> &b,
                                           double s) {  // components/interpolation.rs:68-90
    std::vector<BoxShadow> r;
    size_t n = std::min(a.size(), b.size());
    for (size_t i = 0; i < n; i++)
        r.push_back({lerp_f32(a[i].offset_x, b[i].offset_x, s), lerp_f32(a[i].offset_y, b[i].offset_y, s),
                     lerp_f32(a[i].blur_radius, b[i].blur_radius, s), b[i].color});
    for (size_t i = n; i < b.size(); i++) r.push_back(b[i]);
    return r;
}
static Padding lerp_padding(const Padding &a, const Padding &b, double s) {
    return {lerp_f32(a.top, b.top, s), lerp_f32(a.right, b.right, s), lerp_f32(a.bottom, b.bottom, s),
            lerp_f32(a.left, b.left, s)};
}
static ViewParam lerp_view(const ViewParam &a, const ViewParam &b, double s) {  // view_component/interpolation.rs
    ViewParam r = b;
    r.position = lerp_position(a.position, b.position, s);
    r.border_radius = lerp_radius(a.border_radius, b.border_radius, s);
    r.border_width = lerp_f32(a.border_width, b.border_width, s);
    r.box_shadow = lerp_shadows(a.box_shadow, b.box_shadow, s);
    r.padding = lerp_padding(a.padding, b.padding, s);
    return r;
}
static RescalerParam lerp_rescaler(const RescalerParam &a, const RescalerParam &b, double s) {
    RescalerParam r = b;
    r.position = lerp_position(a.position, b.position, s);
    r.border_radius = lerp_radius(a.border_radius, b.border_radius, s);
    r.border_width = lerp_f32(a.border_width, b.border_width, s);
    r.box_shadow = lerp_shadows(a.box_shadow, b.box_shadow, s);
    return r;
}

// tiles_component/interpolation.rs:16-86
static bool positions_equal(const Tile &l, const Tile &r) {
    const float tol = 0.001f;
    return std::fabs(l.top - r.top) <= tol && std::fabs(l.left - r.left) <= tol &&
           std::fabs(l.width - r.width) <= tol && std::fabs(l.height - r.height) <= tol;
}
static std::vector<OptTile> lerp_tiles(const std::vector<OptTile> &start, const std::vector<OptTile> &end, double s) {
    if (s >= 1.0) return end;
    std::vector<OptTile> out;
    for (const OptTile &ot : end) {
        if (!ot) { out.push_back(std::nullopt); continue; }
        const Tile &tile = *ot;
        // start_id_map is a HashMap collected in order: a later duplicate id overwrites an earlier one
        const OptTile *old_slot = nullptr;
        for (const OptTile &st : start)
            if (st && st->id == tile.id) old_slot = &st;
        if (old_slot && *old_slot) {
            const Tile &o = **old_slot;
            Tile t;
            t.id = tile.id;
            t.top = lerp_f32(o.top, tile.top, s);
            t.left = lerp_f32(o.left, tile.left, s);
            t.width = lerp_f32(o.width, tile.width, s);
            t.height = lerp_f32(o.height, tile.height, s);
            out.push_back(t);
            continue;
        }
        OptTile res;
        for (const OptTile &st : start) {
            if (!st || !positions_equal(*st, tile)) continue;
            bool still_exists = false;
            for (const OptTile &e : end)
                if (e && e->id == st->id) still_exists = true;
            if (!still_exists) res = tile;
            break;  // .find(): first match decides
        }
        out.push_back(res);
    }
    return out;
}

// ------------------------------------------------------------------------------------------------
// Stateful accessors
// ------------------------------------------------------------------------------------------------
static ViewParam view_at(const Stateful &c, uint64_t pts) {  // view_component.rs:47-53
    if (c.transition && c.view_start) return lerp_view(*c.view_start, c.view_end, c.transition->state(pts));
    return c.view_end;
}
static RescalerParam rescaler_at(const Stateful &c, uint64_t pts) {  // rescaler_component.rs:48-54
    if (c.transition && c.rescaler_start) return lerp_rescaler(*c.rescaler_start, c.rescaler_end, c.transition->state(pts));
    return c.rescaler_end;
}

const std::optional<std::string> &Stateful::component_id() const {
    switch (kind) {
        case InputStream:
        case Text:
        case Image:
        case WebView:
        case Shader: return leaf_component_id;
        case View: return view_end.id;
        case Rescaler: return rescaler_end.id;
        default: return tiles.id;
    }
}

Position Stateful::position(uint64_t pts) const {
    switch (kind) {
        case View: {  // view_component.rs:63-69
            ViewParam v = view_at(*this, pts);
            return v.position.with_border(v.border_width).with_padding(v.padding);
        }
        case Rescaler: {  // rescaler_component.rs:64-67
            RescalerParam r = rescaler_at(*this, pts);
            return r.position.with_border(r.border_width);
        }
        case Tiles: {  // tiles_component.rs:71-76
            Position p;
            p.width = tiles.width;
            p.height = tiles.height;
            return p;
        }
        default: {
            Position p;
            p.width = size.width;
            p.height = size.height;
            return p;
        }
    }
}

OptF Stateful::width(uint64_t pts) const {
    if (!is_layout()) return OptF(size.width);
    return position(pts).width;
}
OptF Stateful::height(uint64_t pts) const {
    if (!is_layout()) return OptF(size.height);
    return position(pts).height;
}

void Stateful::node_children(std::vector<const Stateful *> &out) const {
    for (const Stateful &c : children) {
        if (c.is_layout()) c.node_children(out);
        else out.push_back(&c);
    }
}
size_t Stateful::node_children_count() const {
    size_t n = 0;
    for (const Stateful &c : children) n += c.is_layout() ? c.node_children_count() : 1;
    return n;
}

void Stateful::update_state(const std::optional<Resolution> *inputs, size_t n) {  // scene/layout.rs:105-137
    size_t off = 0;
    for (Stateful &c : children) {
        if (c.kind == InputStream) {
            if (off < n && inputs[off]) c.size = {(float)inputs[off]->width, (float)inputs[off]->height};
            else c.size = {0.0f, 0.0f};
            off += 1;
        } else if (!c.is_layout()) {
            off += 1;   // Text, Image, WebView, Shader: no state
        } else {
            size_t cnt = c.node_children_count();
            c.update_state(inputs + std::min(off, n), off < n ? std::min(cnt, n - off) : 0);
            off += cnt;
        }
    }
}

// scene/layout.rs:139-158
static LayoutContent layout_content(const Stateful &c, size_t index) {
    LayoutContent lc;
    if (c.is_layout()) { lc.kind = LayoutContent::None; return lc; }
    lc.kind = LayoutContent::ChildNode;
    lc.index = index;
    lc.size = c.size;
    return lc;
}

static NestedLayout wrap_child(float top, float left, float width, float height, float rotation,
                               Stateful &child, uint64_t pts) {
    // shared tail of layout_static_child / layout_absolute_position_child / tiles layout_child
    NestedLayout nl;
    nl.top = top; nl.left = left; nl.width = width; nl.height = height;
    nl.rotation_degrees = rotation;
    if (child.is_layout()) {
        NestedLayout inner = child.layout({width, height}, pts);
        nl.content.kind = LayoutContent::None;
        nl.child_nodes_count = inner.child_nodes_count;
        nl.children.push_back(std::move(inner));
    } else {
        nl.content = layout_content(child, 0);
        nl.child_nodes_count = 1;
    }
    return nl;
}

// scene/layout.rs:160-237
static NestedLayout layout_absolute_child(Stateful &child, const Position &pos, Size parent, uint64_t pts) {
    float width = pos.width ? *pos.width : parent.width;
    float height = pos.height ? *pos.height : parent.height;
    float top = pos.from_bottom ? parent.height - pos.vertical_offset - height : pos.vertical_offset;
    float left = pos.from_right ? parent.width - pos.horizontal_offset - width : pos.horizontal_offset;
    return wrap_child(top, left, width, height, pos.rotation_degrees, child, pts);
}

// ------------------------------------------------------------------------------------------------
// View (scene/view_component/layout.rs)
// ------------------------------------------------------------------------------------------------
namespace {
struct ViewLayouter {
    const ViewParam &p;
    uint64_t pts;

    bool is_static(const Stateful &c) const {  // static_children_iter :272-284
        if (!c.is_layout()) return true;
        return !c.position(pts).absolute;
    }
    float sum_static_children_sizes(const std::vector<Stateful> &children) const {  // :260-270
        float sum = 0.0f;
        for (const Stateful &c : children) {
            if (!is_static(c)) continue;
            OptF v = p.direction == SMR_DIRECTION_ROW ? c.width(pts) : c.height(pts);
            sum += v ? *v : 0.0f;
        }
        return sum;
    }
    float static_child_size(Size size, const std::vector<Stateful> &children) const {  // :203-229
        float max_size = p.direction == SMR_DIRECTION_ROW ? size.width - p.padding.horizontal()
                                                          : size.height - p.padding.vertical();
        size_t unknown = 0;
        for (const Stateful &c : children) {
            if (!is_static(c)) continue;
            OptF v = p.direction == SMR_DIRECTION_ROW ? c.width(pts) : c.height(pts);
            if (!v) unknown++;
        }
        float sum = sum_static_children_sizes(children);
        if (unknown == 0) return 0.0f;
        return std::fmax(0.0f, (max_size - sum) / (float)unknown);
    }
    float scale_factor_for_overflow_fit(Size content, const std::vector<Stateful> &children) const {  // :231-258
        float sum_size = std::fmax(sum_static_children_sizes(children), 0.000000001f);
        float max_size = p.direction == SMR_DIRECTION_ROW ? content.width : content.height;
        float max_alt = p.direction == SMR_DIRECTION_ROW ? content.height : content.width;
        bool any = false;
        float best = 0.0f;
        for (const Stateful &c : children) {
            if (!is_static(c)) continue;
            OptF v = p.direction == SMR_DIRECTION_ROW ? c.height(pts) : c.width(pts);
            float val = v ? *v : 0.0f;
            // Iterator::max_by keeps the LAST of equal maxima; value-wise irrelevant
            if (!any || !(val < best)) best = val;
            any = true;
        }
        float max_alt_child = std::fmax(any ? best : 0.0f, 0.000000001f);
        return std::fmin(1.0f, std::fmin(max_size / sum_size, max_alt / max_alt_child));
    }
};
}  // namespace

static NestedLayout view_layout(const ViewParam &p, Size size, std::vector<Stateful> &children, uint64_t pts) {
    ViewLayouter L{p, pts};
    Size content = {std::fmax(size.width - 2.0f * p.border_width, 0.0f),
                    std::fmax(size.height - 2.0f * p.border_width, 0.0f)};
    BorderRadius border_radius = p.border_radius.clip_to_size(size);
    float static_child_size = L.static_child_size(content, children);
    float scale = 1.0f;
    std::optional<Mask> mask;
    if (p.overflow != SMR_OVERFLOW_VISIBLE) {
        if (p.overflow == SMR_OVERFLOW_FIT) scale = L.scale_factor_for_overflow_fit(content, children);
        Mask m;
        m.radius = border_radius - p.border_width;
        m.top = p.border_width; m.left = p.border_width;
        m.width = content.width; m.height = content.height;
        mask = m;
    }
    float static_offset = p.border_width / scale;
    float parent_border_width = p.border_width / scale;

    NestedLayout out;
    for (Stateful &child : children) {
        Position pos;
        if (child.is_layout()) pos = child.position(pts);
        else { pos.width = child.width(pts); pos.height = child.height(pts); }
        if (pos.absolute) {
            out.children.push_back(layout_absolute_child(child, pos, size, pts));
            continue;
        }
        // layout_static_child :129-197
        float top, left, width, height;
        if (p.direction == SMR_DIRECTION_ROW) {
            width = pos.width ? *pos.width : static_child_size;
            height = pos.height ? *pos.height : content.height - p.padding.vertical();
            top = parent_border_width + p.padding.top;
            left = static_offset + p.padding.left;
            static_offset += width;
        } else {
            height = pos.height ? *pos.height : static_child_size;
            width = pos.width ? *pos.width : content.width - p.padding.horizontal();
            top = static_offset + p.padding.top;
            left = parent_border_width + p.padding.left;
            static_offset += height;
        }
        out.children.push_back(wrap_child(top, left, width, height, 0.0f, child, pts));
    }
    out.top = 0.0f; out.left = 0.0f;
    out.width = size.width; out.height = size.height;
    out.scale_x = scale; out.scale_y = scale;
    out.mask = mask;
    out.content.kind = LayoutContent::Color;
    out.content.color = p.background_color;
    for (const NestedLayout &c : out.children) out.child_nodes_count += c.child_nodes_count;
    out.border_width = p.border_width;
    out.border_color = p.border_color;
    out.border_radius = border_radius;
    out.box_shadow = p.box_shadow;
    return out;
}

// ------------------------------------------------------------------------------------------------
// Rescaler (scene/rescaler_component/layout.rs)
// ------------------------------------------------------------------------------------------------
static NestedLayout rescaler_layout_with_scale(const RescalerParam &p, Size max_size, BorderRadius border_radius,
                                               Stateful &child, uint64_t pts, float scale) {  // :59-161
    OptF child_width = child.width(pts), child_height = child.height(pts);
    NestedLayout inner;
    if (child.is_layout()) {
        Size cs = {child_width ? *child_width : max_size.width / scale,
                   child_height ? *child_height : max_size.height / scale};
        NestedLayout cl = child.layout(cs, pts);
        inner.content.kind = LayoutContent::None;
        inner.child_nodes_count = cl.child_nodes_count;
        inner.children.push_back(std::move(cl));
    } else {
        inner.content = layout_content(child, 0);
        inner.child_nodes_count = 1;
    }
    OptF ch = child.height(pts), cw = child.width(pts);
    float top = 0.0f, left = 0.0f;
    switch (p.vertical_align) {
        case SMR_VALIGN_TOP: top = 0.0f; break;
        case SMR_VALIGN_BOTTOM: top = ch ? max_size.height - (*ch * scale) : 0.0f; break;
        default: top = ch ? (max_size.height - (*ch * scale)) / 2.0f : 0.0f; break;
    }
    switch (p.horizontal_align) {
        case SMR_HALIGN_LEFT: left = 0.0f; break;
        case SMR_HALIGN_RIGHT: left = cw ? max_size.width - (*cw * scale) : 0.0f; break;
        default: left = cw ? (max_size.width - (*cw * scale)) / 2.0f : 0.0f; break;
    }
    float width = cw ? *cw * scale : max_size.width;
    float height = ch ? *ch * scale : max_size.height;

    inner.top = top + p.border_width;
    inner.left = left + p.border_width;
    inner.width = width; inner.height = height;
    inner.scale_x = scale; inner.scale_y = scale;

    NestedLayout out;
    out.width = max_size.width + (p.border_width * 2.0f);
    out.height = max_size.height + (p.border_width * 2.0f);
    Mask m;
    m.radius = border_radius - p.border_width;
    m.top = p.border_width; m.left = p.border_width;
    m.width = max_size.width; m.height = max_size.height;
    out.mask = m;
    out.content.kind = LayoutContent::None;
    out.child_nodes_count = inner.child_nodes_count;
    out.children.push_back(std::move(inner));
    out.border_width = p.border_width;
    out.border_color = p.border_color;
    out.border_radius = border_radius;
    out.box_shadow = p.box_shadow;
    return out;
}

static NestedLayout rescaler_layout(const RescalerParam &p, Size size, Stateful &child, uint64_t pts) {  // :14-57
    Size content = {std::fmax(size.width - (2.0f * p.border_width), 0.0f),
                    std::fmax(size.height - (2.0f * p.border_width), 0.0f)};
    OptF cw = child.width(pts), ch = child.height(pts);
    BorderRadius br = p.border_radius.clip_to_size(size);
    float scale = 1.0f;
    if (!cw && ch) scale = content.height / *ch;
    else if (cw && !ch) scale = content.width / *cw;
    else if (cw && ch) {
        float sx = content.width / *cw, sy = content.height / *ch;
        scale = p.mode == SMR_RESCALE_FIT ? std::fmin(sx, sy) : std::fmax(sx, sy);
    }
    return rescaler_layout_with_scale(p, content, br, child, pts, scale);
}

// ------------------------------------------------------------------------------------------------
// Tiles (scene/tiles_component/{tiles,layout}.rs)
// ------------------------------------------------------------------------------------------------
namespace {
struct RowsCols { uint32_t rows, columns; };
}

static Size tile_size(const TilesParam &p, RowsCols rc, Size layout) {  // tiles.rs:81-99
    float x_padding = (float)rc.columns * 2.0f * p.padding;
    float y_padding = (float)rc.rows * 2.0f * p.padding;
    float x_margin = ((float)rc.columns + 1.0f) * p.margin;
    float y_margin = ((float)rc.rows + 1.0f) * p.margin;
    float x_scale = std::fmax(layout.width - x_padding - x_margin, 0.0f) / (float)rc.columns / (float)p.aspect_w;
    float y_scale = std::fmax(layout.height - y_padding - y_margin, 0.0f) / (float)rc.rows / (float)p.aspect_h;
    float scale = x_scale < y_scale ? x_scale : y_scale;
    return {(float)p.aspect_w * scale, (float)p.aspect_h * scale};
}

static RowsCols optimal_row_column_count(const TilesParam &p, uint32_t inputs, Size layout) {  // tiles.rs:59-79
    auto from_rows = [&](uint32_t rows) { return RowsCols{rows, (inputs + rows - 1) / rows}; };
    RowsCols best = from_rows(1);
    float best_w = 0.0f;
    for (uint32_t rows = 1; rows <= inputs; rows++) {
        RowsCols rc = from_rows(rows);
        float w = tile_size(p, rc, layout).width;
        if (w > best_w) { best = rc; best_w = w; }
    }
    return best;
}

static std::vector<OptTile> tiles_end_state(const TilesParam &p, Size size, const std::vector<Stateful> &children) {
    // tiles.rs:29-55 + tiles_positions :101-165
    uint32_t count = (uint32_t)children.size();
    std::vector<OptTile> out;
    if (count == 0) return out;
    RowsCols rc = optimal_row_column_count(p, count, size);
    Size ts = tile_size(p, rc, size);
    float additional_y = size.height - (ts.height + 2.0f * p.padding) * (float)rc.rows - (p.margin * ((float)rc.rows + 1.0f));
    float add_top = 0.0f, just_y = 0.0f;
    switch (p.vertical_align) {
        case SMR_VALIGN_TOP: break;
        case SMR_VALIGN_CENTER: add_top = additional_y / 2.0f; break;
        case SMR_VALIGN_BOTTOM: add_top = additional_y; break;
        default: just_y = additional_y / ((float)rc.rows + 1.0f); break;
    }
    float top = add_top + just_y + p.padding + p.margin;
    size_t anon_index = 0, child_i = 0;
    for (uint32_t row = 0; row < rc.rows; row++) {
        uint32_t in_row = row < rc.rows - 1 ? rc.columns : count - ((rc.rows - 1) * rc.columns);
        float additional_x = size.width - (ts.width + 2.0f * p.padding) * (float)in_row - (p.margin * ((float)in_row + 1.0f));
        float add_left = 0.0f, just_x = 0.0f;
        switch (p.horizontal_align) {
            case SMR_HALIGN_LEFT: break;
            case SMR_HALIGN_RIGHT: add_left = additional_x; break;
            case SMR_HALIGN_JUSTIFIED: just_x = additional_x / (float)(in_row + 1); break;
            default: add_left = additional_x / 2.0f; break;
        }
        float left = add_left + just_x + p.margin + p.padding;
        for (uint32_t col = 0; col < in_row && child_i < children.size(); col++, child_i++) {
            Tile t;
            t.top = top; t.left = left; t.width = ts.width; t.height = ts.height;
            const std::optional<std::string> &cid = children[child_i].component_id();
            if (cid) { t.id.is_component = true; t.id.component_id = *cid; }
            else { t.id.index = anon_index++; }
            out.push_back(t);
            left += ts.width + p.margin + p.padding * 2.0f + just_x;
        }
        top += ts.height + p.margin + p.padding * 2.0f + just_y;
    }
    return out;
}

static std::vector<OptTile> resize_tiles(const std::vector<OptTile> &tiles, Size orig, Size desired) {  // layout.rs:130-151
    float scale = std::fmin(desired.width / orig.width, desired.height / orig.height);
    std::vector<OptTile> out;
    for (const OptTile &t : tiles) {
        if (!t) { out.push_back(std::nullopt); continue; }
        Tile r = *t;
        r.top = t->top * scale; r.left = t->left * scale; r.width = t->width * scale; r.height = t->height * scale;
        out.push_back(r);
    }
    return out;
}

static Tile fit_into_tile(const Tile &tile, const Stateful &c, uint64_t pts) {  // layout.rs:107-128
    OptF w = c.width(pts), h = c.height(pts);
    if (!w || !h) return tile;
    float sw = tile.width / *w, sh = tile.height / *h;
    float sf = std::fmin(sw, sh);  // f32::min: NaN-ignoring like fminf
    float top_off = (tile.height - sf * *h) / 2.0f;
    float left_off = (tile.width - sf * *w) / 2.0f;
    Tile r = tile;
    r.top = tile.top + top_off; r.left = tile.left + left_off;
    r.width = sf * *w; r.height = sf * *h;
    return r;
}

static NestedLayout tiles_layout(Stateful &self, Size size, uint64_t pts) {  // tiles_component.rs:62-69,109-120
    std::vector<OptTile> tiles = tiles_end_state(self.tiles, size, self.children);
    if (self.tiles_start && self.transition) {
        std::vector<OptTile> start = resize_tiles(self.tiles_start->first, self.tiles_start->second, size);
        tiles = lerp_tiles(start, tiles, self.transition->state(pts));
    }
    NestedLayout out;
    out.width = size.width; out.height = size.height;
    out.content.kind = LayoutContent::Color;
    out.content.color = self.tiles.background_color;
    for (size_t i = 0; i < self.children.size() && i < tiles.size(); i++) {  // zip
        Stateful &child = self.children[i];
        if (!tiles[i]) {
            size_t cnt = child.is_layout() ? child.node_children_count() : 1;
            out.children.push_back(NestedLayout::child_nodes_placeholder(cnt));
        } else if (child.is_layout()) {
            const Tile &t = *tiles[i];
            out.children.push_back(wrap_child(t.top, t.left, t.width, t.height, 0.0f, child, pts));
        } else {
            Tile f = fit_into_tile(*tiles[i], child, pts);
            out.children.push_back(wrap_child(f.top, f.left, f.width, f.height, 0.0f, child, pts));
        }
    }
    for (const NestedLayout &c : out.children) out.child_nodes_count += c.child_nodes_count;
    self.tiles_last_layout = TilesSnapshot(tiles, size);
    return out;
}

NestedLayout Stateful::layout(Size sz, uint64_t pts) {
    switch (kind) {
        case View: { ViewParam v = view_at(*this, pts); return view_layout(v, sz, children, pts); }
        case Rescaler: { RescalerParam r = rescaler_at(*this, pts); return rescaler_layout(r, sz, children[0], pts); }
        case Tiles: return tiles_layout(*this, sz, pts);
        default: return NestedLayout();
    }
}

NestedLayout NestedLayout::child_nodes_placeholder(size_t n) {
    NestedLayout l;
    l.content.kind = LayoutContent::None;
    l.child_nodes_count = n;
    return l;
}

// ------------------------------------------------------------------------------------------------
// flatten (transformations/layout/flatten.rs)
// ------------------------------------------------------------------------------------------------
namespace {
struct Flattener {
    static RenderLayout render_layout(const NestedLayout &s, const std::vector<Mask> &parent_masks) {  // :311-347
        RenderLayout r;
        r.top = s.top; r.left = s.left; r.width = s.width; r.height = s.height;
        r.rotation_degrees = s.rotation_degrees;
        r.border_radius = s.border_radius;
        r.masks = parent_masks;
        r.border_color = s.border_color;
        r.border_width = s.border_width;
        switch (s.content.kind) {
            case LayoutContent::Color: r.kind = RenderLayout::Color; r.color = s.content.color; break;
            case LayoutContent::ChildNode:
                r.kind = RenderLayout::ChildNode;
                r.index = s.content.index;
                r.crop = {0.0f, 0.0f, s.content.size.width, s.content.size.height};
                break;
            default: r.kind = RenderLayout::Color; r.color = RGBA{0, 0, 0, 0}; break;
        }
        return r;
    }
    static RenderLayout box_shadow_layout(const NestedLayout &s, const BoxShadow &b, const std::vector<Mask> &pm) {  // :350-362
        RenderLayout r;
        r.top = s.top + b.offset_y; r.left = s.left + b.offset_x;
        r.width = s.width; r.height = s.height;
        r.rotation_degrees = s.rotation_degrees;
        r.border_radius = s.border_radius + (b.blur_radius / 2.0f);
        r.kind = RenderLayout::BoxShadow;
        r.color = b.color;
        r.blur_radius = b.blur_radius;
        r.masks = pm;
        return r;
    }
    static std::vector<Mask> child_parent_masks(const NestedLayout &s, const std::vector<Mask> &masks) {  // :365-376
        std::vector<Mask> out;
        for (const Mask &m : masks) {
            Mask r;
            r.radius = m.radius / std::fmin(s.scale_x, s.scale_y);
            r.top = (m.top - s.top) / s.scale_y;
            r.left = (m.left - s.left) / s.scale_x;
            r.width = m.width / s.scale_x;
            r.height = m.height / s.scale_y;
            out.push_back(r);
        }
        return out;
    }
    static std::vector<Mask> parent_parent_masks(const NestedLayout &s, const std::vector<Mask> &masks) {  // :379-389
        std::vector<Mask> out;
        for (const Mask &m : masks) {
            Mask r;
            r.radius = m.radius * std::fmin(s.scale_x, s.scale_y);
            r.top = (m.top * s.scale_y) + s.top;
            r.left = (m.left * s.scale_x) + s.left;
            r.width = m.width * s.scale_x;
            r.height = m.height * s.scale_y;
            out.push_back(r);
        }
        return out;
    }
    static RenderLayout flatten_child(const NestedLayout &s, const RenderLayout &child) {  // :167-305
        float unified = std::fmin(s.scale_x, s.scale_y);
        RenderLayout r = child;
        r.rotation_degrees = child.rotation_degrees + s.rotation_degrees;
        r.border_radius = child.border_radius * unified;
        r.masks = parent_parent_masks(s, child.masks);
        if (!s.crop) {
            r.top = s.top + (child.top * s.scale_y);
            r.left = s.left + (child.left * s.scale_x);
            r.width = child.width * s.scale_x;
            r.height = child.height * s.scale_y;
            if (child.kind == RenderLayout::BoxShadow) r.blur_radius = child.blur_radius * unified;
            else r.border_width = child.border_width * unified;
            return r;
        }
        const Crop &crop = *s.crop;
        float cropped_top = std::fmax(child.top - crop.top, 0.0f);
        float cropped_left = std::fmax(child.left - crop.left, 0.0f);
        float cropped_bottom = std::fmin(child.top + child.height - crop.top, crop.height);
        float cropped_right = std::fmin(child.left + child.width - crop.left, crop.width);
        float cropped_width = cropped_right - cropped_left;
        float cropped_height = cropped_bottom - cropped_top;
        r.top = s.top + (cropped_top * s.scale_y);
        r.left = s.left + (cropped_left * s.scale_x);
        r.width = cropped_width * s.scale_x;
        r.height = cropped_height * s.scale_y;
        if (child.kind == RenderLayout::Color) {
            r.border_width = child.border_width * unified;
        } else if (child.kind == RenderLayout::BoxShadow) {
            r.blur_radius = child.blur_radius * unified;
        } else {
            float top_diff = std::fmax(crop.top - child.top, 0.0f);
            float left_diff = std::fmax(crop.left - child.left, 0.0f);
            float hsf = child.crop.width / child.width;
            float vsf = child.crop.height / child.height;
            r.crop.top = child.crop.top + (top_diff * vsf);
            r.crop.left = child.crop.left + (left_diff * hsf);
            r.crop.width = cropped_width * hsf;
            r.crop.height = cropped_height * vsf;
            r.border_width = child.border_width;  // flatten.rs:265-282: not scaled in the cropped branch
        }
        return r;
    }

    // returns (own box shadows, [self, children shadows, children])
    static void inner_flatten(const NestedLayout &s_in, size_t child_index_offset, const std::vector<Mask> &parent_masks,
                              std::vector<RenderLayout> &shadows, std::vector<RenderLayout> &layouts) {  // :24-82
        NestedLayout s = s_in;  // content index is rewritten
        s.children.clear();
        if (s.content.kind == LayoutContent::ChildNode) {
            s.content.index += child_index_offset;
            child_index_offset += 1;
        }
        RenderLayout self_layout = render_layout(s, parent_masks);
        for (const BoxShadow &b : s.box_shadow) shadows.push_back(box_shadow_layout(s, b, parent_masks));

        std::vector<Mask> masks = parent_masks;
        if (s.mask) masks.push_back(*s.mask);
        masks = child_parent_masks(s, masks);

        std::vector<RenderLayout> ch_shadows, ch_layouts;
        for (const NestedLayout &child : s_in.children) {
            inner_flatten(child, child_index_offset, masks, ch_shadows, ch_layouts);
            child_index_offset += child.child_nodes_count;
        }
        layouts.push_back(self_layout);
        for (const RenderLayout &l : ch_shadows) layouts.push_back(flatten_child(s, l));
        for (const RenderLayout &l : ch_layouts) layouts.push_back(flatten_child(s, l));
    }

    static bool should_render(const RenderLayout &l, const std::vector<std::optional<Resolution>> &inputs,
                              Resolution res) {  // :121-164
        if (l.width <= 0.0f || l.height <= 0.0f || l.top > (float)res.height || l.left > (float)res.width) return false;
        switch (l.kind) {
            case RenderLayout::Color:
                if (l.color.a == 0) return l.border_color.a != 0 || l.border_width > 0.0f;
                return true;
            case RenderLayout::ChildNode: {
                if (l.index < inputs.size() && inputs[l.index]) {
                    const Resolution &sz = *inputs[l.index];
                    if (l.crop.left > (float)sz.width || l.crop.top > (float)sz.height) return false;
                }
                if (l.crop.top + l.crop.height < 0.0f || l.crop.left + l.crop.width < 0.0f) return false;
                return true;
            }
            default: return l.color.a != 0;
        }
    }

    static void fix_final(RenderLayout &l) {  // :87-116
        if (l.kind != RenderLayout::BoxShadow && l.border_width < 1.0f) l.border_width = 0.0f;
        std::vector<Mask> kept;
        for (const Mask &m : l.masks) {
            float max_top = std::fmax(m.radius.top_left, m.radius.top_right);
            float max_bottom = std::fmax(m.radius.bottom_left, m.radius.bottom_right);
            float max_left = std::fmax(m.radius.top_left, m.radius.bottom_left);
            float max_right = std::fmax(m.radius.top_right, m.radius.bottom_right);
            bool skip = m.top + max_top <= l.top && m.left + max_left <= l.left &&
                        m.left + m.width - max_right >= l.left + l.width &&
                        m.top + m.height - max_bottom >= l.top + l.height;
            if (!skip) kept.push_back(m);
        }
        l.masks = std::move(kept);
    }
};
}  // namespace

std::vector<RenderLayout> NestedLayout::flatten(const std::vector<std::optional<Resolution>> &inputs,
                                                Resolution resolution) const {
    std::vector<RenderLayout> shadows, layouts, out;
    Flattener::inner_flatten(*this, 0, {}, shadows, layouts);
    for (std::vector<RenderLayout> *v : {&shadows, &layouts})
        for (RenderLayout &l : *v) {
            if (!Flattener::should_render(l, inputs, resolution)) continue;
            Flattener::fix_final(l);
            out.push_back(std::move(l));
        }
    return out;
}

// ------------------------------------------------------------------------------------------------
// SceneState (scene/scene_state.rs)
// ------------------------------------------------------------------------------------------------
namespace {
struct BuildCtx {
    std::map<std::string, const Stateful *> prev_state;
    uint64_t last_render_pts;
    const std::map<std::string, Resolution> *input_resolutions;
    const std::map<std::string, std::shared_ptr<const ImageAsset>> *images;
    const std::map<std::string, std::shared_ptr<WebInstance>> *webs;
    const std::map<std::string, std::shared_ptr<const ShaderProgram>> *shaders;
    std::string *err;   // the first SceneError of the build
};

// `as usize` of an f32: saturating, NaN -> 0
static size_t f32_as_usize(float v) {
    if (!(v > 0.0f)) return 0;
    if (v >= 1.8446744e19f) return (size_t)-1;
    return (size_t)v;
}

// ImageComponent::stateful_component's resolution (image_component.rs:67-89), literally: the aspect ratio is a usize
// division, so it is 1 for 640 x 360 and 0 for a portrait asset
static Resolution image_resolution(const ImageAsset &a, const OptF &w, const OptF &h) {
    const size_t aspect = (size_t)a.width / (size_t)a.height;
    if (w && h) return {f32_as_usize(roundf(*w)), f32_as_usize(roundf(*h))};
    if (w) return {f32_as_usize(roundf(*w)), f32_as_usize(roundf(*w / (float)aspect))};
    if (h) return {f32_as_usize(roundf(*h * (float)aspect)), f32_as_usize(roundf(*h))};
    return {a.width, a.height};
}

static void gather_components_with_id(const Stateful &c, std::map<std::string, const Stateful *> &out) {  // :259-311
    const std::optional<std::string> &id = c.component_id();
    if (id) out[*id] = &c;
    for (const Stateful &ch : c.children) gather_components_with_id(ch, out);
}

static bool did_child_order_change(const std::vector<Stateful> &prev, const std::vector<Stateful> &cur) {
    if (cur.size() != prev.size()) return true;
    for (size_t i = 0; i < cur.size(); i++)
        if (prev[i].component_id() != cur[i].component_id()) return true;
    return false;
}

// validate_params (transformations/shader/validation.rs:314-520) over the types a smr_shader_param_type can describe;
// `why` names the first mismatch
static void validate_shader_param(const ShaderParamValue &v, const ShaderParamType &t, std::string &why) {
    static const char *names[] = {"F32", "U32", "I32", "List", "Struct", "Vector", "Matrix"};
    if (t.kind == kShaderParamVector || t.kind == kShaderParamMatrix) {   // validate_vector / validate_matrix (:450-520)
        const char *what = t.kind == kShaderParamVector ? "a vector" : "a matrix";
        if (v.kind != SMR_SHADER_PARAM_LIST) {
            why = std::string("expected ") + what + " (a List), got " + names[v.kind];
            return;
        }
        if (v.items.size() != t.length) {
            why = std::string(what) + " needs exactly " + std::to_string(t.length) + (t.kind == kShaderParamVector ? " items" : " rows") +
                  ", got " + std::to_string(v.items.size());
            return;
        }
        for (size_t i = 0; i < v.items.size() && why.empty(); i++) validate_shader_param(v.items[i], t.items[0], why);
        return;
    }
    if (v.kind != t.kind) {
        why = std::string("expected ") + names[t.kind] + ", got " + names[v.kind];
        return;
    }
    if (t.kind == SMR_SHADER_PARAM_LIST) {
        if (v.items.size() > t.length) {
            why = "list too long: expected at most " + std::to_string(t.length) + ", got " + std::to_string(v.items.size());
            return;
        }
        for (size_t i = 0; i < v.items.size() && why.empty(); i++) validate_shader_param(v.items[i], t.items[0], why);
    } else if (t.kind == SMR_SHADER_PARAM_STRUCT) {
        if (v.items.size() != t.items.size()) {
            why = "expected " + std::to_string(t.items.size()) + " fields, got " + std::to_string(v.items.size());
            return;
        }
        for (size_t i = 0; i < v.items.size() && why.empty(); i++) {
            if (v.items[i].field_name != t.items[i].name) {
                why = "field " + std::to_string(i) + " is \"" + t.items[i].name + "\", got \"" + v.items[i].field_name + "\"";
                return;
            }
            validate_shader_param(v.items[i], t.items[i], why);
        }
    }
}

static Stateful build_stateful(const Component &c, const BuildCtx &ctx) {
    Stateful s;
    auto prev_of = [&](Stateful::Kind k) -> const Stateful * {
        if (!c.id) return nullptr;
        auto it = ctx.prev_state.find(*c.id);
        if (it == ctx.prev_state.end() || it->second->kind != k) return nullptr;
        return it->second;
    };
    switch (c.type) {
        case SMR_COMPONENT_INPUT_STREAM: {  // input_stream_component.rs:24-44
            s.kind = Stateful::InputStream;
            s.input_id = c.input_id;
            s.leaf_component_id = c.id;
            auto it = ctx.input_resolutions->find(c.input_id);
            if (it != ctx.input_resolutions->end()) s.size = {(float)it->second.width, (float)it->second.height};
            return s;
        }
        case SMR_COMPONENT_TEXT: {  // text_component.rs:36-53: the size is the caller's layout resolution
            s.kind = Stateful::Text;
            s.leaf_component_id = c.id;
            s.text = c.text;
            s.size = {(float)c.text->width, (float)c.text->height};
            return s;
        }
        case SMR_COMPONENT_IMAGE: {  // image_component.rs:57-124
            s.kind = Stateful::Image;
            s.leaf_component_id = c.id;
            s.image_id = c.image_id; s.image_width = c.image_width; s.image_height = c.image_height;
            auto it = ctx.images->find(c.image_id);
            if (it == ctx.images->end()) {
                if (ctx.err->empty()) *ctx.err = "Image \"" + c.image_id + "\" is not registered";
                return s;
            }
            const Stateful *prev = prev_of(Stateful::Image);
            if (prev && prev->image_id == s.image_id && prev->image_width == s.image_width && prev->image_height == s.image_height &&
                prev->image.asset == it->second) {
                s.image = prev->image;
            } else {
                s.image = {it->second, ctx.last_render_pts, image_resolution(*it->second, c.image_width, c.image_height)};
            }
            const Resolution &r = s.image.resolution;
            // the reference cannot create such a node texture
            if ((r.width == 0 || r.width > 16384 || r.height == 0 || r.height > 16384) && ctx.err->empty())
                *ctx.err = "Image \"" + c.image_id + "\" resolves to a node of " + std::to_string(r.width) + " x " + std::to_string(r.height);
            s.size = {(float)r.width, (float)r.height};
            return s;
        }
        case SMR_COMPONENT_WEB_VIEW: {  // web_view_component.rs:41-71: the instance, then the children, then their ids
            s.kind = Stateful::WebView;
            s.leaf_component_id = c.id;
            auto it = ctx.webs->find(c.web_renderer_id);
            if (it == ctx.webs->end()) {
                if (ctx.err->empty()) *ctx.err = "Web renderer \"" + c.web_renderer_id + "\" does not exist";
                return s;
            }
            s.web = it->second;
            s.size = {(float)s.web->width, (float)s.web->height};
            for (const Component &ch : c.children) s.children.push_back(build_stateful(ch, ctx));
            for (const Stateful &ch : s.children)
                if (!ch.component_id() && ctx.err->empty())
                    *ctx.err = "Web view \"" + c.web_renderer_id + "\" has a child without an id";
            return s;
        }
        case SMR_COMPONENT_SHADER: {  // shader_component.rs:43-72: the shader, the parameter, then the children
            s.kind = Stateful::Shader;
            s.leaf_component_id = c.id;
            auto it = ctx.shaders->find(c.shader_id);
            if (it == ctx.shaders->end()) {
                if (ctx.err->empty()) *ctx.err = "Shader \"" + c.shader_id + "\" not found";
                return s;
            }
            s.shader = it->second;
            s.shader_param = c.shader_param;
            if (c.shader_param && ctx.err->empty()) {
                std::string why;
                if (!s.shader->param_type) why = "the shader declares no parameter (NoBindingInShader)";
                else validate_shader_param(*c.shader_param, *s.shader->param_type, why);
                if (!why.empty()) *ctx.err = "Shader \"" + c.shader_id + "\": parameters do not match: " + why;
            }
            for (const Component &ch : c.children) s.children.push_back(build_stateful(ch, ctx));
            s.size = {c.shader_width, c.shader_height};
            const Resolution r{f32_as_usize(c.shader_width), f32_as_usize(c.shader_height)};
            if ((r.width == 0 || r.width > 16384 || r.height == 0 || r.height > 16384) && ctx.err->empty())
                *ctx.err = "Shader \"" + c.shader_id + "\" node of " + std::to_string(r.width) + " x " + std::to_string(r.height);
            return s;
        }
        case SMR_COMPONENT_VIEW: {  // view_component.rs:103-160
            s.kind = Stateful::View;
            const Stateful *prev = prev_of(Stateful::View);
            if (prev) s.view_start = view_at(*prev, ctx.last_render_pts);
            ViewParam &e = s.view_end;
            e.id = c.id; e.direction = c.direction; e.position = c.position; e.overflow = c.overflow;
            e.background_color = c.background_color; e.border_radius = c.border_radius;
            e.border_width = c.border_width; e.border_color = c.border_color; e.box_shadow = c.box_shadow;
            e.padding = c.padding;
            bool changed = prev ? !(prev->view_end == e) : false;
            bool interrupt = c.transition ? c.transition->should_interrupt : false;
            s.transition = TransitionState::create(c.transition, prev ? prev->transition : std::nullopt, changed,
                                                   interrupt, ctx.last_render_pts);
            break;
        }
        case SMR_COMPONENT_RESCALER: {  // rescaler_component.rs:96-147
            s.kind = Stateful::Rescaler;
            const Stateful *prev = prev_of(Stateful::Rescaler);
            if (prev) s.rescaler_start = rescaler_at(*prev, ctx.last_render_pts);
            RescalerParam &e = s.rescaler_end;
            e.id = c.id; e.position = c.position; e.mode = c.rescale_mode;
            e.horizontal_align = c.horizontal_align; e.vertical_align = c.vertical_align;
            e.border_radius = c.border_radius; e.border_width = c.border_width; e.border_color = c.border_color;
            e.box_shadow = c.box_shadow;
            bool changed = prev ? !(prev->rescaler_end == e) : false;
            bool interrupt = c.transition ? c.transition->should_interrupt : false;
            s.transition = TransitionState::create(c.transition, prev ? prev->transition : std::nullopt, changed,
                                                   interrupt, ctx.last_render_pts);
            break;
        }
        default: {  // Tiles, tiles_component.rs:123-181
            s.kind = Stateful::Tiles;
            const Stateful *prev = prev_of(Stateful::Tiles);
            if (prev) { s.tiles_start = prev->tiles_last_layout; s.tiles_last_layout = prev->tiles_last_layout; }
            TilesParam &e = s.tiles;
            e.id = c.id; e.width = c.tiles_width; e.height = c.tiles_height;
            e.background_color = c.background_color; e.aspect_w = c.tile_aspect_w; e.aspect_h = c.tile_aspect_h;
            e.margin = c.tiles_margin; e.padding = c.tiles_padding;
            e.horizontal_align = c.horizontal_align; e.vertical_align = c.vertical_align;
            for (const Component &ch : c.children) s.children.push_back(build_stateful(ch, ctx));
            bool changed = prev ? (!(prev->tiles == e) || did_child_order_change(prev->children, s.children)) : false;
            bool interrupt = c.transition ? c.transition->should_interrupt : false;
            s.transition = TransitionState::create(c.transition, prev ? prev->transition : std::nullopt, changed,
                                                   interrupt, ctx.last_render_pts);
            return s;
        }
    }
    for (const Component &ch : c.children) s.children.push_back(build_stateful(ch, ctx));
    return s;
}

static bool visit_ids(const Component &c, std::set<std::string> &ids, std::string &dup) {  // validation.rs:47-70
    if (c.id) {
        if (ids.count(*c.id)) { dup = *c.id; return false; }
        ids.insert(*c.id);
    }
    for (const Component &ch : c.children)
        if (!visit_ids(ch, ids, dup)) return false;
    return true;
}

static bool visit_web_ids(const Component &c, std::set<std::string> &ids, std::string &dup) {  // validation.rs:74-100
    if (c.type == SMR_COMPONENT_WEB_VIEW) {
        if (ids.count(c.web_renderer_id)) { dup = c.web_renderer_id; return false; }
        ids.insert(c.web_renderer_id);
    }
    for (const Component &ch : c.children)
        if (!visit_web_ids(ch, ids, dup)) return false;
    return true;
}

static int depth_of(const OutputNode &out, const NodeRef &k) {
    switch (k.kind) {
        case NodeRef::Shader: return out.shaders[k.index].depth;
        case NodeRef::Layout: return out.nested[k.index].depth;
        case NodeRef::Web: return out.webs[k.index].depth;
        default: return 0;
    }
}

static NodeRef node_child(const Stateful &l, OutputNode &out, uint64_t pts, std::string &err);

// The layout node of layout component `l` at `size` (scene_state.rs:206-228): the render graph's clone of `l`, and its node
// children appended to `out` in DFS order
static LayoutParams layout_node(const Stateful &l, Size size, OutputNode &out, uint64_t pts, std::string &err) {
    LayoutParams p;
    p.size = size;
    p.root = l;
    std::vector<const Stateful *> leaves;
    l.node_children(leaves);
    for (const Stateful *c : leaves) {
        const NodeRef k = node_child(*c, out, pts, err);
        p.depth = std::max(p.depth, depth_of(out, k) + 1);
        p.children.push_back(k);
    }
    return p;
}

// A node child of the render graph (build_tree, scene_state.rs:154-196): an input, or a text, image, web, shader or layout
// node appended to `out`, whose own children come first in DFS order.  A layout node's size is node_size at `pts`; a layout
// root without width and height is UnknownDimensionsForLayoutNodeRoot (scene_state.rs:206-228), reported in `err`.
static NodeRef node_child(const Stateful &l, OutputNode &out, uint64_t pts, std::string &err) {
    NodeRef ch;
    if (l.kind == Stateful::Text) {
        ch = {NodeRef::Text, (int)out.texts.size()};
        out.texts.push_back(l.text);
    } else if (l.kind == Stateful::Image) {
        ch = {NodeRef::Image, (int)out.images.size()};
        out.images.push_back(l.image);
    } else if (l.kind == Stateful::WebView) {
        WebParams w;
        w.instance = l.web;
        for (const Stateful &c : l.children) {
            const NodeRef k = node_child(c, out, pts, err);
            w.depth = std::max(w.depth, depth_of(out, k) + 1);
            w.children.push_back(k);
        }
        ch = {NodeRef::Web, (int)out.webs.size()};
        out.webs.push_back(std::move(w));
    } else if (l.kind == Stateful::Shader) {
        ShaderParams p;
        p.shader = l.shader;
        if (l.shader_param) l.shader_param->to_bytes(p.param_bytes);
        // a WGSL shader reads its whole uniform: bytes a short list (or no parameter) leaves out read as zero
        if (p.shader->wgsl && p.param_bytes.size() < p.shader->uniform_size) p.param_bytes.resize(p.shader->uniform_size, 0);
        p.resolution = {f32_as_usize(l.size.width), f32_as_usize(l.size.height)};
        for (const Stateful &c : l.children) {
            const NodeRef k = node_child(c, out, pts, err);
            p.depth = std::max(p.depth, depth_of(out, k) + 1);
            p.children.push_back(k);
        }
        ch = {NodeRef::Shader, (int)out.shaders.size()};
        out.shaders.push_back(std::move(p));
    } else if (l.is_layout()) {
        const Position pos = l.position(pts);
        if (!pos.width || !pos.height) {
            if (err.empty()) {
                const std::optional<std::string> &id = l.component_id();
                err = "Unknown dimensions for layout node root: " +
                      (id ? "Please provide width and height values for component with id \"" + *id + "\"" : std::string("Please provide width and height values."));
            }
            return ch;
        }
        LayoutParams p = layout_node(l, {*pos.width, *pos.height}, out, pts, err);
        ch = {NodeRef::Layout, (int)out.nested.size()};
        out.nested.push_back(std::move(p));
    } else {
        ch.input_id = l.input_id;
    }
    return ch;
}

// recalculate_layout (scene_state.rs:233-262): every layout component whose parent is not a layout is laid out at its size
// (the output's resolution for the root, its own width and height otherwise), which refreshes Tiles::last_layout
static void recalculate_layout(Stateful &c, std::optional<Size> size, uint64_t pts, bool parent_is_layout) {
    const OptF w = c.width(pts), h = c.height(pts);
    if (c.is_layout()) {
        if (!parent_is_layout) {
            if (!size && w && h) size = Size{*w, *h};
            if (size) c.layout(*size, pts);
        }
        for (Stateful &k : c.children) recalculate_layout(k, std::nullopt, pts, true);
    } else {
        for (Stateful &k : c.children) recalculate_layout(k, std::nullopt, pts, false);
    }
}
}  // namespace

void SceneState::register_render_event(uint64_t pts, std::map<std::string, Resolution> res) {
    last_pts_ns_ = pts;
    input_resolutions_ = std::move(res);
}

void SceneState::unregister_output(const std::string &id) {
    output_scenes_.erase(id);
    output_states_.erase(id);
}

bool SceneState::update_scene(const std::string &output_id, const Component &root, Resolution resolution,
                              OutputNode &out, std::string &err, const std::function<bool(OutputNode &)> &accept) {  // scene_state.rs:74-126
    {
        std::set<std::string> ids;
        std::string dup;
        if (!visit_ids(root, ids, dup)) {
            err = "More than one component has an id \"" + dup + "\". Component IDs in scene definition need to be unique.";
            return false;
        }
        ids.clear();   // one web renderer instance per WebView, across the outputs as they would be after the update
        for (const auto &kv : output_scenes_)
            if (kv.first != output_id && !visit_web_ids(kv.second, ids, dup)) break;
        if (dup.empty()) visit_web_ids(root, ids, dup);
        if (!dup.empty()) {
            err = "Instance of web renderer \"" + dup + "\" is used more than once; one WebView per instance is allowed.";
            return false;
        }
    }
    // recalculate_layout on every output at last_pts (refreshes Tiles::last_layout), :87-94,198-230
    for (auto &kv : output_states_) {
        OutputSceneState &st = kv.second;
        recalculate_layout(st.root, Size{(float)st.resolution.width, (float)st.resolution.height}, last_pts_ns_, false);
    }
    BuildCtx ctx;
    auto prev = output_states_.find(output_id);
    if (prev != output_states_.end()) gather_components_with_id(prev->second.root, ctx.prev_state);
    ctx.last_render_pts = last_pts_ns_;
    ctx.input_resolutions = &input_resolutions_;
    ctx.images = &images_;
    ctx.webs = &webs_;
    ctx.shaders = &shaders_;
    std::string build_err;
    ctx.err = &build_err;

    OutputSceneState st;
    st.root = build_stateful(root, ctx);
    if (!build_err.empty()) { err = build_err; return false; }
    st.resolution = resolution;

    // intermediate_node().build_tree(Some(resolution), last_pts), :154-196
    err.clear();
    out = OutputNode();
    out.resolution = resolution;
    if (!st.root.is_layout())
        out.root = node_child(st.root, out, last_pts_ns_, err);
    else
        out.root_layout = layout_node(st.root, {(float)resolution.width, (float)resolution.height}, out, last_pts_ns_, err);
    if (!err.empty()) return false;
    if (accept && !accept(out)) return false;
    output_scenes_[output_id] = root;
    output_states_[output_id] = std::move(st);
    return true;
}

bool SceneState::register_image(const std::string &image_id, std::shared_ptr<const ImageAsset> asset) {
    return images_.emplace(image_id, std::move(asset)).second;
}

bool SceneState::unregister_image(const std::string &image_id) { return images_.erase(image_id) != 0; }

bool SceneState::register_web(const std::string &instance_id, std::shared_ptr<WebInstance> instance) {
    return webs_.emplace(instance_id, std::move(instance)).second;
}

bool SceneState::unregister_web(const std::string &instance_id) { return webs_.erase(instance_id) != 0; }

bool SceneState::register_shader(const std::string &shader_id, std::shared_ptr<const ShaderProgram> shader) {
    return shaders_.emplace(shader_id, std::move(shader)).second;
}

bool SceneState::unregister_shader(const std::string &shader_id) { return shaders_.erase(shader_id) != 0; }

WebInstance *SceneState::web_instance(const std::string &instance_id) const {
    auto it = webs_.find(instance_id);
    return it == webs_.end() ? nullptr : it->second.get();
}

size_t ImageAsset::frame_at(uint64_t pts, uint64_t start_pts) const {
    const uint64_t animation_pts = (pts > start_pts ? pts - start_pts : 0) % duration;
    size_t best = 0;
    uint64_t best_d = UINT64_MAX;
    for (size_t i = 0; i < frame_pts.size(); i++) {   // min_by_key: the first of equal keys
        const uint64_t d = frame_pts[i] > animation_pts ? frame_pts[i] - animation_pts : animation_pts - frame_pts[i];
        if (d < best_d) { best_d = d; best = i; }
    }
    return best;
}

Resolution LayoutParams::resolution(uint64_t pts) const {
    if (given_layouts) return given_resolution;
    Position p = root.position(pts);
    float w = p.width ? *p.width : size.width;
    float h = p.height ? *p.height : size.height;
    return {f32_as_usize(w), f32_as_usize(h)};
}

std::vector<RenderLayout> LayoutParams::layouts(uint64_t pts, const std::vector<std::optional<Resolution>> &inputs) {
    if (given_layouts) return *given_layouts;
    const Resolution res = resolution(pts);
    root.update_state(inputs.data(), inputs.size());
    return root.layout(size, pts).flatten(inputs, res);
}

}  // namespace smr
