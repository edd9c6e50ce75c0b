// interior.h -- the composite's interior proof: where every alpha factor of fs_main is exactly 1, so the fragment is the
// layer's bare colour or sample.  The host (Renderer::prepare_layer: a layer's two bars, which pick its fast class and its
// direct tiles) and the composite kernel (shade_blend: the per-pixel shortcut of the general path) both use this rule.
#pragma once

#include <cfloat>
#include <cmath>

#include "kernels.h"

#ifdef __CUDACC__
#define SMR_HD __host__ __device__
#else
#define SMR_HD
#endif

namespace smr {
namespace dev {

// One rounded rect of fs_main -- the layer itself or one of its masks.  At a pixel centre at least `edge` inside all four
// straight edges and outside the four corner squares of side `corner`, the rect's alpha factor is exactly 1 and, for the
// layer, the border colour does not mix in.  `core` >= both: how far in the host's bars start across a corner.
struct InteriorRect { float edge, corner, core; };

// Why: with (dx, dy) the centre's offset from the rect's centre, r its corner's radius and q = (|d| - half size) + r,
// rounded_rect_sdf is max(qx, qy) - r when both q <= 0 and qx - r (or qy - r) when one is positive, because sqrt(q * q)
// == q.  Outside the corner squares at most one q is positive, so in exact arithmetic the SDF is the plain straight-edge
// distance, for a radius of either sign.  In f32 the vertex stage's coordinates, the SDF's sums (r included) and this
// rule's own sums each round by at most half an ulp of a value below S = |left| + |top| + |w| + |h| + max |r|: together
// less than S * 2^-20.  The margin m = max(2, 1 + S * 2^-19) therefore leaves the SDF more than half a pixel beyond
// what the smoothstep needs (-sdf >= 0.5 without a border; >= bw + 1 with one).  A corner square grows with |r|, so a
// radius as large as the rect (where its rounding would swamp the margin) leaves no interior at all.
// border_width: the layer's (a mask passes 0).  False: no interior (a non-finite field).
SMR_HD inline bool interior_rect(float left, float top, float w, float h, const float radius[4], float border_width,
                                 InteriorRect &k) {
    const float R = fmaxf(fmaxf(fabsf(radius[0]), fabsf(radius[1])), fmaxf(fabsf(radius[2]), fabsf(radius[3])));
    const float S = fabsf(left) + fabsf(top) + fabsf(w) + fabsf(h) + R;
    // fs_main's border branch is taken unless bw < 1: a NaN width draws the border colour everywhere
    const float border = border_width < 1.0f ? 0.0f : border_width + 1.0f;
    // a NaN or infinite field, or a sum that overflows, leaves no interior (fmaxf above skips NaN radii: test them here)
    if (!(S <= FLT_MAX) || !(fabsf(border_width) <= FLT_MAX) || !(radius[0] == radius[0]) || !(radius[1] == radius[1]) ||
        !(radius[2] == radius[2]) || !(radius[3] == radius[3]))
        return false;
    const float m = fmaxf(2.0f, 1.0f + S * (1.0f / 524288.0f));
    k.edge = m + border;
    k.corner = R + m;
    k.core = k.edge + R;
    return true;
}

// interior_rect's margins as the kernel reads them (LayerDev::int_edge / int_corner, MaskDev::edge / corner): an edge of
// +inf proves no pixel
SMR_HD inline void interior_margins(float left, float top, float w, float h, const float radius[4], float border_width,
                                    float &edge, float &corner) {
    InteriorRect k;
    const bool ok = interior_rect(left, top, w, h, radius, border_width, k);
    edge = ok ? k.edge : INFINITY;
    corner = ok ? k.corner : INFINITY;
}

// The rect (left, top, w, h) with these margins proves the pixel centre (pcx, pcy).
SMR_HD inline bool interior_pixel(float left, float top, float w, float h, float edge, float corner, float pcx, float pcy) {
    const float hx = w * 0.5f, hy = h * 0.5f;
    const float dx = fabsf(pcx - (left + hx)), dy = fabsf(pcy - (top + hy));
    const bool inside = dx <= hx - edge && dy <= hy - edge;
    const bool in_corner = dx > hx - corner && dy > hy - corner;
    return inside && !in_corner;
}

// The per-pixel shortcut of the composite's general path: pixel (X, Y) of an axis-aligned colour or texture layer whose
// rect and masks (masks[0 .. L.mask_count)) all prove it.
SMR_HD inline bool interior_shortcut(const LayerDev &L, const MaskDev *masks, int X, int Y) {
    if (L.rotated || L.type == 2) return false;
    const float pcx = (float)X + 0.5f, pcy = (float)Y + 0.5f;
    if (!interior_pixel(L.left, L.top, L.content_w, L.content_h, L.int_edge, L.int_corner, pcx, pcy)) return false;
    for (int i = 0; i < L.mask_count; i++) {
        const MaskDev &mk = masks[i];
        if (!interior_pixel(mk.left, mk.top, mk.width, mk.height, mk.edge, mk.corner, pcx, pcy)) return false;
    }
    return true;
}

}  // namespace dev
}  // namespace smr
