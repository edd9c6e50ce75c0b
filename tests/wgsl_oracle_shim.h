/*
 * wgsl_oracle_shim.h -- CPU restatement of a WGSL shader node's draw, for the WGSL shader oracle (TEST INFRASTRUCTURE
 * ONLY, NOT PRODUCT CODE).  A test's hand-written C++ restatement of one WGSL module defines
 *   WO_NVARY, wo_interp[]  the varyings: count and interpolation (0 perspective, 1 linear, 2 flat)
 *   wo_vs(b, params, position, tex_coords, pos, vary)          vs_main
 *   wo_fs(b, params, tex, fragment position, vary, out) -> bool fs_main (false: discard)
 * between this file's two parts (WO_PRE defined: the types; not defined: the rasteriser).  It is compiled after
 * shader_oracle_shim.h (tests/c_oracles.py), whose sampling and blending it uses.  The rasteriser restates the
 * contract of smr_register_wgsl_shader (include/smelter_b200.h) independently of the product's kernel:
 *   window x = fmaf(x/w, W/2, W/2), y = fmaf(-(y/w), H/2, H/2), snapped to 1/256 px; a plane with a vertex of w <= 0 or a
 *   window coordinate beyond 2^20 px is not drawn; triangles (0,1,2), (2,3,0); the doubled area from the snapped
 *   vertices is negative for a front face; back faces and degenerate triangles are not drawn; a pixel centre is inside
 *   when every barycentric numerator is > 0, or 0 on a top-left edge; b_i = num_i / area in f32; depth
 *   (b0 z0 + b1 z1) + b2 z2 in [0, 1]; varyings as the contract states; blend and 8-bit store per fragment.
 */
#ifdef WO_PRE
struct wo_base { int plane_id; float time; unsigned res[2]; unsigned count; };

__device__ float4 smr_fragment(smr_fragment_in, const smr_base_params &, const void *, const smr_textures &) {
    return make_float4(0.0f, 0.0f, 0.0f, 0.0f);
}
#else

struct wo_vtx { float clip[4]; float vary[WO_NVARY > 0 ? WO_NVARY : 1]; long long X, Y; float z; };

static long long wo_cross(long long ax, long long ay, long long bx, long long by, long long cx, long long cy) {
    return (bx - ax) * (cy - ay) - (by - ay) * (cx - ax);
}

extern "C" void orc_render_wgsl(int W, int H, int mode, float time, const void *params, const uint8_t *const *tex,
                                const int *tw, const int *th, int n, uint8_t *out) {
    init_tables();
    memset(out, 0, (size_t)W * H * 4);
    smr_textures t = {tex, tw, th, (unsigned)n, mode};
    static const float mesh[4][5] = {{1, -1, 0, 1, 1}, {1, 1, 0, 1, 0}, {-1, 1, 0, 0, 0}, {-1, -1, 0, 0, 1}};
    static const int tris[2][3] = {{0, 1, 2}, {2, 3, 0}};
    for (int p = 0; p < (n > 0 ? n : 1); p++) {
        wo_base b = {n > 0 ? p : -1, time, {(unsigned)W, (unsigned)H}, (unsigned)n};
        wo_vtx v[4];
        bool ok = true;
        for (int k = 0; k < 4; k++) {
            wo_vs(b, params, mesh[k], mesh[k] + 3, v[k].clip, v[k].vary);
            float w = v[k].clip[3];
            if (!(w > 0.0f)) { ok = false; continue; }
            float xw = fmaf(v[k].clip[0] / w, (float)W / 2.0f, (float)W / 2.0f);
            float yw = fmaf(-(v[k].clip[1] / w), (float)H / 2.0f, (float)H / 2.0f);
            if (!(fabsf(xw) <= 1048576.0f && fabsf(yw) <= 1048576.0f)) { ok = false; continue; }
            v[k].X = (long long)rintf(xw * 256.0f);
            v[k].Y = (long long)rintf(yw * 256.0f);
            v[k].z = v[k].clip[2] / w;
        }
        if (!ok) continue;
        for (int tr = 0; tr < 2; tr++) {
            const wo_vtx &a = v[tris[tr][0]], &c1 = v[tris[tr][1]], &c2 = v[tris[tr][2]];
            const wo_vtx *V[3] = {&a, &c1, &c2};
            long long area = wo_cross(a.X, a.Y, c1.X, c1.Y, c2.X, c2.Y);
            if (area >= 0) continue;
            area = -area;
            for (int y = 0; y < H; y++)
                for (int x = 0; x < W; x++) {
                    long long px = 256LL * x + 128, py = 256LL * y + 128, num[3];
                    bool in = true;
                    for (int k = 0; k < 3; k++) {
                        const wo_vtx &s = *V[(k + 1) % 3], &e = *V[(k + 2) % 3];
                        num[k] = -wo_cross(s.X, s.Y, e.X, e.Y, px, py);
                        // the interior side of edge s -> e points along (e.Y - s.Y, s.X - e.X)
                        long long nx = e.Y - s.Y, ny = s.X - e.X;
                        bool tl = nx > 0 || (nx == 0 && ny > 0);
                        if (!(num[k] > 0 || (num[k] == 0 && tl))) in = false;
                    }
                    if (!in) continue;
                    float A = (float)area, bb[3];
                    for (int k = 0; k < 3; k++) bb[k] = (float)num[k] / A;
                    float depth = (bb[0] * V[0]->z + bb[1] * V[1]->z) + bb[2] * V[2]->z;
                    if (!(depth >= 0.0f && depth <= 1.0f)) continue;
                    float q[3];
                    for (int k = 0; k < 3; k++) q[k] = bb[k] / V[k]->clip[3];
                    float s = (q[0] + q[1]) + q[2];
                    float vary[WO_NVARY > 0 ? WO_NVARY : 1];
                    for (int j = 0; j < WO_NVARY; j++) {
                        if (wo_interp[j] == 2) vary[j] = V[0]->vary[j];
                        else if (wo_interp[j] == 1) vary[j] = (bb[0] * V[0]->vary[j] + bb[1] * V[1]->vary[j]) + bb[2] * V[2]->vary[j];
                        else vary[j] = ((q[0] * V[0]->vary[j] + q[1] * V[1]->vary[j]) + q[2] * V[2]->vary[j]) / s;
                    }
                    float fpos[4] = {(float)x + 0.5f, (float)y + 0.5f, depth, s};
                    float4 c;
                    if (wo_fs(b, params, t, fpos, vary, c)) blend_fragment(out + ((size_t)y * W + x) * 4, c, mode);
                }
        }
    }
}
#endif
