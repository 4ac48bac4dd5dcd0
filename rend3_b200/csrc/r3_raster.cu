// r3_raster.cu — software rasteriser for the opaque forward pass and the shadow-map passes.
//
// Replaces the fixed-function half of ForwardRoutine::add_forward_to_graph
// (rend3-routine/src/forward.rs:192-315, pipeline state :331-365): vertex pulling of the packed index lists
// produced by the triangle cull (opaque.wgsl::vs_main :91-135 / depth.wgsl::vs_main :51-87 up to clip space),
// clipping, triangle setup, coverage and the reverse-Z GreaterEqual depth test.
//
// Design: a visibility buffer instead of immediate shading.  Every covered sample performs ONE 64-bit
// atomicMax on  (depth bits << 32) | (pass << 31) | triangle-record  — reverse-Z depth in [0,1] orders like its
// bit pattern, so the depth test, the "later draw wins ties" rule and the predicted/residual pass order collapse
// into one integer max in L2.  fs_main then runs once per pixel (r3_shade.cu) instead of once per fragment.
// Shadow maps are the same kernels with a 32-bit atomicMax on the depth bits of the atlas.
//   * setup kernel: persistent grid (every resident CTA of the GPU), one thread per listed triangle; small triangles (bounding box
//     <= 64 pixels) are rasterised inline by the thread with incremental 64-bit edge functions; medium ones
//     (box <= 32x32) are handed to the whole warp: ballot, broadcast the setup by shuffle, 32 pixels per step;
//   * larger ones are split into 16-row bands and queued; the band kernel gives each band to one warp, lanes
//     span 32 consecutive pixels so the visibility-buffer atomics of a warp hit one or two 128-byte lines,
//     and 32x16 blocks entirely outside an edge are skipped with one corner evaluation per edge.
// All setup / coverage / depth arithmetic is __f*_rn in the order of the oracle's RASTER RULES R1-R5
// (oracle/r3_oracle_forward.inc), integer edge functions with the top-left rule — bit-exact by construction.
#include "r3_common.cuh"
#include "r3_scan.cuh"
#include "r3_texture.cuh"

namespace {

constexpr int RS_THREADS = 256;
constexpr float GUARD = 64.0f;
constexpr int SMALL_AREA = 64;           // inline raster when the pixel bounding box covers at most 64 pixels
constexpr int MEDIUM_MAX = 32;           // warp-cooperative raster up to a 32 x 32 pixel box (<= 32 steps of 32 lanes)
constexpr int COOP_MAX_LANES = 33;       // >32 = never: measured on C3/C5, the cooperative walk wins even when every lane holds a medium triangle
constexpr int BAND_ROWS = 16;
constexpr uint32_t LARGE_CAP = 1u << 22; // queued large sub-triangles (160 MB)
constexpr uint32_t BAND_CAP = 1u << 24;  // queued (sub-triangle, band) items (128 MB)
// A sub-triangle that does not fit the queues is rasterised by the set-up kernel instead.  Its band reservation is one atomicAdd
// and may straddle BAND_CAP; raster_band_kernel walks every slot below min(counters[1], BAND_CAP), and the scratch they live in is
// never cleared, so the reservation that crosses the cap fills its in-range slots with BAND_SKIP and the band kernel skips them.
// (A reservation that never overshoots needs a compare-and-swap loop on the counter every large sub-triangle contends for.)
constexpr uint32_t BAND_SKIP = 0xFFFFFFFFu;   // band item whose sub-triangle index is >= LARGE_CAP: nothing to rasterise
constexpr int MODE_COLOUR = 0;           // opaque + cutout forward routines into the visibility buffer
constexpr int MODE_DEPTH = 1;            // shadow passes into the atlas
constexpr int MODE_BLEND = 2;            // blend routine: collect per-sample fragment lists
constexpr int MODE_MSAA = 4;             // or-ed onto MODE_COLOUR / MODE_BLEND: SampleCount::Four (R7); keeps the 4-sample code out of the common kernels
constexpr int MODE_ALPHA = 8;            // or-ed on when some cutout material discards per fragment (texture / vertex alpha): the call into the
                                         // texture sampler would otherwise set the register budget of every kernel (80 -> 128 for the shadow passes)

struct SubTri { int32_t x[3], y[3]; float z[3]; uint32_t rec; };   // oriented (area > 0), snapped 24.8; rec bit 31 = per-fragment alpha test
constexpr uint32_t REC_ALPHA_TESTED = 0x80000000u;
static_assert(sizeof(SubTri) == 40, "SubTri");

struct RasterParams {
    // draw source
    const r3_batch_data* batches; const r3_region* regions; const uint32_t* header;   // header[2] = n_regions (device-side count)
    const r3_indirect_call* calls; const uint32_t* indices; uint64_t index_elems;
    const unsigned long long* tri_prefix;      // [n_regions + 1] exclusive prefix of the listed triangles of the regions in [key_lo, key_hi]
    const r3_object* objects; uint32_t n_slots;
    const r3_object_matrices* matrices; uint32_t matrices_cap;
    const uint32_t* mesh; uint64_t mesh_words;
    const r3_material* materials; uint32_t n_materials;
    TexTable tt;                                   // albedo textures of cutout materials (per-fragment discard)
    // target
    float ox, oy, vw, vh; int32_t x0, y0, x1, y1; uint32_t pitch; int positive_visible;
    uint32_t samples;                              // 1 or 4 (R7: standard 4x pattern); shadow passes are always single-sampled
    unsigned long long* vis; uint32_t pass_bit;   // colour passes
    uint32_t* depth_bits;                          // depth-only passes (shadow atlas)
    r3_tri_record* records;
    // queues
    SubTri* large; uint2* bands; uint32_t* counters;   // [0] n_large, [1] n_bands, [2] band ticket, [3] blend fragment nodes, [4] setup ticket
    uint32_t* frag_heads; uint4* frag_nodes; uint32_t frag_cap;   // blend routine
    unsigned long long key_lo, key_hi;                 // material keys of the routine(s) drawing (forward.rs:286-313)
    unsigned long long* stats;
};

__device__ __forceinline__ uint32_t mesh_word(const RasterParams& p, uint64_t i) { return i < p.mesh_words ? __ldg(&p.mesh[i]) : 0u; }

__device__ __forceinline__ float plane_dist(int plane, const float4 v) {
    switch (plane) {
        case 0: return v.z;
        case 1: return sub_rn(v.w, v.z);
        case 2: return add_rn(v.x, mul_rn(GUARD, v.w));
        case 3: return sub_rn(mul_rn(GUARD, v.w), v.x);
        case 4: return add_rn(v.y, mul_rn(GUARD, v.w));
        default: return sub_rn(mul_rn(GUARD, v.w), v.y);
    }
}
__device__ __forceinline__ float4 clip_lerp(const float4 in, const float4 out, float din, float dout) {
    const float t = div_rn(din, sub_rn(din, dout));
    return make_float4(add_rn(in.x, mul_rn(t, sub_rn(out.x, in.x))), add_rn(in.y, mul_rn(t, sub_rn(out.y, in.y))),
                       add_rn(in.z, mul_rn(t, sub_rn(out.z, in.z))), add_rn(in.w, mul_rn(t, sub_rn(out.w, in.w))));
}
// R1 — Sutherland-Hodgman against every violated plane; returns the polygon size (0 = clipped away)
__device__ __noinline__ int clip_polygon(float4* poly, int n) {
    for (int plane = 0; plane < 6 && n >= 3; ++plane) {
        bool any_out = false;
        for (int i = 0; i < n; ++i) any_out |= plane_dist(plane, poly[i]) < 0.0f;
        if (!any_out) continue;
        float4 outp[12];
        int m = 0;
        for (int i = 0; i < n; ++i) {
            const float4 a = poly[i], b = poly[(i + 1) % n];
            const float da = plane_dist(plane, a), db = plane_dist(plane, b);
            if (da >= 0.0f) {
                outp[m++] = a;
                if (db < 0.0f) outp[m++] = clip_lerp(a, b, da, db);
            } else if (db >= 0.0f) {
                outp[m++] = clip_lerp(b, a, db, da);
            }
        }
        n = m;
        for (int i = 0; i < n; ++i) poly[i] = outp[i];
    }
    return n >= 3 ? n : 0;
}

// Edge functions are evaluated in 64-bit integers in general (24.8 coordinates, guard band 64 x the viewport).  They are
// translation invariant, so a triangle whose vertices and pixel box lie within +-11585 sub-pixel units (45 pixels) of its
// first pixel centre can use 32-bit arithmetic relative to that centre: |E| <= 2 * (2 * 11585)^2 < 2^31.  Same integers,
// same float conversions, half the integer instructions and no 64-bit I2F — that covers nearly every small and medium triangle.
constexpr int FITS32_REACH = 11585;
template <typename T>
struct EdgeSetupT {
    T e0, e1, e2;          // biased edge values at the first pixel centre: >= 0 means inside
    T sx0, sx1, sx2;       // step for +1 pixel in x
    T sy0, sy1, sy2;       // step for +1 pixel in y
    int b0, b1, b2;        // top-left biases folded into e* (0 for top/left edges, 1 otherwise)
    float inv_area;
};
__device__ __forceinline__ float to_float_rn(long long v) { return __ll2float_rn(v); }
__device__ __forceinline__ float to_float_rn(int v) { return __int2float_rn(v); }
__device__ __forceinline__ long long edge_fn(int ax, int ay, int bx, int by, long long px, long long py) {
    return (long long)(bx - ax) * (py - ay) - (long long)(by - ay) * (px - ax);
}
__device__ __forceinline__ int not_top_left(int ax, int ay, int bx, int by) {
    const int dx = bx - ax, dy = by - ay;
    return ((dy < 0) || (dy == 0 && dx > 0)) ? 0 : 1;
}
__device__ __forceinline__ bool fits32(const SubTri& s, int px0, int py0, int px1, int py1) {
    const int ox = px0 * 256 + 128, oy = py0 * 256 + 128;
    int reach = max((px1 - px0) * 256 + 128, (py1 - py0) * 256 + 128);   // +128: multisample offsets stay inside the pixel
#pragma unroll
    for (int k = 0; k < 3; ++k) reach = max(reach, max(abs(s.x[k] - ox), abs(s.y[k] - oy)));
    return reach <= FITS32_REACH && abs(px0) < (1 << 20) && abs(py0) < (1 << 20);
}
// edge functions E_ab, E_bc, E_ca at pixel (px, py): e0 = E_bc (weight of a), e1 = E_ca (weight of b), e2 = E_ab (weight of c)
template <typename T>
__device__ __forceinline__ EdgeSetupT<T> make_edges(const SubTri& s, int px, int py) {
    EdgeSetupT<T> e;
    e.b0 = not_top_left(s.x[1], s.y[1], s.x[2], s.y[2]);
    e.b1 = not_top_left(s.x[2], s.y[2], s.x[0], s.y[0]);
    e.b2 = not_top_left(s.x[0], s.y[0], s.x[1], s.y[1]);
    // vertices relative to the first pixel centre (exact: the edge functions only see differences)
    const int ox = px * 256 + 128, oy = py * 256 + 128;
    const T x0 = (T)s.x[0] - ox, y0 = (T)s.y[0] - oy, x1 = (T)s.x[1] - ox, y1 = (T)s.y[1] - oy, x2 = (T)s.x[2] - ox, y2 = (T)s.y[2] - oy;
    // E(a, b, p) = (bx - ax) * (py - ay) - (by - ay) * (px - ax) at p = 0
    e.e0 = (x2 - x1) * (-y1) - (y2 - y1) * (-x1) - e.b0;
    e.e1 = (x0 - x2) * (-y2) - (y0 - y2) * (-x2) - e.b1;
    e.e2 = (x1 - x0) * (-y0) - (y1 - y0) * (-x0) - e.b2;
    e.sx0 = -(y2 - y1) * 256; e.sy0 = (x2 - x1) * 256;
    e.sx1 = -(y0 - y2) * 256; e.sy1 = (x0 - x2) * 256;
    e.sx2 = -(y1 - y0) * 256; e.sy2 = (x1 - x0) * 256;
    const T area = (x1 - x0) * (y2 - y0) - (y1 - y0) * (x2 - x0);
    e.inv_area = div_rn(1.0f, to_float_rn(area));
    return e;
}
// R5 depth of a covered sample from the (biased) edge values
template <typename T>
__device__ __forceinline__ float sample_depth(const SubTri& s, const EdgeSetupT<T>& e, T e0, T e1, T e2) {
    const float la = mul_rn(to_float_rn((T)(e0 + e.b0)), e.inv_area), lb = mul_rn(to_float_rn((T)(e1 + e.b1)), e.inv_area),
                lc = mul_rn(to_float_rn((T)(e2 + e.b2)), e.inv_area);
    const float z = add_rn(add_rn(mul_rn(la, s.z[0]), mul_rn(lb, s.z[1])), mul_rn(lc, s.z[2]));
    return fminf(fmaxf(z, 0.0f), 1.0f);
}
template <int MODE>
__device__ __forceinline__ uint32_t write_sample(const RasterParams& p, int px, int py, uint32_t k, float z, uint32_t rec) {
    // the result of the atomic is never read, so it compiles to a fire-and-forget RED.MAX: a thread can have
    // hundreds of samples in flight instead of one L2 round trip per sample
    const size_t pi = (size_t)py * p.pitch + px;
    if ((MODE & 3) == MODE_DEPTH) {
        atomicMax(&p.depth_bits[pi], __float_as_uint(z));
    } else if ((MODE & 3) == MODE_COLOUR) {
        const unsigned long long key = ((unsigned long long)__float_as_uint(z) << 32) | ((unsigned long long)p.pass_bit << 31) | (rec & ~REC_ALPHA_TESTED);
        atomicMax(&p.vis[pi * p.samples + k], key);
    } else {
        // blend routine: fragments must be applied in draw order, so they are only collected here (one list per sample).
        // The depth buffer of a sample never decreases, so a fragment behind the opaque depth can never pass.
        const size_t si = pi * p.samples + k;
        if (__float_as_uint(z) >= (uint32_t)(p.vis[si] >> 32)) {
            const uint32_t node = atomicAdd(&p.counters[3], 1u);
            if (node < p.frag_cap) {
                const uint32_t next = atomicExch(&p.frag_heads[si], node + 1u);
                p.frag_nodes[node] = make_uint4(rec & ~REC_ALPHA_TESTED, __float_as_uint(z), next, 0u);
            }
        }
        return 0u;
    }
    return 1u;   // statistics count rasterised (covered) samples
}

// R7: sample offsets from the pixel centre in 1/256 pixel (standard 4x pattern)
__device__ __constant__ int c_sample_dx[4] = {-32, 96, -96, 32};
__device__ __constant__ int c_sample_dy[4] = {-96, -32, 32, 96};

// alpha of the cutout routines' fragment at the centre of pixel (px, py) against the material's threshold: true = discard.
//   colour passes (opaque.wgsl:203-235, discard variant): albedo alpha of get_pixel_data_inner — coords through uv_transform0, the
//     material's sampler, times vertex alpha when ALBEDO_BLEND, times material.albedo.a;
//   depth passes  (depth.wgsl:101-127): the RAW coords0, uvdy = dpdx(coords) like uvdx (sic), always the linear sampler.
// Same operation order as the oracle (this translation unit is compiled without contraction; the mip fraction comes from rule R9's
// log2_r9, a fixed sequence of IEEE operations): the decision is bit-identical.
template <int MODE>
__device__ __noinline__ bool cutout_discards(const RasterParams& p, uint32_t rec, int px, int py) {
    // the record was written earlier in THIS launch (by this thread, or by another lane of the warp before a __syncwarp): plain loads
    const r3_tri_record* tp = p.records + ((rec & ~REC_ALPHA_TESTED) - 1u);
    const float4 q0 = reinterpret_cast<const float4*>(tp)[0], q1 = reinterpret_cast<const float4*>(tp)[1], q2 = reinterpret_cast<const float4*>(tp)[2];
    const uint4 q3 = reinterpret_cast<const uint4*>(tp)[3];
    const float p0[3] = {q0.x, q0.y, q0.z}, p1[3] = {q0.w, q1.x, q1.y}, p2[3] = {q1.z, q1.w, q2.x};
    const uint32_t oid = __float_as_uint(q2.y);
    const uint32_t vid[3] = {__float_as_uint(q2.z), __float_as_uint(q2.w), q3.x};
    const r3_object* obj = &p.objects[oid];
    const r3_material* m = &p.materials[obj->material_index < p.n_materials ? obj->material_index : 0u];
    const uint32_t flags = m->flags;
    float alpha = 1.0f;
    if (flags & R3_MAT_ALBEDO_ACTIVE) {
        const float hw = p.vw * 0.5f, hh = p.vh * 0.5f;
        float b[3][3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float fx = ((float)px - p.ox) + (k == 1 ? 1.5f : 0.5f), fy = ((float)py - p.oy) + (k == 2 ? 1.5f : 0.5f);
            const float nx = fx / hw - 1.0f, ny = 1.0f - fy / hh;
            const float b0 = ((p1[1] * p2[2] - p1[2] * p2[1]) * nx + (p1[2] * p2[0] - p1[0] * p2[2]) * ny) + (p1[0] * p2[1] - p1[1] * p2[0]);
            const float b1 = ((p2[1] * p0[2] - p2[2] * p0[1]) * nx + (p2[2] * p0[0] - p2[0] * p0[2]) * ny) + (p2[0] * p0[1] - p2[1] * p0[0]);
            const float b2 = ((p0[1] * p1[2] - p0[2] * p1[1]) * nx + (p0[2] * p1[0] - p0[0] * p1[2]) * ny) + (p0[0] * p1[1] - p0[1] * p1[0]);
            const float sum = (b0 + b1) + b2;
            b[k][0] = b0 / sum; b[k][1] = b1 / sum; b[k][2] = b2 / sum;
        }
        const uint32_t albedo_tex = m->textures[R3_TEX_ALBEDO];
        if (albedo_tex) {
            float uv[3][2] = {{0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}};
            const uint32_t uv_off = obj->attr_offset[3];
            if (uv_off != R3_ATTR_ABSENT) {
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    const uint64_t w = (uint64_t)(uv_off >> 2) + (uint64_t)vid[k] * 2u;
                    uv[k][0] = __uint_as_float(mesh_word(p, w)); uv[k][1] = __uint_as_float(mesh_word(p, w + 1));
                }
            }
            float co[3][2];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float u = (b[k][0] * uv[0][0] + b[k][1] * uv[1][0]) + b[k][2] * uv[2][0];
                const float v = (b[k][0] * uv[0][1] + b[k][1] * uv[1][1]) + b[k][2] * uv[2][1];
                if ((MODE & 3) == MODE_DEPTH) { co[k][0] = u; co[k][1] = v; }
                else {
                    co[k][0] = (m->uv_transform0[0][0] * u + m->uv_transform0[1][0] * v) + m->uv_transform0[2][0];
                    co[k][1] = (m->uv_transform0[0][1] * u + m->uv_transform0[1][1] * v) + m->uv_transform0[2][1];
                }
            }
            TexCoords tc;
            tc.u = co[0][0]; tc.v = co[0][1];
            tc.dudx = co[1][0] - co[0][0]; tc.dvdx = co[1][1] - co[0][1];
            if ((MODE & 3) == MODE_DEPTH) { tc.dudy = tc.dudx; tc.dvdy = tc.dvdx; }
            else { tc.dudy = co[2][0] - co[0][0]; tc.dvdy = co[2][1] - co[0][1]; }
            alpha = texture_sample_grad(p.tt, albedo_tex, (MODE & 3) != MODE_DEPTH && (flags & R3_MAT_NEAREST), tc).w;
        }
        if (flags & R3_MAT_ALBEDO_BLEND) {
            float va[3] = {1.0f, 1.0f, 1.0f};
            const uint32_t col_off = obj->attr_offset[5];
            if (col_off != R3_ATTR_ABSENT) {
#pragma unroll
                for (int k = 0; k < 3; ++k) va[k] = (float)(mesh_word(p, (uint64_t)(col_off >> 2) + vid[k]) >> 24) / 255.0f;
            }
            alpha *= (b[0][0] * va[0] + b[0][1] * va[1]) + b[0][2] * va[2];
        }
    }
    return alpha * m->albedo[3] < m->alpha_cutout;
}

// coverage + depth of one pixel given the biased edge values at its centre
template <int MODE, typename T>
__device__ __forceinline__ void emit_pixel(const RasterParams& p, const SubTri& s, const EdgeSetupT<T>& e, int px, int py, T c0, T c1, T c2, uint32_t& frags) {
    if (!(MODE & MODE_MSAA)) {
        if ((c0 | c1 | c2) >= 0) {
            // cutout routines: the fragment shader `discard`s (opaque.wgsl:231-235, depth.wgsl:101-127)
            if ((MODE & MODE_ALPHA) && (s.rec & REC_ALPHA_TESTED) && cutout_discards<MODE>(p, s.rec, px, py)) return;
            frags += write_sample<MODE>(p, px, py, 0u, sample_depth<T>(s, e, c0, c1, c2), s.rec);
        }
        return;
    }
    bool tested = !(MODE & MODE_ALPHA) || !(s.rec & REC_ALPHA_TESTED);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        // E(centre + o) = E(centre) + (step_x * o.x + step_y * o.y) / 256 (the steps are exact multiples of 256)
        const T a0 = c0 + (e.sx0 >> 8) * c_sample_dx[k] + (e.sy0 >> 8) * c_sample_dy[k];
        const T a1 = c1 + (e.sx1 >> 8) * c_sample_dx[k] + (e.sy1 >> 8) * c_sample_dy[k];
        const T a2 = c2 + (e.sx2 >> 8) * c_sample_dx[k] + (e.sy2 >> 8) * c_sample_dy[k];
        if ((a0 | a1 | a2) >= 0) {
            if (!tested) {   // once per pixel and primitive: a discard removes every sample
                if (cutout_discards<MODE>(p, s.rec, px, py)) return;
                tested = true;
            }
            frags += write_sample<MODE>(p, px, py, (uint32_t)k, sample_depth<T>(s, e, a0, a1, a2), s.rec);
        }
    }
}

__device__ __forceinline__ void pixel_bounds(const RasterParams& p, const SubTri& s, int& px0, int& py0, int& px1, int& py1) {
    const int minx = min(s.x[0], min(s.x[1], s.x[2])), maxx = max(s.x[0], max(s.x[1], s.x[2]));
    const int miny = min(s.y[0], min(s.y[1], s.y[2])), maxy = max(s.y[0], max(s.y[1], s.y[2]));
    if (p.samples == 1u) {
        px0 = max((minx - 128 + 255) >> 8, p.x0); px1 = min((maxx - 128) >> 8, p.x1 - 1);
        py0 = max((miny - 128 + 255) >> 8, p.y0); py1 = min((maxy - 128) >> 8, p.y1 - 1);
    } else {   // any sample of a touched pixel may be covered
        px0 = max(minx >> 8, p.x0); px1 = min(maxx >> 8, p.x1 - 1);
        py0 = max(miny >> 8, p.y0); py1 = min(maxy >> 8, p.y1 - 1);
    }
}

// one thread walks the pixel box of its own sub-triangle with incremental edge functions
template <int MODE, typename T>
__device__ __forceinline__ void raster_inline_t(const RasterParams& p, const SubTri& s, int px0, int py0, int px1, int py1, uint32_t& frags) {
    const EdgeSetupT<T> e = make_edges<T>(s, px0, py0);
    T r0 = e.e0, r1 = e.e1, r2 = e.e2;
    for (int py = py0; py <= py1; ++py) {
        T c0 = r0, c1 = r1, c2 = r2;
        for (int px = px0; px <= px1; ++px) {
            emit_pixel<MODE, T>(p, s, e, px, py, c0, c1, c2, frags);
            c0 += e.sx0; c1 += e.sx1; c2 += e.sx2;
        }
        r0 += e.sy0; r1 += e.sy1; r2 += e.sy2;
    }
}
template <int MODE>
__device__ __forceinline__ void raster_inline(const RasterParams& p, const SubTri& s, int px0, int py0, int px1, int py1, uint32_t& frags) {
    if (fits32(s, px0, py0, px1, py1)) raster_inline_t<MODE, int>(p, s, px0, py0, px1, py1, frags);
    else raster_inline_t<MODE, long long>(p, s, px0, py0, px1, py1, frags);
}

// R2-R4 for one sub-triangle: snap, orient, then pick the raster path by the size of its pixel bounding box:
//   small  (<= 8x8 .. 64 px)   : inline, by the thread that set it up;
//   medium (<= 32 x 32)         : handed back through `defer` and rasterised by the whole warp (32 pixels per step);
//   large                       : split into 16-row bands and queued for raster_band_kernel.
template <int MODE>
__device__ bool process_subtriangle(const RasterParams& p, const float4 a, const float4 b, const float4 c, uint32_t rec, uint32_t& frags, SubTri* defer,
                                    bool* deferred) {
    const float4 v[3] = {a, b, c};
    int sx[3], sy[3];
    float sz[3];
    const float hw = mul_rn(p.vw, 0.5f), hh = mul_rn(p.vh, 0.5f);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        if (!(v[k].w > 0.0f)) return false;
        // x / 1.0f == x bit for bit: orthographic cameras (every shadow pass) skip the three IEEE divisions per vertex
        const bool unit_w = v[k].w == 1.0f;
        const float nx = unit_w ? v[k].x : div_rn(v[k].x, v[k].w), ny = unit_w ? v[k].y : div_rn(v[k].y, v[k].w), nz = unit_w ? v[k].z : div_rn(v[k].z, v[k].w);
        const float fx = add_rn(p.ox, mul_rn(add_rn(nx, 1.0f), hw)), fy = add_rn(p.oy, mul_rn(sub_rn(1.0f, ny), hh));
        const float qx = rintf(mul_rn(fx, 256.0f)), qy = rintf(mul_rn(fy, 256.0f));
        if (!(fabsf(qx) < 1.0e9f) || !(fabsf(qy) < 1.0e9f)) return false;
        sx[k] = (int)qx; sy[k] = (int)qy; sz[k] = nz;
    }
    const long long area = (long long)(sx[1] - sx[0]) * (sy[2] - sy[0]) - (long long)(sx[2] - sx[0]) * (sy[1] - sy[0]);
    if (area == 0) return false;
    const bool visible = p.positive_visible ? (area < 0) : (area > 0);   // y-down area has the opposite sign of the NDC area
    if (!visible) return false;
    SubTri s;
    if (area > 0) {
#pragma unroll
        for (int k = 0; k < 3; ++k) { s.x[k] = sx[k]; s.y[k] = sy[k]; s.z[k] = sz[k]; }
    } else {
        s.x[0] = sx[0]; s.y[0] = sy[0]; s.z[0] = sz[0]; s.x[1] = sx[2]; s.y[1] = sy[2]; s.z[1] = sz[2]; s.x[2] = sx[1]; s.y[2] = sy[1]; s.z[2] = sz[1];
    }
    s.rec = rec;
    int px0, py0, px1, py1;
    pixel_bounds(p, s, px0, py0, px1, py1);
    if (px0 > px1 || py0 > py1) return true;   // set up, but no sample inside the target rectangle
    const int w = px1 - px0 + 1, h = py1 - py0 + 1;
    bool inline_raster = (w * h <= SMALL_AREA);
    if (!inline_raster && defer && w <= MEDIUM_MAX && h <= MEDIUM_MAX) {
        *defer = s;
        *deferred = true;
        return true;
    }
    if (!inline_raster) {
        const uint32_t nb = (uint32_t)((py1 / BAND_ROWS) - (py0 / BAND_ROWS) + 1);
        const uint32_t li = atomicAdd(&p.counters[0], 1u);
        uint32_t bi = 0;
        bool queued = li < LARGE_CAP;
        if (queued) {
            bi = atomicAdd(&p.counters[1], nb);
            queued = bi + nb <= BAND_CAP;
            if (!queued) for (uint32_t k = bi; k < BAND_CAP; ++k) p.bands[k] = make_uint2(BAND_SKIP, 0u);   // the one reservation that straddles the cap
        }
        if (queued) {
            p.large[li] = s;
            for (uint32_t k = 0; k < nb; ++k) p.bands[bi + k] = make_uint2(li, (uint32_t)(py0 / BAND_ROWS) + k);
            return true;
        }
        if (defer) {   // queues full: stay correct, let the warp rasterise it
            *defer = s;
            *deferred = true;
            return true;
        }
        inline_raster = true;
    }
    raster_inline<MODE>(p, s, px0, py0, px1, py1, frags);
    return true;
}

// medium triangles: all 32 lanes rasterise one sub-triangle; the lane grid is 32x1, 16x2 or 8x4 pixels depending on the box width
template <int MODE, typename T>
__device__ __forceinline__ void raster_cooperative_t(const RasterParams& p, const SubTri& s, int lane, int px0, int py0, int px1, int py1, uint32_t& frags) {
    const int w = px1 - px0 + 1;
    const int lw = w <= 8 ? 8 : (w <= 16 ? 16 : 32), lh = 32 / lw, lx = lane % lw, ly = lane / lw;
    const EdgeSetupT<T> e = make_edges<T>(s, px0, py0);
    for (int py = py0 + ly; py <= py1; py += lh) {
        const T dy = py - py0;
        T c0 = e.e0 + dy * e.sy0 + (T)lx * e.sx0, c1 = e.e1 + dy * e.sy1 + (T)lx * e.sx1, c2 = e.e2 + dy * e.sy2 + (T)lx * e.sx2;
        for (int px = px0 + lx; px <= px1; px += lw) {
            emit_pixel<MODE, T>(p, s, e, px, py, c0, c1, c2, frags);
            c0 += lw * e.sx0; c1 += lw * e.sx1; c2 += lw * e.sx2;
        }
    }
}
template <int MODE>
__device__ __forceinline__ void raster_cooperative(const RasterParams& p, const SubTri& s, int lane, uint32_t& frags) {
    int px0, py0, px1, py1;
    pixel_bounds(p, s, px0, py0, px1, py1);
    if (fits32(s, px0, py0, px1, py1)) raster_cooperative_t<MODE, int>(p, s, lane, px0, py0, px1, py1, frags);   // warp-uniform: same triangle in every lane
    else raster_cooperative_t<MODE, long long>(p, s, lane, px0, py0, px1, py1, frags);
}

// vertex stage up to clip space, clipping and setup of listed triangle i; medium sub-triangles come back through `defer`
template <int MODE>
__device__ void setup_listed_triangle(const RasterParams& p, unsigned long long i, uint32_t n_regions, uint32_t& frags, uint32_t& set_up, SubTri* defer, bool* deferred) {
    // region of listed triangle i: last r with tri_prefix[r] <= i
    // (a warp-cooperative 32-ary bracket search was tried for the many-region case: no gain on config 3, and its extra live
    //  state slowed the shadow passes of config 5)
    uint32_t lo = 0, hi = n_regions;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (p.tri_prefix[mid] <= i) lo = mid; else hi = mid;
    }
    const uint32_t r = lo;
    const uint32_t t = (uint32_t)(i - p.tri_prefix[r]);
    const uint64_t e = (uint64_t)p.calls[r].base_index + (uint64_t)t * 3u;
    if (e + 2 >= p.index_elems) return;
    const uint32_t k0 = p.indices[e], k1 = p.indices[e + 1], k2 = p.indices[e + 2];
    if (k0 == R3_INVALID_VERTEX || k1 == R3_INVALID_VERTEX || k2 == R3_INVALID_VERTEX) return;   // opaque.wgsl:97-101
    const r3_batch_data* batch = &p.batches[p.regions[r].job_index];
    const uint32_t oid = batch->object_culling_information[k0 >> 24].object_id;                  // unpack_vertex_index (shader.rs:249-316)
    if (oid >= p.n_slots || oid >= p.matrices_cap) return;
    const r3_object* obj = &p.objects[oid];
    if (obj->enabled == 0u) return;                                                               // opaque.wgsl:108-112
    bool alpha_tested = false;
    if (p.regions[r].material_key == 1ull) {
        // cutout routine (pbr/routine.rs:97-133, `discard` variant): untextured alpha = material.albedo.a, constant over the
        // object unless the vertex colour is blended in, so the discard (opaque.wgsl:231-235, depth.wgsl:186-207) is per triangle
        const r3_material* m = &p.materials[obj->material_index < p.n_materials ? obj->material_index : 0u];
        // alpha varies inside the object only through the albedo texture or a blended vertex colour: then the discard is
        // evaluated per pixel (cutout_discards); otherwise alpha = material.albedo.a for every fragment of the object
        alpha_tested = (m->flags & R3_MAT_ALBEDO_ACTIVE) && (m->textures[R3_TEX_ALBEDO] != 0u || ((m->flags & R3_MAT_ALBEDO_BLEND) && obj->attr_offset[5] != R3_ATTR_ABSENT));
        if (!alpha_tested && m->albedo[3] < m->alpha_cutout) return;
        if (!(MODE & MODE_ALPHA) || !p.records) alpha_tested = false;   // (run_raster picks the MODE_ALPHA kernels and provides records whenever such materials exist)
    }
    const uint32_t pos_off = obj->attr_offset[0] >> 2;
    float mvp[16];
    {
        const float4* m4 = reinterpret_cast<const float4*>(p.matrices[oid].model_view_proj);   // 64-byte aligned: four 16-byte loads instead of sixteen 4-byte ones
#pragma unroll
        for (int q = 0; q < 4; ++q) { const float4 c4 = __ldg(&m4[q]); mvp[4 * q] = c4.x; mvp[4 * q + 1] = c4.y; mvp[4 * q + 2] = c4.z; mvp[4 * q + 3] = c4.w; }
    }
    const uint32_t vid[3] = {k0 & 0xFFFFFFu, k1 & 0xFFFFFFu, k2 & 0xFFFFFFu};
    float4 clip[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const uint64_t f = (uint64_t)pos_off + (uint64_t)vid[k] * 3u;
        if (f + 2u < p.mesh_words) clip[k] = mat_point_rn(mvp, __uint_as_float(__ldg(&p.mesh[f])), __uint_as_float(__ldg(&p.mesh[f + 1])), __uint_as_float(__ldg(&p.mesh[f + 2])));
        else clip[k] = mat_point_rn(mvp, __uint_as_float(mesh_word(p, f)), __uint_as_float(mesh_word(p, f + 1)), __uint_as_float(mesh_word(p, f + 2)));   // robust access at the buffer end
    }
    // trivial reject + clip need (R1)
    bool ox0 = true, ox1 = true, oy0 = true, oy1 = true, oz0 = true, oz1 = true, need_clip = false, nan = false;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float4 v = clip[k];
        ox0 &= v.x < -v.w; ox1 &= v.x > v.w; oy0 &= v.y < -v.w; oy1 &= v.y > v.w; oz0 &= v.z < 0.0f; oz1 &= v.z > v.w;
#pragma unroll
        for (int pl = 0; pl < 6; ++pl) need_clip |= plane_dist(pl, v) < 0.0f;
        nan |= !(v.w == v.w);
    }
    if (nan || ox0 || ox1 || oy0 || oy1 || oz0 || oz1) return;
    const uint32_t rec = (uint32_t)(i + 1) | (alpha_tested ? REC_ALPHA_TESTED : 0u);
    const auto store_record = [&]() {
        r3_tri_record tr;
#pragma unroll
        for (int k = 0; k < 3; ++k) { tr.xyw[k][0] = clip[k].x; tr.xyw[k][1] = clip[k].y; tr.xyw[k][2] = clip[k].w; tr.vid[k] = vid[k]; }
        tr.object_id = oid; tr._pad[0] = tr._pad[1] = tr._pad[2] = 0u;
        float4* dst = reinterpret_cast<float4*>(&p.records[i]);
        const float4* src = reinterpret_cast<const float4*>(&tr);
        dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2]; dst[3] = src[3];
    };
    if (alpha_tested) store_record();   // the per-fragment discard reads it while this triangle is being rasterised
    bool any = false;
    if (!need_clip) {
        any = process_subtriangle<MODE>(p, clip[0], clip[1], clip[2], rec, frags, defer, deferred);
    } else {
        float4 poly[12];
        poly[0] = clip[0]; poly[1] = clip[1]; poly[2] = clip[2];
        const int n = clip_polygon(poly, 3);
        for (int q = 1; q + 1 < n; ++q) any |= process_subtriangle<MODE>(p, poly[0], poly[q], poly[q + 1], rec, frags, nullptr, nullptr);
    }
    if (any) {
        set_up++;
        if ((MODE & 3) != MODE_DEPTH && !alpha_tested) store_record();
    }
}

// depth-only set-up is a chain of dependent gathers: 64 registers buy a fourth resident CTA per SM
template <int MODE>
__global__ void __launch_bounds__(RS_THREADS, MODE == MODE_DEPTH ? 4 : 1) raster_setup_kernel(const __grid_constant__ RasterParams p) {
    const uint32_t n_regions = p.header[2];
    const unsigned long long total = p.tri_prefix[n_regions];
    const int lane = threadIdx.x & 31;
    uint32_t frags = 0, set_up = 0;
    // every iteration a warp draws a ticket for 32 consecutive listed triangles: the cost of a triangle varies by orders of
    // magnitude (culled / a few pixels / a 32 x 32 box walked by the whole warp), so a static stride leaves most warps idle
    // behind the slowest one (the config-5 shadow passes ran with few active warps that way)
    for (;;) {
        uint32_t tile = 0;
        if (lane == 0) tile = atomicAdd(&p.counters[4], 1u);
        tile = __shfl_sync(0xFFFFFFFFu, tile, 0);
        const unsigned long long base = (unsigned long long)tile * 32ull;
        if (base >= total) break;
        const unsigned long long i = base + lane;
        SubTri med;
        bool has_med = false;
        if (i < total) setup_listed_triangle<MODE>(p, i, n_regions, frags, set_up, &med, &has_med);
        if (MODE & MODE_ALPHA) __syncwarp();   // records of alpha-tested triangles are read by the other lanes below
        uint32_t m = __ballot_sync(0xFFFFFFFFu, has_med);
        if (__popc(m) >= COOP_MAX_LANES) {
            // most lanes hold a medium triangle: 32 boxes walked in parallel beat 32 boxes walked one after the other
            if (has_med) {
                int px0, py0, px1, py1;
                pixel_bounds(p, med, px0, py0, px1, py1);
                raster_inline<MODE>(p, med, px0, py0, px1, py1, frags);
            }
            m = 0;
        }
        while (m) {
            const int src = __ffs(m) - 1;
            m &= m - 1;
            SubTri s;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                s.x[k] = __shfl_sync(0xFFFFFFFFu, med.x[k], src); s.y[k] = __shfl_sync(0xFFFFFFFFu, med.y[k], src); s.z[k] = __shfl_sync(0xFFFFFFFFu, med.z[k], src);
            }
            s.rec = __shfl_sync(0xFFFFFFFFu, med.rec, src);
            raster_cooperative<MODE>(p, s, lane, frags);
        }
    }
    // statistics: one atomic per warp
    frags = warp_reduce(frags);
    set_up = warp_reduce(set_up);
    if (lane == 0 && p.stats) {
        if (set_up) atomicAdd(&p.stats[0], (unsigned long long)set_up);
        if (frags) atomicAdd(&p.stats[1], (unsigned long long)frags);
    }
}

// one warp per (large sub-triangle, 16-row band); lanes = 32 consecutive pixels
template <int MODE>
__global__ void __launch_bounds__(RS_THREADS) raster_band_kernel(const __grid_constant__ RasterParams p) {
    const int lane = threadIdx.x & 31;
    uint32_t n_bands = p.counters[1];
    if (n_bands > BAND_CAP) n_bands = BAND_CAP;
    uint32_t frags = 0;
    for (;;) {
        uint32_t item = 0;
        if (lane == 0) item = atomicAdd(&p.counters[2], 1u);
        item = __shfl_sync(0xFFFFFFFFu, item, 0);
        if (item >= n_bands) break;
        const uint2 it = p.bands[item];
        if (it.x >= LARGE_CAP) continue;   // BAND_SKIP
        const SubTri s = p.large[it.x];
        int px0, py0, px1, py1;
        pixel_bounds(p, s, px0, py0, px1, py1);
        const int by0 = max(py0, (int)it.y * BAND_ROWS), by1 = min(py1, (int)it.y * BAND_ROWS + BAND_ROWS - 1);
        if (by0 > by1) continue;
        const EdgeSetupT<long long> e = make_edges<long long>(s, px0, by0);
        const int rows = by1 - by0 + 1;
        for (int bx = px0; bx <= px1; bx += 32) {
            // skip the 32 x rows block when it lies entirely outside one edge: evaluate the corner that maximises E
            const long long dx = bx - px0, wx = min(31, px1 - bx), hy = rows - 1;
            // multisampling: a sample sits up to 96/256 pixel from the centre, widen the block by half a pixel per axis
            const long long k0 = p.samples == 1u ? 0 : (llabs(e.sx0) + llabs(e.sy0)) / 2, k1 = p.samples == 1u ? 0 : (llabs(e.sx1) + llabs(e.sy1)) / 2,
                            k2 = p.samples == 1u ? 0 : (llabs(e.sx2) + llabs(e.sy2)) / 2;
            const long long m0 = k0 + e.e0 + dx * e.sx0 + (e.sx0 > 0 ? wx * e.sx0 : 0) + (e.sy0 > 0 ? hy * e.sy0 : 0);
            const long long m1 = k1 + e.e1 + dx * e.sx1 + (e.sx1 > 0 ? wx * e.sx1 : 0) + (e.sy1 > 0 ? hy * e.sy1 : 0);
            const long long m2 = k2 + e.e2 + dx * e.sx2 + (e.sx2 > 0 ? wx * e.sx2 : 0) + (e.sy2 > 0 ? hy * e.sy2 : 0);
            if ((m0 | m1 | m2) < 0) continue;
            const int px = bx + lane;
            long long c0 = e.e0 + (dx + lane) * e.sx0, c1 = e.e1 + (dx + lane) * e.sx1, c2 = e.e2 + (dx + lane) * e.sx2;
            for (int py = by0; py <= by1; ++py) {
                if (px <= px1) emit_pixel<MODE, long long>(p, s, e, px, py, c0, c1, c2, frags);
                c0 += e.sy0; c1 += e.sy1; c2 += e.sy2;
            }
        }
    }
    frags = warp_reduce(frags);
    if (lane == 0 && frags && p.stats) atomicAdd(&p.stats[1], (unsigned long long)frags);
}

// exclusive prefix over the regions the routines with material keys in [key_lo, key_hi] draw (forward.rs:286-313)
constexpr int RP_THREADS = 1024;
__global__ void __launch_bounds__(RP_THREADS) region_prefix_kernel(const r3_region* __restrict__ regions, const r3_indirect_call* __restrict__ calls,
                                                                   const uint32_t* __restrict__ header, unsigned long long* __restrict__ prefix,
                                                                   unsigned long long key_lo, unsigned long long key_hi) {
    __shared__ unsigned long long s_warp[RP_THREADS / 32 + 1];
    const uint32_t n_regions = header[2];
    const unsigned long long total = block_scan_excl_chunked<RP_THREADS>(
        n_regions, s_warp,
        [&](uint32_t r) {
            return regions[r].material_key >= key_lo && regions[r].material_key <= key_hi ? (unsigned long long)(calls[r].vertex_count / 3u) : 0ull;
        },
        [&](uint32_t r, unsigned long long e) { prefix[r] = e; });
    if (threadIdx.x == 0) prefix[n_regions] = total;
}

}  // namespace

// ------------------------------------------------------------------ host side
// CTAs of kernel K that are resident at once on the whole GPU (CTAs per SM are a property of the binary: asked once per kernel)
template <void (*K)(const RasterParams)>
static int resident_grid(const r3_ctx* c) {
    static int per_sm = 0;
    if (!per_sm && (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, K, RS_THREADS, 0) != cudaSuccess || per_sm < 1)) { cudaGetLastError(); per_sm = 1; }
    return c->sm_count * per_sm;
}
struct DrawSource { const r3_jobs* jobs; const r3_indirect_call* calls; const uint32_t* indices; uint64_t index_elems; };

static bool draw_source_for(r3_camera* cam, int jobs_idx, int partition, DrawSource* ds) {
    if (!cam->index_buffer.created || jobs_idx < 0) return false;
    const r3_jobs* j = &cam->jobs[jobs_idx];
    if (!j->valid || (!j->device_built && j->n_regions == 0)) return false;
    const r3_iobuf& ib = cam->index_buffer; const r3_iobuf& db = cam->draw_call_buffer;
    if (j->n_regions > db.capacity_elements / 2) return false;
    ds->jobs = j;
    ds->indices = (const uint32_t*)ib.d + (partition ? ib.in_off() : ib.out_off());
    ds->index_elems = ib.capacity_elements / 2;
    ds->calls = (const r3_indirect_call*)db.d + (partition ? db.in_off() : db.out_off());
    return true;
}

static int ensure_raster_scratch(r3_ctx* c) {
    // layout: counters[4] | tri_prefix[...] handled separately | large[LARGE_CAP] | bands[BAND_CAP]
    const uint64_t need = 64 + (uint64_t)LARGE_CAP * sizeof(SubTri) + (uint64_t)BAND_CAP * sizeof(uint2);
    return r3_reserve(c, &c->d_scratch, &c->scratch_cap, need, 1, false, false);
}

static int run_raster(r3_ctx* c, r3_camera* cam, const DrawSource& ds, int mode, int pass, float ox, float oy, float vw, float vh,
                      int x0, int y0, int x1, int y1, uint32_t pitch) {
    const bool depth_only = mode == MODE_DEPTH;
    const r3_jobs* j = ds.jobs;
    R3_TRY(ensure_raster_scratch(c));
    uint32_t* counters = (uint32_t*)c->d_scratch;
    SubTri* large = (SubTri*)((uint8_t*)c->d_scratch + 64);
    uint2* bands = (uint2*)((uint8_t*)large + (size_t)LARGE_CAP * sizeof(SubTri));
    R3_CUDA(c, cudaMemsetAsync(counters, 0, 64, c->stream));
    R3_TRY(r3_reserve_t(c, &cam->d_block_sums, &cam->block_sums_cap, (uint64_t)j->n_regions + 2));
    const unsigned long long key_lo = mode == MODE_BLEND ? 2ull : 0ull, key_hi = mode == MODE_BLEND ? 2ull : 1ull;
    region_prefix_kernel<<<1, RP_THREADS, 0, c->stream>>>(j->d_regions, ds.calls, j->d_header, cam->d_block_sums, key_lo, key_hi);
    R3_CHECK_LAUNCH(c, "region_prefix_kernel");

    RasterParams p;
    p.batches = j->d_batches; p.regions = j->d_regions; p.header = j->d_header;
    p.calls = ds.calls; p.indices = ds.indices; p.index_elems = ds.index_elems; p.tri_prefix = cam->d_block_sums;
    p.objects = c->d_objects; p.n_slots = c->n_slots; p.matrices = cam->d_matrices; p.matrices_cap = cam->matrices_cap;
    p.mesh = c->d_mesh; p.mesh_words = c->mesh_words; p.materials = c->d_materials; p.n_materials = c->n_materials;
    p.ox = ox; p.oy = oy; p.vw = vw; p.vh = vh; p.x0 = x0; p.y0 = y0; p.x1 = x1; p.y1 = y1; p.pitch = pitch;
    p.positive_visible = (cam->header.flags & R3_PCU_POSITIVE_AREA_VISIBLE) ? 1 : 0;
    p.samples = depth_only ? 1u : c->samples;
    p.vis = c->d_vis; p.pass_bit = (uint32_t)(pass & 1); p.depth_bits = (uint32_t*)c->d_atlas;
    p.frag_heads = c->d_frag_heads; p.frag_nodes = c->d_frag_nodes; p.frag_cap = (uint32_t)c->frag_nodes_cap; p.key_lo = key_lo; p.key_hi = key_hi;
    p.large = large; p.bands = bands; p.counters = counters; p.stats = mode == MODE_COLOUR ? c->d_stats : nullptr;   // statistics describe the opaque + cutout passes
    p.tt.tex = c->d_tex_descs; p.tt.n_tex = c->n_textures; p.tt.texels = c->d_texels; p.tt.clamp_to_edge = 0u;
    p.records = nullptr;
    if (depth_only && c->any_frag_alpha) {
        // cutout materials whose alpha comes from a texture / vertex colour: the shadow pass needs the triangle records too
        R3_TRY(r3_reserve_t(c, &c->d_tris[3], &c->tris_cap[3], (uint64_t)j->total_invocations + 1));
        p.records = c->d_tris[3];
    }
    if (!depth_only) {
        // one record slot per listed triangle; the listed total is bounded by the partition size
        const uint64_t max_tris = (uint64_t)j->total_invocations;
        if (max_tris >= (1ull << 31)) return r3_fail(c, R3_E_INVALID, "more than 2^31 triangles in one pass");
        R3_TRY(r3_reserve_t(c, &c->d_tris[pass], &c->tris_cap[pass], max_tris + 1));
        c->n_tris[pass] = max_tris;
        p.records = c->d_tris[pass];
    }
    // persistent grids: exactly the CTAs that are resident at once (SMs x the kernel's CTAs per SM).  A fixed SMs x 8 left the colour
    // kernels (one resident CTA per SM) seven waves of CTAs that start only to find the tickets gone.
    const int variant = mode | ((mode != MODE_DEPTH && c->samples == 4u) ? MODE_MSAA : 0) | ((c->any_frag_alpha && mode != MODE_BLEND) ? MODE_ALPHA : 0);
#define R3_RASTER_ONE(KERNEL, M) KERNEL<M><<<resident_grid<KERNEL<M>>(c), RS_THREADS, 0, c->stream>>>(p)
#define R3_RASTER_LAUNCH(KERNEL)                                                                                          \
    switch (variant) {                                                                                                    \
        case MODE_DEPTH: R3_RASTER_ONE(KERNEL, MODE_DEPTH); break;                                                        \
        case MODE_COLOUR: R3_RASTER_ONE(KERNEL, MODE_COLOUR); break;                                                      \
        case MODE_BLEND: R3_RASTER_ONE(KERNEL, MODE_BLEND); break;                                                        \
        case MODE_COLOUR | MODE_MSAA: R3_RASTER_ONE(KERNEL, MODE_COLOUR | MODE_MSAA); break;                              \
        case MODE_BLEND | MODE_MSAA: R3_RASTER_ONE(KERNEL, MODE_BLEND | MODE_MSAA); break;                                \
        case MODE_DEPTH | MODE_ALPHA: R3_RASTER_ONE(KERNEL, MODE_DEPTH | MODE_ALPHA); break;                              \
        case MODE_COLOUR | MODE_ALPHA: R3_RASTER_ONE(KERNEL, MODE_COLOUR | MODE_ALPHA); break;                            \
        default: R3_RASTER_ONE(KERNEL, MODE_COLOUR | MODE_MSAA | MODE_ALPHA); break;                                      \
    }
    r3_stage_begin(c, depth_only ? R3_STAGE_RASTER_SETUP_DEPTH : R3_STAGE_RASTER_SETUP_COLOUR);
    R3_RASTER_LAUNCH(raster_setup_kernel)
    r3_stage_end(c);
    R3_CHECK_LAUNCH(c, "raster_setup_kernel");
    r3_stage_begin(c, R3_STAGE_RASTER_BANDS);
    R3_RASTER_LAUNCH(raster_band_kernel)
    r3_stage_end(c);
    R3_CHECK_LAUNCH(c, "raster_band_kernel");
#undef R3_RASTER_LAUNCH
#undef R3_RASTER_ONE
    return R3_OK;
}

R3_EXPORT int r3_forward_pass(r3_ctx* c, int source) {
    if (!c || !c->d_vis) return r3_fail(c, R3_E_STATE, "forward_pass before set_render_target");
    cudaSetDevice(c->device);
    r3_camera* cam = &c->cams[0];
    DrawSource ds;
    if (source == 0) {
        if (cam->cache_idx < 0) return R3_OK;                                   // forward.rs:224-231
        if (!draw_source_for(cam, cam->cache_idx, 0, &ds)) return R3_OK;        // Output partition, pre-swap (forward.rs:251)
    } else {
        if (!cam->has_draw_call_set) return R3_OK;                              // forward.rs:212-216
        if (!draw_source_for(cam, cam->cur, 1, &ds)) return R3_OK;              // Input partition, post-swap
    }
    R3_TRY(run_raster(c, cam, ds, MODE_COLOUR, source ? 1 : 0, 0.0f, 0.0f, (float)c->width, (float)c->height, 0, (int)c->row_begin, (int)c->width,
                      (int)c->row_end, c->width));
    if (source == 1) cam->cache_idx = cam->cur;                                 // draw_call_set_cache.insert (forward.rs:219)
    return R3_OK;
}

R3_EXPORT int r3_shadow_pass(r3_ctx* c, uint32_t shadow_index, uint32_t ox, uint32_t oy, uint32_t size) {
    if (!c || !c->d_atlas) return r3_fail(c, R3_E_STATE, "shadow_pass before set_directional_lights");
    if (shadow_index >= R3_MAX_SHADOWS) return r3_fail(c, R3_E_INVALID, "bad shadow index");
    if ((uint64_t)ox + size > c->atlas_w || (uint64_t)oy + size > c->atlas_h) return r3_fail(c, R3_E_INVALID, "shadow viewport outside the atlas");
    cudaSetDevice(c->device);
    r3_camera* cam = &c->cams[shadow_index + 1];
    DrawSource ds;
    if (!cam->has_draw_call_set || !draw_source_for(cam, cam->cur, 0, &ds)) return R3_OK;
    return run_raster(c, cam, ds, MODE_DEPTH, 0, (float)ox, (float)oy, (float)size, (float)size, (int)ox, (int)oy, (int)(ox + size), (int)(oy + size), c->atlas_w);
}

// blend routine, first half: rasterise the key-2 regions of this frame's residual list into per-sample fragment lists.
// The pool holds every fragment that is not behind the opaque depth; when it is too small the pass is repeated with a
// larger one (the only host round trip of the frame, and only in frames with transparent objects).
int r3_blend_collect(r3_ctx* c, bool* ran) {
    *ran = false;
    r3_camera* cam = &c->cams[0];
    DrawSource ds;
    if (!c->any_blend || !cam->has_draw_call_set || !draw_source_for(cam, cam->cur, 1, &ds)) return R3_OK;   // CullingSource::Residual
    const uint64_t n_samples = (uint64_t)c->width * c->height * c->samples;
    R3_TRY(r3_reserve_t(c, &c->d_frag_heads, &c->frag_heads_cap, n_samples));
    if (c->frag_nodes_cap == 0) R3_TRY(r3_reserve_t(c, &c->d_frag_nodes, &c->frag_nodes_cap, n_samples < (1u << 20) ? (1u << 20) : n_samples));
    for (int attempt = 0; attempt < 2; ++attempt) {
        R3_CUDA(c, cudaMemsetAsync(c->d_frag_heads, 0, n_samples * 4, c->stream));
        R3_TRY(run_raster(c, cam, ds, MODE_BLEND, 2, 0.0f, 0.0f, (float)c->width, (float)c->height, 0, (int)c->row_begin, (int)c->width, (int)c->row_end,
                          c->width));
        uint32_t used = 0;
        R3_CUDA(c, cudaMemcpyAsync(&used, (const uint32_t*)c->d_scratch + 3, 4, cudaMemcpyDeviceToHost, c->stream));
        R3_CUDA(c, r3_stream_sync(c));
        if (used <= c->frag_nodes_cap) { *ran = true; return R3_OK; }
        if (attempt == 1 || used >= 0xFFFFFFF0u) break;
        R3_TRY(r3_reserve_t(c, &c->d_frag_nodes, &c->frag_nodes_cap, (uint64_t)used + (used >> 3)));
    }
    return r3_fail(c, R3_E_OOM, "forward_blend: fragment pool overflow");
}
