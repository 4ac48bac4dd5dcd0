// r3_shade.cu — deferred fs_main over the visibility buffer, hi-Z pyramid, HDR->LDR blit, render targets.
//
// Replaces (reference paths):
//   * opaque.wgsl::vs_main outputs + fs_main + surface_shading   rend3-routine/shaders/src/opaque.wgsl:91-135,203-551
//     BRDF terms math/brdf.wgsl:3-33, PCF5 shadow/pcf.wgsl:1-9, sRGB decode math/color.wgsl:3-9
//   * hi_z.wgsl::fs_main min-downsample chain                    rend3-routine/src/hi_z.rs:161-234, hi_z.wgsl:18-33
//   * blit.wgsl fs_main_scene / fs_main_monitor                  rend3-routine/src/tonemapping.rs:108-147, blit.wgsl:21-31
//
// The resolve kernel runs fs_main ONCE per covered pixel: it reads the 64-bit visibility key, fetches the
// winning triangle's 64-byte record, re-runs the vertex stage for its three vertices (vertex pulling from the
// mesh megabuffer), interpolates with perspective-correct weights (raster rule R6) and shades.  Lights are
// staged in shared memory per CTA after a one-block "light prep" kernel has moved them to view space
// (view_mat3 * -direction, view * position, light.view_proj * inv_view) — work the WGSL repeats per fragment.
// This translation unit is compiled WITH fused multiply-add: shaded pixels are checked to 1e-4, not bit-exact.
#include <cuda_fp16.h>

#include "r3_common.cuh"
#include "r3_texture.cuh"

namespace {

constexpr float R3_PI = 3.14159265359f;   // math/consts.wgsl:1
constexpr int MAX_SMEM_DIR = 8, MAX_SMEM_POINT = 128;

struct DirPrep { float lm[16]; float l[3]; float color[3]; float inv_res[2]; float offset[2]; float size[2]; float _pad[4]; };   // 32 floats
struct PointPrep { float pos[3]; float radius; float color[3]; float _pad; };                                                     // 8 floats
static_assert(sizeof(DirPrep) == 128 && sizeof(PointPrep) == 32, "prep layouts");

struct ShadeParams {
    const unsigned long long* vis;
    const r3_tri_record* tris0; const r3_tri_record* tris1; unsigned long long n_tris0, n_tris1;
    const r3_object* objects; const r3_object_matrices* matrices;
    const uint32_t* mesh; uint64_t mesh_words;
    const r3_material* materials; uint32_t n_materials;
    TexTable tt;                                                          // bindless d2 texture table (r3_set_textures)
    TexTable sky; r3_texture_desc sky_desc; float inv_origin_view_proj[16];   // skybox routine (r3_set_skybox)
    const DirPrep* dir; uint32_t n_dir; const PointPrep* point;
    const uint32_t* point_count;                                          // ShaderPointLightBuffer's count (@0), written on the device
    const float* atlas; uint32_t atlas_w, atlas_h;
    // blend routine (r3_forward_blend): triangle records of the key-2 regions + the per-sample fragment lists
    const r3_tri_record* tris2; unsigned long long n_tris2; const uint32_t* frag_heads; const uint4* frag_nodes;
    float ambient[4]; float clear[4];
    uint32_t width, height, row_begin, row_end, samples;
    float4* hdr32; uint2* hdr16; float* depth;
    unsigned long long* stats;
};

__device__ __forceinline__ uint32_t mesh_word(const ShadeParams& p, uint64_t i) { return i < p.mesh_words ? __ldg(&p.mesh[i]) : 0u; }
__device__ __forceinline__ float3 fetch3(const ShadeParams& p, uint32_t byte_off, uint32_t vid) {
    const uint64_t f = (uint64_t)(byte_off >> 2) + (uint64_t)vid * 3u;
    return make_float3(__uint_as_float(mesh_word(p, f)), __uint_as_float(mesh_word(p, f + 1)), __uint_as_float(mesh_word(p, f + 2)));
}
__device__ __forceinline__ float dot3(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ float3 normalize3(float3 a) { const float r = rsqrtf(dot3(a, a)); return make_float3(a.x * r, a.y * r, a.z * r); }
__device__ __forceinline__ float saturate(float v) { return fminf(fmaxf(v, 0.0f), 1.0f); }

struct Pixel { float3 diffuse_pi, f0, normal; float roughness, f90; };   // diffuse_pi = diffuse_color * (1/pi)

// MUFU-based approximations (<= 2 ulp): the shaded result is checked to 1e-4, not bit-exact
__device__ __forceinline__ float sqrt_approx(float x) { float r; asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float rcp_approx(float x) { float r; asm("rcp.approx.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

// surface_shading (opaque.wgsl:440-468) with brdf_d_ggx / brdf_f_schlick / brdf_v_smith_ggx_correlated / brdf_fd_lambert.
// When roughness > 0 and n.v is a number every term is finite, so a light with n.l <= 0 contributes exactly 0 and is skipped.
// With roughness == 0 the reference's 0 * inf = NaN must survive to the caller's max(), so the full path runs; so it does for a
// NaN normal (a zero vertex normal, an axis scaled by 0, a normal map without tangents): saturate() turns n.l into 0 but n.v stays
// NaN, the reference's term is NaN, and fs_main's final max() then yields ambient * albedo, not max(ambient * albedo, 0).
__device__ __forceinline__ float3 surface_shading(const float3 l, const float3 intensity, const Pixel& px, const float3 v, float nov, float occlusion) {
    const float nol = saturate(dot3(px.normal, l));
    const float a = px.roughness, a2 = a * a;
    if (nol <= 0.0f && a2 > 0.0f && nov == nov) return make_float3(0.f, 0.f, 0.f);
    const float3 h = normalize3(make_float3(v.x + l.x, v.y + l.y, v.z + l.z));
    const float noh = saturate(dot3(px.normal, h));
    const float loh = saturate(dot3(l, h));
    const float fd = (noh * a2 - noh) * noh + 1.0f;
    const float d = a2 * rcp_approx(R3_PI * fd * fd);
    const float om = 1.0f - loh, om2 = om * om, pw = om2 * om2 * om;   // pow(1 - loh, 5)
    const float3 f = make_float3(px.f0.x + (px.f90 - px.f0.x) * pw, px.f0.y + (px.f90 - px.f0.y) * pw, px.f0.z + (px.f90 - px.f0.z) * pw);
    const float ggxl = nov * sqrt_approx((-nol * a2 + nol) * nol + a2);
    const float ggxv = nol * sqrt_approx((-nov * a2 + nov) * nov + a2);
    const float dv = d * (0.5f * rcp_approx(ggxl + ggxv));
    const float s = nol * occlusion;
    return make_float3((px.diffuse_pi.x + dv * f.x) * intensity.x * s, (px.diffuse_pi.y + dv * f.y) * intensity.y * s,
                       (px.diffuse_pi.z + dv * f.z) * intensity.z * s);
}

// shadow_sample_pcf5 (shadow/pcf.wgsl:1-9): five textureSampleCompareLevel taps (centre, +-1 texel in x and y) with the
// linear, GreaterEqual, Repeat-addressed comparison sampler (common/samplers.rs:24,42-56), in the oracle's rounding: each tap
// takes its own coordinate (u * W + offset) - 0.5, bilinear weights lerp the 0/1 compares, and the taps are summed in source order.
// One footprint shared by the five taps is not the same: next to a power of two u * W + 1 or u * W - 1 rounds where u * W does not,
// and that tap's fraction moves by an ulp.  So each axis keeps the three coordinates of its offsets -1, 0, +1.
__device__ __forceinline__ int wrap_texel(int i, int n) {
    if ((unsigned)i < (unsigned)n) return i;   // common case: no division
    const int m = i % n;
    return m < 0 ? m + n : m;
}
struct TapAxis { int i[3]; float f[3]; };   // floor and fraction of (u * n + o) - 0.5 for the offsets o = -1, 0, +1
__device__ __forceinline__ TapAxis tap_axis(float u, uint32_t n) {
    const float un = mul_rn(u, (float)n);
    TapAxis a;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float x = sub_rn(add_rn(un, (float)(k - 1)), 0.5f), fl = floorf(x);
        a.f[k] = sub_rn(x, fl);
        // clamp before the int conversion: coordinates far outside the atlas only arise for fragments outside the light volume
        a.i[k] = (int)fminf(fmaxf(fl, -1.0e9f), 1.0e9f);
    }
    return a;
}
// one tap: (c00 * (1 - fx) + c10 * fx) * (1 - fy) + (c01 * (1 - fx) + c11 * fx) * fy
__device__ __forceinline__ float bilinear_rn(float c00, float c10, float c01, float c11, float fx, float fy) {
    const float gx = sub_rn(1.0f, fx);
    return add_rn(mul_rn(add_rn(mul_rn(c00, gx), mul_rn(c10, fx)), sub_rn(1.0f, fy)), mul_rn(add_rn(mul_rn(c01, gx), mul_rn(c11, fx)), fy));
}
__device__ __forceinline__ float texel_ge(const ShadeParams& p, float ref, int x, int y) {
    return ref >= __ldg(&p.atlas[(size_t)y * p.atlas_w + x]) ? 1.0f : 0.0f;
}
// the taps at offsets (0,0), (0,1), (0,-1), (1,0), (-1,0), summed in that order, times 0.2
__device__ __forceinline__ float pcf5_sum(float centre, float up, float down, float right, float left) {
    return mul_rn(add_rn(add_rn(add_rn(add_rn(centre, up), down), right), left), 0.2f);
}
// the general case: every tap reads its own four texels
__device__ __noinline__ float shadow_pcf5_taps(const ShadeParams& p, const TapAxis ax, const TapAxis ay, float ref) {
    const int W = (int)p.atlas_w, H = (int)p.atlas_h;
    const int ox[5] = {0, 0, 0, 1, -1}, oy[5] = {0, 1, -1, 0, 0};
    float t[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        const int a = ox[k] + 1, b = oy[k] + 1;
        const int x0 = wrap_texel(ax.i[a], W), x1 = wrap_texel(ax.i[a] + 1, W), y0 = wrap_texel(ay.i[b], H), y1 = wrap_texel(ay.i[b] + 1, H);
        t[k] = bilinear_rn(texel_ge(p, ref, x0, y0), texel_ge(p, ref, x1, y0), texel_ge(p, ref, x0, y1), texel_ge(p, ref, x1, y1), ax.f[a], ay.f[b]);
    }
    return pcf5_sum(t[0], t[1], t[2], t[3], t[4]);
}
__device__ __forceinline__ float shadow_pcf5(const ShadeParams& p, float u, float v, float ref) {
    const TapAxis ax = tap_axis(u, p.atlas_w), ay = tap_axis(v, p.atlas_h);
    // almost always the offsets -1 and +1 land one texel either side of the centre tap's floor: then the 20 compares are the 12
    // distinct texels of a 4x4 neighbourhood without corners (each tap still with its own fractions)
    if (ax.i[0] != ax.i[1] - 1 || ax.i[2] != ax.i[1] + 1 || ay.i[0] != ay.i[1] - 1 || ay.i[2] != ay.i[1] + 1) return shadow_pcf5_taps(p, ax, ay, ref);
    const int W = (int)p.atlas_w, H = (int)p.atlas_h;
    int xs[4], ys[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { xs[k] = wrap_texel(ax.i[1] - 1 + k, W); ys[k] = wrap_texel(ay.i[1] - 1 + k, H); }
    float c[4][4];   // c[row][col] = ref >= texel ? 1 : 0
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const bool corner = (r == 0 || r == 3) && (q == 0 || q == 3);
            c[r][q] = corner ? 0.0f : texel_ge(p, ref, xs[q], ys[r]);
        }
    const float centre = bilinear_rn(c[1][1], c[1][2], c[2][1], c[2][2], ax.f[1], ay.f[1]);
    const float up = bilinear_rn(c[2][1], c[2][2], c[3][1], c[3][2], ax.f[1], ay.f[2]);
    const float down = bilinear_rn(c[0][1], c[0][2], c[1][1], c[1][2], ax.f[1], ay.f[0]);
    const float right = bilinear_rn(c[1][2], c[1][3], c[2][2], c[2][3], ax.f[2], ay.f[1]);
    const float left = bilinear_rn(c[1][0], c[1][1], c[2][0], c[2][1], ax.f[0], ay.f[1]);
    return pcf5_sum(centre, up, down, right, left);
}

// one perspective weight numerator of raster rule R6, oracle order: ((c.x * nx + c.y * ny) + c.z) with c = cross(a, b) over (x, y, w)
__device__ __forceinline__ float cross_term_rn(const float3 a, const float3 b, float nx, float ny) {
    const float cx = sub_rn(mul_rn(a.y, b.z), mul_rn(a.z, b.y)), cy = sub_rn(mul_rn(a.z, b.x), mul_rn(a.x, b.z)), cz = sub_rn(mul_rn(a.x, b.y), mul_rn(a.y, b.x));
    return add_rn(add_rn(mul_rn(cx, nx), mul_rn(cy, ny)), cz);
}
__device__ __forceinline__ float lerp3_rn(float b0, float b1, float b2, float a0, float a1, float a2) {
    return add_rn(add_rn(mul_rn(b0, a0), mul_rn(b1, a1)), mul_rn(b2, a2));
}

struct VsOut { float4 view_position; float3 normal; float4 color; };
// vs_main for one vertex (opaque.wgsl:114-134) + get_vertices defaults (rend3/src/shader.rs:249-316)
__device__ __forceinline__ VsOut vertex_stage(const ShadeParams& p, const uint32_t* attr_offset, const float* __restrict__ mv, const float3 iss, uint32_t vid) {
    VsOut o;
    const float3 pos = fetch3(p, attr_offset[0], vid);
    float3 n = make_float3(0.f, 0.f, 0.f);
    if (attr_offset[1] != R3_ATTR_ABSENT) n = fetch3(p, attr_offset[1], vid);
    o.color = make_float4(1.f, 1.f, 1.f, 1.f);
    if (attr_offset[5] != R3_ATTR_ABSENT) {   // unpack4x8unorm
        const uint32_t w = mesh_word(p, (uint64_t)(attr_offset[5] >> 2) + vid);
        o.color = make_float4((float)(w & 0xFFu) / 255.0f, (float)((w >> 8) & 0xFFu) / 255.0f, (float)((w >> 16) & 0xFFu) / 255.0f, (float)(w >> 24) / 255.0f);
    }
    o.view_position = mat_point_rn(mv, pos.x, pos.y, pos.z);
    const float3 sn = make_float3(iss.x * n.x, iss.y * n.y, iss.z * n.z);
    o.normal = normalize3(make_float3(mv[0] * sn.x + mv[4] * sn.y + mv[8] * sn.z, mv[1] * sn.x + mv[5] * sn.y + mv[9] * sn.z, mv[2] * sn.x + mv[6] * sn.y + mv[10] * sn.z));
    return o;
}

// vs_main outputs interpolated at the centre of a pixel: what fs_main receives
struct FragIn { float4 vp; float3 vnormal; float4 vcolor; uint32_t material_index; };
struct LightMask { uint32_t w[MAX_SMEM_POINT / 32]; };   // point lights (the shared-memory resident ones) a fragment has to visit

// vs_main for the three vertices of triangle record `tp` + interpolation at the centre of pixel (px, py)
__device__ __forceinline__ FragIn fragment_inputs(const ShadeParams& p, const r3_tri_record* tp, uint32_t px, uint32_t py) {
    const float4 q0 = __ldg(reinterpret_cast<const float4*>(tp)), q1 = __ldg(reinterpret_cast<const float4*>(tp) + 1),
                 q2 = __ldg(reinterpret_cast<const float4*>(tp) + 2);
    const uint4 q3 = __ldg(reinterpret_cast<const uint4*>(tp) + 3);
    // xyw[3][3] = q0.xyz | q0.w q1.xy | q1.zw q2.x ; object_id = q2.y ; vid = q2.z q2.w q3.x
    const float3 p0 = make_float3(q0.x, q0.y, q0.z), p1 = make_float3(q0.w, q1.x, q1.y), p2 = make_float3(q1.z, q1.w, q2.x);
    const uint32_t oid = __float_as_uint(q2.y), vid0 = __float_as_uint(q2.z), vid1 = __float_as_uint(q2.w), vid2 = q3.x;
    // R6: perspective-correct weights b_i ~ cross(p_j, p_k) . (ndc_x, ndc_y, 1)
    const float nx = sub_rn(div_rn((float)px + 0.5f, (float)p.width * 0.5f), 1.0f), ny = sub_rn(1.0f, div_rn((float)py + 0.5f, (float)p.height * 0.5f));
    // The chain b_i -> view_position -> shadow-space depth feeds the (discontinuous) shadow compare, so it is evaluated in
    // source order without contraction, exactly like the oracle; so is the rest of the shadow lookup (shade_inputs: region bounds,
    // atlas-coordinate mix; shadow_pcf5: per-tap coordinates, bilinear weights, tap sum), which makes the shadow factor the oracle's
    // bit for bit.  Everything downstream of the lookup is continuous.
    float b0 = cross_term_rn(p1, p2, nx, ny), b1 = cross_term_rn(p2, p0, nx, ny), b2 = cross_term_rn(p0, p1, nx, ny);
    const float bsum = add_rn(add_rn(b0, b1), b2);
    b0 = div_rn(b0, bsum); b1 = div_rn(b1, bsum); b2 = div_rn(b2, bsum);

    const r3_object* obj = &p.objects[oid];
    const uint4 oa = __ldg(reinterpret_cast<const uint4*>(obj) + 5);   // bytes 80..95 : first_index, index_count, material_index, attr[0]
    const uint4 ob = __ldg(reinterpret_cast<const uint4*>(obj) + 6);   // bytes 96..111: attr[1..4]
    const uint4 oc = __ldg(reinterpret_cast<const uint4*>(obj) + 7);   // bytes 112..127: attr[5], enabled
    const uint32_t attr[6] = {oa.w, ob.x, ob.y, ob.z, ob.w, oc.x};
    const uint32_t material_index = oa.z;
    float mv[16];
    {
        const float4* m4 = reinterpret_cast<const float4*>(p.matrices[oid].model_view);
#pragma unroll
        for (int k = 0; k < 4; ++k) { const float4 c4 = __ldg(&m4[k]); mv[4 * k] = c4.x; mv[4 * k + 1] = c4.y; mv[4 * k + 2] = c4.z; mv[4 * k + 3] = c4.w; }
    }
    const float3 iss = make_float3(1.0f / (mv[0] * mv[0] + mv[1] * mv[1] + mv[2] * mv[2]), 1.0f / (mv[4] * mv[4] + mv[5] * mv[5] + mv[6] * mv[6]),
                                   1.0f / (mv[8] * mv[8] + mv[9] * mv[9] + mv[10] * mv[10]));   // math/matrix.wgsl:1-7
    const VsOut v0 = vertex_stage(p, attr, mv, iss, vid0), v1 = vertex_stage(p, attr, mv, iss, vid1), v2 = vertex_stage(p, attr, mv, iss, vid2);
    const float4 vp = make_float4(lerp3_rn(b0, b1, b2, v0.view_position.x, v1.view_position.x, v2.view_position.x),
                                  lerp3_rn(b0, b1, b2, v0.view_position.y, v1.view_position.y, v2.view_position.y),
                                  lerp3_rn(b0, b1, b2, v0.view_position.z, v1.view_position.z, v2.view_position.z),
                                  lerp3_rn(b0, b1, b2, v0.view_position.w, v1.view_position.w, v2.view_position.w));
    const float3 vnormal = make_float3(b0 * v0.normal.x + b1 * v1.normal.x + b2 * v2.normal.x, b0 * v0.normal.y + b1 * v1.normal.y + b2 * v2.normal.y,
                                       b0 * v0.normal.z + b1 * v1.normal.z + b2 * v2.normal.z);
    const float4 vcolor = make_float4(b0 * v0.color.x + b1 * v1.color.x + b2 * v2.color.x, b0 * v0.color.y + b1 * v1.color.y + b2 * v2.color.y,
                                      b0 * v0.color.z + b1 * v1.color.z + b2 * v2.color.z, b0 * v0.color.w + b1 * v1.color.w + b2 * v2.color.w);

    FragIn f;
    f.vp = vp; f.vnormal = vnormal; f.vcolor = vcolor; f.material_index = material_index;
    return f;
}

// what get_pixel_data_inner (opaque.wgsl:203-424) hands to the lighting code
struct PixelInputs { float4 albedo; float3 normal; float ao, perceptual, metallic, reflectance, clear_coat, cc_rough; float3 emissive; };

// get_pixel_data_inner for a material that references textures: texture coordinates + derivatives (R9: forward differences of the
// primitive's own interpolation), tangent frame, every texture slot and layout flag
__device__ __noinline__ void textured_pixel_data(const ShadeParams& p, const r3_material* m, const FragIn& f, const r3_tri_record* tp, uint32_t px, uint32_t py,
                                                 PixelInputs* out) {
    const float4 q0 = __ldg(reinterpret_cast<const float4*>(tp)), q1 = __ldg(reinterpret_cast<const float4*>(tp) + 1), q2 = __ldg(reinterpret_cast<const float4*>(tp) + 2);
    const uint4 q3 = __ldg(reinterpret_cast<const uint4*>(tp) + 3);
    const float3 p0 = make_float3(q0.x, q0.y, q0.z), p1 = make_float3(q0.w, q1.x, q1.y), p2 = make_float3(q1.z, q1.w, q2.x);
    const uint32_t oid = __float_as_uint(q2.y);
    const uint32_t vid[3] = {__float_as_uint(q2.z), __float_as_uint(q2.w), q3.x};
    const r3_object* obj = &p.objects[oid];
    const uint32_t tangent_off = __ldg(&obj->attr_offset[2]), uv_off = __ldg(&obj->attr_offset[3]);
    const uint32_t flags = __ldg(&m->flags);
    const bool nearest = flags & R3_MAT_NEAREST;
    uint32_t tex[10];
#pragma unroll
    for (int k = 0; k < 10; ++k) tex[k] = __ldg(&m->textures[k]);

    // perspective weights at the pixel centre and at the centres of the right / lower neighbours
    float b[3][3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float fx = (float)px + (k == 1 ? 1.5f : 0.5f), fy = (float)py + (k == 2 ? 1.5f : 0.5f);
        const float nx = sub_rn(div_rn(fx, (float)p.width * 0.5f), 1.0f), ny = sub_rn(1.0f, div_rn(fy, (float)p.height * 0.5f));
        const float b0 = cross_term_rn(p1, p2, nx, ny), b1 = cross_term_rn(p2, p0, nx, ny), b2 = cross_term_rn(p0, p1, nx, ny);
        const float sum = add_rn(add_rn(b0, b1), b2);
        b[k][0] = div_rn(b0, sum); b[k][1] = div_rn(b1, sum); b[k][2] = div_rn(b2, sum);
    }
    float uv[3][2] = {{0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}};
    if (uv_off != R3_ATTR_ABSENT) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const uint64_t w = (uint64_t)(uv_off >> 2) + (uint64_t)vid[k] * 2u;
            uv[k][0] = __uint_as_float(mesh_word(p, w)); uv[k][1] = __uint_as_float(mesh_word(p, w + 1));
        }
    }
    const float4 ut0 = __ldg(reinterpret_cast<const float4*>(m->uv_transform0[0])), ut1 = __ldg(reinterpret_cast<const float4*>(m->uv_transform0[1])),
                 ut2 = __ldg(reinterpret_cast<const float4*>(m->uv_transform0[2]));
    float co[3][2];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float u = lerp3_rn(b[k][0], b[k][1], b[k][2], uv[0][0], uv[1][0], uv[2][0]), v = lerp3_rn(b[k][0], b[k][1], b[k][2], uv[0][1], uv[1][1], uv[2][1]);
        co[k][0] = add_rn(add_rn(mul_rn(ut0.x, u), mul_rn(ut1.x, v)), ut2.x);
        co[k][1] = add_rn(add_rn(mul_rn(ut0.y, u), mul_rn(ut1.y, v)), ut2.y);
    }
    TexCoords tc;
    tc.u = co[0][0]; tc.v = co[0][1];
    tc.dudx = sub_rn(co[1][0], co[0][0]); tc.dvdx = sub_rn(co[1][1], co[0][1]); tc.dudy = sub_rn(co[2][0], co[0][0]); tc.dvdy = sub_rn(co[2][1], co[0][1]);

    PixelInputs o;
    const float4 malbedo = __ldg(reinterpret_cast<const float4*>(m->albedo));
    o.albedo = make_float4(0.f, 0.f, 0.f, 1.f);
    if (flags & R3_MAT_ALBEDO_ACTIVE) {
        o.albedo = tex[R3_TEX_ALBEDO] ? texture_sample_grad(p.tt, tex[R3_TEX_ALBEDO], nearest, tc) : make_float4(1.f, 1.f, 1.f, 1.f);
        if (flags & R3_MAT_ALBEDO_BLEND) {
            const float4 vc = (flags & R3_MAT_ALBEDO_VERTEX_SRGB) ? make_float4(srgb_to_linear(f.vcolor.x), srgb_to_linear(f.vcolor.y), srgb_to_linear(f.vcolor.z), f.vcolor.w) : f.vcolor;
            o.albedo = make_float4(o.albedo.x * vc.x, o.albedo.y * vc.y, o.albedo.z * vc.z, o.albedo.w * vc.w);
        }
    }
    o.albedo = make_float4(o.albedo.x * malbedo.x, o.albedo.y * malbedo.y, o.albedo.z * malbedo.z, o.albedo.w * malbedo.w);
    o.normal = f.vnormal;
    if (tex[R3_TEX_NORMAL] && !(flags & R3_MAT_UNLIT)) {                               // opaque.wgsl:244-276
        const float4 t = texture_sample_grad(p.tt, tex[R3_TEX_NORMAL], nearest, tc);
        float3 n;
        if (flags & R3_MAT_BICOMPONENT_NORMAL) {
            const float bx = ((flags & R3_MAT_SWIZZLED_NORMAL) ? t.w : t.x) * 2.0f - 1.0f, by = t.y * 2.0f - 1.0f;
            n = make_float3(bx, by, sqrtf((1.0f - bx * bx) - by * by));
        } else n = normalize3(make_float3(t.x * 2.0f - 1.0f, t.y * 2.0f - 1.0f, t.z * 2.0f - 1.0f));
        if (flags & R3_MAT_YDOWN_NORMAL) n.y = -n.y;
        // vs_out.tangent = normalize(mv3 * (inv_scale_sq * tangent)) per vertex, interpolated (opaque.wgsl:128)
        float mv[12];
        {
            const float4* m4 = reinterpret_cast<const float4*>(p.matrices[oid].model_view);
#pragma unroll
            for (int k = 0; k < 3; ++k) { const float4 c4 = __ldg(&m4[k]); mv[4 * k] = c4.x; mv[4 * k + 1] = c4.y; mv[4 * k + 2] = c4.z; mv[4 * k + 3] = c4.w; }
        }
        const float3 iss = make_float3(1.0f / (mv[0] * mv[0] + mv[1] * mv[1] + mv[2] * mv[2]), 1.0f / (mv[4] * mv[4] + mv[5] * mv[5] + mv[6] * mv[6]),
                                       1.0f / (mv[8] * mv[8] + mv[9] * mv[9] + mv[10] * mv[10]));
        float3 vt[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            vt[k] = make_float3(0.f, 0.f, 0.f);
            if (tangent_off != R3_ATTR_ABSENT) {
                const float3 t3 = fetch3(p, tangent_off, vid[k]);
                const float3 st = make_float3(iss.x * t3.x, iss.y * t3.y, iss.z * t3.z);
                vt[k] = normalize3(make_float3(mv[0] * st.x + mv[4] * st.y + mv[8] * st.z, mv[1] * st.x + mv[5] * st.y + mv[9] * st.z, mv[2] * st.x + mv[6] * st.y + mv[10] * st.z));
            }
        }
        const float3 vtan = make_float3(b[0][0] * vt[0].x + b[0][1] * vt[1].x + b[0][2] * vt[2].x, b[0][0] * vt[0].y + b[0][1] * vt[1].y + b[0][2] * vt[2].y,
                                        b[0][0] * vt[0].z + b[0][1] * vt[1].z + b[0][2] * vt[2].z);
        const float3 nn = normalize3(f.vnormal), tn = normalize3(vtan);
        const float3 bt = make_float3(nn.y * tn.z - tn.y * nn.z, nn.z * tn.x - tn.z * nn.x, nn.x * tn.y - tn.x * nn.y);
        o.normal = make_float3(tn.x * n.x + bt.x * n.y + nn.x * n.z, tn.y * n.x + bt.y * n.y + nn.y * n.z, tn.z * n.x + bt.z * n.y + nn.z * n.z);
    }
    const float4 mA = __ldg(reinterpret_cast<const float4*>(m->emissive));        // emissive.xyz, roughness
    const float4 mB = __ldg(reinterpret_cast<const float4*>(&m->metallic));       // metallic, reflectance, clear_coat, clear_coat_roughness
    const float m_ao = __ldg(&m->ambient_occlusion);
    o.ao = m_ao; o.perceptual = mA.w; o.metallic = mB.x;
    if (!(flags & R3_MAT_UNLIT)) {
        if (flags & R3_MAT_AOMR_COMBINED) {                                            // opaque.wgsl:280-295
            if (tex[R3_TEX_ROUGHNESS]) { const float4 t = texture_sample_grad(p.tt, tex[R3_TEX_ROUGHNESS], nearest, tc); o.ao = m_ao * t.x; o.perceptual = mA.w * t.y; o.metallic = mB.x * t.z; }
        } else if (flags & R3_MAT_AOMR_BW_SPLIT) {
            if (tex[R3_TEX_ROUGHNESS]) o.perceptual = mA.w * texture_sample_grad(p.tt, tex[R3_TEX_ROUGHNESS], nearest, tc).x;
            if (tex[R3_TEX_METALLIC]) o.metallic = mB.x * texture_sample_grad(p.tt, tex[R3_TEX_METALLIC], nearest, tc).x;
            if (tex[R3_TEX_AMBIENT_OCCLUSION]) o.ao = m_ao * texture_sample_grad(p.tt, tex[R3_TEX_AMBIENT_OCCLUSION], nearest, tc).x;
        } else {
            if (tex[R3_TEX_ROUGHNESS]) {
                const float4 t = texture_sample_grad(p.tt, tex[R3_TEX_ROUGHNESS], nearest, tc);
                const bool sw = flags & R3_MAT_AOMR_SWIZZLED_SPLIT;
                o.perceptual = mA.w * (sw ? t.y : t.x); o.metallic = mB.x * (sw ? t.z : t.y);
            }
            if (tex[R3_TEX_AMBIENT_OCCLUSION]) o.ao = m_ao * texture_sample_grad(p.tt, tex[R3_TEX_AMBIENT_OCCLUSION], nearest, tc).x;
        }
        o.reflectance = mB.y;
        if (tex[R3_TEX_REFLECTANCE]) o.reflectance = mB.y * texture_sample_grad(p.tt, tex[R3_TEX_REFLECTANCE], nearest, tc).x;
        o.clear_coat = mB.z; o.cc_rough = mB.w;
        if (flags & R3_MAT_CC_GLTF_COMBINED) {
            if (tex[R3_TEX_CLEAR_COAT]) { const float4 t = texture_sample_grad(p.tt, tex[R3_TEX_CLEAR_COAT], nearest, tc); o.clear_coat = mB.z * t.x; o.cc_rough = mB.w * t.y; }
        } else {
            if (tex[R3_TEX_CLEAR_COAT]) o.clear_coat = mB.z * texture_sample_grad(p.tt, tex[R3_TEX_CLEAR_COAT], nearest, tc).x;
            if (tex[R3_TEX_CLEAR_COAT_ROUGHNESS]) {
                const float4 t = texture_sample_grad(p.tt, tex[R3_TEX_CLEAR_COAT_ROUGHNESS], nearest, tc);
                o.cc_rough = mB.w * ((flags & R3_MAT_CC_GLTF_SPLIT) ? t.y : t.x);
            }
        }
        o.emissive = make_float3(mA.x, mA.y, mA.z);
        if (tex[R3_TEX_EMISSIVE]) { const float4 t = texture_sample_grad(p.tt, tex[R3_TEX_EMISSIVE], nearest, tc); o.emissive = make_float3(mA.x * t.x, mA.y * t.y, mA.z * t.z); }
    }
    *out = o;
}

// fs_main (opaque.wgsl:470-551).  `mask` lists the point lights that can reach the fragment (a conservative superset is fine:
// every listed light still takes the exact per-fragment range test below).
// skybox.wgsl::fs_main (rend3-routine/shaders/src/skybox.wgsl:24-36) at the centre of pixel (px, py); cube sampling by rule R10 of the
// oracle (face + (s, t) by the major axis, forward-difference derivatives on the same face, trilinear, texels clamped to the face)
__device__ __forceinline__ float3 skybox_direction(const ShadeParams& p, float fx, float fy) {
    const float cx = sub_rn(div_rn(fx, (float)p.width * 0.5f), 1.0f), cy = sub_rn(1.0f, div_rn(fy, (float)p.height * 0.5f));
    const float4 wu = mat_vec_rn(p.inv_origin_view_proj, cx, cy, 1.0f, 1.0f);
    const float wx = div_rn(wu.x, wu.w), wy = div_rn(wu.y, wu.w), wz = div_rn(wu.z, wu.w);
    const float len = sqrtf(add_rn(add_rn(mul_rn(wx, wx), mul_rn(wy, wy)), mul_rn(wz, wz)));
    return make_float3(div_rn(wx, len), div_rn(wy, len), div_rn(wz, len));
}
__device__ __forceinline__ float2 cube_face_coords(const float3 d, int face) {
    float sc, tc, ma;
    switch (face) {
        case 0: sc = -d.z; tc = -d.y; ma = fabsf(d.x); break;
        case 1: sc = d.z; tc = -d.y; ma = fabsf(d.x); break;
        case 2: sc = d.x; tc = d.z; ma = fabsf(d.y); break;
        case 3: sc = d.x; tc = -d.z; ma = fabsf(d.y); break;
        case 4: sc = d.x; tc = -d.y; ma = fabsf(d.z); break;
        default: sc = -d.x; tc = -d.y; ma = fabsf(d.z); break;
    }
    return make_float2(mul_rn(0.5f, add_rn(div_rn(sc, ma), 1.0f)), mul_rn(0.5f, add_rn(div_rn(tc, ma), 1.0f)));
}
__device__ __noinline__ float4 skybox_at_pixel(const ShadeParams& p, uint32_t px, uint32_t py) {
    const float3 d0 = skybox_direction(p, (float)px + 0.5f, (float)py + 0.5f);
    const float3 dx = skybox_direction(p, (float)px + 1.5f, (float)py + 0.5f), dy = skybox_direction(p, (float)px + 0.5f, (float)py + 1.5f);
    const float ax = fabsf(d0.x), ay = fabsf(d0.y), az = fabsf(d0.z);
    int face;
    if (ax >= ay && ax >= az) face = d0.x > 0.0f ? 0 : 1;
    else if (ay >= az) face = d0.y > 0.0f ? 2 : 3;
    else face = d0.z > 0.0f ? 4 : 5;
    const float2 st = cube_face_coords(d0, face), stx = cube_face_coords(dx, face), sty = cube_face_coords(dy, face);
    TexCoords tc;
    tc.u = st.x; tc.v = st.y; tc.dudx = sub_rn(stx.x, st.x); tc.dvdx = sub_rn(stx.y, st.y); tc.dudy = sub_rn(sty.x, st.x); tc.dvdy = sub_rn(sty.y, st.y);
    r3_texture_desc fd = p.sky_desc;
    const unsigned long long bpp = fd.format == R3_TEXFMT_RGBA32_FLOAT ? 16ull : 4ull;
    unsigned long long face_bytes = 0;
    for (uint32_t l = 0; l < fd.mip_count; ++l) { const unsigned long long w = max(fd.width >> l, 1u); face_bytes += w * w * bpp; }
    fd.byte_offset += (unsigned long long)face * face_bytes;
    const float4 t = sample_grad_desc(p.sky, fd, false, tc);
    return make_float4(t.x, t.y, t.z, 1.0f);
}

// TEX = the context holds a texture table: kernels are instantiated with and without the texture path, so that scenes without
// textures keep the register budget (80 instead of 128 on sm_90a) of the lean kernel.
template <bool TEX>
__device__ __forceinline__ float4 shade_inputs(const ShadeParams& p, const DirPrep* __restrict__ s_dir, const PointPrep* __restrict__ s_point, const FragIn& f,
                                               const LightMask& mask, const r3_tri_record* tp, uint32_t px, uint32_t py, uint32_t* lights_evaluated = nullptr) {
    const float4 vp = f.vp; const float4 vcolor = f.vcolor; const uint32_t material_index = f.material_index;
    float3 vnormal = f.vnormal;
    const r3_material* m = &p.materials[material_index < p.n_materials ? material_index : 0u];
    const float4 malbedo = __ldg(reinterpret_cast<const float4*>(m->albedo));
    float4 mA = __ldg(reinterpret_cast<const float4*>(m->emissive));              // emissive.xyz, roughness
    float4 mB = __ldg(reinterpret_cast<const float4*>(&m->metallic));             // metallic, reflectance, clear_coat, clear_coat_roughness
    float4 mC = __ldg(reinterpret_cast<const float4*>(&m->anisotropy));           // anisotropy, ambient_occlusion, alpha_cutout, flags
    const uint32_t flags = __float_as_uint(mC.w);
    float4 albedo = make_float4(0.f, 0.f, 0.f, 1.f);
    const uint4 ta = __ldg(reinterpret_cast<const uint4*>(m->textures)), tb = __ldg(reinterpret_cast<const uint4*>(m->textures) + 1);
    const uint2 tc2 = __ldg(reinterpret_cast<const uint2*>(m->textures) + 4);
    if (TEX && (ta.x | ta.y | ta.z | ta.w | tb.x | tb.y | tb.z | tb.w | tc2.x | tc2.y) != 0u) {
        // the material references textures: get_pixel_data_inner out of line, results funnelled into the same variables
        PixelInputs pi;
        textured_pixel_data(p, m, f, tp, px, py, &pi);
        albedo = pi.albedo; vnormal = pi.normal;
        mA = make_float4(pi.emissive.x, pi.emissive.y, pi.emissive.z, pi.perceptual);
        mB = make_float4(pi.metallic, pi.reflectance, pi.clear_coat, pi.cc_rough);
        mC.y = pi.ao;
    } else {
        // get_pixel_data_inner for untextured materials (opaque.wgsl:203-424)
        if (flags & R3_MAT_ALBEDO_ACTIVE) {
            albedo = make_float4(1.f, 1.f, 1.f, 1.f);
            if (flags & R3_MAT_ALBEDO_BLEND) {
                if (flags & R3_MAT_ALBEDO_VERTEX_SRGB) albedo = make_float4(srgb_to_linear(vcolor.x), srgb_to_linear(vcolor.y), srgb_to_linear(vcolor.z), vcolor.w);
                else albedo = vcolor;
            }
        }
        albedo = make_float4(albedo.x * malbedo.x, albedo.y * malbedo.y, albedo.z * malbedo.z, albedo.w * malbedo.w);
    }
    if (flags & R3_MAT_UNLIT) {
        return albedo;                                                             // opaque.wgsl:476-478
    } else {
        Pixel pxl;
        pxl.normal = normalize3(vnormal);
        const float ao = mC.y, metallic = mB.x, reflectance = mB.y, clear_coat = mB.z, cc_rough = mB.w;
        float perceptual = mA.w;
        const float om = 1.0f - metallic;
        const float inv_pi = 1.0f / R3_PI;
        pxl.diffuse_pi = make_float3(albedo.x * om * inv_pi, albedo.y * om * inv_pi, albedo.z * om * inv_pi);
        const float rterm = (0.16f * reflectance * reflectance) * om;
        pxl.f0 = make_float3(albedo.x * metallic + rterm, albedo.y * metallic + rterm, albedo.z * metallic + rterm);
        if (clear_coat != 0.0f) {
            const float base = fmaxf(perceptual, cc_rough);
            perceptual = perceptual * (1.0f - clear_coat) + base * clear_coat;
        }
        pxl.roughness = perceptual * perceptual;
        pxl.f90 = saturate((pxl.f0.x + pxl.f0.y + pxl.f0.z) * 16.5f);
        const float3 nvp = normalize3(make_float3(vp.x, vp.y, vp.z));
        const float3 v = make_float3(-nvp.x, -nvp.y, -nvp.z);
        const float nov = fabsf(dot3(pxl.normal, v)) + 0.00001f;
        float3 color = make_float3(mA.x, mA.y, mA.z);
        for (uint32_t i = 0; i < p.n_dir; ++i) {                                   // opaque.wgsl:487-522
            const DirPrep& L = i < MAX_SMEM_DIR ? s_dir[i] : p.dir[i];
            const float4 sn = mat_vec_rn(L.lm, vp.x, vp.y, vp.z, vp.w);
            const float snx = sn.x, sny = sn.y, snz = sn.z;
            const float flx = add_rn(mul_rn(snx, 0.5f), 0.5f), fly = add_rn(mul_rn(sny, 0.5f), 0.5f), locy = sub_rn(1.0f, fly);
            float tlx = L.offset[0], tly = L.offset[1], trx = add_rn(tlx, L.size[0]), try_ = add_rn(tly, L.size[1]);
            const float cu = add_rn(mul_rn(tlx, sub_rn(1.0f, flx)), mul_rn(trx, flx)), cv = add_rn(mul_rn(tly, sub_rn(1.0f, locy)), mul_rn(try_, locy));   // mix
            const float bx = mul_rn(L.inv_res[0], 1.5f), by = mul_rn(L.inv_res[1], 1.5f);
            tlx = add_rn(tlx, bx); tly = add_rn(tly, by); trx = sub_rn(trx, bx); try_ = sub_rn(try_, by);
            float shadow = 1.0f;
            if ((flx >= tlx || fly >= tly) && (flx <= trx || fly <= try_) && snz >= 0.0f && snz <= 1.0f)   // literal any() quirk (opaque.wgsl:509-514)
                shadow = shadow_pcf5(p, cu, cv, snz);
            const float3 s = surface_shading(make_float3(L.l[0], L.l[1], L.l[2]), make_float3(L.color[0], L.color[1], L.color[2]), pxl, v, nov, shadow * ao);
            color.x += s.x; color.y += s.y; color.z += s.z;
        }
        uint32_t n_eval = p.n_dir;
        // loaded here, where the loop starts, rather than kept live from the kernel's staging: the register budget stays as it was
        const uint32_t n_point = *p.point_count;
        const uint32_t n_smem_point = min(n_point, (uint32_t)MAX_SMEM_POINT);
        for (uint32_t base = 0; base < n_point; base += 32u) {                     // opaque.wgsl:524-546, ascending light order
            uint32_t m = base < n_smem_point ? mask.w[base >> 5] : 0xFFFFFFFFu;
            if (n_point - base < 32u) m &= (1u << (n_point - base)) - 1u;
            while (m) {
                const uint32_t i = base + (uint32_t)__ffs(m) - 1u;
                m &= m - 1u;
                const PointPrep& L = i < MAX_SMEM_POINT ? s_point[i] : p.point[i];
                const float3 delta = make_float3(L.pos[0] - vp.x, L.pos[1] - vp.y, L.pos[2] - vp.z);
                const float d2 = dot3(delta, delta);
                // att = (1 - s^2)^2 / (1 + s^2) with s = saturate(d / radius) is exactly 0 at and beyond a positive radius; a
                // negative or NaN radius saturates d / radius to 0, so that light reaches every fragment with att = 1
                if (L.radius > 0.0f && d2 >= L.radius * L.radius && pxl.roughness > 0.0f) continue;
                const float inv_d = rsqrtf(d2), d = d2 * inv_d;
                const float sdist = saturate(d * rcp_approx(L.radius)), s2 = sdist * sdist, inv_s2 = 1.0f - s2;
                const float att = inv_s2 * inv_s2 * rcp_approx(1.0f + s2);
                const float3 s = surface_shading(make_float3(delta.x * inv_d, delta.y * inv_d, delta.z * inv_d),
                                                 make_float3(L.color[0] * att, L.color[1] * att, L.color[2] * att), pxl, v, nov, ao);
                color.x += fmaxf(s.x, 0.0f); color.y += fmaxf(s.y, 0.0f); color.z += fmaxf(s.z, 0.0f);
                n_eval++;
            }
        }
        if (lights_evaluated) *lights_evaluated = n_eval;
        return make_float4(fmaxf(p.ambient[0] * albedo.x, color.x), fmaxf(p.ambient[1] * albedo.y, color.y), fmaxf(p.ambient[2] * albedo.z, color.z),
                          fmaxf(p.ambient[3] * albedo.w, albedo.w));
    }
}

// vs_main + fs_main for triangle record `tp` at pixel (px, py), every point light considered
template <bool TEX>
__device__ __forceinline__ float4 shade_fragment(const ShadeParams& p, const DirPrep* __restrict__ s_dir, const PointPrep* __restrict__ s_point,
                                                 const r3_tri_record* tp, uint32_t px, uint32_t py) {
    LightMask all;
#pragma unroll
    for (int k = 0; k < MAX_SMEM_POINT / 32; ++k) all.w[k] = 0xFFFFFFFFu;
    return shade_inputs<TEX>(p, s_dir, s_point, fragment_inputs(p, tp, px, py), all, tp, px, py);
}

template <int SAMPLES, bool TEX>
__global__ void __launch_bounds__(256) resolve_kernel(const __grid_constant__ ShadeParams p) {
    __shared__ DirPrep s_dir[MAX_SMEM_DIR];
    __shared__ PointPrep s_point[MAX_SMEM_POINT];
    // the point-light count, loaded once for the staging and the tile test (shade_inputs reads the same word for its loop)
    const uint32_t n_point = *p.point_count;
    {
        const uint32_t nd = min(p.n_dir, (uint32_t)MAX_SMEM_DIR) * 32u, np = min(n_point, (uint32_t)MAX_SMEM_POINT) * 8u;
        const float* gd = reinterpret_cast<const float*>(p.dir); const float* gp = reinterpret_cast<const float*>(p.point);
        float* sd = reinterpret_cast<float*>(s_dir); float* sp = reinterpret_cast<float*>(s_point);
        for (uint32_t i = threadIdx.x; i < nd; i += blockDim.x) sd[i] = gd[i];
        for (uint32_t i = threadIdx.x; i < np; i += blockDim.x) sp[i] = gp[i];
        __syncthreads();
    }
    // CTA = 32 x 8 pixels: a warp is 32 consecutive pixels of one row (coalesced key reads / colour writes)
    const uint32_t px = blockIdx.x * 32u + (threadIdx.x & 31u), py = p.row_begin + blockIdx.y * 8u + (threadIdx.x >> 5);
    const bool in_target = px < p.width && py < p.row_end;
    const size_t pi = (size_t)py * p.width + px;
    float4 out;
    float depth;
    uint32_t n_shaded = 0, n_lights = 0;   // n_lights: surface_shading evaluations of this fragment (statistics: flops of the pass)
    if (SAMPLES == 1) {
        // tiled light culling: the CTA bounds the view-space positions of its fragments, then 32 lights per warp are tested
        // against that box; fragments only visit the survivors (in ascending light order, so the sums are unchanged).  A light
        // whose sphere misses the box by a 0.1% margin is beyond its radius for every fragment of the tile, where its
        // attenuation is exactly 0 — unless a roughness-0 material needs the reference's 0 * inf = NaN (then nothing is culled).
        __shared__ float s_box[8][6];
        __shared__ uint32_t s_mask[MAX_SMEM_POINT / 32];
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        const unsigned long long key = in_target ? p.vis[pi] : 0ull;
        const uint32_t rec = (uint32_t)(key & 0x7FFFFFFFull), pass = (uint32_t)((key >> 31) & 1ull);
        const bool covered = in_target && rec != 0u && rec <= (pass ? p.n_tris1 : p.n_tris0);
        FragIn f;
        f.vp = make_float4(0.f, 0.f, 0.f, 1.f); f.vnormal = make_float3(0.f, 0.f, 1.f); f.vcolor = make_float4(1.f, 1.f, 1.f, 1.f); f.material_index = 0u;
        bool mirror = false;
        if (covered) {
            f = fragment_inputs(p, (pass ? p.tris1 : p.tris0) + (rec - 1u), px, py);
            const r3_material* m = &p.materials[f.material_index < p.n_materials ? f.material_index : 0u];
            // pixel.roughness as shade_inputs derives it (opaque.wgsl:392-399); anything not safely positive disables the culling
            float perceptual = __ldg(&m->roughness);
            const float cc = __ldg(&m->clear_coat);
            if (cc != 0.0f) perceptual = perceptual * (1.0f - cc) + fmaxf(perceptual, __ldg(&m->clear_coat_roughness)) * cc;
            mirror = !(perceptual * perceptual > 1.0e-30f);
        }
        const bool no_cull = __syncthreads_or(mirror ? 1 : 0) != 0;
        if (n_point != 0u && !no_cull) {
            const float big = 3.0e38f;
            float lo[3] = {covered ? f.vp.x : big, covered ? f.vp.y : big, covered ? f.vp.z : big};
            float hi[3] = {covered ? f.vp.x : -big, covered ? f.vp.y : -big, covered ? f.vp.z : -big};
#pragma unroll
            for (int a = 0; a < 3; ++a)
#pragma unroll
                for (int sft = 16; sft > 0; sft >>= 1) {
                    lo[a] = fminf(lo[a], __shfl_xor_sync(0xFFFFFFFFu, lo[a], sft));
                    hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xFFFFFFFFu, hi[a], sft));
                }
            if (lane == 0) { s_box[warp][0] = lo[0]; s_box[warp][1] = lo[1]; s_box[warp][2] = lo[2]; s_box[warp][3] = hi[0]; s_box[warp][4] = hi[1]; s_box[warp][5] = hi[2]; }
            __syncthreads();
            const uint32_t n_smem_point = min(n_point, (uint32_t)MAX_SMEM_POINT);
            if (threadIdx.x < MAX_SMEM_POINT) {
                bool reach = false;
                if (threadIdx.x < n_smem_point) {
                    float blo[3] = {big, big, big}, bhi[3] = {-big, -big, -big};
#pragma unroll
                    for (int w = 0; w < 8; ++w)
#pragma unroll
                        for (int a = 0; a < 3; ++a) { blo[a] = fminf(blo[a], s_box[w][a]); bhi[a] = fmaxf(bhi[a], s_box[w][3 + a]); }
                    const PointPrep& L = s_point[threadIdx.x];
                    float d2 = 0.0f;
#pragma unroll
                    for (int a = 0; a < 3; ++a) {
                        const float c = L.pos[a], e = fmaxf(fmaxf(blo[a] - c, c - bhi[a]), 0.0f);   // distance to the box along this axis
                        d2 += e * e;
                    }
                    // only a positive radius bounds a light (see shade_inputs); a NaN radius fails every comparison
                    reach = blo[0] <= bhi[0] && (!(L.radius > 0.0f) || d2 <= L.radius * L.radius * 1.001f);
                }
                const uint32_t bal = __ballot_sync(0xFFFFFFFFu, reach);
                if (lane == 0) s_mask[warp] = bal;
            }
            __syncthreads();
        }
        LightMask mask;
#pragma unroll
        for (int k = 0; k < MAX_SMEM_POINT / 32; ++k) mask.w[k] = (n_point != 0u && !no_cull) ? s_mask[k] : 0xFFFFFFFFu;
        if (!in_target) return;
        out = make_float4(p.clear[0], p.clear[1], p.clear[2], p.clear[3]);
        if (covered) { out = shade_inputs<TEX>(p, s_dir, s_point, f, mask, (pass ? p.tris1 : p.tris0) + (rec - 1u), px, py, &n_lights); n_shaded = 1; }
        depth = __uint_as_float((uint32_t)(key >> 32));
    } else {
        if (!in_target) return;
        // SampleCount::Four: a primitive is shaded once per pixel for all the samples it owns; the rgba16f samples are box-filtered
        // ((s0 + s1) + (s2 + s3)) * 0.25 like the resolve attachment (base.rs:245-255); depth resolves to the MIN over the samples
        unsigned long long keys[4];
        float4 col[4];
        float4 sky = make_float4(0.f, 0.f, 0.f, 1.f);
        bool have_sky = false;
        depth = 1.0f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            keys[k] = p.vis[pi * 4u + k];
            depth = fminf(depth, __uint_as_float((uint32_t)(keys[k] >> 32)));
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t id = (uint32_t)keys[k], rec = id & 0x7FFFFFFFu, pass = id >> 31;
            col[k] = make_float4(p.clear[0], p.clear[1], p.clear[2], p.clear[3]);
            if (p.sky.texels && (uint32_t)(keys[k] >> 32) == 0u) {
                // SkyboxRoutine (skybox.rs:80-110, base.rs:175): depth 0, GreaterEqual -> every sample still at the clear depth
                if (!have_sky) { sky = skybox_at_pixel(p, px, py); have_sky = true; }
                col[k] = sky;
            } else if (rec != 0u && rec <= (pass ? p.n_tris1 : p.n_tris0)) {
                int reuse = -1;
                for (int q = 0; q < k; ++q) if ((uint32_t)keys[q] == id && (uint32_t)(keys[q] >> 32) != 0u && reuse < 0) reuse = q;
                if (reuse >= 0) col[k] = col[reuse];
                else { col[k] = shade_fragment<TEX>(p, s_dir, s_point, (pass ? p.tris1 : p.tris0) + (rec - 1u), px, py); n_shaded++; }
            }
            // each sample lives in the rgba16f multisampled target
            col[k] = make_float4(__half2float(__float2half_rn(col[k].x)), __half2float(__float2half_rn(col[k].y)), __half2float(__float2half_rn(col[k].z)),
                                 __half2float(__float2half_rn(col[k].w)));
        }
        out = make_float4(((col[0].x + col[1].x) + (col[2].x + col[3].x)) * 0.25f, ((col[0].y + col[1].y) + (col[2].y + col[3].y)) * 0.25f,
                          ((col[0].z + col[1].z) + (col[2].z + col[3].z)) * 0.25f, ((col[0].w + col[1].w) + (col[2].w + col[3].w)) * 0.25f);
    }
    if (p.hdr32) p.hdr32[pi] = out;   // pre-rounding shading result: only when the parity target is enabled (r3_set_parity_target)
    const __half2 h01 = __floats2half2_rn(out.x, out.y), h23 = __floats2half2_rn(out.z, out.w);
    p.hdr16[pi] = make_uint2(*reinterpret_cast<const uint32_t*>(&h01), *reinterpret_cast<const uint32_t*>(&h23));
    p.depth[pi] = depth;
    const uint32_t active = __activemask();
    const uint32_t total = __reduce_add_sync(active, n_shaded), total_lights = __reduce_add_sync(active, n_lights);
    if ((threadIdx.x & 31u) == (uint32_t)(__ffs(active) - 1) && total) { atomicAdd(&p.stats[2], (unsigned long long)total); atomicAdd(&p.stats[6], (unsigned long long)total_lights); }
}


__device__ __forceinline__ float f16_round(float v) { return __half2float(__float2half_rn(v)); }

// pbr_forward_rendering_transparent (base.rs:181,450-466), second half: apply the collected fragments of a pixel in draw
// order (= record order: non-atomic regions keep their slots, cull.wgsl:374-380).  Per sample: depth test GreaterEqual with
// depth write (forward.rs:331-365), then BlendState::ALPHA_BLENDING (pbr/routine.rs:115-118) into the rgba16f target —
// rule R8 of the oracle: rgb' = (src.rgb * src.a) + (dst.rgb * (1 - src.a)), a' = src.a + dst.a * (1 - src.a), rounded to
// half precision after every primitive.  A primitive is shaded once per pixel for all the samples it covers (R7).
template <int SAMPLES, bool TEX>
__global__ void __launch_bounds__(256) blend_apply_kernel(const __grid_constant__ ShadeParams p) {
    __shared__ DirPrep s_dir[MAX_SMEM_DIR];
    __shared__ PointPrep s_point[MAX_SMEM_POINT];
    const uint32_t n_point = *p.point_count;   // for the staging (shade_inputs reads the same word for its loop)
    {
        const uint32_t nd = min(p.n_dir, (uint32_t)MAX_SMEM_DIR) * 32u, np = min(n_point, (uint32_t)MAX_SMEM_POINT) * 8u;
        const float* gd = reinterpret_cast<const float*>(p.dir); const float* gp = reinterpret_cast<const float*>(p.point);
        float* sd = reinterpret_cast<float*>(s_dir); float* sp = reinterpret_cast<float*>(s_point);
        for (uint32_t i = threadIdx.x; i < nd; i += blockDim.x) sd[i] = gd[i];
        for (uint32_t i = threadIdx.x; i < np; i += blockDim.x) sp[i] = gp[i];
        __syncthreads();
    }
    const uint32_t px = blockIdx.x * 32u + (threadIdx.x & 31u), py = p.row_begin + blockIdx.y * 8u + (threadIdx.x >> 5);
    if (px >= p.width || py >= p.row_end) return;
    const size_t pi = (size_t)py * p.width + px;
    uint32_t head[SAMPLES];
    bool any = false;
#pragma unroll
    for (int k = 0; k < SAMPLES; ++k) { head[k] = p.frag_heads[pi * SAMPLES + k]; any |= head[k] != 0u; }
    if (!any) return;

    // destination samples as the colour target holds them (rgba16f) + their depth
    float4 dst[SAMPLES];
    uint32_t zdst[SAMPLES];
    if (SAMPLES == 1) {
        const uint2 h = p.hdr16[pi];
        const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&h.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&h.y));
        dst[0] = make_float4(a.x, a.y, b.x, b.y);
        zdst[0] = (uint32_t)(p.vis[pi] >> 32);
    } else {
        // the multisampled target is not kept after the box filter: the opaque samples of the (few) pixels that carry
        // transparent fragments are shaded again, exactly as resolve_kernel<4> did
        uint32_t ids[SAMPLES];
#pragma unroll
        for (int k = 0; k < SAMPLES; ++k) {
            const unsigned long long key = p.vis[pi * SAMPLES + k];
            ids[k] = (uint32_t)key; zdst[k] = (uint32_t)(key >> 32);
            const uint32_t rec = ids[k] & 0x7FFFFFFFu, pass = ids[k] >> 31;
            float4 col = make_float4(p.clear[0], p.clear[1], p.clear[2], p.clear[3]);
            if (p.sky.texels && zdst[k] == 0u) col = skybox_at_pixel(p, px, py);
            else if (rec != 0u && rec <= (pass ? p.n_tris1 : p.n_tris0)) {
                int reuse = -1;
                for (int q = 0; q < k; ++q) if (ids[q] == ids[k] && zdst[q] != 0u && reuse < 0) reuse = q;
                if (reuse >= 0) col = dst[reuse];
                else col = shade_fragment<TEX>(p, s_dir, s_point, (pass ? p.tris1 : p.tris0) + (rec - 1u), px, py);
            }
            dst[k] = make_float4(f16_round(col.x), f16_round(col.y), f16_round(col.z), f16_round(col.w));
        }
    }

    uint32_t last = 0u, n_blended = 0u;
    for (;;) {
        // next primitive in draw order over all the samples of the pixel
        uint32_t next = 0xFFFFFFFFu;
#pragma unroll
        for (int k = 0; k < SAMPLES; ++k)
            for (uint32_t n = head[k]; n != 0u;) {
                const uint4 node = __ldg(&p.frag_nodes[n - 1u]);
                if (node.x > last && node.x < next) next = node.x;
                n = node.z;
            }
        if (next == 0xFFFFFFFFu) break;
        last = next;
        if (next > p.n_tris2) continue;
        bool shaded = false;
        float4 src = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int k = 0; k < SAMPLES; ++k) {
            uint32_t z = 0u; bool found = false;
            for (uint32_t n = head[k]; n != 0u && !found;) {
                const uint4 node = __ldg(&p.frag_nodes[n - 1u]);
                if (node.x == next) { z = node.y; found = true; }
                n = node.z;
            }
            if (!found || z < zdst[k]) continue;   // GreaterEqual (reverse-Z bits order like the floats)
            zdst[k] = z;                            // depth write
            if (!shaded) { src = shade_fragment<TEX>(p, s_dir, s_point, p.tris2 + (next - 1u), px, py); shaded = true; }
            const float inv_a = sub_rn(1.0f, src.w);
            dst[k] = make_float4(f16_round(add_rn(mul_rn(src.x, src.w), mul_rn(dst[k].x, inv_a))), f16_round(add_rn(mul_rn(src.y, src.w), mul_rn(dst[k].y, inv_a))),
                                 f16_round(add_rn(mul_rn(src.z, src.w), mul_rn(dst[k].z, inv_a))), f16_round(add_rn(src.w, mul_rn(dst[k].w, inv_a))));
            n_blended++;
        }
    }
    if (n_blended) {
        float4 out;
        float depth;
        if (SAMPLES == 1) { out = dst[0]; depth = __uint_as_float(zdst[0]); }
        else {
            out = make_float4(((dst[0].x + dst[1 % SAMPLES].x) + (dst[2 % SAMPLES].x + dst[3 % SAMPLES].x)) * 0.25f,
                              ((dst[0].y + dst[1 % SAMPLES].y) + (dst[2 % SAMPLES].y + dst[3 % SAMPLES].y)) * 0.25f,
                              ((dst[0].z + dst[1 % SAMPLES].z) + (dst[2 % SAMPLES].z + dst[3 % SAMPLES].z)) * 0.25f,
                              ((dst[0].w + dst[1 % SAMPLES].w) + (dst[2 % SAMPLES].w + dst[3 % SAMPLES].w)) * 0.25f);
            depth = 1.0f;
#pragma unroll
            for (int k = 0; k < SAMPLES; ++k) depth = fminf(depth, __uint_as_float(zdst[k]));
        }
        if (p.hdr32) p.hdr32[pi] = out;
        const __half2 h01 = __floats2half2_rn(out.x, out.y), h23 = __floats2half2_rn(out.z, out.w);
        p.hdr16[pi] = make_uint2(*reinterpret_cast<const uint32_t*>(&h01), *reinterpret_cast<const uint32_t*>(&h23));
        p.depth[pi] = depth;
        atomicAdd(&p.stats[3], (unsigned long long)n_blended);
    }
}

// SkyboxRoutine for single-sampled targets: a pass of its own after the opaque resolve (base.rs:175), so that resolve_kernel<1, .>
// keeps its register budget — every pixel still at the clear depth takes the cube-map colour
__global__ void __launch_bounds__(256) skybox_kernel(const __grid_constant__ ShadeParams p) {
    const uint32_t px = blockIdx.x * 32u + (threadIdx.x & 31u), py = p.row_begin + blockIdx.y * 8u + (threadIdx.x >> 5);
    if (px >= p.width || py >= p.row_end) return;
    const size_t pi = (size_t)py * p.width + px;
    if ((uint32_t)(p.vis[pi] >> 32) != 0u) return;
    const float4 out = skybox_at_pixel(p, px, py);
    if (p.hdr32) p.hdr32[pi] = out;
    const __half2 h01 = __floats2half2_rn(out.x, out.y), h23 = __floats2half2_rn(out.z, out.w);
    p.hdr16[pi] = make_uint2(*reinterpret_cast<const uint32_t*>(&h01), *reinterpret_cast<const uint32_t*>(&h23));
}

// light prep: one thread per light (opaque.wgsl:491,519,528 hoisted out of the fragment loop).  The grid covers the point lights'
// capacity; the buffer's count (@0 of `point_buf`, at most that capacity) says how many exist this frame.
__global__ void light_prep_kernel(const r3_directional_light* dir, uint32_t n_dir, const uint8_t* point_buf,
                                  const __grid_constant__ r3_frame_uniforms u, DirPrep* out_dir, PointPrep* out_point) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t n_point = *reinterpret_cast<const uint32_t*>(point_buf);
    const r3_point_light* point = reinterpret_cast<const r3_point_light*>(point_buf + 16);
    if (i < n_dir) {
        const r3_directional_light L = dir[i];
        DirPrep o;
        for (int j = 0; j < 4; ++j) {   // light.view_proj * uniforms.inv_view, column j
            const float4 c4 = mat_vec_rn(L.view_proj, u.inv_view[4 * j], u.inv_view[4 * j + 1], u.inv_view[4 * j + 2], u.inv_view[4 * j + 3]);
            o.lm[4 * j] = c4.x; o.lm[4 * j + 1] = c4.y; o.lm[4 * j + 2] = c4.z; o.lm[4 * j + 3] = c4.w;
        }
        const float nx = -L.direction[0], ny = -L.direction[1], nz = -L.direction[2];
        const float lx = u.view[0] * nx + u.view[4] * ny + u.view[8] * nz, ly = u.view[1] * nx + u.view[5] * ny + u.view[9] * nz,
                    lz = u.view[2] * nx + u.view[6] * ny + u.view[10] * nz;
        const float len = sqrtf(lx * lx + ly * ly + lz * lz);
        o.l[0] = lx / len; o.l[1] = ly / len; o.l[2] = lz / len;
        for (int k = 0; k < 3; ++k) o.color[k] = L.color[k];
        for (int k = 0; k < 2; ++k) { o.inv_res[k] = L.inv_resolution[k]; o.offset[k] = L.atlas_offset[k]; o.size[k] = L.atlas_size[k]; }
        o._pad[0] = o._pad[1] = o._pad[2] = o._pad[3] = 0.f;
        out_dir[i] = o;
    }
    if (i < n_point) {
        const r3_point_light L = point[i];
        const float4 v = mat_vec_rn(u.view, L.position[0], L.position[1], L.position[2], L.position[3]);
        PointPrep o;
        o.pos[0] = v.x; o.pos[1] = v.y; o.pos[2] = v.z; o.radius = L.radius;
        o.color[0] = L.color[0]; o.color[1] = L.color[1]; o.color[2] = L.color[2]; o._pad = 0.f;
        out_point[i] = o;
    }
}

// hi-Z pyramid (hi_z.rs:161-234): mip 0 = depth bits of the visibility buffer (multisampled: resolve_depth_min.wgsl:18-27 keeps the MIN
// over the samples); every further level = hi_z.wgsl::fs_main (:18-33): MIN over a 2 x 2 footprint, +1 column / row when the source
// size is odd, texels outside the source skipped.  The chain runs in two launches instead of one per level (12 at 4K).
// hiz_head_kernel: a CTA owns a 32 x 32 tile of mip 0, every thread a
// 2 x 2 quad — mip 0 from the visibility buffer, then up to three further levels through shared memory, as long as the source level has
// even dimensions (then the 2 x 2 footprints tile exactly and no `+1 on odd sizes` column crosses a tile).  hiz_tail_kernel: one CTA
// walks the remaining small levels (<= 1/64 of the pixels) with a barrier between them.  Same min() over the same texels: bit-identical.
__global__ void __launch_bounds__(256) hiz_head_kernel(const unsigned long long* __restrict__ vis, uint32_t samples, float* const* __restrict__ mips, const uint32_t* __restrict__ dims,
                                                       uint32_t fused) {
    __shared__ float s1[16][16];
    __shared__ float s2[8][8];
    const uint32_t w0 = dims[0], h0 = dims[1];
    const uint32_t tx = threadIdx.x & 15u, ty = threadIdx.x >> 4;
    const uint32_t x0 = blockIdx.x * 32u + tx * 2u, y0 = blockIdx.y * 32u + ty * 2u;
    float m = 1.0f;                                    // hi_z.wgsl starts from 1.0 and takes min over the texels that exist
#pragma unroll
    for (uint32_t dy = 0; dy < 2; ++dy)
#pragma unroll
        for (uint32_t dx = 0; dx < 2; ++dx) {
            const uint32_t x = x0 + dx, y = y0 + dy;
            if (x < w0 && y < h0) {
                const size_t i = (size_t)y * w0 + x;
                float d = 1.0f;
                for (uint32_t k = 0; k < samples; ++k) d = fminf(d, __uint_as_float((uint32_t)(vis[i * samples + k] >> 32)));
                mips[0][i] = d;
                m = fminf(m, d);
            }
        }
    if (fused < 1u) return;
    const uint32_t w1 = dims[2], h1 = dims[3], x1 = x0 >> 1, y1 = y0 >> 1;
    if (x1 < w1 && y1 < h1) mips[1][(size_t)y1 * w1 + x1] = m;
    if (fused < 2u) return;
    s1[ty][tx] = m;
    __syncthreads();
    if (threadIdx.x < 64u) {
        const uint32_t qx = threadIdx.x & 7u, qy = threadIdx.x >> 3;
        const float v = fminf(fminf(s1[2 * qy][2 * qx], s1[2 * qy][2 * qx + 1]), fminf(s1[2 * qy + 1][2 * qx], s1[2 * qy + 1][2 * qx + 1]));
        const uint32_t w2 = dims[4], h2 = dims[5], x2 = blockIdx.x * 8u + qx, y2 = blockIdx.y * 8u + qy;
        if (x2 < w2 && y2 < h2) mips[2][(size_t)y2 * w2 + x2] = v;
        s2[qy][qx] = v;
    }
    if (fused < 3u) return;
    __syncthreads();
    if (threadIdx.x < 16u) {
        const uint32_t qx = threadIdx.x & 3u, qy = threadIdx.x >> 2;
        const float v = fminf(fminf(s2[2 * qy][2 * qx], s2[2 * qy][2 * qx + 1]), fminf(s2[2 * qy + 1][2 * qx], s2[2 * qy + 1][2 * qx + 1]));
        const uint32_t w3 = dims[6], h3 = dims[7], x3 = blockIdx.x * 4u + qx, y3 = blockIdx.y * 4u + qy;
        if (x3 < w3 && y3 < h3) mips[3][(size_t)y3 * w3 + x3] = v;
    }
}
// one level, one thread per destination texel: the levels between the fused head and the single-CTA tail that are still large
__global__ void hiz_downsample_kernel(const float* __restrict__ src, uint32_t sw, uint32_t sh, float* __restrict__ dst, uint32_t dw, uint32_t dh) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= dw || y >= dh) return;
    const uint32_t oddx = sw & 1u, oddy = sh & 1u;
    float nearest = 1.0f;
    for (uint32_t dx = 0; dx < 2u + oddx; ++dx)
        for (uint32_t dy = 0; dy < 2u + oddy; ++dy) {
            const uint32_t sx = 2u * x + dx, sy = 2u * y + dy;
            if (sx < sw && sy < sh) nearest = fminf(nearest, src[(size_t)sy * sw + sx]);
        }
    dst[(size_t)y * dw + x] = nearest;
}
__global__ void __launch_bounds__(1024) hiz_tail_kernel(float* const* __restrict__ mips, const uint32_t* __restrict__ dims, uint32_t first, uint32_t n_mips) {
    for (uint32_t m = first; m < n_mips; ++m) {
        const uint32_t sw = dims[2 * (m - 1)], sh = dims[2 * (m - 1) + 1], dw = dims[2 * m], dh = dims[2 * m + 1];
        const float* src = mips[m - 1];
        float* dst = mips[m];
        const uint32_t oddx = sw & 1u, oddy = sh & 1u;
        for (uint32_t i = threadIdx.x; i < dw * dh; i += blockDim.x) {
            const uint32_t x = i % dw, y = i / dw;
            float nearest = 1.0f;
            for (uint32_t dx = 0; dx < 2u + oddx; ++dx)
                for (uint32_t dy = 0; dy < 2u + oddy; ++dy) {
                    const uint32_t sx = 2u * x + dx, sy = 2u * y + dy;
                    if (sx < sw && sy < sh) nearest = fminf(nearest, src[(size_t)sy * sw + sx]);
                }
            dst[i] = nearest;
        }
        __syncthreads();   // the level just written is the next one's source (same CTA: block-scope visibility is enough)
    }
}

// blit.wgsl: fs_main_scene into an *Srgb target (exact OETF) or fs_main_monitor (x^0.4166 approximation)
__global__ void tonemap_kernel(const uint2* __restrict__ hdr16, uchar4* __restrict__ ldr, size_t n, int srgb_target) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint2 h = hdr16[i];
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&h.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&h.y));
    const float in[4] = {a.x, a.y, b.x, b.y};
    uint8_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float x = in[k];
        float e;
        if (k == 3) e = x;
        else if (srgb_target) e = x <= 0.0031308f ? x * 12.92f : 1.055f * powf(x, 1.0f / 2.4f) - 0.055f;
        else e = x > 0.0031308f ? 1.055f * powf(x, 0.4166f) - 0.055f : x * 12.92f;
        e = fminf(fmaxf(e, 0.0f), 1.0f);
        o[k] = (uint8_t)floorf(e * 255.0f + 0.5f);
    }
    ldr[i] = make_uchar4(o[0], o[1], o[2], o[3]);
}

}  // namespace

// ------------------------------------------------------------------ host side
R3_EXPORT int r3_set_render_target(r3_ctx* c, uint32_t w, uint32_t h, uint32_t samples, const float clear[4]) {
    if (!c || !w || !h || !clear) return r3_fail(c, R3_E_INVALID, "set_render_target: bad arguments");
    if (samples != 1 && samples != 4) return r3_fail(c, R3_E_INVALID, "SampleCount must be One or Four");
    cudaSetDevice(c->device);
    if (w != c->width || h != c->height || samples != c->samples || !c->d_vis) {
        R3_CUDA(c, r3_stream_sync(c));
        cudaFree(c->d_vis); cudaFree(c->d_hdr32); cudaFree(c->d_hdr16); cudaFree(c->d_depth); cudaFree(c->d_ldr);
        for (float* p : c->d_hiz) cudaFree(p);
        c->d_hiz.clear(); c->hiz_w.clear(); c->hiz_h.clear();
        cudaFree(c->d_hiz_ptrs); cudaFree(c->d_hiz_dims);
        c->d_vis = nullptr; c->d_hdr32 = nullptr; c->d_hdr16 = nullptr; c->d_depth = nullptr; c->d_ldr = nullptr; c->d_hiz_ptrs = nullptr; c->d_hiz_dims = nullptr;
        const size_t n = (size_t)w * h;
        R3_CUDA(c, cudaMalloc((void**)&c->d_vis, n * 8 * samples));
        if (c->parity_target) R3_CUDA(c, cudaMalloc((void**)&c->d_hdr32, n * 16));
        R3_CUDA(c, cudaMalloc((void**)&c->d_hdr16, n * 8));
        R3_CUDA(c, cudaMalloc((void**)&c->d_depth, n * 4));
        R3_CUDA(c, cudaMalloc((void**)&c->d_ldr, n * 4));
        R3_CUDA(c, cudaMemsetAsync(c->d_vis, 0, n * 8 * samples, c->stream));
        // single_sample_mipped depth, cleared to 0.0 (base.rs:256-263, hi_z.rs:170-171)
        uint32_t m = w > h ? w : h, mips = 0;
        while (m) { mips++; m >>= 1; }
        std::vector<uint32_t> dims;
        for (uint32_t i = 0; i < mips; ++i) {
            const uint32_t mw = (w >> i) ? (w >> i) : 1u, mh = (h >> i) ? (h >> i) : 1u;
            float* p = nullptr;
            R3_CUDA(c, cudaMalloc((void**)&p, (size_t)mw * mh * 4));
            R3_CUDA(c, cudaMemsetAsync(p, 0, (size_t)mw * mh * 4, c->stream));
            c->d_hiz.push_back(p); c->hiz_w.push_back(mw); c->hiz_h.push_back(mh);
            dims.push_back(mw); dims.push_back(mh);
        }
        R3_CUDA(c, cudaMalloc((void**)&c->d_hiz_ptrs, mips * sizeof(float*)));
        R3_CUDA(c, cudaMalloc((void**)&c->d_hiz_dims, mips * 8));
        R3_CUDA(c, cudaMemcpyAsync(c->d_hiz_ptrs, c->d_hiz.data(), mips * sizeof(float*), cudaMemcpyHostToDevice, c->stream));
        R3_CUDA(c, cudaMemcpyAsync(c->d_hiz_dims, dims.data(), mips * 8, cudaMemcpyHostToDevice, c->stream));
        R3_CUDA(c, r3_stream_sync(c));
    }
    c->width = w; c->height = h; c->samples = samples;
    memcpy(c->clear_color, clear, 16);
    c->row_begin = 0; c->row_end = h;
    return R3_OK;
}
R3_EXPORT int r3_set_parity_target(r3_ctx* c, int enabled) {
    if (!c) return R3_E_INVALID;
    cudaSetDevice(c->device);
    c->parity_target = enabled != 0;
    if (!c->parity_target && c->d_hdr32) { R3_CUDA(c, r3_stream_sync(c)); cudaFree(c->d_hdr32); c->d_hdr32 = nullptr; }
    if (c->parity_target && !c->d_hdr32 && c->d_vis) {
        R3_CUDA(c, cudaMalloc((void**)&c->d_hdr32, (size_t)c->width * c->height * 16));
        R3_CUDA(c, cudaMemsetAsync(c->d_hdr32, 0, (size_t)c->width * c->height * 16, c->stream));
    }
    return R3_OK;
}
R3_EXPORT int r3_set_scissor_rows(r3_ctx* c, uint32_t a, uint32_t b) {
    if (!c || a > b || b > c->height) return r3_fail(c, R3_E_INVALID, "set_scissor_rows: bad range");
    c->row_begin = a; c->row_end = b;
    return R3_OK;
}
R3_EXPORT int r3_clear_shadow_atlas(r3_ctx* c) {
    if (!c) return R3_E_INVALID;
    cudaSetDevice(c->device);
    if (c->d_atlas) R3_CUDA(c, cudaMemsetAsync(c->d_atlas, 0, (size_t)c->atlas_w * c->atlas_h * 4, c->stream));
    return R3_OK;
}
R3_EXPORT int r3_forward_begin(r3_ctx* c) {
    if (!c || !c->d_vis) return r3_fail(c, R3_E_STATE, "forward_begin before set_render_target");
    cudaSetDevice(c->device);
    R3_CUDA(c, cudaMemsetAsync(c->d_vis, 0, (size_t)c->width * c->height * 8 * c->samples, c->stream));
    R3_CUDA(c, cudaMemsetAsync(c->d_stats, 0, 32, c->stream));
    R3_CUDA(c, cudaMemsetAsync(c->d_stats + 6, 0, 8, c->stream));
    c->n_tris[0] = c->n_tris[1] = c->n_tris[2] = 0;
    return R3_OK;
}
R3_EXPORT int r3_hiz_build(r3_ctx* c) {
    if (!c || !c->d_vis || c->d_hiz.empty()) return r3_fail(c, R3_E_STATE, "hiz_build before set_render_target");
    cudaSetDevice(c->device);
    // levels fused into the head kernel: as long as the source level has even dimensions (and the level exists), at most three
    const uint32_t n_mips = (uint32_t)c->d_hiz.size();
    uint32_t fused = 0;
    while (fused < 3u && fused + 1u < n_mips && !(c->hiz_w[fused] & 1u) && !(c->hiz_h[fused] & 1u)) fused++;
    const dim3 grid((c->width + 31) / 32, (c->height + 31) / 32);
    hiz_head_kernel<<<grid, 256, 0, c->stream>>>(c->d_vis, c->samples, c->d_hiz_ptrs, c->d_hiz_dims, fused);
    R3_CHECK_LAUNCH(c, "hiz_head_kernel");
    uint32_t m = fused + 1u;
    for (; m < n_mips && (uint64_t)c->hiz_w[m] * c->hiz_h[m] > 4096u; ++m) {   // still large: one launch per level, thousands of threads
        const dim3 block(32, 8), dgrid((c->hiz_w[m] + 31) / 32, (c->hiz_h[m] + 7) / 8);
        hiz_downsample_kernel<<<dgrid, block, 0, c->stream>>>(c->d_hiz[m - 1], c->hiz_w[m - 1], c->hiz_h[m - 1], c->d_hiz[m], c->hiz_w[m], c->hiz_h[m]);
        R3_CHECK_LAUNCH(c, "hiz_downsample_kernel");
    }
    if (m < n_mips) {                                                            // the small rest: one CTA walks the levels
        hiz_tail_kernel<<<1, 1024, 0, c->stream>>>(c->d_hiz_ptrs, c->d_hiz_dims, m, n_mips);
        R3_CHECK_LAUNCH(c, "hiz_tail_kernel");
    }
    return R3_OK;
}
static void fill_shade_params(r3_ctx* c, ShadeParams* out) {
    r3_camera* cam = &c->cams[0];
    ShadeParams& p = *out;
    DirPrep* d_dir = reinterpret_cast<DirPrep*>(c->d_light_mats);
    PointPrep* d_point = reinterpret_cast<PointPrep*>(c->d_light_mats + (size_t)c->n_dir * 32);
    p.vis = c->d_vis;
    p.tris0 = c->d_tris[0]; p.tris1 = c->d_tris[1]; p.n_tris0 = c->n_tris[0]; p.n_tris1 = c->n_tris[1];
    p.tris2 = c->d_tris[2]; p.n_tris2 = c->n_tris[2]; p.frag_heads = c->d_frag_heads; p.frag_nodes = c->d_frag_nodes;
    p.objects = c->d_objects; p.matrices = cam->d_matrices; p.mesh = c->d_mesh; p.mesh_words = c->mesh_words;
    p.materials = c->d_materials; p.n_materials = c->n_materials;
    p.tt.tex = c->d_tex_descs; p.tt.n_tex = c->n_textures; p.tt.texels = c->d_texels; p.tt.clamp_to_edge = 0u;
    p.sky.tex = nullptr; p.sky.n_tex = 0; p.sky.texels = c->has_skybox ? c->d_sky_texels : nullptr; p.sky.clamp_to_edge = 1u;
    p.sky_desc = c->sky_desc; memcpy(p.inv_origin_view_proj, c->uniforms.inv_origin_view_proj, 64);
    p.dir = d_dir; p.n_dir = c->n_dir; p.point = d_point; p.point_count = reinterpret_cast<const uint32_t*>(c->d_point);
    p.atlas = c->d_atlas; p.atlas_w = c->atlas_w; p.atlas_h = c->atlas_h;
    memcpy(p.ambient, c->uniforms.ambient, 16); memcpy(p.clear, c->clear_color, 16);
    p.width = c->width; p.height = c->height; p.row_begin = c->row_begin; p.row_end = c->row_end; p.samples = c->samples;
    p.hdr32 = reinterpret_cast<float4*>(c->d_hdr32); p.hdr16 = reinterpret_cast<uint2*>(c->d_hdr16); p.depth = c->d_depth; p.stats = c->d_stats;
}
R3_EXPORT int r3_forward_resolve(r3_ctx* c) {
    if (!c || !c->d_vis) return r3_fail(c, R3_E_STATE, "forward_resolve before set_render_target");
    if (!c->uniforms_set) return r3_fail(c, R3_E_STATE, "forward_resolve before set_frame_uniforms");
    if (c->point_eval_pending) return r3_fail(c, R3_E_STATE, "forward_resolve: point lights set or updated since the last evaluate_point_lights");
    if (c->dir_eval_pending) return r3_fail(c, R3_E_STATE, "forward_resolve: directional lights updated since the last evaluate_shadow_cameras");
    cudaSetDevice(c->device);
    const uint64_t need_floats = (uint64_t)c->n_dir * 32 + (uint64_t)c->point_capacity * 8 + 64;
    static_assert(sizeof(DirPrep) == 32 * 4 && sizeof(PointPrep) == 8 * 4, "prep sizes");
    R3_TRY(r3_reserve_t(c, &c->d_light_mats, &c->light_mats_cap, need_floats));
    float* prep = c->d_light_mats;
    DirPrep* d_dir = reinterpret_cast<DirPrep*>(prep);
    PointPrep* d_point = reinterpret_cast<PointPrep*>(prep + (size_t)c->n_dir * 32);
    const uint32_t nl = c->n_dir > c->point_capacity ? c->n_dir : c->point_capacity;
    if (nl) {
        light_prep_kernel<<<(nl + 127) / 128, 128, 0, c->stream>>>(c->d_dir, c->n_dir, c->d_point, c->uniforms, d_dir, d_point);
        R3_CHECK_LAUNCH(c, "light_prep_kernel");
    }
    ShadeParams p;
    fill_shade_params(c, &p);
    const uint32_t rows = c->row_end - c->row_begin;
    if (rows) {
        const dim3 grid((c->width + 31) / 32, (rows + 7) / 8);
        const bool tex = c->n_textures != 0;
        r3_stage_begin(c, R3_STAGE_RESOLVE);
        if (c->samples == 1) { if (tex) resolve_kernel<1, true><<<grid, 256, 0, c->stream>>>(p); else resolve_kernel<1, false><<<grid, 256, 0, c->stream>>>(p); }
        else { if (tex) resolve_kernel<4, true><<<grid, 256, 0, c->stream>>>(p); else resolve_kernel<4, false><<<grid, 256, 0, c->stream>>>(p); }
        r3_stage_end(c);
        R3_CHECK_LAUNCH(c, "resolve_kernel");
        if (c->has_skybox && c->samples == 1) {
            skybox_kernel<<<grid, 256, 0, c->stream>>>(p);
            R3_CHECK_LAUNCH(c, "skybox_kernel");
        }
    }
    return R3_OK;
}
R3_EXPORT int r3_forward_blend(r3_ctx* c) {
    if (!c || !c->d_vis) return r3_fail(c, R3_E_STATE, "forward_blend before set_render_target");
    if (!c->uniforms_set) return r3_fail(c, R3_E_STATE, "forward_blend before set_frame_uniforms");
    if (c->point_eval_pending) return r3_fail(c, R3_E_STATE, "forward_blend: point lights set or updated since the last evaluate_point_lights");
    if (c->dir_eval_pending) return r3_fail(c, R3_E_STATE, "forward_blend: directional lights updated since the last evaluate_shadow_cameras");
    cudaSetDevice(c->device);
    bool ran = false;
    R3_TRY(r3_blend_collect(c, &ran));
    const uint32_t rows = c->row_end - c->row_begin;
    if (!ran || !rows) return R3_OK;
    ShadeParams p;
    fill_shade_params(c, &p);   // the lights were prepared by r3_forward_resolve of this frame
    const dim3 grid((c->width + 31) / 32, (rows + 7) / 8);
    const bool tex = c->n_textures != 0;
    if (c->samples == 1) { if (tex) blend_apply_kernel<1, true><<<grid, 256, 0, c->stream>>>(p); else blend_apply_kernel<1, false><<<grid, 256, 0, c->stream>>>(p); }
    else { if (tex) blend_apply_kernel<4, true><<<grid, 256, 0, c->stream>>>(p); else blend_apply_kernel<4, false><<<grid, 256, 0, c->stream>>>(p); }
    R3_CHECK_LAUNCH(c, "blend_apply_kernel");
    return R3_OK;
}
R3_EXPORT int r3_tonemap(r3_ctx* c, int srgb_target) {
    if (!c || !c->d_hdr16) return r3_fail(c, R3_E_STATE, "tonemap before set_render_target");
    cudaSetDevice(c->device);
    const size_t n = (size_t)c->width * c->height;
    tonemap_kernel<<<(unsigned)((n + 255) / 256), 256, 0, c->stream>>>(reinterpret_cast<const uint2*>(c->d_hdr16), reinterpret_cast<uchar4*>(c->d_ldr), n, srgb_target);
    R3_CHECK_LAUNCH(c, "tonemap_kernel");
    return R3_OK;
}

static int copy_out(r3_ctx* c, const void* src, void* out, uint64_t cap, uint64_t count, size_t elem) {
    if (!src) return r3_fail(c, R3_E_STATE, "readback before the stage ran");
    if (!out || cap < count) return r3_fail(c, R3_E_INVALID, "readback: capacity too small");
    cudaSetDevice(c->device);
    R3_CUDA(c, cudaMemcpyAsync(out, src, count * elem, cudaMemcpyDeviceToHost, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    return R3_OK;
}
R3_EXPORT int r3_readback_hdr_f32(r3_ctx* c, float* out, uint64_t cap) {
    if (!c) return R3_E_INVALID;
    if (!c->parity_target) return r3_fail(c, R3_E_STATE, "readback_hdr_f32: the rgba32f parity target is off (r3_set_parity_target)");
    return copy_out(c, c->d_hdr32, out, cap, (uint64_t)c->width * c->height * 4, 4);
}
R3_EXPORT int r3_readback_hdr_f16(r3_ctx* c, uint16_t* out, uint64_t cap) { return c ? copy_out(c, c->d_hdr16, out, cap, (uint64_t)c->width * c->height * 4, 2) : R3_E_INVALID; }
R3_EXPORT int r3_readback_depth(r3_ctx* c, float* out, uint64_t cap) { return c ? copy_out(c, c->d_depth, out, cap, (uint64_t)c->width * c->height, 4) : R3_E_INVALID; }
R3_EXPORT int r3_readback_ldr(r3_ctx* c, uint8_t* out, uint64_t cap) { return c ? copy_out(c, c->d_ldr, out, cap, (uint64_t)c->width * c->height * 4, 1) : R3_E_INVALID; }
R3_EXPORT int r3_readback_shadow_atlas(r3_ctx* c, float* out, uint64_t cap) { return c ? copy_out(c, c->d_atlas, out, cap, (uint64_t)c->atlas_w * c->atlas_h, 4) : R3_E_INVALID; }
R3_EXPORT int r3_readback_hiz(r3_ctx* c, uint32_t mip, float* out, uint64_t cap, uint32_t* w, uint32_t* h) {
    if (!c || mip >= c->d_hiz.size()) return r3_fail(c, R3_E_INVALID, "readback_hiz: mip");
    if (w) *w = c->hiz_w[mip];
    if (h) *h = c->hiz_h[mip];
    if (!out) return R3_OK;
    return copy_out(c, c->d_hiz[mip], out, cap, (uint64_t)c->hiz_w[mip] * c->hiz_h[mip], 4);
}
R3_EXPORT int r3_forward_light_evaluations(r3_ctx* c, uint64_t* n) {
    if (!c || !n) return R3_E_INVALID;
    cudaSetDevice(c->device);
    R3_CUDA(c, cudaMemcpyAsync(n, c->d_stats + 6, 8, cudaMemcpyDeviceToHost, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    return R3_OK;
}
R3_EXPORT int r3_forward_stats(r3_ctx* c, uint64_t stats[4]) {
    if (!c || !stats) return R3_E_INVALID;
    cudaSetDevice(c->device);
    R3_CUDA(c, cudaMemcpyAsync(stats, c->d_stats, 32, cudaMemcpyDeviceToHost, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    return R3_OK;
}
