// r3_mesh_deform.cu — meshes that deform every frame: r3_set_deformable_meshes, r3_deform_meshes, r3_deform_meshes_device,
// r3_readback_deformable_mesh_spheres.
//
// rend3's meshes are immutable; the reference deforms one by rebuilding it (MeshBuilder::build: smooth normals and tangents,
// rend3-types/src/lib.rs:477-512, 617-837), re-adding it (MeshManager::add: BoundingSphere::from_mesh, mesh.rs:169, util/frustum.rs:15-56)
// and re-adding its objects (ObjectManager::add, object.rs:267-284).  Here the set is described once and each deform runs four kernels
// that write what that rebuild would produce, bit for bit (rule R15, DESIGN.md §2; -fmad=false and the _rn intrinsics):
//   deform_vertex_kernel   one thread per vertex: walks the vertex's corner list (the triangles that name it, ascending, a triangle
//                          twice when it names the vertex twice), recomputes each face's normal / tangent vector from the new
//                          positions (they stay in L2: no scratch), sums them from +0.0, normalises, Gram-Schmidt, stores position,
//                          normal and tangent, and leaves the CTA's bounding-box partial (below);
//   deform_bbox_kernel     one CTA per mesh: folds the mesh's CTA partials in order into the box, centre = (max + min) / 2;
//   deform_radius_kernel   one thread per vertex again: f32::max(0, |p - centre|) into the mesh's radius (atomicMax on the bits);
//   deform_objects_kernel  one thread per listed slot: mesh sphere, world sphere (sphere_apply_transform_rn, shared with
//                          object_transforms_kernel) into the record, the cull + bake's copies and the centre bit; sort location.
//
// The bounding box is Vec3A::max / min on SSE2 (_mm_max_ps(acc, p) = acc > p ? acc : p): a NaN or a tie takes the later vertex.  Per
// component that fold equals "the NaN if the last vertex is NaN, else the largest vertex after the last NaN, ties to the later one",
// which a reduction can compute with an associative, non-commutative operator over 64-bit keys (reset_max below).  CTAs never straddle
// meshes, so a CTA's partial belongs to one mesh and the partials of a mesh are consecutive.
#include <algorithm>
#include <cstring>
#include <vector>

#include "r3_common.cuh"
#include "r3_scan.cuh"
#include "../../include/r3_anim_check.h"

namespace {

constexpr uint32_t DF_THREADS = 256;
constexpr uint32_t DF_WARPS = DF_THREADS / 32;
constexpr uint32_t DF_ALL_FLAGS = R3_DEFORM_LEFT_HANDED | R3_DEFORM_NORMALS | R3_DEFORM_TANGENTS;

// one mesh of the set as the kernels read it
struct deform_mesh_dev {
    r3_deformable_mesh m;
    uint32_t vertex_base;   // the mesh's first vertex in the set (the position array and the corner lists)
    uint32_t block_first;   // its first CTA of the vertex and radius kernels
    uint32_t n_blocks;      // ceil(vertex_count / DF_THREADS)
    uint32_t _pad;
};
static_assert(sizeof(deform_mesh_dev) == 48, "deform_mesh_dev");

// Bounding-box key of one vertex component: bit 63 = the run holds a NaN (reset), bits 31-62 = the value's order (0: NaN), bits 0-30 =
// the vertex.  order(x) is monotone in x with -0.0 == +0.0, from 1 up: a larger key is a larger value, or the same value later.  The
// min fold uses ~order.  Key 0 is the identity.
constexpr unsigned long long KEY_RESET = 1ull << 63;
constexpr unsigned long long KEY_VALUE = KEY_RESET - 1;
__device__ __forceinline__ uint32_t float_order(float x) {
    const uint32_t u = x == 0.0f ? 0u : __float_as_uint(x);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ void bbox_keys(float x, uint32_t v, unsigned long long& kmax, unsigned long long& kmin) {
    if (isnan(x)) { kmax = kmin = KEY_RESET | v; return; }
    const uint32_t o = float_order(x);
    kmax = ((unsigned long long)o << 31) | v;
    kmin = ((unsigned long long)(~o) << 31) | v;
}
// fold(earlier run, later run): a later run that holds a NaN starts over; otherwise the larger key, the reset bit kept.  Called as
// op(later, earlier), the order warp_scan_incl applies it in.
struct reset_max {
    __device__ __forceinline__ unsigned long long operator()(unsigned long long later, unsigned long long earlier) const {
        if (later & KEY_RESET) return later;
        const unsigned long long a = later & KEY_VALUE, b = earlier & KEY_VALUE;
        return (earlier & KEY_RESET) | (a > b ? a : b);
    }
};

// the ordered fold of the block's six keys per thread (thread order), in thread DF_THREADS - 1
__device__ __forceinline__ void block_fold_keys(unsigned long long (&k)[6], unsigned long long (*s_warp)[DF_WARPS]) {
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
#pragma unroll
    for (int j = 0; j < 6; ++j) {
        k[j] = warp_scan_incl(k[j], reset_max());
        if (lane == 31) s_warp[j][warp] = k[j];
    }
    __syncthreads();
    if (warp == DF_WARPS - 1) {
#pragma unroll
        for (int j = 0; j < 6; ++j) k[j] = warp_scan_incl(lane < DF_WARPS ? s_warp[j][lane] : 0ull, reset_max());
    }
}

struct f3 { float x, y, z; };
__device__ __forceinline__ f3 ld3(const float* p) { return {__ldg(p), __ldg(p + 1), __ldg(p + 2)}; }
__device__ __forceinline__ f3 ldw3(const uint32_t* mesh, uint64_t w) {
    return {__uint_as_float(__ldg(mesh + w)), __uint_as_float(__ldg(mesh + w + 1)), __uint_as_float(__ldg(mesh + w + 2))};
}
__device__ __forceinline__ void stw3(uint32_t* mesh, uint64_t w, f3 v) {
    mesh[w] = __float_as_uint(v.x); mesh[w + 1] = __float_as_uint(v.y); mesh[w + 2] = __float_as_uint(v.z);
}
__device__ __forceinline__ f3 sub3(f3 a, f3 b) { return {sub_rn(a.x, b.x), sub_rn(a.y, b.y), sub_rn(a.z, b.z)}; }
__device__ __forceinline__ f3 add3(f3 a, f3 b) { return {add_rn(a.x, b.x), add_rn(a.y, b.y), add_rn(a.z, b.z)}; }
__device__ __forceinline__ f3 scale3(f3 a, float s) { return {mul_rn(a.x, s), mul_rn(a.y, s), mul_rn(a.z, s)}; }
__device__ __forceinline__ float dot3(f3 a, f3 b) { return add_rn(add_rn(mul_rn(a.x, b.x), mul_rn(a.y, b.y)), mul_rn(a.z, b.z)); }
// Vec3::cross (glam.py::cross): (a.y b.z - b.y a.z, a.z b.x - b.z a.x, a.x b.y - b.x a.y)
__device__ __forceinline__ f3 cross3(f3 a, f3 b) {
    return {sub_rn(mul_rn(a.y, b.z), mul_rn(b.y, a.z)), sub_rn(mul_rn(a.z, b.x), mul_rn(b.z, a.x)), sub_rn(mul_rn(a.x, b.y), mul_rn(b.x, a.y))};
}
// Vec3::normalize_or_zero: rcp = 1 / sqrt(dot(v, v)); v * rcp when rcp is finite and > 0, else zero
__device__ __forceinline__ f3 normalize_or_zero3(f3 v) {
    const float rcp = div_rn(1.0f, __fsqrt_rn(dot3(v, v)));
    if (isfinite(rcp) && rcp > 0.0f) return scale3(v, rcp);
    return {0.0f, 0.0f, 0.0f};
}

__global__ void __launch_bounds__(DF_THREADS)
deform_vertex_kernel(const deform_mesh_dev* __restrict__ meshes, const uint32_t* __restrict__ block_mesh, const float* __restrict__ pos_in,
                     const uint32_t* __restrict__ corner_start, const uint32_t* __restrict__ corners, uint32_t* mesh,
                     unsigned long long* __restrict__ partials) {
    __shared__ unsigned long long s_warp[6][DF_WARPS];
    const deform_mesh_dev md = meshes[__ldg(block_mesh + blockIdx.x)];
    const uint32_t v = (blockIdx.x - md.block_first) * DF_THREADS + threadIdx.x;
    unsigned long long k[6] = {0, 0, 0, 0, 0, 0};   // max x, y, z, min x, y, z
    if (v < md.m.vertex_count) {
        const uint64_t g = (uint64_t)md.vertex_base + v;
        const f3 p = ld3(pos_in + 3 * g);
        const uint32_t flags = md.m.flags;
        f3 n = {0.0f, 0.0f, 0.0f}, t = {0.0f, 0.0f, 0.0f};   // sums start from +0.0
        if (flags & (R3_DEFORM_NORMALS | R3_DEFORM_TANGENTS)) {
            const uint32_t c1 = __ldg(corner_start + g + 1);
            const float* base = pos_in + 3 * (uint64_t)md.vertex_base;
            for (uint32_t c = __ldg(corner_start + g); c < c1; ++c) {
                const uint64_t w = (uint64_t)md.m.first_index + 3ull * __ldg(corners + c);
                const uint32_t i0 = __ldg(mesh + w), i1 = __ldg(mesh + w + 1), i2 = __ldg(mesh + w + 2);
                const f3 p1 = ld3(base + 3ull * i0), p2 = ld3(base + 3ull * i1), p3 = ld3(base + 3ull * i2);
                const f3 e1 = sub3(p2, p1), e2 = sub3(p3, p1);
                if (flags & R3_DEFORM_NORMALS) n = add3(n, (flags & R3_DEFORM_LEFT_HANDED) ? cross3(e1, e2) : cross3(e2, e1));
                if (flags & R3_DEFORM_TANGENTS) {
                    const uint64_t uw = md.m.uv0_offset / 4;
                    const float t1x = __uint_as_float(__ldg(mesh + uw + 2ull * i0)), t1y = __uint_as_float(__ldg(mesh + uw + 2ull * i0 + 1));
                    const float t2x = __uint_as_float(__ldg(mesh + uw + 2ull * i1)), t2y = __uint_as_float(__ldg(mesh + uw + 2ull * i1 + 1));
                    const float t3x = __uint_as_float(__ldg(mesh + uw + 2ull * i2)), t3y = __uint_as_float(__ldg(mesh + uw + 2ull * i2 + 1));
                    const float u1x = sub_rn(t2x, t1x), u1y = sub_rn(t2y, t1y), u2x = sub_rn(t3x, t1x), u2y = sub_rn(t3y, t1y);
                    const float r = div_rn(1.0f, sub_rn(mul_rn(u1x, u2y), mul_rn(u1y, u2x)));
                    // (edge1 * uv2.y) - (edge2 * uv1.y) * r: r scales the second term only (lib.rs:826)
                    t = add3(t, sub3(scale3(e1, u2y), scale3(scale3(e2, u1y), r)));
                }
            }
        }
        stw3(mesh, md.m.position_offset / 4 + 3ull * v, p);
        if (flags & R3_DEFORM_NORMALS) {
            n = normalize_or_zero3(n);
            stw3(mesh, md.m.normal_offset / 4 + 3ull * v, n);
        }
        if (flags & R3_DEFORM_TANGENTS) {
            if (!(flags & R3_DEFORM_NORMALS)) n = ldw3(mesh, md.m.normal_offset / 4 + 3ull * v);   // the mesh's own normal
            t = normalize_or_zero3(sub3(t, scale3(n, dot3(n, t))));                                 // Gram-Schmidt (lib.rs:832-835)
            stw3(mesh, md.m.tangent_offset / 4 + 3ull * v, t);
        }
        bbox_keys(p.x, v, k[0], k[3]);
        bbox_keys(p.y, v, k[1], k[4]);
        bbox_keys(p.z, v, k[2], k[5]);
    }
    block_fold_keys(k, s_warp);
    if (threadIdx.x == DF_THREADS - 1) {
#pragma unroll
        for (int j = 0; j < 6; ++j) partials[(size_t)blockIdx.x * 6 + j] = k[j];
    }
}

// one CTA per mesh: thread i folds a contiguous run of the mesh's partials, the runs in thread order; then the box's vertices are read
// back for their bits (NaN payloads and the sign of zero included) and centre = (max + min) / 2.  The radius starts at +0.0.
__global__ void __launch_bounds__(DF_THREADS)
deform_bbox_kernel(const deform_mesh_dev* __restrict__ meshes, const float* __restrict__ pos_in, const unsigned long long* __restrict__ partials,
                   float4* __restrict__ spheres) {
    __shared__ unsigned long long s_warp[6][DF_WARPS];
    const deform_mesh_dev md = meshes[blockIdx.x];
    const uint32_t per = (md.n_blocks + DF_THREADS - 1) / DF_THREADS, q0 = threadIdx.x * per, q1 = min(q0 + per, md.n_blocks);
    unsigned long long k[6] = {0, 0, 0, 0, 0, 0};
    for (uint32_t q = q0; q < q1; ++q)
#pragma unroll
        for (int j = 0; j < 6; ++j) k[j] = reset_max()(partials[(size_t)(md.block_first + q) * 6 + j], k[j]);
    block_fold_keys(k, s_warp);
    if (threadIdx.x != DF_THREADS - 1) return;
    float4 s = make_float4(0.0f, 0.0f, 0.0f, 0.0f);   // an empty mesh: Vec3A::ZERO, radius 0
    if (md.m.vertex_count) {
        const float* base = pos_in + 3 * (uint64_t)md.vertex_base;
        float c[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const float mx = base[3ull * (uint32_t)(k[j] & 0x7FFFFFFFu) + j], mn = base[3ull * (uint32_t)(k[j + 3] & 0x7FFFFFFFu) + j];
            c[j] = div_rn(add_rn(mx, mn), 2.0f);
        }
        s = make_float4(c[0], c[1], c[2], 0.0f);
    }
    spheres[blockIdx.x] = s;
}

// find_mesh_bounding_sphere_radius: fold of f32::max(distance, |p - centre|) from 0.0.  f32::max ignores a NaN as fmaxf does, and the
// lengths are +0.0 or more, so the fold is the largest length, which the bits order like unsigned integers.
__global__ void __launch_bounds__(DF_THREADS)
deform_radius_kernel(const deform_mesh_dev* __restrict__ meshes, const uint32_t* __restrict__ block_mesh, const float* __restrict__ pos_in,
                     float4* spheres) {
    const uint32_t mi = __ldg(block_mesh + blockIdx.x);
    const deform_mesh_dev md = meshes[mi];
    const uint32_t v = (blockIdx.x - md.block_first) * DF_THREADS + threadIdx.x;
    float r = 0.0f;
    if (v < md.m.vertex_count) {
        const float4 s = spheres[mi];
        const f3 d = sub3(ld3(pos_in + 3 * ((uint64_t)md.vertex_base + v)), f3{s.x, s.y, s.z});
        r = fmaxf(0.0f, __fsqrt_rn(dot3(d, d)));
    }
    const uint32_t bits = warp_reduce(__float_as_uint(r), r3_op_max());
    if ((threadIdx.x & 31u) == 0 && bits) atomicMax(reinterpret_cast<uint32_t*>(&spheres[mi].w), bits);
}

// ObjectManager::add's sphere and location for every listed slot (object.rs:267-284), with the slot's current transform
__global__ void __launch_bounds__(DF_THREADS)
deform_objects_kernel(const uint32_t* __restrict__ slots, const uint32_t* __restrict__ object_mesh, uint32_t n, uint32_t n_slots,
                      const float4* __restrict__ spheres, float4* __restrict__ mesh_spheres, float4* __restrict__ objects,
                      float4* __restrict__ hot_spheres, float* __restrict__ radii, uint32_t* __restrict__ centre_bits, float* __restrict__ sort_loc,
                      uint32_t sort_n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = __ldg(slots + i);
    if (s >= n_slots) return;
    const float4 ms = spheres[__ldg(object_mesh + i)];
    mesh_spheres[s] = ms;
    float x[4], y[4], z[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float4 col = objects[(size_t)s * 8 + j];
        x[j] = col.x; y[j] = col.y; z[j] = col.z;
    }
    const float4 sph = sphere_apply_transform_rn(x, y, z, ms);
    objects[(size_t)s * 8 + 4] = sph;
    hot_spheres[s] = sph;
    radii[s] = sph.w;
    const uint32_t bit = 1u << (s & 31u);
    if (centre_is_translation(sph.x, sph.y, sph.z, x[3], y[3], z[3])) atomicOr(&centre_bits[s >> 5], bit);
    else atomicAnd(&centre_bits[s >> 5], ~bit);
    if (sort_loc && s < sort_n) {   // location = the world sphere's centre (object.rs:273)
        float* l = sort_loc + 3 * (size_t)s;
        l[0] = sph.x; l[1] = sph.y; l[2] = sph.z;
    }
}

}  // namespace

struct r3_deform_state {
    bool valid = false;                       // a set exists and no mesh-buffer write has invalidated its corner lists
    uint32_t n_meshes = 0, n_objects = 0, n_blocks = 0, max_slot = 0;
    uint64_t n_vertices = 0;
    std::vector<r3_deformable_mesh> meshes;   // host copy: the index ranges r3_update_mesh_buffer must not write
    deform_mesh_dev* d_meshes = nullptr; uint32_t meshes_cap = 0;
    uint32_t* d_block_mesh = nullptr; uint32_t block_mesh_cap = 0;
    unsigned long long* d_partials = nullptr; uint64_t partials_cap = 0;
    uint32_t* d_corner_start = nullptr; uint64_t corner_start_cap = 0;
    uint32_t* d_corners = nullptr; uint64_t corners_cap = 0;
    float4* d_spheres = nullptr; uint32_t spheres_cap = 0;
    uint32_t* d_slots = nullptr; uint32_t slots_cap = 0;
    uint32_t* d_object_mesh = nullptr; uint32_t object_mesh_cap = 0;
};

void r3_deform_destroy(r3_ctx* c) {
    r3_deform_state* d = c->deform;
    if (!d) return;
    cudaFree(d->d_meshes); cudaFree(d->d_block_mesh); cudaFree(d->d_partials); cudaFree(d->d_corner_start); cudaFree(d->d_corners);
    cudaFree(d->d_spheres); cudaFree(d->d_slots); cudaFree(d->d_object_mesh);
    delete d;
    c->deform = nullptr;
}

void r3_deform_note_mesh_write(r3_ctx* c, bool whole_buffer, uint64_t byte_offset, uint64_t nbytes) {
    r3_deform_state* d = c->deform;
    if (!d || !d->valid) return;
    if (whole_buffer) { d->valid = false; return; }
    for (const r3_deformable_mesh& m : d->meshes) {
        const uint64_t a = (uint64_t)m.first_index * 4, b = a + (uint64_t)m.index_count * 4;
        if (m.index_count && byte_offset < b && a < byte_offset + nbytes) { d->valid = false; return; }
    }
}

namespace {

// a byte range [a, b) of the mesh buffer; `write` ranges must not meet any other range of the set
struct byte_range { uint64_t a, b; };

int check_ranges(r3_ctx* c, std::vector<byte_range>& writes, std::vector<byte_range>& reads) {
    // the reads may overlap each other (two meshes may share uv0): merge them, then every range of writes + merged reads is disjoint
    std::sort(reads.begin(), reads.end(), [](const byte_range& x, const byte_range& y) { return x.a < y.a; });
    std::vector<uint64_t> r;
    r.reserve(2 * (writes.size() + reads.size()));
    for (const byte_range& w : writes) { r.push_back(w.a); r.push_back(w.b); }
    for (size_t i = 0; i < reads.size();) {
        uint64_t a = reads[i].a, b = reads[i].b;
        for (++i; i < reads.size() && reads[i].a < b; ++i) b = std::max(b, reads[i].b);
        r.push_back(a); r.push_back(b);
    }
    const char* msg = "";
    if (r3_anim_check_disjoint(r.data(), r.size() / 2, "set_deformable_meshes: a written range overlaps another range of the set", &msg) != R3_OK)
        return r3_fail(c, R3_E_INVALID, msg);
    return R3_OK;
}

int check_deform_state(r3_ctx* c, const char* who_state) {
    r3_deform_state* d = c->deform;
    if (!d || !d->valid) return r3_fail(c, R3_E_STATE, who_state);
    if (c->objects_borrowed) return r3_fail(c, R3_E_STATE, "deform_meshes: the object buffer is borrowed (r3_set_objects_device)");
    if (d->n_objects) {
        if (!c->d_objects || !c->hot_valid || d->max_slot >= c->n_slots) return r3_fail(c, R3_E_STATE, "deform_meshes: a listed slot is past the slot count");
        if (d->max_slot >= c->n_mesh_spheres) return r3_fail(c, R3_E_STATE, "deform_meshes: r3_set_object_mesh_spheres does not cover every listed slot");
    }
    return R3_OK;
}

int launch_deform(r3_ctx* c, const float* d_pos) {
    r3_deform_state* d = c->deform;
    if (d->n_blocks) {
        deform_vertex_kernel<<<d->n_blocks, DF_THREADS, 0, c->stream>>>(d->d_meshes, d->d_block_mesh, d_pos, d->d_corner_start, d->d_corners, c->d_mesh, d->d_partials);
        R3_CHECK_LAUNCH(c, "deform_vertex_kernel");
    }
    deform_bbox_kernel<<<d->n_meshes, DF_THREADS, 0, c->stream>>>(d->d_meshes, d_pos, d->d_partials, d->d_spheres);
    R3_CHECK_LAUNCH(c, "deform_bbox_kernel");
    if (d->n_blocks) {
        deform_radius_kernel<<<d->n_blocks, DF_THREADS, 0, c->stream>>>(d->d_meshes, d->d_block_mesh, d_pos, d->d_spheres);
        R3_CHECK_LAUNCH(c, "deform_radius_kernel");
    }
    if (d->n_objects) {
        const uint32_t sort_n = c->have_live ? (uint32_t)c->sort_key.size() : 0u;
        deform_objects_kernel<<<(d->n_objects + DF_THREADS - 1) / DF_THREADS, DF_THREADS, 0, c->stream>>>(
            d->d_slots, d->d_object_mesh, d->n_objects, c->n_slots, d->d_spheres, c->d_mesh_spheres, reinterpret_cast<float4*>(c->d_objects),
            c->d_hot_sphere, c->d_hot_radius, c->d_centre_bits, sort_n ? c->d_sort_loc : nullptr, sort_n);
        R3_CHECK_LAUNCH(c, "deform_objects_kernel");
        r3_new_frame_epoch(c);                   // a frame-wide sort made before the deform is stale
        if (sort_n) c->locations_moved = true;   // the host batching's mirror c->sort_loc is behind the device's
    }
    return R3_OK;
}

}  // namespace

R3_EXPORT int r3_set_deformable_meshes(r3_ctx* c, const r3_deformable_mesh* meshes, uint32_t n_meshes, const uint32_t* object_slots,
                                       const uint32_t* object_meshes, uint32_t n_objects) {
    if (!c) return R3_E_INVALID;
    if ((!meshes && n_meshes) || ((!object_slots || !object_meshes) && n_objects)) return r3_fail(c, R3_E_INVALID, "set_deformable_meshes: null");
    if (n_meshes == 0) {
        if (n_objects) return r3_fail(c, R3_E_INVALID, "set_deformable_meshes: objects without meshes");
        if (c->deform) { c->deform->valid = false; c->deform->meshes.clear(); }
        return R3_OK;
    }
    if (!c->d_objects || !c->hot_valid) return r3_fail(c, R3_E_STATE, "set_deformable_meshes before set_objects");
    if (c->objects_borrowed) return r3_fail(c, R3_E_STATE, "set_deformable_meshes: the object buffer is borrowed (r3_set_objects_device)");
    // ---- the records, against the mesh buffer as it is
    const uint64_t buf = c->mesh_words * 4;
    uint64_t n_vertices = 0, n_indices = 0, idx_lo = ~0ull, idx_hi = 0;
    std::vector<byte_range> writes, reads;
    const auto inside = [buf](uint64_t off, uint64_t bytes) { return off + bytes <= buf; };
    for (uint32_t i = 0; i < n_meshes; ++i) {
        const r3_deformable_mesh m = meshes[i];
        const uint64_t vb = 12ull * m.vertex_count;
        if (m.flags & ~DF_ALL_FLAGS) return r3_fail(c, R3_E_INVALID, "set_deformable_meshes: unknown flag bits");
        if (m.position_offset == R3_ATTR_ABSENT) return r3_fail(c, R3_E_INVALID, "set_deformable_meshes: a mesh without positions");
        if ((m.flags & R3_DEFORM_NORMALS) && m.normal_offset == R3_ATTR_ABSENT) return r3_fail(c, R3_E_INVALID, "set_deformable_meshes: normals recomputed without a normal range");
        if ((m.flags & R3_DEFORM_TANGENTS) && (m.tangent_offset == R3_ATTR_ABSENT || m.uv0_offset == R3_ATTR_ABSENT || m.normal_offset == R3_ATTR_ABSENT))
            return r3_fail(c, R3_E_INVALID, "set_deformable_meshes: tangents recomputed without tangent, uv0 and normal ranges");
        for (uint32_t off : {m.position_offset, m.normal_offset, m.tangent_offset, m.uv0_offset})
            if (off != R3_ATTR_ABSENT && (off & 3u)) return r3_fail(c, R3_E_INVALID, "set_deformable_meshes: an offset that is not a multiple of 4");
        if (m.index_count % 3) return r3_fail(c, R3_E_INVALID, "set_deformable_meshes: index_count is not a multiple of 3");
        const uint64_t ia = (uint64_t)m.first_index * 4, ib = 4ull * m.index_count;
        const bool tangents = m.flags & R3_DEFORM_TANGENTS, normals = m.flags & R3_DEFORM_NORMALS;
        if (!inside(m.position_offset, vb) || !inside(ia, ib) || ((normals || tangents) && !inside(m.normal_offset, vb)) ||
            (tangents && (!inside(m.tangent_offset, vb) || !inside(m.uv0_offset, 8ull * m.vertex_count))))
            return r3_fail(c, R3_E_INVALID, "set_deformable_meshes: a range outside the mesh buffer");
        n_vertices += m.vertex_count;
        n_indices += m.index_count;
        if (m.vertex_count) {
            writes.push_back({m.position_offset, m.position_offset + vb});
            if (normals) writes.push_back({m.normal_offset, m.normal_offset + vb});
            if (tangents) {
                writes.push_back({m.tangent_offset, m.tangent_offset + vb});
                reads.push_back({m.uv0_offset, m.uv0_offset + 8ull * m.vertex_count});
                if (!normals) reads.push_back({m.normal_offset, m.normal_offset + vb});
            }
        }
        if (m.index_count) {
            reads.push_back({ia, ia + ib});
            idx_lo = std::min(idx_lo, (uint64_t)m.first_index);
            idx_hi = std::max(idx_hi, (uint64_t)m.first_index + m.index_count);
        }
    }
    if (n_vertices > 0x7FFFFFFFull || n_indices > 0xFFFFFFFFull) return r3_fail(c, R3_E_INVALID, "set_deformable_meshes: more than 2^31 - 1 vertices or 2^32 - 1 indices");
    R3_TRY(check_ranges(c, writes, reads));
    // ---- the objects
    uint32_t slot_lo = ~0u, slot_hi = 0;
    {
        std::vector<uint64_t> seen(((size_t)c->n_slots + 63) / 64, 0ull);
        for (uint32_t i = 0; i < n_objects; ++i) {
            const uint32_t s = object_slots[i];
            if (object_meshes[i] >= n_meshes) return r3_fail(c, R3_E_INVALID, "set_deformable_meshes: object mesh out of range");
            if (s >= c->n_slots) return r3_fail(c, R3_E_INVALID, "set_deformable_meshes: slot beyond the object buffer");
            if (seen[s >> 6] & (1ull << (s & 63u))) return r3_fail(c, R3_E_INVALID, "set_deformable_meshes: one slot named twice");
            seen[s >> 6] |= 1ull << (s & 63u);
            slot_lo = std::min(slot_lo, s); slot_hi = std::max(slot_hi, s);
        }
    }
    // ---- read back the indices and the listed records (one copy each: the hull of the ranges) and check them
    cudaSetDevice(c->device);
    std::vector<uint32_t> idx(n_indices ? idx_hi - idx_lo : 0);
    std::vector<r3_object> recs(n_objects ? slot_hi - slot_lo + 1 : 0);
    if (!idx.empty()) R3_CUDA(c, cudaMemcpyAsync(idx.data(), c->d_mesh + idx_lo, idx.size() * 4, cudaMemcpyDeviceToHost, c->stream));
    if (!recs.empty()) R3_CUDA(c, cudaMemcpyAsync(recs.data(), c->d_objects + slot_lo, recs.size() * sizeof(r3_object), cudaMemcpyDeviceToHost, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    for (uint32_t i = 0; i < n_meshes; ++i) {
        const r3_deformable_mesh& m = meshes[i];
        const uint32_t* ix = idx.data() + (m.first_index - idx_lo);
        for (uint32_t j = 0; j < m.index_count; ++j)
            if (ix[j] >= m.vertex_count) return r3_fail(c, R3_E_INVALID, "set_deformable_meshes: an index >= vertex_count");
    }
    for (uint32_t i = 0; i < n_objects; ++i) {
        const r3_object& o = recs[object_slots[i] - slot_lo];
        const r3_deformable_mesh& m = meshes[object_meshes[i]];
        if (o.first_index != m.first_index || o.index_count != m.index_count || o.attr_offset[R3_ATTR_POSITION] != m.position_offset)
            return r3_fail(c, R3_E_INVALID, "set_deformable_meshes: a slot's record does not draw its mesh");
    }
    // ---- vertex -> corner lists: a stable counting sort of the indices by vertex, so each list is in ascending triangle order (a triangle
    // that names a vertex twice is listed twice); start[g] .. start[g + 1] is global vertex g's list
    std::vector<deform_mesh_dev> dev(n_meshes);
    std::vector<uint32_t> start(n_vertices + 1, 0u), corners(n_indices), block_mesh;
    uint32_t vb = 0, blocks = 0;
    for (uint32_t i = 0; i < n_meshes; ++i) {
        const r3_deformable_mesh& m = meshes[i];
        const uint32_t nb = (m.vertex_count + DF_THREADS - 1) / DF_THREADS;
        dev[i] = deform_mesh_dev{m, vb, blocks, nb, 0u};
        block_mesh.insert(block_mesh.end(), nb, i);
        const uint32_t* ix = idx.data() + (m.first_index - idx_lo);
        for (uint32_t j = 0; j < m.index_count; ++j) start[vb + ix[j] + 1]++;
        vb += m.vertex_count; blocks += nb;
    }
    for (uint64_t g = 0; g < n_vertices; ++g) start[g + 1] += start[g];
    {
        std::vector<uint32_t> fill(start.begin(), start.end() - 1);
        for (uint32_t i = 0; i < n_meshes; ++i) {
            const r3_deformable_mesh& m = meshes[i];
            const uint32_t* ix = idx.data() + (m.first_index - idx_lo);
            uint32_t* f = fill.data() + dev[i].vertex_base;
            for (uint32_t j = 0; j < m.index_count; ++j) corners[f[ix[j]]++] = j / 3;
        }
    }
    // ---- upload
    if (!c->deform) c->deform = new r3_deform_state();
    r3_deform_state* d = c->deform;
    d->valid = false;
    R3_TRY(r3_reserve_t(c, &d->d_meshes, &d->meshes_cap, n_meshes));
    R3_TRY(r3_reserve_t(c, &d->d_block_mesh, &d->block_mesh_cap, std::max(blocks, 1u)));
    R3_TRY(r3_reserve_t(c, &d->d_partials, &d->partials_cap, 6ull * std::max(blocks, 1u)));
    R3_TRY(r3_reserve_t(c, &d->d_corner_start, &d->corner_start_cap, n_vertices + 1));
    R3_TRY(r3_reserve_t(c, &d->d_corners, &d->corners_cap, std::max<uint64_t>(n_indices, 1)));
    R3_TRY(r3_reserve_t(c, &d->d_spheres, &d->spheres_cap, n_meshes));
    R3_TRY(r3_reserve_t(c, &d->d_slots, &d->slots_cap, std::max(n_objects, 1u)));
    R3_TRY(r3_reserve_t(c, &d->d_object_mesh, &d->object_mesh_cap, std::max(n_objects, 1u)));
    R3_CUDA(c, cudaMemcpyAsync(d->d_meshes, dev.data(), dev.size() * sizeof(deform_mesh_dev), cudaMemcpyHostToDevice, c->stream));
    if (blocks) R3_CUDA(c, cudaMemcpyAsync(d->d_block_mesh, block_mesh.data(), (size_t)blocks * 4, cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, cudaMemcpyAsync(d->d_corner_start, start.data(), start.size() * 4, cudaMemcpyHostToDevice, c->stream));
    if (n_indices) R3_CUDA(c, cudaMemcpyAsync(d->d_corners, corners.data(), corners.size() * 4, cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, cudaMemsetAsync(d->d_spheres, 0, (size_t)n_meshes * 16, c->stream));
    if (n_objects) {
        R3_CUDA(c, cudaMemcpyAsync(d->d_slots, object_slots, (size_t)n_objects * 4, cudaMemcpyHostToDevice, c->stream));
        R3_CUDA(c, cudaMemcpyAsync(d->d_object_mesh, object_meshes, (size_t)n_objects * 4, cudaMemcpyHostToDevice, c->stream));
    }
    R3_CUDA(c, r3_stream_sync(c));   // host pointers are only borrowed for the call
    d->meshes.assign(meshes, meshes + n_meshes);
    d->n_meshes = n_meshes; d->n_objects = n_objects; d->n_blocks = blocks; d->n_vertices = n_vertices;
    d->max_slot = n_objects ? slot_hi : 0;
    d->valid = true;
    return R3_OK;
}

R3_EXPORT int r3_deform_meshes(r3_ctx* c, const float* positions, uint64_t n_floats) {
    if (!c) return R3_E_INVALID;
    R3_TRY(check_deform_state(c, "deform_meshes before set_deformable_meshes, or after a mesh-buffer write that replaced its indices"));
    if (n_floats != 3 * c->deform->n_vertices) return r3_fail(c, R3_E_INVALID, "deform_meshes: n_floats is not 3 x the set's vertex count");
    if (!positions && n_floats) return r3_fail(c, R3_E_INVALID, "deform_meshes: null");
    cudaSetDevice(c->device);
    R3_TRY(r3_reserve(c, &c->d_scratch, &c->scratch_cap, std::max<uint64_t>(n_floats * 4, 4), 1, false, false));
    if (n_floats) R3_CUDA(c, cudaMemcpyAsync(c->d_scratch, positions, n_floats * 4, cudaMemcpyHostToDevice, c->stream));
    R3_TRY(launch_deform(c, (const float*)c->d_scratch));
    R3_CUDA(c, r3_stream_sync(c));   // host pointer is only borrowed for the call; the only drain
    return R3_OK;
}

R3_EXPORT int r3_deform_meshes_device(r3_ctx* c, const float* d_positions, uint64_t n_floats) {
    if (!c) return R3_E_INVALID;
    R3_TRY(check_deform_state(c, "deform_meshes_device before set_deformable_meshes, or after a mesh-buffer write that replaced its indices"));
    if (n_floats != 3 * c->deform->n_vertices) return r3_fail(c, R3_E_INVALID, "deform_meshes_device: n_floats is not 3 x the set's vertex count");
    if ((!d_positions && n_floats) || ((uintptr_t)d_positions & 3u)) return r3_fail(c, R3_E_INVALID, "deform_meshes_device: null or misaligned positions (4 bytes)");
    cudaSetDevice(c->device);
    return launch_deform(c, d_positions);
}

R3_EXPORT int r3_readback_deformable_mesh_spheres(r3_ctx* c, float* out, uint32_t first, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (!c->deform || !c->deform->n_meshes || c->deform->meshes.empty()) return r3_fail(c, R3_E_STATE, "readback_deformable_mesh_spheres before set_deformable_meshes");
    if ((!out && n) || (uint64_t)first + n > c->deform->n_meshes) return r3_fail(c, R3_E_INVALID, "readback_deformable_mesh_spheres: range outside the set");
    if (n == 0) return R3_OK;
    cudaSetDevice(c->device);
    R3_CUDA(c, cudaMemcpyAsync(out, c->deform->d_spheres + first, (size_t)n * 16, cudaMemcpyDeviceToHost, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    return R3_OK;
}
