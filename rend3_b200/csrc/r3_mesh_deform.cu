// r3_mesh_deform.cu — meshes that deform every frame: r3_set_deformable_meshes, r3_deform_meshes, r3_deform_meshes_device,
// r3_readback_deformable_mesh_spheres; and meshes whose topology changes every frame: r3_set_remeshable_meshes, r3_remesh_meshes,
// r3_remesh_meshes_device, r3_readback_remesh_status.
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
//
// The vertex -> corner lists are built on the device for both kinds of set: one key per corner, (global vertex << 32 | triangle), in
// index order, then a stable LSD radix sort on the vertex bits (r3_radix.cuh, the batching sort's tiles) and a lower-bound search per
// vertex for the list starts.  Stability gives each list in ascending triangle order, which is the order R15 sums in.  A remesh runs,
// before the four kernels above: Mesh::validate per mesh (remesh_counts_kernel, remesh_indices_kernel), the counts in force and a skip bit
// (remesh_apply_kernel), the corner keys (which also copy the indices into the mesh buffer), the sort, and the supplied attribute streams
// (remesh_copy_kernel).  Every grid is sized by the capacities, so the counts can vary on the device inside a frame graph.
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "r3_common.cuh"
#include "r3_radix.cuh"
#include "r3_scan.cuh"
#include "../../include/r3_anim_check.h"

namespace {

constexpr uint32_t DF_THREADS = 256;
constexpr uint32_t DF_WARPS = DF_THREADS / 32;
constexpr uint32_t DF_ALL_FLAGS = R3_DEFORM_LEFT_HANDED | R3_DEFORM_NORMALS | R3_DEFORM_TANGENTS;

// one mesh of the set as the kernels read it; a remesh set's ranges and streams are laid out by the capacities
struct deform_mesh_dev {
    r3_deformable_mesh m;     // m.vertex_count, m.index_count: the counts in force (a remesh writes them, r3_readback_remesh_status)
    uint32_t vertex_base;     // the mesh's first vertex in the set (the vertex streams and the corner lists)
    uint32_t block_first;     // its first CTA of the vertex and radius kernels
    uint32_t n_blocks;        // ceil(vertex capacity / DF_THREADS)
    uint32_t skip;            // the last remesh rejected the mesh: no kernel writes anything of it
    uint32_t index_base;      // its first index in the set
    uint32_t vertex_capacity, index_capacity;
    uint32_t color0_offset;   // R3_ATTR_ABSENT in a deformable set
};
static_assert(sizeof(deform_mesh_dev) == 64, "deform_mesh_dev");

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
    if (md.skip) return;   // CTAs never straddle meshes: uniform
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
    if (md.skip) return;   // the mesh sphere stays
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
    if (md.skip) return;
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

// ObjectManager::add's sphere and location for every listed slot (object.rs:267-284), with the slot's current transform, and for a remesh
// set its index_count; nothing for a slot whose mesh the last remesh rejected.  A deform leaves index_count alone: its value is the
// set's by definition, and a record rewritten since the set was made must keep what the host gave it, which the invocation bound counts.
__global__ void __launch_bounds__(DF_THREADS)
deform_objects_kernel(const deform_mesh_dev* __restrict__ meshes, const uint32_t* __restrict__ slots, const uint32_t* __restrict__ object_mesh,
                      uint32_t n, uint32_t n_slots, uint32_t store_index_count, const float4* __restrict__ spheres, float4* __restrict__ mesh_spheres, float4* __restrict__ objects,
                      float4* __restrict__ hot_spheres, float* __restrict__ radii, uint32_t* __restrict__ centre_bits, float* __restrict__ sort_loc,
                      uint32_t sort_n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = __ldg(slots + i), mi = __ldg(object_mesh + i);
    if (s >= n_slots || meshes[mi].skip) return;
    const float4 ms = spheres[mi];
    mesh_spheres[s] = ms;
    if (store_index_count) reinterpret_cast<uint32_t*>(objects + (size_t)s * 8)[offsetof(r3_object, index_count) / 4] = meshes[mi].m.index_count;
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
    slot_bit_assign(centre_bits, s, centre_is_translation(sph.x, sph.y, sph.z, x[3], y[3], z[3]));
    if (sort_loc && s < sort_n) {   // location = the world sphere's centre (object.rs:273)
        float* l = sort_loc + 3 * (size_t)s;
        l[0] = sph.x; l[1] = sph.y; l[2] = sph.z;
    }
}

// ---- the vertex -> corner lists
// the mesh whose index range holds set index j: the last one with index_base <= j (index_base ascending; empty meshes share a base)
__device__ __forceinline__ uint32_t mesh_of_index(const uint32_t* __restrict__ index_base, uint32_t n_meshes, uint32_t j) {
    uint32_t lo = 0, hi = n_meshes;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldg(index_base + mid) <= j) lo = mid; else hi = mid;
    }
    return lo;
}

// One key per set index, in index order: (the corner's global vertex << 32) | its triangle in the mesh; (`none` << 32) past the mesh's
// index_count and for a skipped mesh.  `src` (a remesh's index stream, laid out like the set's indices): the index is read there and
// copied into the mesh buffer; nullptr: read from the mesh buffer.
__global__ void __launch_bounds__(DF_THREADS)
corner_keys_kernel(const deform_mesh_dev* __restrict__ meshes, const uint32_t* __restrict__ index_base, uint32_t n_meshes, uint32_t n,
                   const uint32_t* __restrict__ src, uint32_t* mesh, unsigned long long* __restrict__ keys, uint32_t none) {
    const uint64_t j = (uint64_t)blockIdx.x * DF_THREADS + threadIdx.x;
    if (j >= n) return;
    const deform_mesh_dev& md = meshes[mesh_of_index(index_base, n_meshes, (uint32_t)j)];
    const uint32_t k = (uint32_t)j - md.index_base;
    unsigned long long key = (unsigned long long)none << 32;
    if (!md.skip && k < md.m.index_count) {
        const uint64_t w = (uint64_t)md.m.first_index + k;
        uint32_t v;
        if (src) { v = __ldg(src + j); mesh[w] = v; }
        else v = mesh[w];
        key = ((unsigned long long)(md.vertex_base + v) << 32) | (k / 3u);
    }
    keys[j] = key;
}

__global__ void __launch_bounds__(SORT_THREADS) corner_hist_kernel(const unsigned long long* __restrict__ keys, uint32_t n, int shift, uint32_t* __restrict__ hist) {
    radix_tile_hist(keys, n, shift, hist, blockIdx.x, gridDim.x);
}

__global__ void __launch_bounds__(SORT_THREADS) corner_scatter_kernel(const unsigned long long* __restrict__ keys_in, unsigned long long* __restrict__ keys_out,
                                                                      uint32_t n, int shift, const uint32_t* __restrict__ hist_scanned) {
    __shared__ uint32_t s_gbase[256];
    s_gbase[threadIdx.x] = hist_scanned[threadIdx.x * gridDim.x + blockIdx.x];
    radix_tile_scatter(keys_in, keys_out, n, shift, blockIdx.x * SORT_TILE, s_gbase);
}

// from the sorted keys: corners[p] = the triangle of sorted corner p; start[g] = the first sorted corner of vertex g (a lower bound),
// g <= n_vertices, so vertex g's list is corners[start[g] .. start[g + 1])
__global__ void __launch_bounds__(DF_THREADS)
corner_lists_kernel(const unsigned long long* __restrict__ keys, uint32_t n, uint32_t n_vertices, uint32_t* __restrict__ corners,
                    uint32_t* __restrict__ start) {
    const uint64_t i = (uint64_t)blockIdx.x * DF_THREADS + threadIdx.x;
    if (i < n) corners[i] = (uint32_t)keys[i];
    if (i <= n_vertices) {
        uint32_t lo = 0, hi = n;
        while (lo < hi) {
            const uint32_t mid = lo + ((hi - lo) >> 1);
            if ((keys[mid] >> 32) < i) lo = mid + 1; else hi = mid;
        }
        start[i] = lo;
    }
}

// ---- remesh: Mesh::validate (rend3-types/src/lib.rs:533-567) on the new counts and indices, before anything is written
// the count checks, in validate's order: the status word, R3_REMESH_APPLIED when they pass
__global__ void remesh_counts_kernel(const deform_mesh_dev* __restrict__ meshes, const uint32_t* __restrict__ counts, uint32_t n,
                                     uint32_t* __restrict__ status) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t vc = __ldg(counts + 2 * i), ic = __ldg(counts + 2 * i + 1);
    status[i] = vc > meshes[i].vertex_capacity ? R3_REMESH_OVER_CAPACITY : (ic % 3u) ? R3_REMESH_NOT_TRIANGLES
              : ic > meshes[i].index_capacity ? R3_REMESH_OVER_CAPACITY : R3_REMESH_APPLIED;
}

// one thread per set index: an index at or past its mesh's new vertex_count (only where the counts passed: the first reason stays)
__global__ void __launch_bounds__(DF_THREADS)
remesh_indices_kernel(const uint32_t* __restrict__ index_base, uint32_t n_meshes, uint32_t n, const uint32_t* __restrict__ counts,
                      const uint32_t* __restrict__ indices, uint32_t* status) {
    const uint64_t j = (uint64_t)blockIdx.x * DF_THREADS + threadIdx.x;
    if (j >= n) return;
    const uint32_t mi = mesh_of_index(index_base, n_meshes, (uint32_t)j);
    const uint32_t k = (uint32_t)j - __ldg(index_base + mi);
    if (k < __ldg(counts + 2 * mi + 1) && __ldg(indices + j) >= __ldg(counts + 2 * mi) && status[mi] == R3_REMESH_APPLIED)
        status[mi] = R3_REMESH_INDEX_OUT_OF_RANGE;
}

// the counts in force: an applied mesh takes the new ones; a rejected mesh keeps its counts and is skipped by the rest of the call
__global__ void remesh_apply_kernel(deform_mesh_dev* __restrict__ meshes, const uint32_t* __restrict__ counts, const uint32_t* __restrict__ status,
                                    uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bool ok = status[i] == R3_REMESH_APPLIED;
    if (ok) { meshes[i].m.vertex_count = __ldg(counts + 2 * i); meshes[i].m.index_count = __ldg(counts + 2 * i + 1); }
    meshes[i].skip = ok ? 0u : 1u;
}

// the supplied attributes of every applied mesh's first vertex_count vertices into its ranges: normals and tangents the build does not
// recompute, uv0 and color0 (one word).  Before the vertex stage, which reads uv0 and authored normals of other vertices.
__global__ void __launch_bounds__(DF_THREADS)
remesh_copy_kernel(const deform_mesh_dev* __restrict__ meshes, const uint32_t* __restrict__ block_mesh, const uint32_t* __restrict__ normals,
                   const uint32_t* __restrict__ tangents, const uint32_t* __restrict__ uv0, const uint32_t* __restrict__ color0, uint32_t* __restrict__ mesh) {
    const deform_mesh_dev md = meshes[__ldg(block_mesh + blockIdx.x)];
    const uint32_t v = (blockIdx.x - md.block_first) * DF_THREADS + threadIdx.x;
    if (md.skip || v >= md.m.vertex_count) return;
    const uint64_t g = (uint64_t)md.vertex_base + v;
    const uint32_t flags = md.m.flags;
    if (md.m.normal_offset != R3_ATTR_ABSENT && !(flags & R3_DEFORM_NORMALS))
        for (int j = 0; j < 3; ++j) mesh[md.m.normal_offset / 4 + 3ull * v + j] = __ldg(normals + 3 * g + j);
    if (md.m.tangent_offset != R3_ATTR_ABSENT && !(flags & R3_DEFORM_TANGENTS))
        for (int j = 0; j < 3; ++j) mesh[md.m.tangent_offset / 4 + 3ull * v + j] = __ldg(tangents + 3 * g + j);
    if (md.m.uv0_offset != R3_ATTR_ABSENT)
        for (int j = 0; j < 2; ++j) mesh[md.m.uv0_offset / 4 + 2ull * v + j] = __ldg(uv0 + 2 * g + j);
    if (md.color0_offset != R3_ATTR_ABSENT) mesh[md.color0_offset / 4 + (uint64_t)v] = __ldg(color0 + g);
}

}  // namespace

struct r3_deform_state {
    bool valid = false;                       // a set exists and no mesh-buffer write has invalidated it
    bool remesh = false;                      // the set is r3_set_remeshable_meshes' (else r3_set_deformable_meshes')
    uint32_t n_meshes = 0, n_objects = 0, n_blocks = 0, max_slot = 0, sort_passes = 0;
    uint64_t n_vertices = 0, n_indices = 0;   // the set's totals (capacities for a remesh set)
    uint32_t reads = 0;                       // READS_*: the optional streams some mesh of a remesh set reads
    std::vector<r3_deformable_mesh> meshes;   // host copy: the index ranges r3_update_mesh_buffer must not write (a deformable set)
    std::vector<r3_remeshable_mesh> remeshes; // host copy: the capacities the host form validates against (a remesh set)
    deform_mesh_dev* d_meshes = nullptr; uint32_t meshes_cap = 0;
    uint32_t* d_block_mesh = nullptr; uint32_t block_mesh_cap = 0;
    unsigned long long* d_partials = nullptr; uint64_t partials_cap = 0;
    uint32_t* d_corner_start = nullptr; uint64_t corner_start_cap = 0;
    uint32_t* d_corners = nullptr; uint64_t corners_cap = 0;
    float4* d_spheres = nullptr; uint32_t spheres_cap = 0;
    uint32_t* d_slots = nullptr; uint32_t slots_cap = 0;
    uint32_t* d_object_mesh = nullptr; uint32_t object_mesh_cap = 0;
    uint32_t* d_index_base = nullptr; uint32_t index_base_cap = 0;
    unsigned long long* d_keys[2] = {nullptr, nullptr}; uint64_t keys_cap[2] = {0, 0};
    uint32_t* d_hist = nullptr; uint64_t hist_cap = 0;
    uint32_t* d_status = nullptr; uint32_t status_cap = 0;
    std::vector<uint32_t> listed;             // host copy of the listed slots (r3_set_object_variants must not list them)
};

namespace {
// the sort's tiles address keys with 32-bit positions (r3_radix.cuh: tile * SORT_TILE + offset): a set's index total stays a whole
// tile below 2^32
constexpr uint64_t MAX_SET_INDICES = (1ull << 32) - SORT_TILE;
constexpr uint32_t READS_NORMALS = 1, READS_TANGENTS = 2, READS_UV0 = 4, READS_COLOR0 = 8;

// the invocation floors exist only while a remesh set or an object-variant set does; dropping them changes the bound
void drop_floors(r3_ctx* c) {
    if (!c->d_invocation_floor) return;
    cudaFree(c->d_invocation_floor);
    c->d_invocation_floor = nullptr; c->n_invocation_floor = 0; c->invocation_floor_cap = 0;
    c->max_invocations_valid = false;
}

int remove_set(r3_ctx* c) {
    r3_deform_state* d = c->deform;
    if (d) {
        d->valid = false; d->remesh = false; d->n_meshes = 0;
        d->meshes.clear(); d->remeshes.clear(); d->listed.clear();
    }
    return r3_rebuild_invocation_floors(c);   // the object-variant set's floors stay
}

// the invocation floor of every listed slot of a remesh set: its mesh's index_capacity
__global__ void floor_scatter_kernel(const deform_mesh_dev* __restrict__ meshes, const uint32_t* __restrict__ slots, const uint32_t* __restrict__ object_mesh,
                                     uint32_t n, uint32_t* __restrict__ floor) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) floor[slots[i]] = meshes[object_mesh[i]].index_capacity;
}
}  // namespace

int r3_rebuild_invocation_floors(r3_ctx* c) {
    const r3_deform_state* d = c->deform;
    const bool remesh = d && d->remesh && d->n_meshes;
    c->max_invocations_valid = false;
    if (!remesh && !r3_variants_have_set(c)) { drop_floors(c); return R3_OK; }
    const uint32_t n = std::max(c->n_slots, 1u);
    R3_TRY(r3_reserve_t(c, &c->d_invocation_floor, &c->invocation_floor_cap, n));
    R3_CUDA(c, cudaMemsetAsync(c->d_invocation_floor, 0, (size_t)n * 4, c->stream));
    c->n_invocation_floor = c->n_slots;
    if (remesh && d->n_objects) {
        floor_scatter_kernel<<<(d->n_objects + DF_THREADS - 1) / DF_THREADS, DF_THREADS, 0, c->stream>>>(d->d_meshes, d->d_slots, d->d_object_mesh,
                                                                                                       d->n_objects, c->d_invocation_floor);
        R3_CHECK_LAUNCH(c, "floor_scatter_kernel");
    }
    return r3_variants_scatter_floors(c);
}

const std::vector<uint32_t>* r3_deform_listed_slots(r3_ctx* c) { return c->deform && c->deform->n_meshes ? &c->deform->listed : nullptr; }

void r3_deform_destroy(r3_ctx* c) {
    drop_floors(c);
    r3_deform_state* d = c->deform;
    if (!d) return;
    cudaFree(d->d_meshes); cudaFree(d->d_block_mesh); cudaFree(d->d_partials); cudaFree(d->d_corner_start); cudaFree(d->d_corners);
    cudaFree(d->d_spheres); cudaFree(d->d_slots); cudaFree(d->d_object_mesh); cudaFree(d->d_index_base); cudaFree(d->d_keys[0]);
    cudaFree(d->d_keys[1]); cudaFree(d->d_hist); cudaFree(d->d_status);
    delete d;
    c->deform = nullptr;
}

void r3_deform_note_mesh_write(r3_ctx* c, bool whole_buffer, uint64_t byte_offset, uint64_t nbytes) {
    r3_deform_state* d = c->deform;
    if (!d || !d->valid) return;
    if (whole_buffer) { d->valid = false; return; }
    if (d->remesh) return;   // every remesh rebuilds its corner lists from the indices it writes
    for (const r3_deformable_mesh& m : d->meshes) {
        const uint64_t a = (uint64_t)m.first_index * 4, b = a + (uint64_t)m.index_count * 4;
        if (m.index_count && byte_offset < b && a < byte_offset + nbytes) { d->valid = false; return; }
    }
}

int r3_deform_grow_floors(r3_ctx* c, uint32_t n) {
    if (!c->d_invocation_floor || c->n_invocation_floor >= n) return R3_OK;
    R3_TRY(r3_reserve_t(c, &c->d_invocation_floor, &c->invocation_floor_cap, n, true));
    R3_CUDA(c, cudaMemsetAsync(c->d_invocation_floor + c->n_invocation_floor, 0, (size_t)(n - c->n_invocation_floor) * 4, c->stream));
    c->n_invocation_floor = n;
    return R3_OK;
}

namespace {

int fail_s(r3_ctx* c, int code, const std::string& msg) { return r3_fail(c, code, msg.c_str()); }

// a byte range [a, b) of the mesh buffer; `write` ranges must not meet any other range of the set
struct byte_range { uint64_t a, b; };

int check_ranges(r3_ctx* c, std::vector<byte_range>& writes, std::vector<byte_range>& reads, const char* what) {
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
    if (r3_anim_check_disjoint(r.data(), r.size() / 2, what, &msg) != R3_OK) return r3_fail(c, R3_E_INVALID, msg);
    return R3_OK;
}

// The (slot, mesh) pairs: mesh in range, slot below the slot count and named once.  *lo, *hi: the slots' hull.
int check_objects(r3_ctx* c, const char* who, const uint32_t* object_slots, const uint32_t* object_meshes, uint32_t n_objects, uint32_t n_meshes,
                  uint32_t* lo, uint32_t* hi) {
    std::vector<uint64_t> seen(((size_t)c->n_slots + 63) / 64, 0ull);
    *lo = ~0u; *hi = 0;
    for (uint32_t i = 0; i < n_objects; ++i) {
        const uint32_t s = object_slots[i];
        if (object_meshes[i] >= n_meshes) return fail_s(c, R3_E_INVALID, std::string(who) + ": object mesh out of range");
        if (s >= c->n_slots) return fail_s(c, R3_E_INVALID, std::string(who) + ": slot beyond the object buffer");
        if (seen[s >> 6] & (1ull << (s & 63u))) return fail_s(c, R3_E_INVALID, std::string(who) + ": one slot named twice");
        if (r3_variants_list(c, s)) return fail_s(c, R3_E_INVALID, std::string(who) + ": a slot listed by the object-variant set");
        seen[s >> 6] |= 1ull << (s & 63u);
        *lo = std::min(*lo, s); *hi = std::max(*hi, s);
    }
    return R3_OK;
}

int check_deform_state(r3_ctx* c, bool remesh, const char* who_state) {
    r3_deform_state* d = c->deform;
    if (!d || !d->valid || d->remesh != remesh) return r3_fail(c, R3_E_STATE, who_state);
    const char* who = remesh ? "remesh_meshes" : "deform_meshes";
    R3_TRY(r3_check_object_writer(c, who, R3_NEED_OWNED));
    if (d->n_objects) {
        if (!c->d_objects || !c->hot_valid || d->max_slot >= c->n_slots) return fail_s(c, R3_E_STATE, std::string(who) + ": a listed slot is past the slot count");
        if (d->max_slot >= c->n_mesh_spheres) return fail_s(c, R3_E_STATE, std::string(who) + ": r3_set_object_mesh_spheres does not cover every listed slot");
    }
    return R3_OK;
}

// The vertex -> corner lists of the set from its indices (`src`: a remesh's index stream, copied into the mesh buffer on the way; nullptr:
// the mesh buffer): keys, the stable radix sort on the vertex bits, the lists and their starts.
int build_corner_lists(r3_ctx* c, const uint32_t* src) {
    r3_deform_state* d = c->deform;
    const uint32_t n = (uint32_t)d->n_indices, nv = (uint32_t)d->n_vertices;
    int k = 0;
    if (n) {
        corner_keys_kernel<<<(uint32_t)(((uint64_t)n + DF_THREADS - 1) / DF_THREADS), DF_THREADS, 0, c->stream>>>(d->d_meshes, d->d_index_base, d->n_meshes, n, src, c->d_mesh,
                                                                                          d->d_keys[0], nv);
        R3_CHECK_LAUNCH(c, "corner_keys_kernel");
        const uint32_t tiles = (uint32_t)(((uint64_t)n + SORT_TILE - 1) / SORT_TILE);
        for (uint32_t pass = 0; pass < d->sort_passes; ++pass, k ^= 1) {
            const int shift = 32 + 8 * (int)pass;
            corner_hist_kernel<<<tiles, SORT_THREADS, 0, c->stream>>>(d->d_keys[k], n, shift, d->d_hist);
            R3_CHECK_LAUNCH(c, "corner_hist_kernel");
            scan_u32_kernel<<<1, 1024, 0, c->stream>>>(d->d_hist, 256u * tiles);
            R3_CHECK_LAUNCH(c, "scan_u32_kernel");
            corner_scatter_kernel<<<tiles, SORT_THREADS, 0, c->stream>>>(d->d_keys[k], d->d_keys[k ^ 1], n, shift, d->d_hist);
            R3_CHECK_LAUNCH(c, "corner_scatter_kernel");
        }
    }
    const uint64_t threads = std::max<uint64_t>(n, (uint64_t)nv + 1);
    corner_lists_kernel<<<(uint32_t)((threads + DF_THREADS - 1) / DF_THREADS), DF_THREADS, 0, c->stream>>>(d->d_keys[k], n, nv, d->d_corners, d->d_corner_start);
    R3_CHECK_LAUNCH(c, "corner_lists_kernel");
    return R3_OK;
}

void free_sort_scratch(r3_deform_state* d) {
    cudaFree(d->d_keys[0]); cudaFree(d->d_keys[1]); cudaFree(d->d_hist);
    d->d_keys[0] = d->d_keys[1] = nullptr; d->keys_cap[0] = d->keys_cap[1] = 0;
    d->d_hist = nullptr; d->hist_cap = 0;
}

// room for a set of n_meshes meshes, `blocks` vertex CTAs, the vertex and index totals and n_objects listed slots
int reserve_set(r3_ctx* c, uint32_t n_meshes, uint32_t blocks, uint64_t n_vertices, uint64_t n_indices, uint32_t n_objects) {
    if (!c->deform) c->deform = new r3_deform_state();
    r3_deform_state* d = c->deform;
    R3_TRY(r3_reserve_t(c, &d->d_meshes, &d->meshes_cap, n_meshes));
    R3_TRY(r3_reserve_t(c, &d->d_block_mesh, &d->block_mesh_cap, std::max(blocks, 1u)));
    R3_TRY(r3_reserve_t(c, &d->d_partials, &d->partials_cap, 6ull * std::max(blocks, 1u)));
    R3_TRY(r3_reserve_t(c, &d->d_corner_start, &d->corner_start_cap, n_vertices + 1));
    R3_TRY(r3_reserve_t(c, &d->d_corners, &d->corners_cap, std::max<uint64_t>(n_indices, 1)));
    R3_TRY(r3_reserve_t(c, &d->d_keys[0], &d->keys_cap[0], std::max<uint64_t>(n_indices, 1)));
    R3_TRY(r3_reserve_t(c, &d->d_keys[1], &d->keys_cap[1], std::max<uint64_t>(n_indices, 1)));
    R3_TRY(r3_reserve_t(c, &d->d_hist, &d->hist_cap, 256ull * ((n_indices + SORT_TILE - 1) / SORT_TILE) + 1));
    R3_TRY(r3_reserve_t(c, &d->d_index_base, &d->index_base_cap, n_meshes));
    R3_TRY(r3_reserve_t(c, &d->d_status, &d->status_cap, n_meshes));
    R3_TRY(r3_reserve_t(c, &d->d_spheres, &d->spheres_cap, n_meshes));
    R3_TRY(r3_reserve_t(c, &d->d_slots, &d->slots_cap, std::max(n_objects, 1u)));
    R3_TRY(r3_reserve_t(c, &d->d_object_mesh, &d->object_mesh_cap, std::max(n_objects, 1u)));
    return R3_OK;
}

// the uploads both set calls share, on the stream (the caller drains it)
int upload_set(r3_ctx* c, const std::vector<deform_mesh_dev>& dev, const std::vector<uint32_t>& block_mesh, const std::vector<uint32_t>& index_base,
               const uint32_t* object_slots, const uint32_t* object_meshes, uint32_t n_objects) {
    r3_deform_state* d = c->deform;
    R3_CUDA(c, cudaMemcpyAsync(d->d_meshes, dev.data(), dev.size() * sizeof(deform_mesh_dev), cudaMemcpyHostToDevice, c->stream));
    if (!block_mesh.empty()) R3_CUDA(c, cudaMemcpyAsync(d->d_block_mesh, block_mesh.data(), block_mesh.size() * 4, cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, cudaMemcpyAsync(d->d_index_base, index_base.data(), index_base.size() * 4, cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, cudaMemsetAsync(d->d_spheres, 0, dev.size() * 16, c->stream));
    R3_CUDA(c, cudaMemsetAsync(d->d_status, 0, dev.size() * 4, c->stream));
    if (n_objects) {
        R3_CUDA(c, cudaMemcpyAsync(d->d_slots, object_slots, (size_t)n_objects * 4, cudaMemcpyHostToDevice, c->stream));
        R3_CUDA(c, cudaMemcpyAsync(d->d_object_mesh, object_meshes, (size_t)n_objects * 4, cudaMemcpyHostToDevice, c->stream));
    }
    return R3_OK;
}

void commit_set(r3_ctx* c, bool remesh, uint32_t n_meshes, uint32_t n_objects, uint32_t blocks, uint64_t n_vertices, uint64_t n_indices, uint32_t max_slot) {
    r3_deform_state* d = c->deform;
    d->remesh = remesh;
    d->n_meshes = n_meshes; d->n_objects = n_objects; d->n_blocks = blocks; d->n_vertices = n_vertices; d->n_indices = n_indices;
    d->max_slot = max_slot;
    // passes over the bits of the largest key vertex, n_vertices itself (the sentinel of unused indices)
    uint32_t bits = 0;
    while (bits < 32 && (n_vertices >> bits)) ++bits;
    d->sort_passes = (bits + 7) / 8;
    d->valid = true;
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
        const uint32_t sort_n = r3_sort_extent(c);
        deform_objects_kernel<<<(d->n_objects + DF_THREADS - 1) / DF_THREADS, DF_THREADS, 0, c->stream>>>(
            d->d_meshes, d->d_slots, d->d_object_mesh, d->n_objects, c->n_slots, d->remesh ? 1u : 0u, d->d_spheres, c->d_mesh_spheres, reinterpret_cast<float4*>(c->d_objects),
            c->d_hot_sphere, c->d_hot_radius, c->d_centre_bits, sort_n ? c->d_sort_loc : nullptr, sort_n);
        R3_CHECK_LAUNCH(c, "deform_objects_kernel");
        r3_new_frame_epoch(c);                   // a frame-wide sort made before the deform is stale
        if (sort_n) c->locations_moved = true;   // the host batching's mirror c->sort_loc is behind the device's
    }
    return R3_OK;
}

// the streams of one remesh, in device memory
struct remesh_streams { const uint32_t* counts; const float* positions; const uint32_t* indices; const float* normals; const float* tangents; const float* uv0; const uint32_t* color0; };

int launch_remesh(r3_ctx* c, const remesh_streams& s) {
    r3_deform_state* d = c->deform;
    const uint32_t n = (uint32_t)d->n_indices, mb = (d->n_meshes + DF_THREADS - 1) / DF_THREADS;
    remesh_counts_kernel<<<mb, DF_THREADS, 0, c->stream>>>(d->d_meshes, s.counts, d->n_meshes, d->d_status);
    R3_CHECK_LAUNCH(c, "remesh_counts_kernel");
    if (n) {
        remesh_indices_kernel<<<(uint32_t)(((uint64_t)n + DF_THREADS - 1) / DF_THREADS), DF_THREADS, 0, c->stream>>>(d->d_index_base, d->n_meshes, n, s.counts, s.indices, d->d_status);
        R3_CHECK_LAUNCH(c, "remesh_indices_kernel");
    }
    remesh_apply_kernel<<<mb, DF_THREADS, 0, c->stream>>>(d->d_meshes, s.counts, d->d_status, d->n_meshes);
    R3_CHECK_LAUNCH(c, "remesh_apply_kernel");
    R3_TRY(build_corner_lists(c, s.indices));
    if (d->n_blocks && (d->reads & (READS_NORMALS | READS_TANGENTS | READS_UV0 | READS_COLOR0))) {
        remesh_copy_kernel<<<d->n_blocks, DF_THREADS, 0, c->stream>>>(d->d_meshes, d->d_block_mesh, reinterpret_cast<const uint32_t*>(s.normals),
                                                                      reinterpret_cast<const uint32_t*>(s.tangents), reinterpret_cast<const uint32_t*>(s.uv0),
                                                                      s.color0, c->d_mesh);
        R3_CHECK_LAUNCH(c, "remesh_copy_kernel");
    }
    return launch_deform(c, s.positions);
}

// the pointer checks both remesh forms share
int check_remesh_args(r3_ctx* c, const char* who, const remesh_streams& s, uint64_t n_vertices, uint64_t n_indices, uintptr_t align) {
    r3_deform_state* d = c->deform;
    if (n_vertices != d->n_vertices || n_indices != d->n_indices)
        return fail_s(c, R3_E_INVALID, std::string(who) + ": n_vertices and n_indices must be the set's total capacities");
    const bool need_v = n_vertices != 0;
    const struct { const void* p; bool needed; } ptrs[] = {
        {s.counts, true}, {s.positions, need_v}, {s.indices, n_indices != 0}, {s.normals, need_v && (d->reads & READS_NORMALS)},
        {s.tangents, need_v && (d->reads & READS_TANGENTS)}, {s.uv0, need_v && (d->reads & READS_UV0)}, {s.color0, need_v && (d->reads & READS_COLOR0)}};
    for (const auto& q : ptrs) {
        if (q.needed && !q.p) return fail_s(c, R3_E_INVALID, std::string(who) + ": a null stream that some mesh of the set reads");
        if ((uintptr_t)q.p & (align - 1)) return fail_s(c, R3_E_INVALID, std::string(who) + ": a misaligned stream (4 bytes)");
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
        return remove_set(c);
    }
    R3_TRY(r3_check_object_writer(c, "set_deformable_meshes", R3_NEED_HOT | R3_NEED_OWNED));
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
    if (n_vertices > 0x7FFFFFFFull || n_indices > MAX_SET_INDICES) return r3_fail(c, R3_E_INVALID, "set_deformable_meshes: more than 2^31 - 1 vertices or 2^32 - 2^11 indices");
    R3_TRY(check_ranges(c, writes, reads, "set_deformable_meshes: a written range overlaps another range of the set"));
    // ---- the objects
    uint32_t slot_lo, slot_hi;
    R3_TRY(check_objects(c, "set_deformable_meshes", object_slots, object_meshes, n_objects, n_meshes, &slot_lo, &slot_hi));
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
    // ---- upload, and build the vertex -> corner lists from the indices in the mesh buffer
    std::vector<deform_mesh_dev> dev(n_meshes);
    std::vector<uint32_t> block_mesh, index_base(n_meshes);
    uint32_t vb = 0, ib = 0, blocks = 0;
    for (uint32_t i = 0; i < n_meshes; ++i) {
        const r3_deformable_mesh& m = meshes[i];
        const uint32_t nb = (m.vertex_count + DF_THREADS - 1) / DF_THREADS;
        dev[i] = deform_mesh_dev{m, vb, blocks, nb, 0u, ib, m.vertex_count, m.index_count, R3_ATTR_ABSENT};
        index_base[i] = ib;
        block_mesh.insert(block_mesh.end(), nb, i);
        vb += m.vertex_count; ib += m.index_count; blocks += nb;
    }
    R3_TRY(remove_set(c));
    R3_TRY(reserve_set(c, n_meshes, blocks, n_vertices, n_indices, n_objects));
    R3_TRY(upload_set(c, dev, block_mesh, index_base, object_slots, object_meshes, n_objects));
    commit_set(c, false, n_meshes, n_objects, blocks, n_vertices, n_indices, n_objects ? slot_hi : 0);
    c->deform->meshes.assign(meshes, meshes + n_meshes);
    c->deform->listed.assign(object_slots, object_slots + n_objects);
    R3_TRY(build_corner_lists(c, nullptr));
    R3_CUDA(c, r3_stream_sync(c));   // host pointers are only borrowed for the call
    free_sort_scratch(c->deform);    // a deformable set sorts only here; a remesh set sorts in every call
    return R3_OK;
}

R3_EXPORT int r3_deform_meshes(r3_ctx* c, const float* positions, uint64_t n_floats) {
    if (!c) return R3_E_INVALID;
    R3_TRY(check_deform_state(c, false, "deform_meshes before set_deformable_meshes, or after a mesh-buffer write that replaced its indices"));
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
    R3_TRY(check_deform_state(c, false, "deform_meshes_device before set_deformable_meshes, or after a mesh-buffer write that replaced its indices"));
    if (n_floats != 3 * c->deform->n_vertices) return r3_fail(c, R3_E_INVALID, "deform_meshes_device: n_floats is not 3 x the set's vertex count");
    if ((!d_positions && n_floats) || ((uintptr_t)d_positions & 3u)) return r3_fail(c, R3_E_INVALID, "deform_meshes_device: null or misaligned positions (4 bytes)");
    cudaSetDevice(c->device);
    return launch_deform(c, d_positions);
}

R3_EXPORT int r3_readback_deformable_mesh_spheres(r3_ctx* c, float* out, uint32_t first, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (!c->deform || !c->deform->n_meshes) return r3_fail(c, R3_E_STATE, "readback_deformable_mesh_spheres before set_deformable_meshes or set_remeshable_meshes");
    if ((!out && n) || (uint64_t)first + n > c->deform->n_meshes) return r3_fail(c, R3_E_INVALID, "readback_deformable_mesh_spheres: range outside the set");
    if (n == 0) return R3_OK;
    cudaSetDevice(c->device);
    R3_CUDA(c, cudaMemcpyAsync(out, c->deform->d_spheres + first, (size_t)n * 16, cudaMemcpyDeviceToHost, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    return R3_OK;
}

R3_EXPORT int r3_set_remeshable_meshes(r3_ctx* c, const r3_remeshable_mesh* meshes, uint32_t n_meshes, const uint32_t* object_slots,
                                       const uint32_t* object_meshes, uint32_t n_objects) {
    if (!c) return R3_E_INVALID;
    if ((!meshes && n_meshes) || ((!object_slots || !object_meshes) && n_objects)) return r3_fail(c, R3_E_INVALID, "set_remeshable_meshes: null");
    if (n_meshes == 0) {
        if (n_objects) return r3_fail(c, R3_E_INVALID, "set_remeshable_meshes: objects without meshes");
        return remove_set(c);
    }
    R3_TRY(r3_check_object_writer(c, "set_remeshable_meshes", R3_NEED_HOT | R3_NEED_OWNED));
    // ---- the records: every capacity-sized range inside the buffer, and every range (all are written) disjoint from every other
    const uint64_t buf = c->mesh_words * 4;
    uint64_t n_vertices = 0, n_indices = 0;
    uint32_t reads = 0;
    std::vector<byte_range> writes, none;
    for (uint32_t i = 0; i < n_meshes; ++i) {
        const r3_remeshable_mesh m = meshes[i];
        if (m.flags & ~DF_ALL_FLAGS) return r3_fail(c, R3_E_INVALID, "set_remeshable_meshes: unknown flag bits");
        if (m.position_offset == R3_ATTR_ABSENT) return r3_fail(c, R3_E_INVALID, "set_remeshable_meshes: a mesh without positions");
        if ((m.flags & R3_DEFORM_NORMALS) && m.normal_offset == R3_ATTR_ABSENT) return r3_fail(c, R3_E_INVALID, "set_remeshable_meshes: normals recomputed without a normal range");
        if ((m.flags & R3_DEFORM_TANGENTS) && (m.tangent_offset == R3_ATTR_ABSENT || m.uv0_offset == R3_ATTR_ABSENT || m.normal_offset == R3_ATTR_ABSENT))
            return r3_fail(c, R3_E_INVALID, "set_remeshable_meshes: tangents recomputed without tangent, uv0 and normal ranges");
        const struct { uint32_t off; uint32_t bytes; } attrs[] = {{m.position_offset, 12}, {m.normal_offset, 12}, {m.tangent_offset, 12},
                                                                  {m.uv0_offset, 8}, {m.color0_offset, 4}};
        for (const auto& a : attrs) {
            if (a.off == R3_ATTR_ABSENT) continue;
            if (a.off & 3u) return r3_fail(c, R3_E_INVALID, "set_remeshable_meshes: an offset that is not a multiple of 4");
            const uint64_t b = (uint64_t)a.off + (uint64_t)a.bytes * m.vertex_capacity;
            if (b > buf) return r3_fail(c, R3_E_INVALID, "set_remeshable_meshes: a range outside the mesh buffer");
            if (b > a.off) writes.push_back({a.off, b});
        }
        const uint64_t ia = (uint64_t)m.first_index * 4, ib = ia + 4ull * m.index_capacity;
        if (ib > buf) return r3_fail(c, R3_E_INVALID, "set_remeshable_meshes: a range outside the mesh buffer");
        if (ib > ia) writes.push_back({ia, ib});
        if (m.normal_offset != R3_ATTR_ABSENT && !(m.flags & R3_DEFORM_NORMALS)) reads |= READS_NORMALS;
        if (m.tangent_offset != R3_ATTR_ABSENT && !(m.flags & R3_DEFORM_TANGENTS)) reads |= READS_TANGENTS;
        if (m.uv0_offset != R3_ATTR_ABSENT) reads |= READS_UV0;
        if (m.color0_offset != R3_ATTR_ABSENT) reads |= READS_COLOR0;
        n_vertices += m.vertex_capacity;
        n_indices += m.index_capacity;
    }
    if (n_vertices > 0x7FFFFFFFull || n_indices > MAX_SET_INDICES) return r3_fail(c, R3_E_INVALID, "set_remeshable_meshes: more than 2^31 - 1 vertices or 2^32 - 2^11 indices");
    R3_TRY(check_ranges(c, writes, none, "set_remeshable_meshes: a range overlaps another range of the set"));
    uint32_t slot_lo, slot_hi;
    R3_TRY(check_objects(c, "set_remeshable_meshes", object_slots, object_meshes, n_objects, n_meshes, &slot_lo, &slot_hi));
    // ---- the listed records draw their meshes
    cudaSetDevice(c->device);
    std::vector<r3_object> recs(n_objects ? slot_hi - slot_lo + 1 : 0);
    if (!recs.empty()) {
        R3_CUDA(c, cudaMemcpyAsync(recs.data(), c->d_objects + slot_lo, recs.size() * sizeof(r3_object), cudaMemcpyDeviceToHost, c->stream));
        R3_CUDA(c, r3_stream_sync(c));
    }
    for (uint32_t i = 0; i < n_objects; ++i) {
        const r3_object& o = recs[object_slots[i] - slot_lo];
        const r3_remeshable_mesh& m = meshes[object_meshes[i]];
        if (o.first_index != m.first_index || o.index_count > m.index_capacity || o.attr_offset[R3_ATTR_POSITION] != m.position_offset ||
            o.attr_offset[R3_ATTR_NORMAL] != m.normal_offset || o.attr_offset[R3_ATTR_TANGENT] != m.tangent_offset ||
            o.attr_offset[R3_ATTR_UV0] != m.uv0_offset || o.attr_offset[R3_ATTR_COLOR0] != m.color0_offset)
            return r3_fail(c, R3_E_INVALID, "set_remeshable_meshes: a slot's record does not draw its mesh");
    }
    // ---- upload; the counts in force start at 0
    std::vector<deform_mesh_dev> dev(n_meshes);
    std::vector<uint32_t> block_mesh, index_base(n_meshes);
    uint32_t vb = 0, ib = 0, blocks = 0;
    for (uint32_t i = 0; i < n_meshes; ++i) {
        const r3_remeshable_mesh& m = meshes[i];
        const uint32_t nb = (m.vertex_capacity + DF_THREADS - 1) / DF_THREADS;
        const r3_deformable_mesh dm{m.position_offset, m.normal_offset, m.tangent_offset, m.uv0_offset, m.first_index, 0u, 0u, m.flags};
        dev[i] = deform_mesh_dev{dm, vb, blocks, nb, 0u, ib, m.vertex_capacity, m.index_capacity, m.color0_offset};
        index_base[i] = ib;
        block_mesh.insert(block_mesh.end(), nb, i);
        vb += m.vertex_capacity; ib += m.index_capacity; blocks += nb;
    }
    R3_TRY(remove_set(c));
    R3_TRY(reserve_set(c, n_meshes, blocks, n_vertices, n_indices, n_objects));
    R3_TRY(upload_set(c, dev, block_mesh, index_base, object_slots, object_meshes, n_objects));
    commit_set(c, true, n_meshes, n_objects, blocks, n_vertices, n_indices, n_objects ? slot_hi : 0);
    c->deform->listed.assign(object_slots, object_slots + n_objects);
    // the invocation floors: the listed slots' index_capacity (and the object-variant set's), zero elsewhere
    R3_TRY(r3_rebuild_invocation_floors(c));
    c->deform->reads = reads;
    c->deform->remeshes.assign(meshes, meshes + n_meshes);
    R3_CUDA(c, r3_stream_sync(c));   // host pointers are only borrowed for the call
    return R3_OK;
}

R3_EXPORT int r3_remesh_meshes(r3_ctx* c, const uint32_t* counts, const float* positions, const uint32_t* indices, const float* normals,
                               const float* tangents, const float* uv0, const uint32_t* color0, uint64_t n_vertices, uint64_t n_indices) {
    if (!c) return R3_E_INVALID;
    R3_TRY(check_deform_state(c, true, "remesh_meshes before set_remeshable_meshes, or after r3_set_mesh_buffer"));
    const remesh_streams h{counts, positions, indices, normals, tangents, uv0, color0};
    R3_TRY(check_remesh_args(c, "remesh_meshes", h, n_vertices, n_indices, 1));
    r3_deform_state* d = c->deform;
    // Mesh::validate on every mesh before anything is written
    uint64_t ib = 0;
    for (uint32_t i = 0; i < d->n_meshes; ++i) {
        const r3_remeshable_mesh& m = d->remeshes[i];
        const uint32_t vc = counts[2 * i], ic = counts[2 * i + 1];
        if (vc > m.vertex_capacity || ic > m.index_capacity) return r3_fail(c, R3_E_INVALID, "remesh_meshes: a count above its capacity");
        if (ic % 3) return r3_fail(c, R3_E_INVALID, "remesh_meshes: index_count is not a multiple of 3");
        for (uint32_t k = 0; k < ic; ++k)
            if (indices[ib + k] >= vc) return r3_fail(c, R3_E_INVALID, "remesh_meshes: an index >= vertex_count");
        ib += m.index_capacity;
    }
    // one copy per stream into the scratch, 16-byte aligned pieces
    const uint64_t sizes[7] = {8ull * d->n_meshes, 12 * n_vertices, 4 * n_indices, (d->reads & READS_NORMALS) ? 12 * n_vertices : 0,
                               (d->reads & READS_TANGENTS) ? 12 * n_vertices : 0, (d->reads & READS_UV0) ? 8 * n_vertices : 0,
                               (d->reads & READS_COLOR0) ? 4 * n_vertices : 0};
    const void* src[7] = {counts, positions, indices, normals, tangents, uv0, color0};
    uint64_t off[7], total = 0;
    for (int k = 0; k < 7; ++k) { off[k] = total; total += (sizes[k] + 15) & ~15ull; }
    cudaSetDevice(c->device);
    R3_TRY(r3_reserve(c, &c->d_scratch, &c->scratch_cap, std::max<uint64_t>(total, 16), 1, false, false));
    uint8_t* base = (uint8_t*)c->d_scratch;
    for (int k = 0; k < 7; ++k)
        if (sizes[k]) R3_CUDA(c, cudaMemcpyAsync(base + off[k], src[k], sizes[k], cudaMemcpyHostToDevice, c->stream));
    const remesh_streams s{(const uint32_t*)(base + off[0]), (const float*)(base + off[1]), (const uint32_t*)(base + off[2]),
                           (const float*)(base + off[3]), (const float*)(base + off[4]), (const float*)(base + off[5]), (const uint32_t*)(base + off[6])};
    R3_TRY(launch_remesh(c, s));
    R3_CUDA(c, r3_stream_sync(c));   // host pointers are only borrowed for the call; the only drain
    return R3_OK;
}

R3_EXPORT int r3_remesh_meshes_device(r3_ctx* c, const uint32_t* d_counts, const float* d_positions, const uint32_t* d_indices, const float* d_normals,
                                      const float* d_tangents, const float* d_uv0, const uint32_t* d_color0, uint64_t n_vertices, uint64_t n_indices) {
    if (!c) return R3_E_INVALID;
    R3_TRY(check_deform_state(c, true, "remesh_meshes_device before set_remeshable_meshes, or after r3_set_mesh_buffer"));
    const remesh_streams s{d_counts, d_positions, d_indices, d_normals, d_tangents, d_uv0, d_color0};
    R3_TRY(check_remesh_args(c, "remesh_meshes_device", s, n_vertices, n_indices, 4));
    cudaSetDevice(c->device);
    return launch_remesh(c, s);
}

R3_EXPORT int r3_readback_remesh_status(r3_ctx* c, uint32_t* status, uint32_t* counts_or_null, uint32_t first, uint32_t n) {
    if (!c) return R3_E_INVALID;
    r3_deform_state* d = c->deform;
    if (!d || !d->n_meshes || !d->remesh) return r3_fail(c, R3_E_STATE, "readback_remesh_status before set_remeshable_meshes");
    if ((!status && n) || (uint64_t)first + n > d->n_meshes) return r3_fail(c, R3_E_INVALID, "readback_remesh_status: range outside the set");
    if (n == 0) return R3_OK;
    cudaSetDevice(c->device);
    std::vector<deform_mesh_dev> dev(counts_or_null ? n : 0);
    R3_CUDA(c, cudaMemcpyAsync(status, d->d_status + first, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream));
    if (counts_or_null) R3_CUDA(c, cudaMemcpyAsync(dev.data(), d->d_meshes + first, (size_t)n * sizeof(deform_mesh_dev), cudaMemcpyDeviceToHost, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    for (uint32_t i = 0; i < (counts_or_null ? n : 0u); ++i) { counts_or_null[2 * i] = dev[i].m.vertex_count; counts_or_null[2 * i + 1] = dev[i].m.index_count; }
    return R3_OK;
}
