// r3_object_transforms.cu — Renderer::set_object_transform (rend3/src/managers/object.rs:302-316) for many objects at once, from host or
// device memory: r3_set_object_mesh_spheres, r3_set_object_transforms, r3_set_object_transforms_device.
//
// A moved object brings 64 bytes of new information, its matrix; the world bounding sphere (mesh sphere.apply_transform,
// util/frustum.rs:22-32) and the sort location (transform_point3a(ZERO)) are functions of it and of the mesh sphere, which stays
// resident per slot.  One kernel reads matrix, mesh sphere and (sparse form) slot and writes everything that depends on them: float4
// #0-4 of the record, the cull + bake's dense copies (rows_xyz, rows_w, spheres, radii, the affine and centre bits) and the sort
// location — about 260 B per object, HBM-bound.  `enabled`, the cold fields, key and flags are never touched.  Arithmetic: rule R12's object half (DESIGN.md §2),
// one IEEE f32 operation at a time, never contracted (-fmad=false and the _rn intrinsics).
//
// Layout: four lanes per object, lane k owning column k as one float4 (16-byte loads and stores, 64-byte runs per object); a warp walks
// 32 consecutive entries in four steps of eight.  The lanes of an object exchange the columns' xyz by shuffles and each evaluates the
// sums in the rule's order.  In the dense form entry i is slot i, so a warp owns one 32-slot word of the affine and of the centre bits
// and stores them whole; only a ragged last word and the sparse form use atomics, as split_slots_kernel does.
//
// The same unit switches prepared slots on and off (ObjectManager::add into a prepared slot / remove, object.rs:122-160, 330-342):
// r3_set_objects_enabled, r3_set_objects_enabled_device write the record's `enabled` word, the enabled bit and the live bit of each
// listed slot — 4 B + 2 bits per entry, from 1 B (dense) or 5 B (sparse) read.
#include <cstring>
#include <vector>

#include "r3_common.cuh"

namespace {

constexpr uint32_t OT_THREADS = 256;

template <bool SPARSE>
__global__ void __launch_bounds__(OT_THREADS, 4)
object_transforms_kernel(const float4* __restrict__ mats, const uint32_t* __restrict__ slots, uint32_t n, uint32_t n_slots, const float4* __restrict__ mesh_spheres,
                         float4* __restrict__ objects, float* __restrict__ rows_xyz, float* __restrict__ rows_w, float4* __restrict__ spheres,
                         float* __restrict__ radii, uint32_t* __restrict__ affine_bits, uint32_t* __restrict__ centre_bits, float* __restrict__ sort_loc,
                         uint32_t sort_n) {
    const uint32_t lane = threadIdx.x & 31u, k = lane & 3u, g = lane >> 2, first = lane & ~3u;
    const uint32_t wtile = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, base = wtile * 32u;
    if (base >= n) return;   // the whole warp
    uint32_t abits = 0, cbits = 0;
#pragma unroll
    for (uint32_t it = 0; it < 4; ++it) {
        const uint32_t i = base + it * 8u + g;
        uint32_t s = n_slots;
        if (i < n) s = SPARSE ? __ldg(slots + i) : i;
        const bool ok = s < n_slots;   // out-of-range writes are dropped (ScatterCopy's robust access)
        float4 col = make_float4(0.f, 0.f, 0.f, 0.f), ms = col;
        if (ok) { col = __ldcs(&mats[(size_t)i * 4 + k]); ms = __ldg(&mesh_spheres[s]); }
        float x[4], y[4], z[4];   // xyz of the four columns
#pragma unroll
        for (uint32_t j = 0; j < 4; ++j) {
            x[j] = __shfl_sync(0xFFFFFFFFu, col.x, first + j); y[j] = __shfl_sync(0xFFFFFFFFu, col.y, first + j); z[j] = __shfl_sync(0xFFFFFFFFu, col.z, first + j);
        }
        const uint32_t a = __ballot_sync(0xFFFFFFFFu, ok && __float_as_uint(col.w) == affine_w_bits(k));
        const bool affine = ((a >> first) & 0xFu) == 0xFu;
        // BoundingSphere::apply_transform; every lane of the object evaluates it (zeros when !ok)
        const float4 sph = sphere_apply_transform_rn(x, y, z, ms);
        // the four lanes of an object agree, so the ballot carries each object's centre bit four times
        const uint32_t cb = __ballot_sync(0xFFFFFFFFu, ok && centre_is_translation(sph.x, sph.y, sph.z, x[3], y[3], z[3]));
        const bool centred = (cb >> first) & 1u;
        if (!SPARSE) {
#pragma unroll
            for (uint32_t q = 0; q < 8; ++q) {
                abits |= (((a >> (4u * q)) & 0xFu) == 0xFu ? 1u : 0u) << (it * 8u + q);
                cbits |= ((cb >> (4u * q)) & 1u) << (it * 8u + q);
            }
        }
        if (ok) {
            objects[(size_t)s * 8 + k] = col;
            float* xyz = rows_xyz + (size_t)s * 12 + k;
            xyz[0] = col.x; xyz[4] = col.y; xyz[8] = col.z;
            rows_w[(size_t)s * 4 + k] = col.w;
            if (k == 0) objects[(size_t)s * 8 + 4] = sph;
            else if (k == 1) { spheres[s] = sph; radii[s] = sph.w; }
            else if (k == 2) {
                // location = transform_point3a(Vec3A::ZERO): w + ((x * 0 + y * 0) + z * 0) per component — NaN for an inf axis
                if (sort_loc && s < sort_n) {
                    float* l = sort_loc + 3 * (size_t)s;
                    l[0] = add_rn(x[3], add_rn(add_rn(mul_rn(x[0], 0.0f), mul_rn(x[1], 0.0f)), mul_rn(x[2], 0.0f)));
                    l[1] = add_rn(y[3], add_rn(add_rn(mul_rn(y[0], 0.0f), mul_rn(y[1], 0.0f)), mul_rn(y[2], 0.0f)));
                    l[2] = add_rn(z[3], add_rn(add_rn(mul_rn(z[0], 0.0f), mul_rn(z[1], 0.0f)), mul_rn(z[2], 0.0f)));
                }
            } else if (SPARSE) {
                const uint32_t bit = 1u << (s & 31u);   // other slots of the word may be written by other warps
                if (affine) atomicOr(&affine_bits[s >> 5], bit);
                else atomicAnd(&affine_bits[s >> 5], ~bit);
                if (centred) atomicOr(&centre_bits[s >> 5], bit);
                else atomicAnd(&centre_bits[s >> 5], ~bit);
            }
        }
    }
    if (!SPARSE && lane == 0) {
        if (n - base >= 32u) { affine_bits[wtile] = abits; centre_bits[wtile] = cbits; }
        else {   // the last word also holds slots past n: they keep their bits
            const uint32_t mask = (1u << (n - base)) - 1u;
            atomicAnd(&affine_bits[wtile], ~mask | abits);
            atomicOr(&affine_bits[wtile], abits);
            atomicAnd(&centre_bits[wtile], ~mask | cbits);
            atomicOr(&centre_bits[wtile], cbits);
        }
    }
}

__global__ void scatter_mesh_spheres_kernel(const float4* __restrict__ src, const uint32_t* __restrict__ slots, uint32_t n, float4* __restrict__ dst) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[slots[i]] = src[i];
}

// every slot below `limit` and no slot named twice (two entries' stores would land in an unspecified order)
int check_slots(r3_ctx* c, const uint32_t* slots, uint32_t n, uint32_t limit, const char* beyond, const char* twice) {
    std::vector<uint64_t> seen(((size_t)limit + 63) / 64, 0ull);
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t s = slots[i];
        if (s >= limit) return r3_fail(c, R3_E_INVALID, beyond);
        const uint64_t bit = 1ull << (s & 63u);
        if (seen[s >> 6] & bit) return r3_fail(c, R3_E_INVALID, twice);
        seen[s >> 6] |= bit;
    }
    return R3_OK;
}

int check_state(r3_ctx* c) {
    if (!c->d_objects || !c->hot_valid) return r3_fail(c, R3_E_STATE, "set_object_transforms before set_objects");
    if (c->n_mesh_spheres < c->n_slots) return r3_fail(c, R3_E_STATE, "set_object_transforms: r3_set_object_mesh_spheres does not cover every slot");
    if (c->objects_borrowed) return r3_fail(c, R3_E_STATE, "set_object_transforms: the object buffer is borrowed (r3_set_objects_device)");
    return R3_OK;
}

int launch_transforms(r3_ctx* c, const uint32_t* d_slots, const float* d_mats, uint32_t n) {
    const uint32_t sort_n = c->have_live ? (uint32_t)c->sort_key.size() : 0u;
    const uint32_t ctas = (uint32_t)(((uint64_t)n + OT_THREADS - 1) / OT_THREADS);   // a warp walks 32 entries: 256 per CTA
    auto kernel = d_slots ? object_transforms_kernel<true> : object_transforms_kernel<false>;
    kernel<<<ctas, OT_THREADS, 0, c->stream>>>(reinterpret_cast<const float4*>(d_mats), d_slots, n, c->n_slots, c->d_mesh_spheres, reinterpret_cast<float4*>(c->d_objects),
                                               reinterpret_cast<float*>(c->d_hot_xyz), reinterpret_cast<float*>(c->d_hot_w), c->d_hot_sphere, c->d_hot_radius,
                                               c->d_affine_bits, c->d_centre_bits, sort_n ? c->d_sort_loc : nullptr, sort_n);
    R3_CHECK_LAUNCH(c, "object_transforms_kernel");
    r3_new_frame_epoch(c);                       // a frame-wide sort made before the move is stale
    if (sort_n) c->locations_moved = true;       // the host batching's mirror c->sort_loc is behind the device's
    return R3_OK;
}

// ---- ObjectManager::add into a prepared slot / remove: r3_set_objects_enabled, r3_set_objects_enabled_device
// Entry i makes slot s present or absent: the record's `enabled` word (u32 @116), the slot's bit of the cull + bake's enabled bits and,
// below sort_n, its live bit.  Nothing else of the record, the hot arrays or the sort facts changes.
constexpr uint32_t EN_THREADS = 256;
constexpr uint32_t EN_WORD = offsetof(r3_object, enabled) / 4;

// sparse: one thread per entry; slots of one bit word come from different threads, so the words take atomics
__global__ void __launch_bounds__(EN_THREADS)
objects_enabled_sparse_kernel(const uint32_t* __restrict__ slots, const uint8_t* __restrict__ enabled, uint32_t n, uint32_t n_slots,
                              uint32_t* __restrict__ objects, uint32_t* __restrict__ enabled_bits, uint32_t* __restrict__ live_bits, uint32_t sort_n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = __ldg(slots + i);
    if (s >= n_slots) return;   // out-of-range writes are dropped (ScatterCopy's robust access)
    const bool on = __ldg(enabled + i) != 0;
    objects[(size_t)s * 32 + EN_WORD] = on ? 1u : 0u;
    const uint32_t bit = 1u << (s & 31u);
    if (on) atomicOr(&enabled_bits[s >> 5], bit);
    else atomicAnd(&enabled_bits[s >> 5], ~bit);
    if (s < sort_n) {
        if (on) atomicOr(&live_bits[s >> 5], bit);
        else atomicAnd(&live_bits[s >> 5], ~bit);
    }
}

// *word = (*word & ~mask) | (bits & mask): a plain store when the warp owns the whole word, atomics when slots past the range share it
__device__ __forceinline__ void store_bits(uint32_t* word, uint32_t bits, uint32_t mask) {
    if (mask == 0xFFFFFFFFu) *word = bits;
    else if (mask) { atomicAnd(word, ~mask | bits); atomicOr(word, bits & mask); }
}

// dense: entry i is slot i; a warp owns one 32-slot word, ballots the 32 flags and stores the bit words whole
__global__ void __launch_bounds__(EN_THREADS)
objects_enabled_dense_kernel(const uint8_t* __restrict__ enabled, uint32_t n, uint32_t* __restrict__ objects, uint32_t* __restrict__ enabled_bits,
                             uint32_t* __restrict__ live_bits, uint32_t sort_n) {
    const uint32_t lane = threadIdx.x & 31u, wtile = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, base = wtile * 32u;
    if (base >= n) return;   // the whole warp
    const uint32_t s = base + lane;
    const bool on = s < n && __ldg(enabled + s) != 0;
    const uint32_t bits = __ballot_sync(0xFFFFFFFFu, on);
    if (s < n) objects[(size_t)s * 32 + EN_WORD] = on ? 1u : 0u;
    if (lane == 0) {
        const auto below = [base](uint32_t end) { return end >= base + 32u ? 0xFFFFFFFFu : end > base ? (1u << (end - base)) - 1u : 0u; };
        store_bits(&enabled_bits[wtile], bits, below(n));
        if (live_bits) store_bits(&live_bits[wtile], bits, below(n < sort_n ? n : sort_n));
    }
}

int check_presence_state(r3_ctx* c, const char* who) {
    if (!c->d_objects || !c->hot_valid) return r3_fail(c, R3_E_STATE, who);
    if (c->objects_borrowed) return r3_fail(c, R3_E_STATE, "set_objects_enabled: the object buffer is borrowed (r3_set_objects_device)");
    return R3_OK;
}

int launch_enabled(r3_ctx* c, const uint32_t* d_slots, const uint8_t* d_enabled, uint32_t n) {
    const uint32_t sort_n = c->have_live ? (uint32_t)c->sort_key.size() : 0u;
    uint32_t* objects = reinterpret_cast<uint32_t*>(c->d_objects);
    uint32_t* live = sort_n ? c->d_live_bits : nullptr;
    const uint32_t ctas = (uint32_t)(((uint64_t)n + EN_THREADS - 1) / EN_THREADS);
    if (d_slots) objects_enabled_sparse_kernel<<<ctas, EN_THREADS, 0, c->stream>>>(d_slots, d_enabled, n, c->n_slots, objects, c->d_enabled_bits, live, sort_n);
    else objects_enabled_dense_kernel<<<ctas, EN_THREADS, 0, c->stream>>>(d_enabled, n, objects, c->d_enabled_bits, live, sort_n);
    R3_CHECK_LAUNCH(c, "objects_enabled_kernel");
    r3_new_frame_epoch(c);
    return R3_OK;
}

}  // namespace

R3_EXPORT int r3_set_objects_enabled(r3_ctx* c, const uint32_t* slots, const uint8_t* enabled, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (n == 0) return R3_OK;
    if (!enabled) return r3_fail(c, R3_E_INVALID, "set_objects_enabled: null");
    R3_TRY(check_presence_state(c, "set_objects_enabled before set_objects"));
    if (!slots && n > c->n_slots) return r3_fail(c, R3_E_INVALID, "set_objects_enabled: more flags than slots");
    if (slots) R3_TRY(check_slots(c, slots, n, c->n_slots, "set_objects_enabled: slot beyond the object buffer", "set_objects_enabled: one slot named twice"));
    cudaSetDevice(c->device);
    R3_TRY(r3_reserve(c, &c->d_scratch, &c->scratch_cap, (uint64_t)n * 5, 1, false, false));
    uint32_t* d_slots = slots ? (uint32_t*)c->d_scratch : nullptr;
    uint8_t* d_enabled = (uint8_t*)c->d_scratch + (slots ? (size_t)n * 4 : 0);
    if (slots) R3_CUDA(c, cudaMemcpyAsync(d_slots, slots, (size_t)n * 4, cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, cudaMemcpyAsync(d_enabled, enabled, n, cudaMemcpyHostToDevice, c->stream));
    R3_TRY(launch_enabled(c, d_slots, d_enabled, n));
    R3_CUDA(c, r3_stream_sync(c));               // host pointers are only borrowed for the call
    r3_presence_set_host(c, slots, enabled, n);  // the host sees every entry: its mirrors stay exact
    return R3_OK;
}

R3_EXPORT int r3_set_objects_enabled_device(r3_ctx* c, const uint32_t* d_slots, const uint8_t* d_enabled, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (n == 0) return R3_OK;
    if (!d_enabled || ((uintptr_t)d_slots & 3u)) return r3_fail(c, R3_E_INVALID, "set_objects_enabled_device: null or misaligned pointer (slots: 4 bytes)");
    R3_TRY(check_presence_state(c, "set_objects_enabled_device before set_objects"));
    if (!d_slots && n > c->n_slots) return r3_fail(c, R3_E_INVALID, "set_objects_enabled_device: more flags than slots");
    cudaSetDevice(c->device);
    R3_TRY(launch_enabled(c, d_slots, d_enabled, n));
    c->presence_on_device = true;                // which slots are live is now known on the device only
    r3_presence_derive(c);
    return R3_OK;
}

R3_EXPORT int r3_set_object_mesh_spheres(r3_ctx* c, const uint32_t* slots, const float* center_radius, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (!center_radius && n) return r3_fail(c, R3_E_INVALID, "set_object_mesh_spheres: null");
    cudaSetDevice(c->device);
    if (!slots) {
        R3_TRY(r3_reserve_t(c, &c->d_mesh_spheres, &c->mesh_spheres_cap, n));
        if (n) R3_CUDA(c, cudaMemcpyAsync(c->d_mesh_spheres, center_radius, (size_t)n * 16, cudaMemcpyHostToDevice, c->stream));
        R3_CUDA(c, r3_stream_sync(c));           // host pointer is only borrowed for the call
        c->n_mesh_spheres = n;
        return R3_OK;
    }
    if (n == 0) return R3_OK;
    R3_TRY(check_slots(c, slots, n, c->n_mesh_spheres, "set_object_mesh_spheres: slot beyond the mesh spheres", "set_object_mesh_spheres: one slot named twice"));
    R3_TRY(r3_reserve(c, &c->d_scratch, &c->scratch_cap, (uint64_t)n * 20, 1, false, false));
    float4* d_src = (float4*)c->d_scratch;
    uint32_t* d_slots = (uint32_t*)((uint8_t*)c->d_scratch + (size_t)n * 16);
    R3_CUDA(c, cudaMemcpyAsync(d_src, center_radius, (size_t)n * 16, cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, cudaMemcpyAsync(d_slots, slots, (size_t)n * 4, cudaMemcpyHostToDevice, c->stream));
    scatter_mesh_spheres_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>(d_src, d_slots, n, c->d_mesh_spheres);
    R3_CHECK_LAUNCH(c, "scatter_mesh_spheres_kernel");
    R3_CUDA(c, r3_stream_sync(c));
    return R3_OK;
}

R3_EXPORT int r3_set_object_transforms(r3_ctx* c, const uint32_t* slots, const float* mat4s, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (n == 0) return R3_OK;
    if (!mat4s) return r3_fail(c, R3_E_INVALID, "set_object_transforms: null");
    R3_TRY(check_state(c));
    if (!slots && n > c->n_slots) return r3_fail(c, R3_E_INVALID, "set_object_transforms: more matrices than slots");
    if (slots) R3_TRY(check_slots(c, slots, n, c->n_slots, "set_object_transforms: slot beyond the object buffer", "set_object_transforms: one slot named twice"));
    cudaSetDevice(c->device);
    R3_TRY(r3_reserve(c, &c->d_scratch, &c->scratch_cap, (uint64_t)n * 68, 1, false, false));
    float* d_mats = (float*)c->d_scratch;
    uint32_t* d_slots = slots ? (uint32_t*)((uint8_t*)c->d_scratch + (size_t)n * 64) : nullptr;
    R3_CUDA(c, cudaMemcpyAsync(d_mats, mat4s, (size_t)n * 64, cudaMemcpyHostToDevice, c->stream));
    if (slots) R3_CUDA(c, cudaMemcpyAsync(d_slots, slots, (size_t)n * 4, cudaMemcpyHostToDevice, c->stream));
    R3_TRY(launch_transforms(c, d_slots, d_mats, n));
    R3_CUDA(c, r3_stream_sync(c));               // host pointers are only borrowed for the call; the only drain
    return R3_OK;
}

R3_EXPORT int r3_set_object_transforms_device(r3_ctx* c, const uint32_t* d_slots, const float* d_mat4s, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (n == 0) return R3_OK;
    if (!d_mat4s || ((uintptr_t)d_mat4s & 15u) || ((uintptr_t)d_slots & 3u)) return r3_fail(c, R3_E_INVALID, "set_object_transforms_device: null or misaligned pointer (matrices: 16 bytes)");
    R3_TRY(check_state(c));
    if (!d_slots && n > c->n_slots) return r3_fail(c, R3_E_INVALID, "set_object_transforms_device: more matrices than slots");
    cudaSetDevice(c->device);
    return launch_transforms(c, d_slots, d_mat4s, n);
}

// r3_resize_objects: the mesh spheres, once set, grow with the slots; the new ones are zero spheres
int r3_grow_mesh_spheres(r3_ctx* c, uint32_t n) {
    if (!c->d_mesh_spheres || c->n_mesh_spheres >= n) return R3_OK;
    if (n > c->mesh_spheres_cap) R3_TRY(r3_reserve_t(c, &c->d_mesh_spheres, &c->mesh_spheres_cap, r3_hot_capacity(n), true));
    R3_CUDA(c, cudaMemsetAsync(c->d_mesh_spheres + c->n_mesh_spheres, 0, (size_t)(n - c->n_mesh_spheres) * 16, c->stream));
    c->n_mesh_spheres = n;
    return R3_OK;
}

// Host batching sorts by the host mirror c->sort_loc.  After a move the device's locations are ahead of it, and for the device form the
// host does not know which slots moved: stage enqueues a copy of the whole array into the mirror (*staged = true when it did); it is
// complete once the caller has drained the stream, which the host batching does anyway for the visible list.
int r3_stage_moved_locations(r3_ctx* c, bool* staged) {
    *staged = false;
    if (!c->locations_moved) return R3_OK;
    c->locations_moved = false;
    const size_t sort_n = c->have_live ? c->sort_key.size() : 0u;
    if (sort_n == 0 || !c->d_sort_loc) return R3_OK;
    R3_CUDA(c, cudaMemcpyAsync(c->sort_loc.data(), c->d_sort_loc, sort_n * 12, cudaMemcpyDeviceToHost, c->stream));
    *staged = true;
    return R3_OK;
}
