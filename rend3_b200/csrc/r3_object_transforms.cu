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
//
// And it switches objects between prepared mesh and material variants (ObjectManager::add with another mesh kind or material,
// object.rs:122-160, 267-284): r3_set_object_variants, r3_switch_object_variants, r3_switch_object_variants_device.  A switch writes what
// the re-add writes — the record's mesh range, material and attribute offsets, the world sphere of the variant's mesh sphere moved by the
// slot's transform (read from the cull + bake's rows, 48 B), the cull + bake's sphere copies and centre bit, the mesh sphere, and the
// sort key and location — about 190 B per entry from a 64-B variant record that stays in L2.
#include <algorithm>
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
                if (sort_loc && s < sort_n) {
                    float* l = sort_loc + 3 * (size_t)s;
                    l[0] = sort_location_rn(x); l[1] = sort_location_rn(y); l[2] = sort_location_rn(z);
                }
            } else if (SPARSE) {
                slot_bit_assign(affine_bits, s, affine);
                slot_bit_assign(centre_bits, s, centred);
            }
        }
    }
    if (!SPARSE && lane == 0) {   // the last word also holds slots past n: they keep their bits
        const uint32_t mask = n - base >= 32u ? 0xFFFFFFFFu : (1u << (n - base)) - 1u;
        store_bits(&affine_bits[wtile], abits, mask);
        store_bits(&centre_bits[wtile], cbits, mask);
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

int check_state(r3_ctx* c) {   // of two failed preconditions, the mesh spheres' message comes before the borrowed buffer's
    R3_TRY(r3_check_object_writer(c, "set_object_transforms", R3_NEED_HOT | R3_NEED_SPHERES));
    return r3_check_object_writer(c, "set_object_transforms", R3_NEED_OWNED);
}

int launch_transforms(r3_ctx* c, const uint32_t* d_slots, const float* d_mats, uint32_t n) {
    const uint32_t sort_n = r3_sort_extent(c);
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
    slot_bit_assign(enabled_bits, s, on);
    if (s < sort_n) slot_bit_assign(live_bits, s, on);
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

// ---- ObjectManager::add with another mesh kind or material: r3_switch_object_variants, r3_switch_object_variants_device
constexpr uint32_t VR_THREADS = 256;
constexpr uint32_t VR_NONE = 0xFFFFFFFFu;      // slot_group of an unlisted slot; current word of a slot never switched
constexpr uint32_t VR_UNSEEN = 0x80000000u;    // current-word bit: switched by the device form, not yet read by the host
static_assert(sizeof(r3_object_variant) == 64 && offsetof(r3_object_variant, sort_flags) == 36 && offsetof(r3_object_variant, material_key) == 40,
              "the kernel reads a variant as four float4s: record words 20-27, then attr_offset[5], flags, key, then the mesh sphere");

// Entry i switches slot s = slots[i] (dense: i) to variant first + choices[i] of the slot's group; unlisted slots, slots at or past
// n_slots and choices past the group are dropped.  One thread per entry; the dense form's warp owns one 32-slot word of the centre bits
// and stores the bits of the entries it applied (whole words without atomics), the sparse form uses atomics as object_transforms_kernel.
template <bool SPARSE>
__global__ void __launch_bounds__(VR_THREADS)
object_variants_kernel(const uint32_t* __restrict__ slots, const uint32_t* __restrict__ choices, uint32_t n, uint32_t n_slots,
                       const uint32_t* __restrict__ slot_group, const uint4* __restrict__ groups, const float4* __restrict__ variants, uint32_t tag,
                       const float4* __restrict__ rows_xyz, float4* __restrict__ objects, float4* __restrict__ mesh_spheres, float4* __restrict__ spheres,
                       float* __restrict__ radii, uint32_t* __restrict__ centre_bits, uint8_t* __restrict__ key8, float* __restrict__ sort_loc,
                       uint32_t sort_n, uint32_t* __restrict__ current) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if ((SPARSE ? i : (i & ~31u)) >= n) return;   // dense: the whole warp, which ballots below
    uint32_t s = n_slots, v = 0;
    bool ok = false;
    if (i < n) {
        s = SPARSE ? __ldg(slots + i) : i;
        if (s < n_slots) {
            const uint32_t g = __ldg(slot_group + s);
            if (g != VR_NONE) {
                const uint4 gr = __ldg(groups + g);   // first, count, floor
                const uint32_t ch = __ldg(choices + i);
                if (ch < gr.y) { v = gr.x + ch; ok = true; }
            }
        }
    }
    bool centred = false;
    if (ok) {
        const float4 v0 = __ldg(variants + 4 * (size_t)v), v1 = __ldg(variants + 4 * (size_t)v + 1), v2 = __ldg(variants + 4 * (size_t)v + 2),
                     ms = __ldg(variants + 4 * (size_t)v + 3);
        const float4 r0 = rows_xyz[3 * (size_t)s], r1 = rows_xyz[3 * (size_t)s + 1], r2 = rows_xyz[3 * (size_t)s + 2];
        const float x[4] = {r0.x, r0.y, r0.z, r0.w}, y[4] = {r1.x, r1.y, r1.z, r1.w}, z[4] = {r2.x, r2.y, r2.z, r2.w};
        // BoundingSphere::apply_transform (R12), the same function as a move and a deform
        const float4 sph = sphere_apply_transform_rn(x, y, z, ms);
        float4* rec = objects + (size_t)s * 8;
        rec[4] = sph;
        rec[5] = v0;                                                          // first_index, index_count, material_index, attr_offset[0]
        rec[6] = v1;                                                          // attr_offset[1..4]
        reinterpret_cast<uint32_t*>(rec + 7)[0] = __float_as_uint(v2.x);      // attr_offset[5]; `enabled` (@116) stays
        mesh_spheres[s] = ms;
        spheres[s] = sph;
        radii[s] = sph.w;
        centred = centre_is_translation(sph.x, sph.y, sph.z, x[3], y[3], z[3]);
        if (s < sort_n) {
            // key8 as r3_set_object_sort_info builds it (r3_ctx.cu sort_key8); location = the world sphere's centre (object.rs:273)
            const uint32_t flags = __float_as_uint(v2.y), key = __float_as_uint(v2.z);
            key8[s] = (uint8_t)(((((key & 63u) << 1) | ((flags & 2u) ? 0u : 1u)) << 1) | ((flags & 4u) ? 1u : 0u));
            float* l = sort_loc + 3 * (size_t)s;
            l[0] = sph.x; l[1] = sph.y; l[2] = sph.z;
        }
        current[s] = v | tag;
    }
    if (SPARSE) {
        if (ok) slot_bit_assign(centre_bits, s, centred);
    } else {
        const uint32_t applied = __ballot_sync(0xFFFFFFFFu, ok), bits = __ballot_sync(0xFFFFFFFFu, ok && centred);
        if ((threadIdx.x & 31u) == 0) store_bits(&centre_bits[i >> 5], bits, applied);
    }
}

// the listed slots' invocation floors: the largest index_count of the slot's group
__global__ void variant_floors_kernel(const uint32_t* __restrict__ slot_group, const uint4* __restrict__ groups, uint32_t n, uint32_t* __restrict__ floor) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const uint32_t g = slot_group[s];
    if (g != VR_NONE) floor[s] = groups[g].z;
}

// the host has read the current words: clear their VR_UNSEEN bits
__global__ void variant_words_seen_kernel(uint32_t* __restrict__ current, uint32_t n) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) current[s] &= ~VR_UNSEEN;
}

int launch_enabled(r3_ctx* c, const uint32_t* d_slots, const uint8_t* d_enabled, uint32_t n) {
    const uint32_t sort_n = r3_sort_extent(c);
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

struct r3_variant_state {
    uint32_t n_variants = 0, n_groups = 0;
    uint32_t n_slots = 0;                     // length of the per-slot arrays (the slot count when the set was made, grown by resize)
    uint32_t n_words = 0;                     // the highest listed slot + 1: the current words the host batching reads back
    uint64_t index_end = 0;                   // the largest first_index + index_count of the variants (mesh-buffer words)
    std::vector<r3_object_variant> variants;  // host copies: validation, floors and the key mirrors
    std::vector<r3_variant_group> groups;
    std::vector<uint32_t> slot_group;         // per slot: its group, VR_NONE when unlisted
    std::vector<uint32_t> staged;             // current words read back by variants_stage
    float4* d_variants = nullptr; uint32_t variants_cap = 0;
    uint4* d_groups = nullptr; uint32_t groups_cap = 0;   // first, count, floor, 0
    uint32_t* d_slot_group = nullptr; uint32_t* d_current = nullptr; uint32_t slots_cap = 0;
};

namespace {

int check_variant_state(r3_ctx* c, const char* who) {
    const r3_variant_state* V = c->variants;
    if (!V || !V->n_variants) return r3_fail(c, R3_E_STATE, who);
    R3_TRY(r3_check_object_writer(c, "switch_object_variants", R3_NEED_HOT | R3_NEED_OWNED | R3_NEED_SPHERES));
    if (c->mesh_words < V->index_end) return r3_fail(c, R3_E_STATE, "switch_object_variants: the mesh buffer ends before a variant's indices");
    return R3_OK;
}

int launch_variants(r3_ctx* c, const uint32_t* d_slots, const uint32_t* d_choices, uint32_t n, uint32_t tag) {
    const r3_variant_state* V = c->variants;
    const uint32_t sort_n = r3_sort_extent(c);
    const uint32_t n_slots = std::min(c->n_slots, V->n_slots);
    const uint32_t ctas = (uint32_t)(((uint64_t)n + VR_THREADS - 1) / VR_THREADS);
    auto kernel = d_slots ? object_variants_kernel<true> : object_variants_kernel<false>;
    kernel<<<ctas, VR_THREADS, 0, c->stream>>>(d_slots, d_choices, n, n_slots, V->d_slot_group, V->d_groups, V->d_variants, tag, c->d_hot_xyz,
                                               reinterpret_cast<float4*>(c->d_objects), c->d_mesh_spheres, c->d_hot_sphere, c->d_hot_radius,
                                               c->d_centre_bits, sort_n ? c->d_sort_key8 : nullptr, sort_n ? c->d_sort_loc : nullptr, sort_n, V->d_current);
    R3_CHECK_LAUNCH(c, "object_variants_kernel");
    r3_new_frame_epoch(c);                       // a frame-wide sort made before the switch is stale
    if (sort_n) c->locations_moved = true;       // the host batching's mirror c->sort_loc is behind the device's
    return R3_OK;
}

void free_variants(r3_variant_state* V) {
    cudaFree(V->d_variants); cudaFree(V->d_groups); cudaFree(V->d_slot_group); cudaFree(V->d_current);
}

}  // namespace

bool r3_variants_have_set(const r3_ctx* c) { return c->variants && c->variants->n_variants; }
bool r3_variants_list(const r3_ctx* c, uint32_t slot) {
    const r3_variant_state* V = c->variants;
    return V && V->n_variants && slot < V->slot_group.size() && V->slot_group[slot] != VR_NONE;
}

void r3_variants_destroy(r3_ctx* c) {
    if (!c->variants) return;
    free_variants(c->variants);
    delete c->variants;
    c->variants = nullptr;
}

int r3_variants_grow(r3_ctx* c, uint32_t n) {
    r3_variant_state* V = c->variants;
    if (!V || !V->n_variants || V->n_slots >= n) return R3_OK;
    if (n > V->slots_cap) {
        const uint64_t cap = r3_hot_capacity(n);
        uint32_t cap_a = V->slots_cap, cap_b = V->slots_cap;
        R3_TRY(r3_reserve_t(c, &V->d_slot_group, &cap_a, cap, true));
        R3_TRY(r3_reserve_t(c, &V->d_current, &cap_b, cap, true));
        V->slots_cap = cap_a;
    }
    R3_CUDA(c, cudaMemsetAsync(V->d_slot_group + V->n_slots, 0xFF, (size_t)(n - V->n_slots) * 4, c->stream));
    R3_CUDA(c, cudaMemsetAsync(V->d_current + V->n_slots, 0xFF, (size_t)(n - V->n_slots) * 4, c->stream));
    V->slot_group.resize(n, VR_NONE);
    V->n_slots = n;
    return R3_OK;
}

int r3_variants_scatter_floors(r3_ctx* c) {
    const r3_variant_state* V = c->variants;
    if (!V || !V->n_variants) return R3_OK;
    const uint32_t n = std::min(V->n_slots, c->n_invocation_floor);
    if (!n) return R3_OK;
    variant_floors_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>(V->d_slot_group, V->d_groups, n, c->d_invocation_floor);
    R3_CHECK_LAUNCH(c, "variant_floors_kernel");
    return R3_OK;
}

// After r3_switch_object_variants_device the host's key / flag mirrors are behind the device's.  stage enqueues a copy of the listed slots'
// current-variant words to the host and marks them seen on the device (*staged = true when it did; c->variants_on_device stays set until
// apply); once the caller has drained the stream, apply rebuilds the mirrors of the slots switched since.
static int variants_stage(r3_ctx* c, bool* staged) {
    *staged = false;
    if (!c->variants_on_device) return R3_OK;
    r3_variant_state* V = c->variants;
    if (!V || !V->n_variants || !V->n_words) {   // nothing listed: nothing to read
        c->variants_on_device = false;
        r3_presence_derive(c);
        return R3_OK;
    }
    V->staged.resize(V->n_words);
    R3_CUDA(c, cudaMemcpyAsync(V->staged.data(), V->d_current, (size_t)V->n_words * 4, cudaMemcpyDeviceToHost, c->stream));
    variant_words_seen_kernel<<<(V->n_words + 255) / 256, 256, 0, c->stream>>>(V->d_current, V->n_words);
    R3_CHECK_LAUNCH(c, "variant_words_seen_kernel");
    *staged = true;
    return R3_OK;
}

static void variants_apply(r3_ctx* c) {
    const r3_variant_state* V = c->variants;
    const uint32_t sorted = std::min(r3_sort_extent(c), (uint32_t)V->staged.size());
    for (uint32_t s = 0; s < sorted; ++s) {
        const uint32_t w = V->staged[s];
        if (w == VR_NONE || !(w & VR_UNSEEN)) continue;
        const r3_object_variant& v = V->variants[w & ~VR_UNSEEN];
        r3_sort_set_key_flags(c, s, v.material_key, (uint8_t)v.sort_flags);
    }
    c->variants_on_device = false;
    r3_presence_derive(c);
}

int r3_variants_sync_host(r3_ctx* c) {
    bool staged = false;
    R3_TRY(variants_stage(c, &staged));
    if (!staged) return R3_OK;
    R3_CUDA(c, r3_stream_sync(c));
    variants_apply(c);
    return R3_OK;
}

R3_EXPORT int r3_set_object_variants(r3_ctx* c, const r3_object_variant* variants, uint32_t n_variants, const r3_variant_group* groups, uint32_t n_groups,
                                     const uint32_t* slots, const uint32_t* slot_groups, uint32_t n_listed) {
    if (!c) return R3_E_INVALID;
    if ((!variants && n_variants) || (!groups && n_groups) || ((!slots || !slot_groups) && n_listed)) return r3_fail(c, R3_E_INVALID, "set_object_variants: null");
    cudaSetDevice(c->device);
    if (n_variants == 0) {
        if (n_groups || n_listed) return r3_fail(c, R3_E_INVALID, "set_object_variants: groups or slots without variants");
        R3_TRY(r3_variants_sync_host(c));         // device switches the host has not seen settle the mirrors first
        if (c->variants) { free_variants(c->variants); *c->variants = r3_variant_state(); }
        c->variant_key2 = c->variant_wide_key = false;
        R3_TRY(r3_rebuild_invocation_floors(c));
        R3_CUDA(c, r3_stream_sync(c));
        r3_presence_derive(c);
        return R3_OK;
    }
    R3_TRY(r3_check_object_writer(c, "set_object_variants", R3_NEED_HOT | R3_NEED_OWNED | R3_NEED_SPHERES));
    // ---- every argument before anything is written
    uint64_t index_end = 0;
    bool key2 = false, wide = false;
    for (uint32_t i = 0; i < n_variants; ++i) {
        const r3_object_variant& v = variants[i];
        const uint64_t end = (uint64_t)v.first_index + v.index_count;
        if (end > c->mesh_words) return r3_fail(c, R3_E_INVALID, "set_object_variants: an index range outside the mesh buffer");
        if (v.index_count % 3) return r3_fail(c, R3_E_INVALID, "set_object_variants: index_count is not a multiple of 3");
        for (uint32_t off : v.attr_offset)
            if (off != R3_ATTR_ABSENT && (off & 3u)) return r3_fail(c, R3_E_INVALID, "set_object_variants: an offset that is not a multiple of 4");
        if (v.attr_offset[R3_ATTR_POSITION] == R3_ATTR_ABSENT) return r3_fail(c, R3_E_INVALID, "set_object_variants: a variant without positions");
        if (v.sort_flags & ~6u) return r3_fail(c, R3_E_INVALID, "set_object_variants: sort_flags other than bits 1-2");
        index_end = std::max(index_end, end);
        key2 |= v.material_key == 2;
        wide |= v.material_key >= 64;
    }
    std::vector<uint4> dev_groups(n_groups);
    for (uint32_t g = 0; g < n_groups; ++g) {
        const r3_variant_group& gr = groups[g];
        if (gr.count == 0 || (uint64_t)gr.first + gr.count > n_variants) return r3_fail(c, R3_E_INVALID, "set_object_variants: an empty group or one past the variants");
        uint32_t floor = 0;
        for (uint32_t k = 0; k < gr.count; ++k) floor = std::max(floor, variants[gr.first + k].index_count);
        dev_groups[g] = make_uint4(gr.first, gr.count, floor, 0u);
    }
    std::vector<uint32_t> slot_group(c->n_slots, VR_NONE);
    uint32_t n_words = 0;
    for (uint32_t i = 0; i < n_listed; ++i) {
        const uint32_t s = slots[i];
        if (s >= c->n_slots) return r3_fail(c, R3_E_INVALID, "set_object_variants: slot beyond the object buffer");
        if (slot_group[s] != VR_NONE) return r3_fail(c, R3_E_INVALID, "set_object_variants: one slot named twice");
        if (slot_groups[i] >= n_groups) return r3_fail(c, R3_E_INVALID, "set_object_variants: group index out of range");
        slot_group[s] = slot_groups[i];
        n_words = std::max(n_words, s + 1);
    }
    if (const std::vector<uint32_t>* listed = r3_deform_listed_slots(c))
        for (uint32_t s : *listed)
            if (s < slot_group.size() && slot_group[s] != VR_NONE)
                return r3_fail(c, R3_E_INVALID, "set_object_variants: a slot listed by the deformable or remeshable set");
    // ---- the set
    R3_TRY(r3_variants_sync_host(c));
    if (!c->variants) c->variants = new r3_variant_state();
    r3_variant_state* V = c->variants;
    R3_TRY(r3_reserve_t(c, &V->d_variants, &V->variants_cap, 4ull * n_variants));
    R3_TRY(r3_reserve_t(c, &V->d_groups, &V->groups_cap, std::max(n_groups, 1u)));
    const uint32_t n = std::max(c->n_slots, 1u);
    if (n > V->slots_cap || !V->d_slot_group) {
        uint32_t cap_a = 0, cap_b = 0;
        cudaFree(V->d_slot_group); cudaFree(V->d_current);
        V->d_slot_group = V->d_current = nullptr; V->slots_cap = 0;
        R3_TRY(r3_reserve_t(c, &V->d_slot_group, &cap_a, n));
        R3_TRY(r3_reserve_t(c, &V->d_current, &cap_b, n));
        V->slots_cap = cap_a;
    }
    R3_CUDA(c, cudaMemcpyAsync(V->d_variants, variants, (size_t)n_variants * sizeof(r3_object_variant), cudaMemcpyHostToDevice, c->stream));
    if (n_groups) R3_CUDA(c, cudaMemcpyAsync(V->d_groups, dev_groups.data(), (size_t)n_groups * 16, cudaMemcpyHostToDevice, c->stream));
    if (c->n_slots) R3_CUDA(c, cudaMemcpyAsync(V->d_slot_group, slot_group.data(), (size_t)c->n_slots * 4, cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, cudaMemsetAsync(V->d_current, 0xFF, (size_t)n * 4, c->stream));
    V->n_variants = n_variants; V->n_groups = n_groups; V->n_slots = c->n_slots; V->n_words = n_words; V->index_end = index_end;
    V->variants.assign(variants, variants + n_variants);
    V->groups.assign(groups, groups + n_groups);
    V->slot_group.swap(slot_group);
    c->variant_key2 = key2; c->variant_wide_key = wide;
    R3_TRY(r3_rebuild_invocation_floors(c));
    R3_CUDA(c, r3_stream_sync(c));               // host pointers are only borrowed for the call
    r3_presence_derive(c);
    return R3_OK;
}

R3_EXPORT int r3_switch_object_variants(r3_ctx* c, const uint32_t* slots, const uint32_t* choices, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (n == 0) return R3_OK;
    if (!choices) return r3_fail(c, R3_E_INVALID, "switch_object_variants: null");
    R3_TRY(check_variant_state(c, "switch_object_variants before set_object_variants"));
    if (!slots && n > c->n_slots) return r3_fail(c, R3_E_INVALID, "switch_object_variants: more choices than slots");
    if (slots) R3_TRY(check_slots(c, slots, n, c->n_slots, "switch_object_variants: slot beyond the object buffer", "switch_object_variants: one slot named twice"));
    const r3_variant_state* V = c->variants;
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t s = slots ? slots[i] : i;
        const uint32_t g = s < V->slot_group.size() ? V->slot_group[s] : VR_NONE;
        if (g == VR_NONE) return r3_fail(c, R3_E_INVALID, "switch_object_variants: a slot the set does not list");
        if (choices[i] >= V->groups[g].count) return r3_fail(c, R3_E_INVALID, "switch_object_variants: a choice past its group");
    }
    cudaSetDevice(c->device);
    R3_TRY(r3_reserve(c, &c->d_scratch, &c->scratch_cap, (uint64_t)n * 8, 1, false, false));
    uint32_t* d_choices = (uint32_t*)c->d_scratch;
    uint32_t* d_slots = slots ? d_choices + n : nullptr;
    R3_CUDA(c, cudaMemcpyAsync(d_choices, choices, (size_t)n * 4, cudaMemcpyHostToDevice, c->stream));
    if (slots) R3_CUDA(c, cudaMemcpyAsync(d_slots, slots, (size_t)n * 4, cudaMemcpyHostToDevice, c->stream));
    R3_TRY(launch_variants(c, d_slots, d_choices, n, 0u));
    R3_CUDA(c, r3_stream_sync(c));               // host pointers are only borrowed for the call
    R3_TRY(r3_variants_sync_host(c));            // earlier device switches of other slots: their mirrors too
    // the host sees every entry: its key and flag mirrors stay exact
    const uint32_t sorted = r3_sort_extent(c);
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t s = slots ? slots[i] : i;
        if (s >= sorted) continue;
        const r3_object_variant& v = V->variants[V->groups[V->slot_group[s]].first + choices[i]];
        r3_sort_set_key_flags(c, s, v.material_key, (uint8_t)v.sort_flags);
    }
    r3_presence_derive(c);
    return R3_OK;
}

R3_EXPORT int r3_switch_object_variants_device(r3_ctx* c, const uint32_t* d_slots, const uint32_t* d_choices, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (n == 0) return R3_OK;
    if (!d_choices || ((uintptr_t)d_choices & 3u) || ((uintptr_t)d_slots & 3u))
        return r3_fail(c, R3_E_INVALID, "switch_object_variants_device: null or misaligned pointer (4 bytes)");
    R3_TRY(check_variant_state(c, "switch_object_variants_device before set_object_variants"));
    if (!d_slots && n > c->n_slots) return r3_fail(c, R3_E_INVALID, "switch_object_variants_device: more choices than slots");
    cudaSetDevice(c->device);
    R3_TRY(launch_variants(c, d_slots, d_choices, n, VR_UNSEEN));
    c->variants_on_device = true;                // the switched slots' keys are now known on the device only
    r3_presence_derive(c);
    return R3_OK;
}

R3_EXPORT int r3_readback_object_variants(r3_ctx* c, uint32_t* out, uint32_t first, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if ((!out && n) || (uint64_t)first + n > c->n_slots) return r3_fail(c, R3_E_INVALID, "readback_object_variants: range outside the slots");
    if (n == 0) return R3_OK;
    cudaSetDevice(c->device);
    const r3_variant_state* V = c->variants;
    const uint32_t have = V && V->n_variants && first < V->n_slots ? std::min(n, V->n_slots - first) : 0u;
    if (have) R3_CUDA(c, cudaMemcpyAsync(out, V->d_current + first, (size_t)have * 4, cudaMemcpyDeviceToHost, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    for (uint32_t i = 0; i < n; ++i) out[i] = i < have && out[i] != VR_NONE ? out[i] & ~VR_UNSEEN : VR_NONE;
    return R3_OK;
}

R3_EXPORT int r3_set_objects_enabled(r3_ctx* c, const uint32_t* slots, const uint8_t* enabled, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (n == 0) return R3_OK;
    if (!enabled) return r3_fail(c, R3_E_INVALID, "set_objects_enabled: null");
    R3_TRY(r3_check_object_writer(c, "set_objects_enabled", R3_NEED_HOT | R3_NEED_OWNED));
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
    R3_TRY(r3_check_object_writer(c, "set_objects_enabled_device", R3_NEED_HOT));
    R3_TRY(r3_check_object_writer(c, "set_objects_enabled", R3_NEED_OWNED));   // both forms name the host form here
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
static int stage_moved_locations(r3_ctx* c, bool* staged) {
    *staged = false;
    if (!c->locations_moved) return R3_OK;
    c->locations_moved = false;
    const size_t sort_n = r3_sort_extent(c);
    if (sort_n == 0 || !c->d_sort_loc) return R3_OK;
    R3_CUDA(c, cudaMemcpyAsync(c->sort_loc.data(), c->d_sort_loc, sort_n * 12, cudaMemcpyDeviceToHost, c->stream));
    *staged = true;
    return R3_OK;
}

// r3_animation.cu: the posed slots' locations, staged and applied as above (apply does nothing unless stage enqueued a copy)
int r3_anim_stage_posed_locations(r3_ctx* c, bool* staged);
void r3_anim_apply_posed_locations(r3_ctx* c);

int r3_stage_sort_mirrors(r3_ctx* c, bool* pending) {
    bool moved = false, posed = false, switched = false;
    R3_TRY(stage_moved_locations(c, &moved));
    R3_TRY(r3_anim_stage_posed_locations(c, &posed));
    R3_TRY(variants_stage(c, &switched));
    *pending = moved || posed || switched;
    return R3_OK;
}

void r3_apply_sort_mirrors(r3_ctx* c) {
    r3_anim_apply_posed_locations(c);
    if (c->variants_on_device) variants_apply(c);   // still set: variants_stage enqueued a copy
}
