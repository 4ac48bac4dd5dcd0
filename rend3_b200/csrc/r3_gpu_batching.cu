// r3_gpu_batching.cu — batch_objects on the device: sort the visible objects and build the ShaderBatchData records
// without leaving the GPU, so a frame needs no mid-frame host synchronisation.
//
// Replaces the host half of GpuCuller::add_culling_to_graph (rend3-routine/src/culling/culler.rs:682-713):
//   batch_objects            rend3-routine/src/culling/batching.rs:120-250
//   ShaderJobSortingKey::cmp batching.rs:53-79   (material key, sorting reason, distance; bind group is DUMMY)
// The reference does this single-threaded on the CPU, per camera, under the data_core mutex — the object-level
// bottleneck SURVEY §8 (row a4) calls out.  Here:
//   1. key generation: 64-bit key = [material_key:6 | reason:1 | sortable(distance²):32 | position in the visible list:24];
//   2. stable LSD radix sort on the 39 significant bits (5 passes of 8 bits; histogram, scan, stable scatter with
//      __match_any_sync ranking) — ties keep the ascending-handle order of the visible list, the same tie rule the
//      oracle and the host path use;
//   3. batch partition, only for worlds where a batch can reach the dispatch limit of batching.rs:196 (256 x the largest
//      padded triangle count >= max_dispatch_count x 256): where each batch starts, found on the device (see
//      "dispatch-limit partition" below); otherwise a batch is a tile of 256 sorted objects;
//   4. batch build: one CTA per batch (block scans give invocation_start, region boundaries, local ids),
//      one scan over the batches (batch_base_invocation, global region ids), one fix-up pass that also swaps the
//      per-camera previous-invocation map (batching.rs:226,230).
// All counts stay on the device in the job header; the cull / raster kernels read them there.
// Not covered on the device (the host path remains for them): material keys >= 64 and more than 2^24 visible objects (the
// position no longer fits in the low 24 key bits; reported through the overflow flag).
#include <algorithm>
#include <cstring>

#include <cooperative_groups.h>
#include <cuda/atomic>

#include "r3_common.cuh"
#include "r3_radix.cuh"
#include "r3_scan.cuh"

namespace {

constexpr int KEY_SHIFT0 = 24, SORT_PASSES = 5;

// order-preserving map of OrderedFloat's total order (batching.rs:37): every NaN is one value above +inf, -0.0 == +0.0
__device__ __forceinline__ uint32_t sortable_f32(float f) {
    if (f != f) return 0xFFC00000u;                              // the image of the canonical quiet NaN 0x7FC00000
    const uint32_t b = __float_as_uint(f) == 0x80000000u ? 0u : __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ unsigned long long make_sort_key(const uint32_t* __restrict__ visible, const uint8_t* __restrict__ key8, const float* __restrict__ loc,
                                                            float vx, float vy, float vz, uint32_t j) {
    const uint32_t h = visible ? visible[j] : j;                 // visible == nullptr: the frame-wide sort over every slot (see r3_device_batch_objects)
    const uint8_t k = key8[h];                                   // (material_key << 1 | reason) << 1 | back_to_front
    const float dx = sub_rn(vx, loc[3 * (size_t)h]), dy = sub_rn(vy, loc[3 * (size_t)h + 1]), dz = sub_rn(vz, loc[3 * (size_t)h + 2]);
    float d2 = add_rn(add_rn(mul_rn(dx, dx), mul_rn(dy, dy)), mul_rn(dz, dz));   // Vec3A::distance_squared (batching.rs:156-157)
    if (k & 1u) d2 = -d2;                                                        // SortingOrder::BackToFront (batching.rs:158-160)
    return ((unsigned long long)(k >> 1) << 56) | ((unsigned long long)sortable_f32(d2) << 24) | (unsigned long long)j;
}

// (A limit of 12288 keys — 225 KB of shared memory — would put the 10 000-object config on this path, where one CTA sorts more slowly
//  than the cooperative kernel on 5 CTAs; the limit stays at 8192 keys, 161 KB.)
// cap <= SMALL_SORT_MAX: key generation + the same stable LSD radix sort, but by ONE CTA entirely in shared memory — one launch
// instead of 16, which is what a frame with a few thousand objects per camera is made of.  Warp w owns the w-th contiguous
// chunk of the keys; per pass: per-warp digit counts (__match_any_sync, leader adds), a scan over (digit, warp), then the
// warps re-walk their chunks in order and scatter (rank inside the round from the peer mask).  A pass whose digit is the same
// for every key (typical for the material-key byte) is skipped.
constexpr uint32_t SMALL_SORT_MAX = 8192;
constexpr int SMALL_SORT_THREADS = 1024, SMALL_SORT_WARPS = SMALL_SORT_THREADS / 32;
__host__ __device__ inline uint32_t small_sort_pad(uint32_t n) { return ((n + SMALL_SORT_THREADS - 1) / SMALL_SORT_THREADS) * SMALL_SORT_THREADS; }
inline size_t small_sort_smem(uint32_t cap) { return (size_t)small_sort_pad(cap) * 16 + (size_t)SMALL_SORT_WARPS * 256 * 4 + 256 * 4; }
__global__ void __launch_bounds__(SMALL_SORT_THREADS) small_sort_kernel(const uint32_t* __restrict__ visible, const uint32_t* __restrict__ visible_count,
                                                                        const uint8_t* __restrict__ key8, const float* __restrict__ loc, float vx, float vy, float vz,
                                                                        unsigned long long* __restrict__ keys_out, uint32_t* __restrict__ header, uint32_t cap_pad, uint32_t count_imm) {
    extern __shared__ unsigned long long s_keys[];                               // [2][cap_pad]
    uint32_t* s_count = reinterpret_cast<uint32_t*>(s_keys + 2 * (size_t)cap_pad);   // [warps][256]
    uint32_t* s_base = s_count + SMALL_SORT_WARPS * 256;                          // [256]
    __shared__ uint32_t s_wsum[8];
    __shared__ int s_skip;
    const uint32_t nv = min(visible_count ? *visible_count : count_imm, cap_pad);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) { header[0] = nv; header[4] = 0u; }
    for (uint32_t j = threadIdx.x; j < nv; j += SMALL_SORT_THREADS) s_keys[j] = make_sort_key(visible, key8, loc, vx, vy, vz, j);
    const uint32_t rounds = (nv + SMALL_SORT_THREADS - 1) / SMALL_SORT_THREADS, chunk = rounds * 32u;
    int src = 0;
    for (int pass = 0; pass < SORT_PASSES; ++pass) {
        const int shift = KEY_SHIFT0 + 8 * pass;
        const unsigned long long* in = s_keys + (size_t)src * cap_pad;
        unsigned long long* out = s_keys + (size_t)(src ^ 1) * cap_pad;
        for (uint32_t i = threadIdx.x; i < SMALL_SORT_WARPS * 256; i += SMALL_SORT_THREADS) s_count[i] = 0u;
        if (threadIdx.x == 0) s_skip = 0;
        __syncthreads();
        for (uint32_t r = 0; r < rounds; ++r) {
            const uint32_t idx = warp * chunk + r * 32u + lane;
            const bool valid = idx < nv;
            const uint32_t digit = valid ? (uint32_t)(in[idx] >> shift) & 255u : 256u + lane;
            const uint32_t peers = __match_any_sync(0xFFFFFFFFu, digit);
            if (valid && lane == __ffs(peers) - 1) s_count[warp * 256 + digit] += __popc(peers);
            __syncwarp();
        }
        __syncthreads();
        uint32_t total = 0, incl = 0;
        if (threadIdx.x < 256) {
            for (int w = 0; w < SMALL_SORT_WARPS; ++w) { const uint32_t t = s_count[w * 256 + threadIdx.x]; s_count[w * 256 + threadIdx.x] = total; total += t; }
            if (total == nv) s_skip = 1;
            incl = warp_scan_incl(total);   // threads 256-1023 are between the barriers: no block scan here
            if (lane == 31) s_wsum[warp] = incl;
        }
        __syncthreads();
        if (threadIdx.x < 256) {
            uint32_t before = 0;
            for (int w = 0; w < warp; ++w) before += s_wsum[w];
            s_base[threadIdx.x] = before + incl - total;
        }
        __syncthreads();
        const int skip = s_skip;
        __syncthreads();        // s_skip is reset at the top of the next pass
        if (skip) continue;     // block-uniform
        for (uint32_t r = 0; r < rounds; ++r) {
            const uint32_t idx = warp * chunk + r * 32u + lane;
            const bool valid = idx < nv;
            const unsigned long long key = valid ? in[idx] : 0ull;
            const uint32_t digit = valid ? (uint32_t)(key >> shift) & 255u : 256u + lane;
            const uint32_t peers = __match_any_sync(0xFFFFFFFFu, digit);
            if (valid) {
                const uint32_t pos = s_base[digit] + s_count[warp * 256 + digit] + __popc(peers & ((1u << lane) - 1u));
                out[pos] = key;
            }
            __syncwarp();
            if (valid && lane == __ffs(peers) - 1) s_count[warp * 256 + digit] += __popc(peers);
            __syncwarp();
        }
        __syncthreads();
        src ^= 1;
    }
    const unsigned long long* fin = s_keys + (size_t)src * cap_pad;
    for (uint32_t j = threadIdx.x; j < nv; j += SMALL_SORT_THREADS) keys_out[j] = fin[j];
}

__global__ void keygen_kernel(const uint32_t* __restrict__ visible, const uint32_t* __restrict__ visible_count, const uint8_t* __restrict__ key8,
                              const float* __restrict__ loc, float vx, float vy, float vz, unsigned long long* __restrict__ keys, uint32_t* __restrict__ header,
                              uint32_t count_imm) {
    const uint32_t nv = visible_count ? *visible_count : count_imm;
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j == 0) { header[0] = nv; header[4] = (nv >= (1u << 24)) ? 1u : 0u; }
    if (j >= nv) return;
    keys[j] = make_sort_key(visible, key8, loc, vx, vy, vz, j);
}

__global__ void __launch_bounds__(SORT_THREADS) radix_hist_kernel(const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ header,
                                                                  int shift, uint32_t* __restrict__ hist) {
    radix_tile_hist(keys, header[0], shift, hist, blockIdx.x, gridDim.x);
}

__global__ void __launch_bounds__(SORT_THREADS) radix_scatter_kernel(const unsigned long long* __restrict__ keys_in, unsigned long long* __restrict__ keys_out,
                                                                     const uint32_t* __restrict__ header, int shift, const uint32_t* __restrict__ hist_scanned) {
    __shared__ uint32_t s_gbase[256];
    const uint32_t nv = header[0], base = blockIdx.x * SORT_TILE;
    s_gbase[threadIdx.x] = hist_scanned[threadIdx.x * gridDim.x + blockIdx.x];
    if (base >= nv) return;
    radix_tile_scatter(keys_in, keys_out, nv, shift, base, s_gbase);
}

// object slot of sorted position j: the low 24 key bits are the slot (frame-wide sort) or a position in `visible`
__device__ __forceinline__ uint32_t sorted_slot(const unsigned long long* keys, const uint32_t* visible, uint32_t keys_hold_slots, uint32_t j) {
    const uint32_t low = (uint32_t)(keys[j] & 0xFFFFFFull);
    return keys_hold_slots ? low : visible[low];
}

// ---- batch build (batching.rs:180-246), one CTA per batch
struct BuildParams {
    const unsigned long long* keys; const uint32_t* visible; const r3_object* objects;
    r3_batch_data* batches; uint32_t* header;
    uint32_t* batch_inv; uint32_t* batch_regions;         // per batch: total_invocations, number of regions
    const uint32_t* batch_start;                          // [header[1] + 1] first sorted object of each batch (dispatch-limit partition), or
                                                          // nullptr: batch b is the sorted objects [256 b, 256 b + 256)
    r3_region* regions; uint32_t* region_first_inv;
    const uint32_t* prev_map; uint32_t* cur_map; uint32_t map_cap;
    uint64_t dispatch_limit;
    uint32_t keys_hold_slots;                             // low 24 key bits = the object slot (frame-wide sort) instead of a position in `visible`
};

// the sorted objects [*lo, *lo + *n) of batch b; false past the last batch
__device__ __forceinline__ bool batch_range(const BuildParams& p, uint32_t nv, uint32_t b, uint32_t* lo, uint32_t* n) {
    if (p.batch_start) {
        if (b >= p.header[1]) return false;
        *lo = p.batch_start[b];
        *n = min(p.batch_start[b + 1] - *lo, 256u);
    } else {
        if (b * 256u >= nv) return false;
        *lo = b * 256u;
        *n = min(256u, nv - *lo);
    }
    return true;
}

// Mid-sized worlds (more than one CTA's worth, up to 256 tiles = 524288 visible objects): the whole sort — key generation and
// the five histogram / offset / scatter passes — in ONE cooperative launch with grid-wide barriers between the phases instead of
// 16 launches.  Every CTA derives its own scatter bases from the raw digit-major histogram table (one pass over <= 256 columns
// per thread), so no separate scan kernel runs.
constexpr uint32_t COOP_SORT_MAX_BLOCKS = 256;
struct SortCoopParams {
    const uint32_t* visible; const uint32_t* visible_count; const uint8_t* key8; const float* loc; float vx, vy, vz;
    unsigned long long* keys[2]; uint32_t* hist; uint32_t* header; uint32_t count_imm;
};
__global__ void __launch_bounds__(SORT_THREADS) radix_sort_coop_kernel(const __grid_constant__ SortCoopParams p) {
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    __shared__ uint32_t s_gbase[256];
    __shared__ uint32_t s_warp[SORT_THREADS / 32 + 1];
    const uint32_t nv = p.visible_count ? *p.visible_count : p.count_imm, nb = gridDim.x, b = blockIdx.x;
    const uint32_t base = b * SORT_TILE;
    if (b == 0 && threadIdx.x == 0) { p.header[0] = nv; p.header[4] = (nv >= (1u << 24)) ? 1u : 0u; }
#pragma unroll 1
    for (int r = 0; r < SORT_KEYS_PER_THREAD; ++r) {
        const uint32_t i = base + r * SORT_THREADS + threadIdx.x;
        if (i < nv) p.keys[0][i] = make_sort_key(p.visible, p.key8, p.loc, p.vx, p.vy, p.vz, i);
    }
    __syncthreads();
    int src = 0;
    for (int pass = 0; pass < SORT_PASSES; ++pass) {
        const int shift = KEY_SHIFT0 + 8 * pass;
        const unsigned long long* keys_in = p.keys[src];
        unsigned long long* keys_out = p.keys[src ^ 1];
        radix_tile_hist(keys_in, nv, shift, p.hist, b, nb);
        grid.sync();
        // scatter bases of this tile: digits below mine in every tile + my digit in the tiles in front of me
        uint32_t before = 0, total = 0;
        const uint32_t* col = p.hist + threadIdx.x * nb;
        for (uint32_t k = 0; k < nb; ++k) { const uint32_t v = col[k]; total += v; if (k < b) before += v; }
        s_gbase[threadIdx.x] = block_scan_excl<SORT_THREADS>(total, s_warp) + before;
        radix_tile_scatter(keys_in, keys_out, nv, shift, base, s_gbase);
        grid.sync();
        src ^= 1;
    }
}

__global__ void __launch_bounds__(256) batch_build_kernel(const __grid_constant__ BuildParams p) {
    __shared__ uint32_t s_warp[256 / 32 + 1];
    __shared__ uint32_t s_start[256];
    __shared__ uint32_t s_first[256];
    const uint32_t nv = p.header[0], b = blockIdx.x, i = threadIdx.x;
    uint32_t lo, n;
    if (!batch_range(p, nv, b, &lo, &n)) { if (i == 0) { p.batch_inv[b] = 0; p.batch_regions[b] = 0; } return; }
    const uint32_t j = lo + i;
    const bool valid = i < n;
    unsigned long long key = 0ull, prev_key = 0ull;
    uint32_t h = 0, tri = 0;
    if (valid) {
        key = p.keys[j];
        h = sorted_slot(p.keys, p.visible, p.keys_hold_slots, j);
        tri = p.objects[h].index_count / 3u;                                  // batching.rs:192
        if (j > 0) prev_key = p.keys[j - 1];
    }
    const uint32_t k7 = (uint32_t)(key >> 56), mat = k7 >> 1, prev_mat = (uint32_t)(prev_key >> 57);
    const uint32_t padded = valid ? ((tri + 255u) & ~255u) : 0u;              // round_up(invocation_count, WORKGROUP_SIZE) batching.rs:235
    uint32_t total_inv, n_regions;
    const uint32_t start = block_scan_excl<256>(padded, s_warp, &total_inv);
    __syncthreads();
    const uint32_t flag = (valid && (i == 0 || mat != prev_mat)) ? 1u : 0u;  // a region starts at a batch start or a key change (batching.rs:194-204)
    const uint32_t region_local = block_scan_excl<256>(flag, s_warp, &n_regions) + flag - 1u;
    s_start[i] = start;
    // index of the first object of my region: running max of (flag ? i : 0), within the warp, then over the warps in front
    uint32_t first = warp_scan_incl(flag ? i : 0u, r3_op_max());
    __syncthreads();
    if ((i & 31) == 31) s_warp[i >> 5] = first;
    __syncthreads();
    uint32_t wmax = 0;
    for (uint32_t w = 0; w < (i >> 5); ++w) wmax = max(wmax, s_warp[w]);
    first = max(first, wmax);
    s_first[i] = first;
    __syncthreads();
    r3_batch_data* bd = &p.batches[b];
    if (valid) {
        r3_object_culling_info info;
        info.invocation_start = start;
        info.invocation_end = start + tri;
        info.object_id = h;
        info.region_id = region_local;                     // made global by batch_finalize_kernel
        info.base_region_invocation = s_start[first];
        info.local_region_id = i - first;
        info.previous_global_invocation = (h < p.map_cap) ? p.prev_map[h] : R3_NO_PREVIOUS;   // batching.rs:226
        info.atomic_capable = (k7 & 1u) ? 0u : 1u;         // SortingReason::Optimization (batching.rs:227)
        bd->object_culling_information[i] = info;
    }
    if (i == 0) {
        bd->total_objects = n; bd->total_invocations = total_inv; bd->batch_base_invocation = 0;
        p.batch_inv[b] = total_inv;
        p.batch_regions[b] = n ? n_regions : 1u;           // the leading empty batch still closes one region (batching.rs:197-199)
        // without the partition no batch may reach the limit (r3_device_batch_objects only skips it then): tripwire
        if (!p.batch_start && (uint64_t)total_inv >= p.dispatch_limit) atomicExch(&p.header[4], 1u);
    }
}

// one block: exclusive scans over the batches -> batch_base_invocation, global region ids; fills the header.  Both are scanned
// at once as (invocations << 32 | regions): there are fewer regions than objects, so the low half never carries into the high
// half, and the high half wraps exactly as a uint32_t sum of the invocations would.
__global__ void __launch_bounds__(1024) batch_scan_kernel(const __grid_constant__ BuildParams p) {
    __shared__ unsigned long long s_warp[1024 / 32 + 1];
    const uint32_t nv = p.header[0], nb = p.batch_start ? p.header[1] : (nv + 255u) / 256u;
    const unsigned long long tot = block_scan_excl_chunked<1024>(
        nb, s_warp, [&](uint32_t b) { return (unsigned long long)p.batch_inv[b] << 32 | p.batch_regions[b]; },
        [&](uint32_t b, unsigned long long e) { p.batch_inv[b] = (uint32_t)(e >> 32); p.batch_regions[b] = (uint32_t)e; });
    if (threadIdx.x == 0) {
        const uint32_t n_inv = (uint32_t)(tot >> 32), n_reg = (uint32_t)tot;
        p.header[1] = nb; p.header[2] = n_reg; p.header[3] = n_inv;
        p.region_first_inv[n_reg] = n_inv;
    }
}

__global__ void __launch_bounds__(256) batch_finalize_kernel(const __grid_constant__ BuildParams p) {
    const uint32_t nv = p.header[0], b = blockIdx.x, i = threadIdx.x;
    uint32_t lo, n;
    if (!batch_range(p, nv, b, &lo, &n)) return;
    r3_batch_data* bd = &p.batches[b];
    const uint32_t base_inv = p.batch_inv[b], base_reg = p.batch_regions[b];
    if (i == 0) bd->batch_base_invocation = base_inv;
    if (i < n) {
        r3_object_culling_info* info = &bd->object_culling_information[i];
        const uint32_t local_region = info->region_id;
        info->region_id = base_reg + local_region;
        if (info->object_id < p.map_cap) p.cur_map[info->object_id] = info->invocation_start + base_inv;   // batching.rs:230
        if (info->local_region_id == 0) {
            r3_region r;
            r.job_index = b; r.bind_group_index = 0u; r.material_key = p.keys[lo + i] >> 57;
            p.regions[base_reg + local_region] = r;                                                            // batching.rs:199,238
            p.region_first_inv[base_reg + local_region] = base_inv + info->invocation_start;
        }
    } else if (n == 0 && i == 0) {
        // the leading empty batch (the first sorted object alone reaches the dispatch limit): its region carries that object's key
        r3_region r;
        r.job_index = b; r.bind_group_index = 0u; r.material_key = p.keys[lo] >> 57;
        p.regions[base_reg] = r;
        p.region_first_inv[base_reg] = base_inv;
    }
}

// ---- frame-wide sort shared by the cameras of a frame.  batch_objects sorts by (material key, sorting reason, distance to the
// VIEWPORT camera) for every camera, shadow cameras included (batching.rs:156-157 uses viewport_camera_state) — the key of an object
// is the same in all of them, only the visible sets differ.  So the slots are sorted ONCE per frame and each camera takes its
// visible objects out of that order with a stream compaction (ties resolve by slot in both forms: the results are identical).
// On config 3 this replaces five cooperative sorts by one sort and five much shorter compactions.
constexpr int RC_THREADS = 1024;
__device__ __forceinline__ bool rank_visible(const unsigned long long* __restrict__ gkeys, uint32_t r, uint32_t n, const uint32_t* __restrict__ words, uint32_t cap,
                                             unsigned long long* key) {
    if (r >= n) return false;
    const unsigned long long k = gkeys[r];
    const uint32_t slot = (uint32_t)(k & 0xFFFFFFull);
    *key = k;
    return slot < cap && ((__ldg(&words[slot >> 5]) >> (slot & 31u)) & 1u);
}
__global__ void __launch_bounds__(RC_THREADS) rank_count_kernel(const unsigned long long* __restrict__ gkeys, uint32_t n, const uint32_t* __restrict__ words, uint32_t cap,
                                                                uint32_t* __restrict__ tile_counts) {
    unsigned long long k;
    const int c = __syncthreads_count(rank_visible(gkeys, blockIdx.x * RC_THREADS + threadIdx.x, n, words, cap, &k) ? 1 : 0);
    if (threadIdx.x == 0) tile_counts[blockIdx.x] = (uint32_t)c;
}
__global__ void __launch_bounds__(RC_THREADS) rank_scatter_kernel(const unsigned long long* __restrict__ gkeys, uint32_t n, const uint32_t* __restrict__ words, uint32_t cap,
                                                                  const uint32_t* __restrict__ tile_counts, unsigned long long* __restrict__ keys_out,
                                                                  uint32_t* __restrict__ header) {
    __shared__ uint32_t s_warp[32];
    const uint32_t base = block_sum_u32<RC_THREADS>(tile_counts, blockIdx.x, s_warp);
    unsigned long long key = 0ull;
    const bool vis = rank_visible(gkeys, blockIdx.x * RC_THREADS + threadIdx.x, n, words, cap, &key);
    uint32_t total;
    const uint32_t rank = block_flag_rank<RC_THREADS>(vis, s_warp, &total);
    if (vis) keys_out[base + rank] = key;
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) { header[0] = base + total; header[4] = 0u; }
}

// ---- dispatch-limit partition (batching.rs:194-209): where the batches start when a batch can reach L = max_dispatch_count x 256
// invocations.  Over the sorted objects j: T_j = triangles, P_j = round_up(T_j, 256), S_j = exclusive prefix of P.  The batch that
// starts at s ends at next(s) = the first e in (s, min(s + 256, nv)) with S_e - S_s + T_e >= L, else min(s + 256, nv).  S_e + T_e is
// non-decreasing in e (S_e + T_e <= S_e + P_e = S_{e+1}), so next(s) is one binary search.  The batch starts are the chain
// 0 -> next(0) -> ..., marked without the host by pointer doubling: with J = next, K times  mark |= J(mark), J = J o J; after K steps
// every n^i(0), i < 2^K, is marked.  The marks are set in place, read and written with relaxed atomics by the threads of one step: a
// thread that already sees a mark set in the same step only marks a further chain member earlier, so the final set is the same.
// Then the marks are compacted into batch_start[].  When T_0 >= L the reference first closes an EMPTY batch (batching.rs:196 with
// nothing in it): batch_start then begins with a 0 of its own.  Launch counts and grids depend only on the capacity and K.
struct PartitionParams {
    const unsigned long long* keys; const uint32_t* visible; const r3_object* objects; uint32_t keys_hold_slots;
    uint32_t* header;
    uint32_t* s_local; uint32_t* f_local;   // [cap] S_j and S_j + T_j inside j's tile of 256
    uint32_t* tile_sum;                     // [tiles] P summed over each tile, then their exclusive prefix
    uint32_t* jump[2];                      // [cap + 1] J, ping-pong; J[nv] = nv
    uint32_t* mark;                         // [cap + 1]
    uint32_t* mark_count;                   // [cap / 1024 + 1] marks per 1024-object tile
    uint32_t* batch_start;                  // [nb_max + 1]
    uint64_t dispatch_limit; uint32_t nb_max;
};

__global__ void __launch_bounds__(256) partition_tile_kernel(const __grid_constant__ PartitionParams p) {
    __shared__ uint32_t s_warp[256 / 32 + 1];
    const uint32_t nv = p.header[0], j = blockIdx.x * 256u + threadIdx.x;
    if (blockIdx.x * 256u >= nv) return;
    const uint32_t tri = j < nv ? p.objects[sorted_slot(p.keys, p.visible, p.keys_hold_slots, j)].index_count / 3u : 0u;
    uint32_t total;
    const uint32_t s = block_scan_excl<256>((tri + 255u) & ~255u, s_warp, &total);
    if (j < nv) { p.s_local[j] = s; p.f_local[j] = s + tri; }
    if (threadIdx.x == 0) p.tile_sum[blockIdx.x] = total;
}

__global__ void __launch_bounds__(1024) partition_scan_kernel(const __grid_constant__ PartitionParams p) {
    __shared__ uint32_t s_warp[1024 / 32 + 1];
    block_scan_excl_chunked<1024>((p.header[0] + 255u) / 256u, s_warp, [&](uint32_t t) { return p.tile_sum[t]; },
                                  [&](uint32_t t, uint32_t e) { p.tile_sum[t] = e; });
}

// next(s) for every s < nv (S and S + T of the 511 objects from this tile's first on are staged in shared memory), J[nv] = nv, mark = {0}
__global__ void __launch_bounds__(256) partition_next_kernel(const __grid_constant__ PartitionParams p) {
    __shared__ uint32_t s_f[512];
    const uint32_t nv = p.header[0], base = blockIdx.x * 256u, s = base + threadIdx.x;
    if (base > nv) return;
    for (uint32_t k = threadIdx.x; k < 512u; k += 256u) {
        const uint32_t e = base + k;
        s_f[k] = e < nv ? p.tile_sum[e >> 8] + p.f_local[e] : 0u;   // S_e + T_e < 2^32: the padded total is below 2^31
    }
    __syncthreads();
    if (s < nv) {
        const uint32_t ss = p.tile_sum[s >> 8] + p.s_local[s];
        uint32_t lo = s + 1u, hi = min(s + 256u, nv);
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if ((uint64_t)(s_f[mid - base] - ss) >= p.dispatch_limit) hi = mid;
            else lo = mid + 1u;
        }
        p.jump[0][s] = lo;
        p.mark[s] = s == 0u ? 1u : 0u;
    } else if (s == nv) {
        p.jump[0][s] = nv;
        p.mark[s] = 0u;
    }
}

// one doubling step: mark |= J(mark), out = J o J (out == nullptr on the last step)
__global__ void __launch_bounds__(256) partition_jump_kernel(const uint32_t* __restrict__ header, const uint32_t* __restrict__ in, uint32_t* __restrict__ out, uint32_t* mark) {
    using mark_ref = cuda::atomic_ref<uint32_t, cuda::thread_scope_device>;
    const uint32_t s = blockIdx.x * 256u + threadIdx.x;
    if (s > header[0]) return;
    const uint32_t js = in[s];
    if (mark_ref(mark[s]).load(cuda::memory_order_relaxed)) mark_ref(mark[js]).store(1u, cuda::memory_order_relaxed);
    if (out) out[s] = in[js];
}

__global__ void __launch_bounds__(1024) partition_count_kernel(const __grid_constant__ PartitionParams p) {
    const uint32_t nv = p.header[0], j = blockIdx.x * 1024u + threadIdx.x;
    const int c = __syncthreads_count(j < nv && p.mark[j]);
    if (threadIdx.x == 0) p.mark_count[blockIdx.x] = (uint32_t)c;
}

// the marked objects in ascending order -> batch_start[lead + rank]; the last CTA writes the batch count and the closing entry
__global__ void __launch_bounds__(1024) partition_scatter_kernel(const __grid_constant__ PartitionParams p) {
    __shared__ uint32_t s_warp[32];
    const uint32_t nv = p.header[0], j = blockIdx.x * 1024u + threadIdx.x;
    const uint32_t lead = (nv > 0u && (uint64_t)p.f_local[0] >= p.dispatch_limit) ? 1u : 0u;   // T_0 >= L: the leading empty batch
    const uint32_t base = lead + block_sum_u32<1024>(p.mark_count, blockIdx.x, s_warp);
    const bool m = j < nv && p.mark[j];
    uint32_t total;
    const uint32_t pos = base + block_flag_rank<1024>(m, s_warp, &total);
    if (m && pos < p.nb_max) p.batch_start[pos] = j;
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) {
        uint32_t nb = base + total;
        if (nb > p.nb_max) { nb = p.nb_max; atomicExch(&p.header[4], 1u); }   // beyond the bound of r3_device_batch_objects: tripwire
        p.header[1] = nb;
        p.batch_start[nb] = nv;
        if (lead) p.batch_start[0] = 0u;
    }
}

// out[0] = sum over the slots of round_up(triangles, 256), out[1] = the largest such term; a slot's index_count counts as at least its
// floor (slots below n_floor)
__global__ void max_invocations_kernel(const r3_object* __restrict__ objects, uint32_t n, const uint32_t* __restrict__ floor, uint32_t n_floor,
                                       unsigned long long* __restrict__ out) {
    unsigned long long acc = 0, big = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const uint32_t ic = i < n_floor ? max(objects[i].index_count, floor[i]) : objects[i].index_count;
        const unsigned long long v = ((ic / 3u) + 255u) & ~255u;
        acc += v; big = max(big, v);
    }
    acc = warp_reduce(acc);
    big = warp_reduce(big, r3_op_max());
    if ((threadIdx.x & 31) == 0 && acc) { atomicAdd(out, acc); atomicMax(out + 1, big); }
}

}  // namespace

// sum over every slot of round_up(max(index_count, floor) / 3, 256): the bound the culling buffers are sized with when the per-frame
// totals stay on the device.  One small reduction + 8-byte readback at upload time, never per frame.
int r3_compute_max_invocations(r3_ctx* c) {
    if (c->max_invocations_valid) return R3_OK;
    c->max_total_invocations = 0; c->max_object_invocations = 0;
    if (c->n_slots) {
        R3_CUDA(c, cudaMemsetAsync(c->d_stats + 4, 0, 16, c->stream));
        max_invocations_kernel<<<c->sm_count * 4, 256, 0, c->stream>>>(c->d_objects, c->n_slots, c->d_invocation_floor, c->n_invocation_floor, c->d_stats + 4);
        R3_CHECK_LAUNCH(c, "max_invocations_kernel");
        unsigned long long v[2] = {0, 0};
        R3_CUDA(c, cudaMemcpyAsync(v, c->d_stats + 4, 16, cudaMemcpyDeviceToHost, c->stream));
        R3_CUDA(c, r3_stream_sync(c));
        c->max_total_invocations = v[0]; c->max_object_invocations = v[1];
    }
    c->max_invocations_valid = true;
    return R3_OK;
}

R3_EXPORT int r3_debug_invocation_bound(r3_ctx* c, uint64_t out[2]) {
    if (!c || !out) return R3_E_INVALID;
    cudaSetDevice(c->device);
    R3_TRY(r3_compute_max_invocations(c));
    out[0] = c->max_total_invocations; out[1] = c->max_object_invocations;
    return R3_OK;
}

// key generation + stable LSD radix sort of `cap` candidates: the entries of `visible` (count on the device) or, with visible == nullptr,
// the slots [0, cap) themselves.  keys[*src_out] holds the result.
static int r3_launch_sort(r3_ctx* c, const uint32_t* visible, const uint32_t* visible_count, uint32_t cap, const float vp_loc[3], unsigned long long* keys[2],
                          uint32_t** hist, uint64_t* hist_cap, uint32_t* header, int* src_out) {
    int src = 0;
    const uint32_t sort_blocks = (cap + SORT_TILE - 1) / SORT_TILE;
    R3_TRY(r3_reserve_t(c, hist, hist_cap, (uint64_t)sort_blocks * 256 + 1));
    r3_stage_begin(c, R3_STAGE_SORT);
    if (cap <= SMALL_SORT_MAX) {
        // small worlds: key generation + radix sort by one CTA in shared memory, one launch
        const size_t smem = small_sort_smem(cap);
        cudaFuncSetAttribute(small_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)small_sort_smem(SMALL_SORT_MAX));   // per device
        small_sort_kernel<<<1, SMALL_SORT_THREADS, smem, c->stream>>>(visible, visible_count, c->d_sort_key8, c->d_sort_loc, vp_loc[0], vp_loc[1], vp_loc[2], keys[0], header,
                                                                      small_sort_pad(cap), cap);
        R3_CHECK_LAUNCH(c, "small_sort_kernel");
    } else if (sort_blocks <= COOP_SORT_MAX_BLOCKS && c->coop_launch_ok) {
        SortCoopParams sp;
        sp.visible = visible; sp.visible_count = visible_count; sp.key8 = c->d_sort_key8; sp.loc = c->d_sort_loc;
        sp.vx = vp_loc[0]; sp.vy = vp_loc[1]; sp.vz = vp_loc[2];
        sp.keys[0] = keys[0]; sp.keys[1] = keys[1]; sp.hist = *hist; sp.header = header; sp.count_imm = cap;
        void* args[] = {&sp};
        R3_CUDA(c, cudaLaunchCooperativeKernel((const void*)radix_sort_coop_kernel, dim3(sort_blocks), dim3(SORT_THREADS), args, 0, c->stream));
        c->launches++;
        src = SORT_PASSES & 1;
    } else {
        keygen_kernel<<<(cap + 255) / 256, 256, 0, c->stream>>>(visible, visible_count, c->d_sort_key8, c->d_sort_loc, vp_loc[0], vp_loc[1], vp_loc[2], keys[0], header, cap);
        R3_CHECK_LAUNCH(c, "keygen_kernel");
        for (int pass = 0; pass < SORT_PASSES; ++pass) {
            const int shift = KEY_SHIFT0 + 8 * pass;
            radix_hist_kernel<<<sort_blocks, SORT_THREADS, 0, c->stream>>>(keys[src], header, shift, *hist);
            R3_CHECK_LAUNCH(c, "radix_hist_kernel");
            scan_u32_kernel<<<1, 1024, 0, c->stream>>>(*hist, sort_blocks * 256u);
            R3_CHECK_LAUNCH(c, "scan_u32_kernel");
            radix_scatter_kernel<<<sort_blocks, SORT_THREADS, 0, c->stream>>>(keys[src], keys[src ^ 1], header, shift, *hist);
            R3_CHECK_LAUNCH(c, "radix_scatter_kernel");
            src ^= 1;
        }
    }
    r3_stage_end(c);
    *src_out = src;
    return R3_OK;
}

// Should this camera take its order from the frame-wide sort?  Yes when several cameras batch per frame (known from the previous
// frame; on a first frame: when shadow-casting lights exist) and the world is small enough that sorting every slot once beats
// sorting each camera's visible set.  R3_FRAME_SORT=0 / 1 forces the choice (tests run both).
static bool r3_frame_sort_wanted(r3_ctx* c, r3_camera* cam, const float vp_loc[3]) {
    // a camera batching a second time or another viewport location starts a new frame epoch (as do r3_set_frame_uniforms and new sort data)
    if (cam->gsort_epoch_used == c->gsort_epoch || (c->gsort_cameras_this_epoch > 0 && memcmp(c->gsort_loc, vp_loc, 12) != 0)) r3_new_frame_epoch(c);
    if (c->gsort_cameras_this_epoch == 0) memcpy(c->gsort_loc, vp_loc, 12);
    cam->gsort_epoch_used = c->gsort_epoch;
    c->gsort_cameras_this_epoch++;
    const char* force = getenv("R3_FRAME_SORT");
    if (force) return force[0] != '0';
    if (c->n_slots > (1u << 22)) return false;
    return c->gsort_cameras_last_epoch >= 2 || (c->gsort_cameras_last_epoch == 0 && c->n_dir >= 1);
}
static int r3_frame_sort(r3_ctx* c, const float vp_loc[3]) {
    if (c->gsort_valid && c->gsort_sorted_epoch == c->gsort_epoch) return R3_OK;   // the location is fixed within an epoch
    const uint32_t n = (uint32_t)(c->sort_flags.size() < c->n_slots ? c->sort_flags.size() : c->n_slots);
    R3_TRY(r3_reserve_t(c, &c->d_gsort_keys[0], &c->gsort_cap[0], (uint64_t)n + 1));
    R3_TRY(r3_reserve_t(c, &c->d_gsort_keys[1], &c->gsort_cap[1], (uint64_t)n + 1));
    if (!c->d_gsort_header) R3_CUDA(c, cudaMalloc((void**)&c->d_gsort_header, 32));
    int src = 0;
    if (n) R3_TRY(r3_launch_sort(c, nullptr, nullptr, n, vp_loc, c->d_gsort_keys, &c->d_gsort_hist, &c->gsort_hist_cap, c->d_gsort_header, &src));
    c->gsort_src = src; c->gsort_n = n; c->gsort_valid = true; c->gsort_sorted_epoch = c->gsort_epoch;
    return R3_OK;
}

int r3_device_batch_objects(r3_ctx* c, r3_camera* cam, const float vp_loc[3], uint32_t max_dispatch_count) {
    if (!cam->header_set) return r3_fail(c, R3_E_STATE, "batch_objects before object_uniform_upload");
    const uint32_t cap = cam->header.object_count;
    R3_TRY(r3_compute_max_invocations(c));
    if (c->max_total_invocations >= (1ull << 31)) return r3_fail(c, R3_E_INVALID, "more than 2^31 padded invocations");
    const int w = (cam->cache_idx == 0) ? 1 : 0;   // never overwrite the DrawCallSet cached for the predicted pass
    cam->cur = w;
    r3_jobs& j = cam->jobs[w];
    // The partition only runs when some batch can reach the dispatch limit L: 256 objects of the largest padded size reach it.  Bound
    // on the batch count then: at most floor(nv / 256) batches end at the object limit; if batch i ends at the dispatch limit because of
    // object e, batches i and i + 1 hold >= (invocations of i) + T_e >= L invocations together, so every other such batch owns a
    // disjoint pair worth >= L: at most 2 floor(total / L) + 1 of them end at the limit (the leading empty batch included).  With one
    // batch left open at the end, nb <= ceil(nv / 256) + 2 floor(total / L) + 3.  Every batch but the leading empty one holds an object,
    // so also nb <= nv + 1 (the only bound when L = 0).  total = the padded sum over every slot, nv <= cap.
    const uint64_t dispatch_limit = (uint64_t)max_dispatch_count * R3_WORKGROUP_SIZE;
    const bool partition = c->max_object_invocations * R3_BATCH_SIZE >= dispatch_limit;
    uint64_t nb_max = (cap + 255u) / 256u;
    if (partition) {
        nb_max = (uint64_t)cap + 1u;
        if (dispatch_limit) nb_max = std::min<uint64_t>(nb_max, (cap + 255u) / 256u + 2u * (c->max_total_invocations / dispatch_limit) + 3u);
    }
    const uint32_t nb_cap = (uint32_t)nb_max + 1u, nr_cap = nb_cap + 64u;
    R3_TRY(r3_reserve_t(c, &j.d_batches, &j.batches_cap, nb_cap));
    uint32_t rcap = j.regions_cap;
    R3_TRY(r3_reserve_t(c, &j.d_regions, &j.regions_cap, nr_cap));
    if (!j.d_region_first_inv || rcap != j.regions_cap) {
        cudaFree(j.d_region_first_inv);
        j.d_region_first_inv = nullptr;
        R3_CUDA(c, cudaMalloc((void**)&j.d_region_first_inv, ((size_t)j.regions_cap + 2) * 4));
    }
    if (!j.d_header) R3_CUDA(c, cudaMalloc((void**)&j.d_header, 32));
    R3_TRY(r3_reserve_t(c, &cam->d_sort_keys[0], &cam->sort_keys_cap, (uint64_t)cap + 1));
    R3_TRY(r3_reserve_t(c, &cam->d_sort_keys[1], &cam->sort_keys_cap2, (uint64_t)cap + 1));
    const uint32_t sort_blocks = (cap + SORT_TILE - 1) / SORT_TILE;
    R3_TRY(r3_reserve_t(c, &cam->d_sort_hist, &cam->sort_hist_cap, (uint64_t)sort_blocks * 256 + 1));
    // batch scratch: batch_inv[nb] | batch_regions[nb], and with the partition:
    //   batch_start[nb] | s_local[cap] | f_local[cap] | tile_sum[tiles] | jump[2][cap + 1] | mark_count[mtiles] | mark[cap + 1]
    const uint32_t part_tiles = (cap + 255u) / 256u, mark_tiles = (cap + 1023u) / 1024u;
    const uint64_t part_words = partition ? (uint64_t)nb_cap + 2ull * cap + part_tiles + 2ull * (cap + 1u) + mark_tiles + (cap + 1u) : 0u;
    R3_TRY(r3_reserve_t(c, &cam->d_batch_tmp, &cam->batch_tmp_cap, (uint64_t)nb_cap * 2 + part_words));
    if (cam->prev_inv_cap < cap || !cam->d_prev_inv[0]) {
        for (int k = 0; k < 2; ++k) {
            uint32_t* n = nullptr;
            R3_CUDA(c, cudaMalloc((void**)&n, ((size_t)cap + 1) * 4));
            R3_CUDA(c, cudaMemsetAsync(n, 0xFF, ((size_t)cap + 1) * 4, c->stream));
            if (cam->d_prev_inv[k]) {   // keep last frame's entries across a capacity growth
                R3_CUDA(c, cudaMemcpyAsync(n, cam->d_prev_inv[k], (size_t)cam->prev_inv_cap * 4, cudaMemcpyDeviceToDevice, c->stream));
                R3_CUDA(c, r3_stream_sync(c));
                cudaFree(cam->d_prev_inv[k]);
            }
            cam->d_prev_inv[k] = n;
        }
        cam->prev_inv_cap = cap;
    }
    const int prev = cam->prev_inv_cur, cur = prev ^ 1;
    // get_and_reset_camera (batching.rs:111-113): the WHOLE map starts empty, also the entries beyond this frame's object_count
    // (a world that shrinks and grows again must not see invocations from two frames ago)
    R3_CUDA(c, cudaMemsetAsync(cam->d_prev_inv[cur], 0xFF, (size_t)cam->prev_inv_cap * 4, c->stream));
    R3_CUDA(c, cudaMemsetAsync(j.d_header, 0, 32, c->stream));

    if (cap) {
        int src = 0;
        const unsigned long long* sorted_keys = nullptr;
        bool keys_hold_slots = false;
        if (r3_frame_sort_wanted(c, cam, vp_loc)) {
            // one sort for the frame's cameras, then this camera's visible objects in that order
            R3_TRY(r3_frame_sort(c, vp_loc));
            const uint32_t n = c->gsort_n, tiles = (n + RC_THREADS - 1) / RC_THREADS;
            R3_TRY(r3_reserve_t(c, &cam->d_sort_hist, &cam->sort_hist_cap, (uint64_t)tiles + 1));
            if (tiles) {                                   // no sortable slot at all: the zeroed header already says "no visible objects"
                rank_count_kernel<<<tiles, RC_THREADS, 0, c->stream>>>(c->d_gsort_keys[c->gsort_src], n, cam->d_words, cap, cam->d_sort_hist);
                R3_CHECK_LAUNCH(c, "rank_count_kernel");
                rank_scatter_kernel<<<tiles, RC_THREADS, 0, c->stream>>>(c->d_gsort_keys[c->gsort_src], n, cam->d_words, cap, cam->d_sort_hist, cam->d_sort_keys[0], j.d_header);
                R3_CHECK_LAUNCH(c, "rank_scatter_kernel");
            }
            sorted_keys = cam->d_sort_keys[0];
            keys_hold_slots = true;
            cam->batching_path = 3;
        } else {
            R3_TRY(r3_launch_sort(c, cam->d_visible, cam->d_visible_count, cap, vp_loc, cam->d_sort_keys, &cam->d_sort_hist, &cam->sort_hist_cap, j.d_header, &src));
            sorted_keys = cam->d_sort_keys[src];
        }
        BuildParams p;
        p.keys = sorted_keys; p.visible = cam->d_visible; p.objects = c->d_objects; p.keys_hold_slots = keys_hold_slots ? 1u : 0u;
        p.batches = j.d_batches; p.header = j.d_header;
        p.batch_inv = cam->d_batch_tmp; p.batch_regions = p.batch_inv + nb_cap; p.batch_start = nullptr;
        p.regions = j.d_regions; p.region_first_inv = j.d_region_first_inv;
        p.prev_map = cam->d_prev_inv[prev]; p.cur_map = cam->d_prev_inv[cur]; p.map_cap = cam->prev_inv_cap;
        p.dispatch_limit = dispatch_limit;
        if (partition) {
            PartitionParams q;
            q.keys = sorted_keys; q.visible = cam->d_visible; q.objects = c->d_objects; q.keys_hold_slots = p.keys_hold_slots;
            q.header = j.d_header;
            q.batch_start = p.batch_regions + nb_cap;
            q.s_local = q.batch_start + nb_cap; q.f_local = q.s_local + cap; q.tile_sum = q.f_local + cap;
            q.jump[0] = q.tile_sum + part_tiles; q.jump[1] = q.jump[0] + cap + 1; q.mark_count = q.jump[1] + cap + 1;
            q.mark = q.mark_count + mark_tiles;
            q.dispatch_limit = dispatch_limit; q.nb_max = (uint32_t)nb_max;
            const uint32_t jump_blocks = (cap + 1u + 255u) / 256u;
            partition_tile_kernel<<<part_tiles, 256, 0, c->stream>>>(q);
            R3_CHECK_LAUNCH(c, "partition_tile_kernel");
            partition_scan_kernel<<<1, 1024, 0, c->stream>>>(q);
            R3_CHECK_LAUNCH(c, "partition_scan_kernel");
            partition_next_kernel<<<jump_blocks, 256, 0, c->stream>>>(q);
            R3_CHECK_LAUNCH(c, "partition_next_kernel");
            int steps = 0;                                 // K = ceil(log2(nb_max)): 2^K >= the batches a chain can start
            while ((1ull << steps) < nb_max) ++steps;
            for (int k = 0; k < steps; ++k) {
                partition_jump_kernel<<<jump_blocks, 256, 0, c->stream>>>(j.d_header, q.jump[k & 1], k + 1 < steps ? q.jump[(k + 1) & 1] : nullptr, q.mark);
                R3_CHECK_LAUNCH(c, "partition_jump_kernel");
            }
            partition_count_kernel<<<mark_tiles, 1024, 0, c->stream>>>(q);
            R3_CHECK_LAUNCH(c, "partition_count_kernel");
            partition_scatter_kernel<<<mark_tiles, 1024, 0, c->stream>>>(q);
            R3_CHECK_LAUNCH(c, "partition_scatter_kernel");
            p.batch_start = q.batch_start;
        }
        batch_build_kernel<<<nb_cap - 1, 256, 0, c->stream>>>(p);
        R3_CHECK_LAUNCH(c, "batch_build_kernel");
        batch_scan_kernel<<<1, 1024, 0, c->stream>>>(p);
        R3_CHECK_LAUNCH(c, "batch_scan_kernel");
        batch_finalize_kernel<<<nb_cap - 1, 256, 0, c->stream>>>(p);
        R3_CHECK_LAUNCH(c, "batch_finalize_kernel");
    }
    cam->prev_inv_cur = cur;
    j.device_built = true; j.valid = true;
    j.n_batches = nb_cap - 1; j.n_regions = nr_cap - 1;                 // upper bounds; exact counts live in d_header
    j.total_invocations = (uint32_t)c->max_total_invocations;
    j.batches.clear(); j.regions.clear();
    return R3_OK;
}

// device-built jobs -> host vectors (r3_batch_counts / r3_readback_batches / tests); blocks
int r3_download_jobs(r3_ctx* c, r3_camera* cam) {
    r3_jobs& j = cam->jobs[cam->cur];
    if (!j.device_built || !j.batches.empty() || !j.d_header) return R3_OK;
    uint32_t hdr[8] = {0};
    R3_CUDA(c, cudaMemcpyAsync(hdr, j.d_header, 32, cudaMemcpyDeviceToHost, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    if (hdr[4]) return r3_fail(c, R3_E_INVALID, "device batch_objects overflow (batch count beyond its bound, or > 2^24 visible objects): use host batching");
    j.batches.resize(hdr[1]); j.regions.resize(hdr[2]);
    if (hdr[1]) R3_CUDA(c, cudaMemcpyAsync(j.batches.data(), j.d_batches, (size_t)hdr[1] * sizeof(r3_batch_data), cudaMemcpyDeviceToHost, c->stream));
    if (hdr[2]) R3_CUDA(c, cudaMemcpyAsync(j.regions.data(), j.d_regions, (size_t)hdr[2] * sizeof(r3_region), cudaMemcpyDeviceToHost, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    // the 8448-byte records carry 244 bytes of padding the host path leaves zero
    for (auto& b : j.batches) {
        std::memset(b._pad, 0, sizeof b._pad);
        for (uint32_t o = b.total_objects; o < R3_BATCH_SIZE; ++o) std::memset(&b.object_culling_information[o], 0, sizeof(r3_object_culling_info));
    }
    return R3_OK;
}
