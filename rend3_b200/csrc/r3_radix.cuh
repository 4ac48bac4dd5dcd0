// r3_radix.cuh — the stable LSD radix sort's building blocks, shared by the batching sort (r3_gpu_batching.cu) and the vertex ->
// corner lists of the dynamic meshes (r3_mesh_deform.cu): per-tile digit histograms stored digit-major, one in-place exclusive scan
// of that table, and a stable per-tile scatter.  8-bit digits of unsigned long long keys at any shift.
#pragma once
#ifdef __CUDACC__
#include <stdint.h>

#include "r3_scan.cuh"

namespace {

constexpr int SORT_THREADS = 256;
constexpr int SORT_KEYS_PER_THREAD = 8;
constexpr int SORT_TILE = SORT_THREADS * SORT_KEYS_PER_THREAD;   // 2048 keys per block

// Digit histogram of the tile of SORT_TILE keys at `base`, stored digit-major into hist[digit * n_tiles + tile]: a flat
// exclusive scan of that table gives every tile's scatter bases.  SORT_THREADS threads, one digit each.
__device__ __forceinline__ void radix_tile_hist(const unsigned long long* keys, uint32_t nv, int shift, uint32_t* hist, uint32_t tile, uint32_t n_tiles) {
    __shared__ uint32_t s_hist[256];
    s_hist[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t base = tile * SORT_TILE;
#pragma unroll
    for (int r = 0; r < SORT_KEYS_PER_THREAD; ++r) {
        const uint32_t i = base + r * SORT_THREADS + threadIdx.x;
        if (i < nv) atomicAdd(&s_hist[(uint32_t)(keys[i] >> shift) & 0xFFu], 1u);
    }
    __syncthreads();
    hist[threadIdx.x * n_tiles + tile] = s_hist[threadIdx.x];
}

// Stable scatter of the tile at `base`, 256 keys per round: a key goes to s_gbase[digit] (the tile's first position of that
// digit, in shared memory) + the keys of its digit in earlier rounds + those in lower warps of this round + its rank among the
// warp's peers (__match_any_sync).  SORT_THREADS threads, one digit each.
__device__ __forceinline__ void radix_tile_scatter(const unsigned long long* keys_in, unsigned long long* keys_out, uint32_t nv, int shift, uint32_t base,
                                                   const uint32_t* s_gbase) {
    __shared__ uint32_t s_cnt[SORT_THREADS / 32][256];   // per-warp digit counts of the current round
    __shared__ uint32_t s_run[256];                       // digits already emitted by this tile in earlier rounds
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    s_run[threadIdx.x] = 0;
#pragma unroll 1
    for (int r = 0; r < SORT_KEYS_PER_THREAD; ++r) {
#pragma unroll
        for (int w = 0; w < SORT_THREADS / 32; ++w) s_cnt[w][threadIdx.x] = 0;
        __syncthreads();
        const uint32_t i = base + r * SORT_THREADS + threadIdx.x;
        const bool valid = i < nv;
        const unsigned long long key = valid ? keys_in[i] : 0ull;
        const uint32_t d = valid ? ((uint32_t)(key >> shift) & 0xFFu) : 0x100u;     // invalid lanes form their own group
        const uint32_t peers = __match_any_sync(0xFFFFFFFFu, d);
        const uint32_t rank_in_warp = __popc(peers & ((1u << lane) - 1u));
        if (valid && rank_in_warp == 0) s_cnt[warp][d] = __popc(peers);              // one writer per (warp, digit)
        __syncthreads();
        // digit t: exclusive prefix over the warps, then advance the tile's running count
        uint32_t acc = 0;
#pragma unroll
        for (int w = 0; w < SORT_THREADS / 32; ++w) { const uint32_t c = s_cnt[w][threadIdx.x]; s_cnt[w][threadIdx.x] = acc; acc += c; }
        __syncthreads();
        if (valid) keys_out[s_gbase[d] + s_run[d] + s_cnt[warp][d] + rank_in_warp] = key;
        __syncthreads();
        s_run[threadIdx.x] += acc;
        __syncthreads();
    }
}

// in-place exclusive scan by one block: every thread owns a contiguous run (serial sum, one block scan of the 1024 run totals,
// serial write-back) — three barriers in all instead of four per 1024 elements
__global__ void __launch_bounds__(1024) scan_u32_kernel(uint32_t* __restrict__ data, uint32_t n) {
    __shared__ uint32_t s_warp[1024 / 32 + 1];
    const uint32_t per = (((n + 1023u) / 1024u) + 3u) & ~3u;          // multiple of 4: runs start 16-byte aligned
    const uint32_t lo = min(threadIdx.x * per, n), hi = min(lo + per, n);
    uint32_t sum = 0;
    uint32_t i = lo;
    for (; i + 4 <= hi; i += 4) { const uint4 v = *reinterpret_cast<const uint4*>(data + i); sum += v.x + v.y + v.z + v.w; }
    for (; i < hi; ++i) sum += data[i];
    uint32_t run = block_scan_excl<1024>(sum, s_warp);
    for (i = lo; i + 4 <= hi; i += 4) {
        const uint4 v = *reinterpret_cast<const uint4*>(data + i);
        uint4 o;
        o.x = run; o.y = o.x + v.x; o.z = o.y + v.y; o.w = o.z + v.z; run = o.w + v.w;
        *reinterpret_cast<uint4*>(data + i) = o;
    }
    for (; i < hi; ++i) { const uint32_t v = data[i]; data[i] = run; run += v; }
}

}  // namespace

#endif
