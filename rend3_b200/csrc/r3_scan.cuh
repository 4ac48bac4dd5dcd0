// r3_scan.cuh — the integer prefix sums, reductions and stream compactions the kernels share.  Every visible list, batch table,
// triangle index list, draw record and exchange count is built from these.  Templated on the value type (uint32_t, and
// unsigned long long for the packed (hi << 32 | lo) pairs whose halves are summed together) and, where a caller needs it, the operator.
// Warp-level functions need the full warp; block-level functions contain __syncthreads() and need every thread of the block.
#pragma once
#ifdef __CUDACC__
#include <stdint.h>

struct r3_op_sum {
    template <typename T> __device__ __forceinline__ T operator()(T a, T b) const { return a + b; }
};
struct r3_op_max {
    template <typename T> __device__ __forceinline__ T operator()(T a, T b) const { return a > b ? a : b; }
};

// op over lanes [0, lane] of the warp
template <typename T, typename Op = r3_op_sum>
__device__ __forceinline__ T warp_scan_incl(T v, Op op = Op()) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const T t = __shfl_up_sync(0xFFFFFFFFu, v, d);
        if (lane >= d) v = op(v, t);
    }
    return v;
}

// op over the 32 lanes, in every lane
template <typename T, typename Op = r3_op_sum>
__device__ __forceinline__ T warp_reduce(T v, Op op = Op()) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) v = op(v, __shfl_xor_sync(0xFFFFFFFFu, v, s));
    return v;
}

// Exclusive prefix sum over a block of THREADS threads (thread order); *total, when given, receives the block's sum in every thread.
// s_warp: THREADS / 32 + 1 entries, read after the last of the one or two barriers inside, so writing it again (a next call
// included) needs a __syncthreads() first.
template <int THREADS, typename T>
__device__ __forceinline__ T block_scan_excl(T v, T* s_warp, T* total = nullptr) {
    constexpr int WARPS = THREADS / 32;
    static_assert(THREADS % 32 == 0 && WARPS <= 32, "block_scan_excl: whole warps, at most 1024 threads");
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const T incl = warp_scan_incl(v);
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if constexpr (WARPS <= 8) {
        // few warps: every thread adds up the warp totals itself, which saves the second barrier
        T before = 0, tot = 0;
#pragma unroll
        for (int w = 0; w < WARPS; ++w) {
            const T c = s_warp[w];
            if (w < warp) before += c;
            tot += c;
        }
        if (total) *total = tot;
        return before + incl - v;
    } else {
        if (warp == 0) {
            const T w = lane < WARPS ? s_warp[lane] : T(0);
            const T wi = warp_scan_incl(w);
            if (lane < WARPS) s_warp[lane] = wi - w;
            if (total && lane == WARPS - 1) s_warp[WARPS] = wi;
        }
        __syncthreads();
        if (total) *total = s_warp[WARPS];
        return s_warp[warp] + incl - v;
    }
}

// Sum over a block of THREADS threads, in every thread.  s_warp: THREADS / 32 entries.  One barrier; any write to s_warp
// afterwards needs a __syncthreads() first.
template <int THREADS, typename T>
__device__ __forceinline__ T block_reduce(T v, T* s_warp) {
    constexpr int WARPS = THREADS / 32;
    static_assert(THREADS % 32 == 0 && WARPS <= 32, "block_reduce: whole warps, at most 1024 threads");
    v = warp_reduce(v);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = v;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    return warp_reduce(lane < WARPS ? s_warp[lane] : T(0));
}

// counts[0] + ... + counts[n - 1], in every thread: what a compaction CTA adds to its local positions when counts holds the
// per-CTA counts of a previous pass and n is the number of CTAs in front of it.  s_warp is free again on return.
template <int THREADS>
__device__ __forceinline__ uint32_t block_sum_u32(const uint32_t* __restrict__ counts, uint32_t n, uint32_t* s_warp) {
    uint32_t v = 0;
    for (uint32_t i = threadIdx.x; i < n; i += THREADS) v += __ldg(&counts[i]);
    v = block_reduce<THREADS>(v, s_warp);
    __syncthreads();
    return v;
}

// Stream compaction inside a block of THREADS threads: the number of set flags of the threads in front of this one (thread order),
// and the block's count in *total.  s_warp: THREADS / 32 entries; writing it after the call needs a __syncthreads() first.
template <int THREADS>
__device__ __forceinline__ uint32_t block_flag_rank(bool flag, uint32_t* s_warp, uint32_t* total) {
    constexpr int WARPS = THREADS / 32;
    static_assert(THREADS % 32 == 0 && WARPS <= 32, "block_flag_rank: whole warps, at most 1024 threads");
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t bal = __ballot_sync(0xFFFFFFFFu, flag);
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    uint32_t before = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) {
        const uint32_t c = s_warp[w];
        if (w < warp) before += c;
        tot += c;
    }
    *total = tot;
    return before + __popc(bal & ((1u << lane) - 1u));
}

// Ordered expansion of the warp's 32 visibility words (one per lane, lane j's word covering ids id_base + 32 j .. + 31) into
// ascending ids: set bit b of lane j's word goes to position pos_j + (set bits of that word below b), pos_j being lane j's
// exclusive prefix.  store(position, id) writes one entry.
template <typename Store>
__device__ __forceinline__ void warp_expand_words(uint32_t word, uint32_t pos, uint32_t id_base, Store store) {
    const int lane = threadIdx.x & 31;
#pragma unroll 1
    for (int j = 0; j < 32; ++j) {
        const uint32_t wj = __shfl_sync(0xFFFFFFFFu, word, j), ej = __shfl_sync(0xFFFFFFFFu, pos, j);
        if ((wj >> lane) & 1u) store(ej + __popc(wj & ((1u << lane) - 1u)), id_base + j * 32u + lane);
    }
}

// Exclusive prefix sum of n values by ONE block of THREADS threads, THREADS values at a time with the running total carried
// across the chunks: store(i, sum of load(0 .. i - 1)) for every i < n.  Returns the sum of all n values in every thread.
// load(i) is only called for i < n.  s_warp: THREADS / 32 + 1 entries; writing it after the call needs a __syncthreads() first.
template <int THREADS, typename T, typename Load, typename Store>
__device__ __forceinline__ T block_scan_excl_chunked(uint32_t n, T* s_warp, Load load, Store store) {
    T carry = 0;
    for (uint32_t base = 0; base < n; base += THREADS) {
        const uint32_t i = base + threadIdx.x;
        const T v = i < n ? load(i) : T(0);
        T total;
        const T excl = block_scan_excl<THREADS>(v, s_warp, &total);
        if (i < n) store(i, carry + excl);
        carry += total;
        if (base + THREADS < n) __syncthreads();   // s_warp is reused by the next chunk
    }
    return carry;
}

#endif
