// r3_cull_bake.cu — fused per-object frustum cull + object-uniform bake, then ordered visible-list compaction.
//
// Replaces (reference paths):
//   * uniform_prep.wgsl::cs_main          rend3-routine/shaders/src/uniform_prep.wgsl:9-27
//       MV = view * T, MVP = view_proj * T for every enabled slot < object_count
//   * the sphere/frustum filter of batch_objects   rend3-routine/src/culling/batching.rs:144-148
//       Frustum::contains_sphere, 5 planes        rend3/src/util/frustum.rs:148-161
// and emits the visible slots as one ASCENDING u32 list (the canonical, bit-exact artefact).
//
// Design (HBM-bound: 224 flop against 212 algorithmic bytes per object — 84 read + 128 written; on affine transforms whose
// sphere centre is the translation the kernel reads 52 B + 3 bits, 184 B per object by the same count).
//   hot/cold split — the reference's 128-byte Object record (object.rs:23-36) stays the canonical store for the kernels
//     that need its cold fields (first_index, index_count, material, attribute offsets); the fields this path reads
//     (transform, bounding sphere, enabled) are ALSO kept as dense arrays — rows_xyz[3n] float4 (rows 0-2 of the
//     transform, row r of slot o at 3o + r), rows_w[n] float4 (row 3), spheres[n] float4, radii[n] float, enabled, affine
//     and centre 1 bit per slot — filled by split_objects_kernel whenever records are uploaded (r3_set_objects,
//     r3_set_objects_device), by split_slots_kernel when they are scattered (r3_update_objects, the animation posing) and by
//     object_transforms_kernel when objects move (r3_set_object_transforms).  The affine bit is set when row 3 has exactly the
//     bit patterns (+0, +0, +0, 1); rows_w is then never read, because the kernel substitutes those constants.  The centre bit
//     is set when the sphere's centre has exactly the bit patterns of the translation (elements .w of rows 0-2) — true of every
//     world sphere made from a mesh sphere centred at the mesh origin; the cull then takes the centre from the transform tile
//     and reads 4 B of radii instead of 16 B of spheres.  With the AoS records every 32-byte sector of a record is touched,
//     i.e. 128 B read per object; the dense arrays bring that to 52 B + 3 bits for affine, centred slots, 64 B + 3 bits for
//     affine ones with another centre, 80 B + 3 bits at most (and to 16 B + 1 bit for cull-only, which always reads spheres).
//   stream kernel  — no inter-CTA dependency:
//     * a warp owns 32 consecutive slots.  Three fully coalesced 512-byte loads fetch rows 0-2 of their transforms and
//       a transpose through the warp's 1536 bytes of shared memory hands the lane of (slot o, column j) that column; row
//       3 is the affine constant or, for other slots, one float of rows_w.  The lane multiplies the column by `view` and
//       by `view_proj` (operands straight from the constant bank) and stores column j of MV and of MVP — 64-byte runs,
//       whole sectors.  Arithmetic is __fmul_rn/__fadd_rn in WGSL's accumulation order, never contracted: MV/MVP are
//       bit-identical to the CPU oracle;
//     * lane l tests the sphere of slot base+l: with the centre bit, the centre is column 3 of the slot's tile in shared memory
//       and the radius one float of radii; without it, the lane loads the sphere.  The loads are predicated per lane, so a tile
//       of centred slots touches one 128-byte run of radii and none of spheres.  The ballot IS the 32-bit visibility word of
//       the 32 slots (1 bit per object goes to HBM);
//     * each CTA (1024 slots) also leaves its survivor count.
//   compact kernel — one CTA per 32768 objects: sums the CTA counts in front of it (<= 40 KB, L2 resident),
//     scans its 1024 visibility words and writes the surviving slot ids in ascending order.  It moves
//     N/8 + 4*visible bytes, ~1% of the stream kernel's traffic.
// (History: a single-pass kernel with a decoupled look-back lost time to look-back stalls; the
//  two-kernel AoS version ran at the copy bandwidth but moved 256 B per object.)
#include <cstdlib>
#include <type_traits>

#include "r3_common.cuh"
#include "r3_scan.cuh"

namespace {

constexpr int CB_THREADS = 256;
constexpr int CB_WARPS = CB_THREADS / 32;
constexpr int CB_WT = 4;                                   // 32-object warp tiles per warp
constexpr int CB_CTA_OBJECTS = CB_WARPS * CB_WT * 32;      // 1024
constexpr int CP_THREADS = 1024;                           // compact kernel: one visibility word per thread
constexpr int CP_OBJECTS = CP_THREADS * 32;                // 32768 objects per compact CTA
constexpr int CP_CTAS_PER_TILE = CP_OBJECTS / CB_CTA_OBJECTS;   // 32 stream-CTA counts per compact CTA

struct CullBakeParams {
    float view[16];
    float view_proj[16];
    float frustum[5][4];
    uint32_t object_count;
};
// r3_shadow_uniform_upload: the camera lives in device memory (written by r3_evaluate_shadow_cameras in the same stream)
struct DeviceCameraParams {
    const r3_camera_header* cam;
    uint32_t object_count;
};
constexpr int CAM_FLOATS = 52;   // view[16] | view_proj[16] | frustum[5][4], staged in shared memory by DeviceCameraParams launches

// AoS Object records -> the dense hot arrays.  8 lanes per 128-byte record (coalesced 512-byte loads); float4 #0-3 =
// transform columns, #4 = bounding sphere, #7.y = `enabled` (byte 116).  Lane k < 4 holds column k and scatters it into
// element k of rows 0-2 (rows_xyz) and of row 3 (rows_w); lane 4 stores the sphere and its radius and, with column 3 shuffled
// over from lane 3, decides the centre bit.
__global__ void __launch_bounds__(256) split_objects_kernel(const float4* __restrict__ objects, uint32_t n, float* __restrict__ rows_xyz, float* __restrict__ rows_w,
                                                            float4* __restrict__ spheres, float* __restrict__ radii, uint32_t* __restrict__ enabled_bits,
                                                            uint32_t* __restrict__ affine_bits, uint32_t* __restrict__ centre_bits) {
    const int lane = threadIdx.x & 31, k = lane & 7, g = lane >> 3;
    const uint32_t wtile = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, base = wtile * 32u;
    if (base >= n) return;
    uint32_t bits = 0, abits = 0, cbits = 0;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const uint32_t obj = base + it * 4 + g;
        float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
        if (obj < n) {
            r = __ldcs(&objects[(size_t)obj * 8 + k]);
            if (k < 4) {
                float* xyz = rows_xyz + (size_t)obj * 12 + k;
                xyz[0] = r.x; xyz[4] = r.y; xyz[8] = r.z;
                rows_w[(size_t)obj * 4 + k] = r.w;
            } else if (k == 4) { spheres[obj] = r; radii[obj] = r.w; }
        }
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, k == 7 && obj < n && __float_as_uint(r.y) != 0u);   // lanes 7, 15, 23, 31
        bits |= (((b >> 7) & 1u) | (((b >> 15) & 1u) << 1) | (((b >> 23) & 1u) << 2) | (((b >> 31) & 1u) << 3)) << (it * 4);
        const uint32_t a = __ballot_sync(0xFFFFFFFFu, k < 4 && obj < n && __float_as_uint(r.w) == affine_w_bits(k));   // lanes 0-3 of each record
#pragma unroll
        for (int q = 0; q < 4; ++q) abits |= (((a >> (8 * q)) & 0xFu) == 0xFu ? 1u : 0u) << (it * 4 + q);
        const float tx = __shfl_up_sync(0xFFFFFFFFu, r.x, 1), ty = __shfl_up_sync(0xFFFFFFFFu, r.y, 1), tz = __shfl_up_sync(0xFFFFFFFFu, r.z, 1);   // column 3
        const uint32_t cb = __ballot_sync(0xFFFFFFFFu, k == 4 && obj < n && centre_is_translation(r.x, r.y, r.z, tx, ty, tz));   // lanes 4, 12, 20, 28
        cbits |= (((cb >> 4) & 1u) | (((cb >> 12) & 1u) << 1) | (((cb >> 20) & 1u) << 2) | (((cb >> 28) & 1u) << 3)) << (it * 4);
    }
    if (lane == 0) { enabled_bits[wtile] = bits; affine_bits[wtile] = abits; centre_bits[wtile] = cbits; }
}
// the same for the records r3_update_objects has just scattered (ScatterCopy, util/scatter_copy.rs:69-136)
__global__ void __launch_bounds__(256) split_slots_kernel(const float4* __restrict__ objects, const uint32_t* __restrict__ slots, uint32_t n_updates, uint32_t n_slots,
                                                          float* __restrict__ rows_xyz, float* __restrict__ rows_w, float4* __restrict__ spheres, float* __restrict__ radii,
                                                          uint32_t* __restrict__ enabled_bits, uint32_t* __restrict__ affine_bits, uint32_t* __restrict__ centre_bits) {
    const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 3, k = threadIdx.x & 7;
    const uint32_t s = i < n_updates ? slots[i] : n_slots;
    const bool ok = s < n_slots;
    float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ok) {
        r = objects[(size_t)s * 8 + k];
        if (k < 4) {
            float* xyz = rows_xyz + (size_t)s * 12 + k;
            xyz[0] = r.x; xyz[4] = r.y; xyz[8] = r.z;
            rows_w[(size_t)s * 4 + k] = r.w;
        } else if (k == 4) { spheres[s] = r; radii[s] = r.w; }
    }
    // the 8 lanes of a record share i and s; the grid is whole warps
    const uint32_t a = __ballot_sync(0xFFFFFFFFu, ok && k < 4 && __float_as_uint(r.w) == affine_w_bits(k));
    const float tx = __shfl_up_sync(0xFFFFFFFFu, r.x, 1), ty = __shfl_up_sync(0xFFFFFFFFu, r.y, 1), tz = __shfl_up_sync(0xFFFFFFFFu, r.z, 1);   // column 3
    const uint32_t cb = __ballot_sync(0xFFFFFFFFu, ok && k == 4 && centre_is_translation(r.x, r.y, r.z, tx, ty, tz));
    if (ok && k == 7) {
        slot_bit_assign(enabled_bits, s, __float_as_uint(r.y) != 0u);
        slot_bit_assign(affine_bits, s, ((a >> (threadIdx.x & 24u)) & 0xFu) == 0xFu);
        slot_bit_assign(centre_bits, s, (cb >> ((threadIdx.x & 24u) + 4u)) & 1u);
    }
}

template <bool BAKE, bool CULL, bool LIVE, typename Params = CullBakeParams>
__global__ void __launch_bounds__(CB_THREADS)
cull_bake_kernel(const float4* __restrict__ rows_xyz, const float* __restrict__ rows_w, const uint32_t* __restrict__ affine_bits, const float4* __restrict__ spheres,
                 const float* __restrict__ radii, const uint32_t* __restrict__ centre_bits, const uint32_t* __restrict__ enabled_bits, const uint32_t* __restrict__ live_bits, float4* __restrict__ matrices, uint32_t* __restrict__ words,
                 uint32_t* __restrict__ cta_counts, const __grid_constant__ Params p) {
    __shared__ uint32_t s_count[CB_WARPS];
    __shared__ float4 s_rows[BAKE ? CB_WARPS : 1][96];   // per warp: rows 0-2 of its 32 slots
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float* view;
    const float* view_proj;
    const float* frustum;   // [5][4]
    if constexpr (std::is_same<Params, DeviceCameraParams>::value) {
        // one copy per CTA: the operands the constant bank holds for the other instantiations
        __shared__ float s_cam[CAM_FLOATS];
        const float* src = reinterpret_cast<const float*>(p.cam);
        if (threadIdx.x < CAM_FLOATS) s_cam[threadIdx.x] = __ldg(src + (threadIdx.x < 32 ? threadIdx.x : threadIdx.x + 4));   // frustum at float 36
        __syncthreads();
        view = s_cam; view_proj = s_cam + 16; frustum = s_cam + 32;
    } else {
        view = p.view; view_proj = p.view_proj; frustum = &p.frustum[0][0];
    }
    const int col = lane & 3, sub = lane >> 2;   // transform column / slot within an 8-slot group
    uint32_t count = 0;
#pragma unroll 2
    for (int wt = 0; wt < CB_WT; ++wt) {
        const uint32_t wtile = (blockIdx.x * CB_WARPS + warp) * CB_WT + wt;   // visibility word index
        const uint32_t base = wtile * 32u;
        if (base >= p.object_count) break;
        float4 t[3];
        float4 sp = make_float4(0.f, 0.f, 0.f, 0.f);
        uint32_t enabled = 0u, affine = 0u, centred = 0u;
        if (BAKE && CULL) centred = __ldg(&centre_bits[wtile]);
        if (BAKE) {
#pragma unroll
            for (int q = 0; q < 3; ++q) {
                const uint32_t e = q * 32 + lane;   // row e % 3 of slot e / 3
                t[q] = base + e / 3u < p.object_count ? __ldcs(&rows_xyz[(size_t)base * 3 + e]) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
        // a centred slot's sphere is its translation and the radius: the lane loads 4 B of radii instead of 16 B of spheres (per lane,
        // so a warp only touches the sectors of the array its lanes need)
        const bool centre_from_tile = BAKE && CULL && ((centred >> lane) & 1u);
        if (CULL && base + lane < p.object_count) {
            if (centre_from_tile) sp.w = __ldcs(&radii[base + lane]);
            else sp = __ldcs(&spheres[base + lane]);
        }
        if (BAKE || (CULL && !LIVE)) enabled = __ldg(&enabled_bits[wtile]);
        if (BAKE) affine = __ldg(&affine_bits[wtile]);
        if (BAKE) {
            // transpose through shared memory: the lane of (slot, col) reads element col of the slot's rows 0-2, words
            // 12 slot + 4 r + col — 8 slots x 4 columns hit 32 distinct banks
            float4* tile = s_rows[warp];
            __syncwarp();   // every lane has read the previous tile
#pragma unroll
            for (int q = 0; q < 3; ++q) tile[q * 32 + lane] = t[q];
            __syncwarp();
            const float* tf = reinterpret_cast<const float*>(tile);
#pragma unroll
            for (int it = 0; it < 4; ++it) {
                const uint32_t slot = it * 8 + sub, obj = base + slot;
                if (obj < p.object_count && ((enabled >> slot) & 1u)) {   // uniform_prep.wgsl:18-20 skips disabled slots
                    const float* c = tf + slot * 12 + col;
                    // affine slot: row 3 is bit for bit (+0, +0, +0, 1), so the constant is the element it would have read
                    const float w = ((affine >> slot) & 1u) ? (col == 3 ? 1.0f : 0.0f) : __ldcs(&rows_w[(size_t)obj * 4 + col]);
                    float4* dst = &matrices[(size_t)obj * 8 + col];
                    __stcs(dst, mat_vec_rn(view, c[0], c[4], c[8], w));
                    __stcs(dst + 4, mat_vec_rn(view_proj, c[0], c[4], c[8], w));
                }
            }
        }
        if (CULL) {
            // one object per lane: Plane::distance = abc.dot(center) + d with glam's scalar dot order (util/frustum.rs:79-81,148-161)
            const uint32_t live = LIVE ? __ldg(&live_bits[wtile]) : enabled;
            if constexpr (BAKE) {
                if (centre_from_tile) {   // elements .w of rows 0-2 in the transposed tile (zeros past object_count, where the ballot drops the lane)
                    const float* tr = reinterpret_cast<const float*>(s_rows[warp]) + lane * 12 + 3;
                    sp.x = tr[0]; sp.y = tr[4]; sp.z = tr[8];
                }
            }
            const float neg_radius = -sp.w;
            bool inside = true;
#pragma unroll
            for (int pl = 0; pl < 5; ++pl) {
                const float* f = frustum + 4 * pl;
                const float d = add_rn(add_rn(add_rn(mul_rn(f[0], sp.x), mul_rn(f[1], sp.y)), mul_rn(f[2], sp.z)), f[3]);
                inside = inside && (d >= neg_radius);
            }
            const uint32_t word = __ballot_sync(0xFFFFFFFFu, base + lane < p.object_count && ((live >> lane) & 1u) && inside);
            if (lane == 0) words[wtile] = word;
            count += __popc(word);
        }
    }
    if (CULL) {
        if (lane == 0) s_count[warp] = count;
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t t = 0;
#pragma unroll
            for (int w = 0; w < CB_WARPS; ++w) t += s_count[w];
            cta_counts[blockIdx.x] = t;
        }
    }
}

// visible-set exchange fused into the compaction: every word this rank produced is also stored, coalesced, into the gathered
// buffer of every rank (its own included) through NVLink peer mappings — no collective kernel, no extra pass over the words
// Buffer of every rank (one allocation, mapped into every process): [ flags[EX_SLOTS][R3_MAX_EXCHANGE_RANKS] | pad to EX_HEADER_WORDS ] then
// rows[EX_SLOTS][n_ranks][words_per_rank].  A step with epoch e uses slot e % EX_SLOTS (called `parity` below): rank r stores its words into row (e & 1, r) of every
// buffer and then publishes them with flags[e % EX_SLOTS][r] = e (st.release.sys by the last CTA to finish, after every CTA fenced its stores
// at system scope).  A consumer waits with ld.acquire.sys on the flag of the row it needs — on the device, no host barrier — and the
// other row sets keep the previous epochs intact while the next ones are written.
constexpr uint32_t EX_HEADER_WORDS = 256;
constexpr uint32_t EX_SLOTS = R3_EXCHANGE_SLOTS;   // row sets in flight: epoch e uses slot e % EX_SLOTS, so a consumer may lag EX_SLOTS - 1 epochs behind the producers
struct ExchangeParams { uint32_t* peers[R3_MAX_EXCHANGE_RANKS]; uint32_t n_ranks, word_offset, words_per_rank, flag_offset, epoch; uint32_t* done; };

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) { asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) { uint32_t v; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }

__global__ void __launch_bounds__(CP_THREADS)
compact_visible_kernel(const uint32_t* __restrict__ words, const uint32_t* __restrict__ cta_counts, uint32_t n_words, uint32_t n_cta_counts,
                       uint32_t* __restrict__ visible, uint32_t* __restrict__ visible_count, const __grid_constant__ ExchangeParams ex) {
    __shared__ uint32_t s_warp[CP_THREADS / 32 + 1];
    // (1) survivors in front of this tile: sum of the stream CTAs' counts before it
    const uint32_t tile_base = block_sum_u32<CP_THREADS>(cta_counts, min(blockIdx.x * CP_CTAS_PER_TILE, n_cta_counts), s_warp);
    // (2) block-wide exclusive scan of the word popcounts (one word per thread)
    const uint32_t wi = blockIdx.x * CP_THREADS + threadIdx.x;
    const uint32_t word = wi < n_words ? __ldg(&words[wi]) : 0u;
    if (ex.n_ranks && wi < ex.words_per_rank) {
#pragma unroll 1
        for (uint32_t r = 0; r < ex.n_ranks; ++r) ex.peers[r][(size_t)ex.word_offset + wi] = word;
    }
    uint32_t total;
    const uint32_t excl = tile_base + block_scan_excl<CP_THREADS>((uint32_t)__popc(word), s_warp, &total);
    if (threadIdx.x == 0 && blockIdx.x == gridDim.x - 1) *visible_count = tile_base + total;
    // (3) ascending slot ids
    warp_expand_words(word, excl, (blockIdx.x * CP_THREADS + (threadIdx.x & ~31u)) * 32u, [&](uint32_t pos, uint32_t id) { visible[pos] = id; });
    if (ex.n_ranks) {
        // publish the row: the CTA barrier orders every thread's peer stores before thread 0's system-scope fence (cumulative), which
        // orders them before the arrival; the last CTA to arrive writes the epoch flags with release semantics
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence_system();
            const uint32_t arrived = atomicAdd(ex.done, 1u);
            if (arrived == gridDim.x - 1u) {
                *ex.done = 0u;                                  // next launch of this camera starts from zero (stream-ordered)
                __threadfence_system();
                for (uint32_t r = 0; r < ex.n_ranks; ++r) st_release_sys(ex.peers[r] + ex.flag_offset, ex.epoch);
            }
        }
    }
}

// ---- consumer side: the GLOBAL visible list (ascending global object ids) out of the gathered rows, chained on the epoch flags.
//   wait         : one small CTA spins on flags[parity][r] with ld.acquire.sys until every row's epoch has arrived;
//   count        : CTA (row r, tile t) counts the survivors of its 1024 words;
//   expand       : survivors in front of the tile (sum of the counts before it), block scan, ordered expansion — as the local compaction.
struct MergeParams {
    const uint32_t* gathered;            // this rank's buffer (flags + rows)
    uint32_t n_ranks, words_per_rank, parity, epoch, tiles_per_rank;
    uint32_t rank_base[R3_MAX_EXCHANGE_RANKS];   // global id of slot 0 of every rank's shard
    uint32_t rank_objects[R3_MAX_EXCHANGE_RANKS];
    uint32_t* tile_counts; uint32_t* out; uint32_t* out_count; uint32_t out_cap;
};
__device__ __forceinline__ uint32_t merge_word(const MergeParams& p, uint32_t r, uint32_t w) {
    if (w >= p.words_per_rank) return 0u;
    uint32_t word = __ldcg(p.gathered + EX_HEADER_WORDS + ((size_t)p.parity * p.n_ranks + r) * p.words_per_rank + w);   // written by a peer: L2, never a stale L1 line
    const uint32_t n = p.rank_objects[r];                   // bits beyond the shard's object count are never listed
    if (w * 32u >= n) return 0u;
    if (n - w * 32u < 32u) word &= (1u << (n - w * 32u)) - 1u;
    return word;
}
// one small CTA waits for the flags (thread r: rank r's row); the count / expand kernels behind it on the stream then read complete rows.
// (Spinning inside the 1024-thread count CTAs kept hundreds of them resident while a peer was late — and the next cull + bake of THIS rank
//  off the SMs.)
__global__ void exchange_wait_kernel(const uint32_t* __restrict__ flags, uint32_t n_ranks, uint32_t epoch) {
    if (threadIdx.x < n_ranks)
        while ((int32_t)(ld_acquire_sys(flags + threadIdx.x) - epoch) < 0) __nanosleep(100);
}
__global__ void __launch_bounds__(CP_THREADS) exchange_count_kernel(const __grid_constant__ MergeParams p) {
    const uint32_t r = blockIdx.x / p.tiles_per_rank, t = blockIdx.x % p.tiles_per_rank;
    __shared__ uint32_t s_warp[CP_THREADS / 32];
    const uint32_t cnt = block_reduce<CP_THREADS>((uint32_t)__popc(merge_word(p, r, t * CP_THREADS + threadIdx.x)), s_warp);
    if (threadIdx.x == 0) p.tile_counts[blockIdx.x] = cnt;
}
// back-pressure: a consumer that has finished reading epoch e tells every producer so (acks[my_rank] = e in every rank's buffer); a
// producer about to overwrite the slot of epoch e waits until every consumer has acknowledged it
constexpr uint32_t EX_ACK_WORDS = 128;              // word offset of acks[R3_MAX_EXCHANGE_RANKS] inside the buffer header
__global__ void exchange_ack_kernel(const __grid_constant__ ExchangeParams ex, uint32_t epoch) {
    if (threadIdx.x < ex.n_ranks) {
        __threadfence_system();
        st_release_sys(ex.peers[threadIdx.x] + EX_ACK_WORDS + ex.flag_offset, epoch);   // flag_offset carries my rank here
    }
}
// count-only consumer: CTA (rank r, slice s) sums the popcounts of its slice of row r with 16-byte loads and adds them to out[r] and to the
// total out[n_ranks] — one small wave of CTAs (n_ranks x 16 of 256 threads), so that it slips into the tail of the stream kernel instead of
// queueing thousands of CTAs behind it (tile-sized count CTAs made the weak-scaled step on 8 GPUs markedly slower than on one)
constexpr uint32_t RC_SLICES = 16;
constexpr int LC_THREADS = 256;
__global__ void __launch_bounds__(LC_THREADS) exchange_light_count_kernel(const __grid_constant__ MergeParams p, uint32_t* __restrict__ out) {
    __shared__ uint32_t s_warp[LC_THREADS / 32];
    const uint32_t r = blockIdx.x / RC_SLICES, sl = blockIdx.x % RC_SLICES;
    const uint32_t n_words = (p.rank_objects[r] + 31u) / 32u;                        // words of the shard that can hold survivors
    const uint32_t vecs = (p.words_per_rank + 3u) / 4u, per = (vecs + RC_SLICES - 1u) / RC_SLICES;
    const uint32_t v0 = sl * per, v1 = min(v0 + per, vecs);
    const uint4* row = reinterpret_cast<const uint4*>(p.gathered + EX_HEADER_WORDS + ((size_t)p.parity * p.n_ranks + r) * p.words_per_rank);   // rows are 256-byte aligned
    const uint32_t tail_bits = p.rank_objects[r] & 31u;
    uint32_t cnt = 0;
    for (uint32_t v = v0 + threadIdx.x; v < v1; v += blockDim.x) {
        const uint4 q = __ldcg(&row[v]);
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (uint32_t k = 0; k < 4; ++k) {
            const uint32_t wi = v * 4u + k;
            uint32_t word = wi < n_words ? w[k] : 0u;
            if (tail_bits && wi == n_words - 1u) word &= (1u << tail_bits) - 1u;
            cnt += __popc(word);
        }
    }
    const uint32_t t = block_reduce<LC_THREADS>(cnt, s_warp);
    if (threadIdx.x == 0 && t) { atomicAdd(&out[r], t); atomicAdd(&out[p.n_ranks], t); }
}
// per-rank survivor counts (and their total) from the tile counts: one CTA
__global__ void __launch_bounds__(1024) exchange_rank_counts_kernel(const uint32_t* __restrict__ tile_counts, uint32_t tiles_per_rank, uint32_t n_ranks, uint32_t* __restrict__ out) {
    __shared__ uint32_t s_warp[32];
    uint32_t total = 0;
    for (uint32_t r = 0; r < n_ranks; ++r) {
        const uint32_t sum = block_sum_u32<1024>(tile_counts + r * tiles_per_rank, tiles_per_rank, s_warp);
        if (threadIdx.x == 0) out[r] = sum;
        total += sum;
    }
    if (threadIdx.x == 0) out[n_ranks] = total;
}
__global__ void __launch_bounds__(CP_THREADS) exchange_expand_kernel(const __grid_constant__ MergeParams p) {
    __shared__ uint32_t s_warp[CP_THREADS / 32 + 1];
    const uint32_t r = blockIdx.x / p.tiles_per_rank, t = blockIdx.x % p.tiles_per_rank;
    const uint32_t tile_base = block_sum_u32<CP_THREADS>(p.tile_counts, blockIdx.x, s_warp);
    const uint32_t word = merge_word(p, r, t * CP_THREADS + threadIdx.x);
    uint32_t total;
    const uint32_t excl = tile_base + block_scan_excl<CP_THREADS>((uint32_t)__popc(word), s_warp, &total);
    if (threadIdx.x == 0 && blockIdx.x == gridDim.x - 1) *p.out_count = tile_base + total;
    warp_expand_words(word, excl, p.rank_base[r] + (t * CP_THREADS + (threadIdx.x & ~31u)) * 32u, [&](uint32_t pos, uint32_t id) {
        if (pos < p.out_cap) p.out[pos] = id;
    });
}

}  // namespace

static int launch_cull_bake(r3_ctx* c, r3_camera* cam, uint32_t mode, const r3_camera_header* d_header) {
    const uint32_t n = cam->header.object_count;
    const bool bake = mode & R3_CB_BAKE, cull = mode & R3_CB_CULL;
    if (n == 0 || (!bake && !cull)) {
        // with objects, the last CTA of compact_visible_kernel writes the count
        if (cull) R3_CUDA(c, cudaMemsetAsync(cam->d_visible_count, 0, 4, c->stream));
        return R3_OK;
    }
    CullBakeParams p;
    memcpy(p.view, cam->header.view, 64);
    memcpy(p.view_proj, cam->header.view_proj, 64);
    memcpy(p.frustum, cam->header.frustum, 80);
    p.object_count = n;
    const uint32_t n_ctas = (n + CB_CTA_OBJECTS - 1) / CB_CTA_OBJECTS, n_words = (n + 31) / 32;
    // scratch: two sets of { visibility words [n_words] | stream-CTA counts [n_ctas] }, used alternately: the words of
    // call k stay intact while call k+1 runs, so an exchange of the visible set (r3_device_ptr which = 4) can overlap the
    // next cull on another stream.  (d_tile_state is a u64 array; each set is padded to a 256-byte multiple.)
    const uint64_t set_words = (((uint64_t)n_words + n_ctas + 63) / 64) * 64;
    R3_TRY(r3_reserve_t(c, &cam->d_tile_state, &cam->tile_state_cap, set_words + 2));
    if (cull) cam->words_set ^= 1u;
    uint32_t* words = reinterpret_cast<uint32_t*>(cam->d_tile_state) + (size_t)cam->words_set * set_words;
    cam->d_words = words;
    uint32_t* cta_counts = words + n_words;
    if (!c->hot_valid) return r3_fail(c, R3_E_STATE, "object_uniform_upload before set_objects");
    float4* mats = reinterpret_cast<float4*>(cam->d_matrices);
    // the live mask of r3_set_object_sort_info is only trusted when it covers every slot of this launch; a shorter (stale) one would be
    // read out of bounds — then `enabled` decides, as without sort info
    const bool live = c->have_live && cull && c->sort_flags.size() >= (size_t)n;
#define R3_CB_LAUNCH(B, C, L) \
    cull_bake_kernel<B, C, L><<<n_ctas, CB_THREADS, 0, c->stream>>>(c->d_hot_xyz, reinterpret_cast<const float*>(c->d_hot_w), c->d_affine_bits, c->d_hot_sphere, \
                                                                    c->d_hot_radius, c->d_centre_bits, c->d_enabled_bits, c->d_live_bits, mats, words, cta_counts, p)
    r3_stage_begin(c, R3_STAGE_CULL_BAKE);
    if (d_header) {
        // without a live mask the kernel's `live` word is the enabled word, so the LIVE instantiations read the enabled bits instead
        const DeviceCameraParams dp{d_header, n};
        const uint32_t* live_bits = live ? c->d_live_bits : c->d_enabled_bits;
#define R3_CB_DEV_LAUNCH(B, C)                                                                                                                       \
    cull_bake_kernel<B, C, C, DeviceCameraParams><<<n_ctas, CB_THREADS, 0, c->stream>>>(c->d_hot_xyz, reinterpret_cast<const float*>(c->d_hot_w),     \
                                                                                      c->d_affine_bits, c->d_hot_sphere, c->d_hot_radius, c->d_centre_bits, \
                                                                                      c->d_enabled_bits, live_bits, \
                                                                                      mats, words, cta_counts, dp)
        if (bake && cull) R3_CB_DEV_LAUNCH(true, true);
        else if (bake) R3_CB_DEV_LAUNCH(true, false);
        else R3_CB_DEV_LAUNCH(false, true);
#undef R3_CB_DEV_LAUNCH
    } else if (bake && cull) { if (live) R3_CB_LAUNCH(true, true, true); else R3_CB_LAUNCH(true, true, false); }
    else if (bake) R3_CB_LAUNCH(true, false, false);
    else { if (live) R3_CB_LAUNCH(false, true, true); else R3_CB_LAUNCH(false, true, false); }
#undef R3_CB_LAUNCH
    r3_stage_end(c);
    R3_CHECK_LAUNCH(c, "cull_bake_kernel");
    if (cull) {
        const uint32_t n_tiles = (n_words + CP_THREADS - 1) / CP_THREADS;
        ExchangeParams ex{};
        if (cam->ex_connected) {
            if (n_words > cam->ex_words_per_rank) return r3_fail(c, R3_E_INVALID, "object_uniform_upload: more objects than the exchange was created for");
            for (uint32_t r = 0; r < cam->ex_ranks; ++r) ex.peers[r] = cam->ex_peers[r];
            const uint32_t epoch = ++cam->ex_epoch, parity = epoch % EX_SLOTS;
            if (cam->ex_merge_pending[parity]) {   // this rank's consumer of the slot's previous epoch still reads the rows this step overwrites
                R3_CUDA(c, cudaStreamWaitEvent(c->stream, cam->ex_merge_done[parity], 0));
                cam->ex_merge_pending[parity] = false;
            }
            if (epoch > EX_SLOTS && cam->ex_consumed[parity] == epoch - EX_SLOTS) {
                // ... and so may the PEERS' consumers (the protocol is symmetric: an epoch this rank consumed, every rank consumes): wait, on
                // the device, until all of them have acknowledged it.  With EX_SLOTS row sets a consumer may lag three epochs before this blocks.
                exchange_wait_kernel<<<1, 32, 0, c->stream>>>(cam->d_gathered + EX_ACK_WORDS, cam->ex_ranks, epoch - EX_SLOTS);
                R3_CHECK_LAUNCH(c, "exchange_wait_kernel");
            }
            ex.n_ranks = cam->ex_ranks; ex.words_per_rank = cam->ex_words_per_rank;
            ex.word_offset = EX_HEADER_WORDS + (parity * cam->ex_ranks + cam->ex_rank) * cam->ex_words_per_rank;
            ex.flag_offset = parity * R3_MAX_EXCHANGE_RANKS + cam->ex_rank; ex.epoch = epoch; ex.done = cam->d_ex_done;
            cam->ex_objects = n;
        }
        // with an exchange every slot of this rank's row is written each step (the tail beyond n_words as zeros)
        const uint32_t n_tiles_ex = cam->ex_connected ? (cam->ex_words_per_rank + CP_THREADS - 1) / CP_THREADS : 0u;
        compact_visible_kernel<<<n_tiles > n_tiles_ex ? n_tiles : n_tiles_ex, CP_THREADS, 0, c->stream>>>(words, cta_counts, n_words, n_ctas, cam->d_visible, cam->d_visible_count, ex);
        R3_CHECK_LAUNCH(c, "compact_visible_kernel");
    }
    return R3_OK;
}

int r3_launch_cull_bake(r3_ctx* c, r3_camera* cam, uint32_t mode) { return launch_cull_bake(c, cam, mode, nullptr); }
int r3_launch_cull_bake_device_camera(r3_ctx* c, r3_camera* cam, uint32_t mode, const r3_camera_header* d_header) {
    return launch_cull_bake(c, cam, mode, d_header);
}

uint64_t r3_hot_capacity(uint64_t want) {
    uint64_t cap = 1024;
    while (cap < want) cap *= 2;
    if (cap > want + want / 8 && want > (1u << 20)) cap = want + want / 8;   // large worlds: 12.5% head room instead of a power of two
    return cap;
}
// (re)build the dense hot arrays from the AoS records (all slots)
int r3_split_objects(r3_ctx* c) {
    const uint32_t n = c->n_slots;
    const uint64_t want = n ? n : 1;
    if (want > c->hot_cap) {
        cudaFree(c->d_hot_xyz); cudaFree(c->d_hot_w); cudaFree(c->d_hot_sphere); cudaFree(c->d_enabled_bits); cudaFree(c->d_affine_bits);
        cudaFree(c->d_hot_radius); cudaFree(c->d_centre_bits);
        c->d_hot_xyz = nullptr; c->d_hot_w = nullptr; c->d_hot_sphere = nullptr; c->d_enabled_bits = nullptr; c->d_affine_bits = nullptr;
        c->d_hot_radius = nullptr; c->d_centre_bits = nullptr; c->hot_cap = 0;
        const uint64_t cap = r3_hot_capacity(want);
        R3_CUDA(c, cudaMalloc((void**)&c->d_hot_xyz, cap * 48));
        R3_CUDA(c, cudaMalloc((void**)&c->d_hot_w, cap * 16));
        R3_CUDA(c, cudaMalloc((void**)&c->d_hot_sphere, cap * 16));
        R3_CUDA(c, cudaMalloc((void**)&c->d_hot_radius, cap * 4));
        R3_CUDA(c, cudaMalloc((void**)&c->d_enabled_bits, ((cap + 31) / 32 + 1) * 4));
        R3_CUDA(c, cudaMalloc((void**)&c->d_affine_bits, ((cap + 31) / 32 + 1) * 4));
        R3_CUDA(c, cudaMalloc((void**)&c->d_centre_bits, ((cap + 31) / 32 + 1) * 4));
        c->hot_cap = cap;
    }
    if (n) {
        const uint32_t warps = (n + 31) / 32;
        split_objects_kernel<<<(warps + 7) / 8, 256, 0, c->stream>>>(reinterpret_cast<const float4*>(c->d_objects), n, reinterpret_cast<float*>(c->d_hot_xyz),
                                                                      reinterpret_cast<float*>(c->d_hot_w), c->d_hot_sphere, c->d_hot_radius, c->d_enabled_bits,
                                                                      c->d_affine_bits, c->d_centre_bits);
        R3_CHECK_LAUNCH(c, "split_objects_kernel");
    }
    c->hot_valid = true;
    return R3_OK;
}
// refresh the hot copies of the `n` slots listed in d_slots (device pointer) after a scatter
int r3_split_slots(r3_ctx* c, const uint32_t* d_slots, uint32_t n) {
    if (!c->hot_valid || n == 0) return R3_OK;
    split_slots_kernel<<<(n * 8 + 255) / 256, 256, 0, c->stream>>>(reinterpret_cast<const float4*>(c->d_objects), d_slots, n, c->n_slots,
                                                                    reinterpret_cast<float*>(c->d_hot_xyz), reinterpret_cast<float*>(c->d_hot_w), c->d_hot_sphere,
                                                                    c->d_hot_radius, c->d_enabled_bits, c->d_affine_bits, c->d_centre_bits);
    R3_CHECK_LAUNCH(c, "split_slots_kernel");
    return R3_OK;
}
namespace {
__global__ void mask_word_kernel(uint32_t* word_a, uint32_t* word_b, uint32_t* word_c, uint32_t keep_mask) {
    if (word_a) *word_a &= keep_mask;
    if (word_b) *word_b &= keep_mask;
    if (word_c) *word_c &= keep_mask;
}
}  // namespace
int r3_launch_mask_word(r3_ctx* c, uint32_t* word_a, uint32_t* word_b, uint32_t* word_c, uint32_t keep_mask) {
    mask_word_kernel<<<1, 1, 0, c->stream>>>(word_a, word_b, word_c, keep_mask);
    R3_CHECK_LAUNCH(c, "mask_word_kernel");
    return R3_OK;
}
// r3_resize_objects: the hot copies of slots [0, old_n) are kept by a device copy (FreelistDerivedBuffer::apply, buffer.rs:66-83);
// slots [old_n, n) are zero records: rows, row 3, sphere and radius 0, enabled 0, affine 0 (row 3 is not (0, 0, 0, 1)) and centre 0
// — what split_objects_kernel derives from them, except the centre bit, which it would set (a zero centre is the zero translation);
// a clear bit is always correct, since the cull then reads the sphere.  Bits at or past old_n read 0, also in the old last partial word.
int r3_grow_hot(r3_ctx* c, uint32_t old_n, uint32_t n) {
    if (!c->hot_valid) old_n = 0;
    const uint64_t old_words = ((uint64_t)old_n + 31) / 32;
    if ((uint64_t)n > c->hot_cap || !c->d_hot_xyz) {
        const uint64_t cap = r3_hot_capacity(n ? n : 1), bit_words = (cap + 31) / 32 + 1;
        float4 *xyz = nullptr, *w = nullptr, *sph = nullptr;
        float* rad = nullptr;
        uint32_t *en = nullptr, *af = nullptr, *ce = nullptr;
        R3_CUDA(c, cudaMalloc((void**)&xyz, cap * 48));
        R3_CUDA(c, cudaMalloc((void**)&w, cap * 16));
        R3_CUDA(c, cudaMalloc((void**)&sph, cap * 16));
        R3_CUDA(c, cudaMalloc((void**)&rad, cap * 4));
        R3_CUDA(c, cudaMalloc((void**)&en, bit_words * 4));
        R3_CUDA(c, cudaMalloc((void**)&af, bit_words * 4));
        R3_CUDA(c, cudaMalloc((void**)&ce, bit_words * 4));
        if (old_n) {
            R3_CUDA(c, cudaMemcpyAsync(xyz, c->d_hot_xyz, (size_t)old_n * 48, cudaMemcpyDeviceToDevice, c->stream));
            R3_CUDA(c, cudaMemcpyAsync(w, c->d_hot_w, (size_t)old_n * 16, cudaMemcpyDeviceToDevice, c->stream));
            R3_CUDA(c, cudaMemcpyAsync(sph, c->d_hot_sphere, (size_t)old_n * 16, cudaMemcpyDeviceToDevice, c->stream));
            R3_CUDA(c, cudaMemcpyAsync(rad, c->d_hot_radius, (size_t)old_n * 4, cudaMemcpyDeviceToDevice, c->stream));
            R3_CUDA(c, cudaMemcpyAsync(en, c->d_enabled_bits, old_words * 4, cudaMemcpyDeviceToDevice, c->stream));
            R3_CUDA(c, cudaMemcpyAsync(af, c->d_affine_bits, old_words * 4, cudaMemcpyDeviceToDevice, c->stream));
            R3_CUDA(c, cudaMemcpyAsync(ce, c->d_centre_bits, old_words * 4, cudaMemcpyDeviceToDevice, c->stream));
        }
        R3_CUDA(c, r3_stream_sync(c));
        cudaFree(c->d_hot_xyz); cudaFree(c->d_hot_w); cudaFree(c->d_hot_sphere); cudaFree(c->d_enabled_bits); cudaFree(c->d_affine_bits);
        cudaFree(c->d_hot_radius); cudaFree(c->d_centre_bits);
        c->d_hot_xyz = xyz; c->d_hot_w = w; c->d_hot_sphere = sph; c->d_enabled_bits = en; c->d_affine_bits = af; c->hot_cap = cap;
        c->d_hot_radius = rad; c->d_centre_bits = ce;
    }
    const uint64_t first_word = old_n / 32, new_words = ((uint64_t)n + 31) / 32;
    if (n > old_n) {
        R3_CUDA(c, cudaMemsetAsync(c->d_hot_xyz + (size_t)old_n * 3, 0, (size_t)(n - old_n) * 48, c->stream));
        R3_CUDA(c, cudaMemsetAsync(c->d_hot_w + old_n, 0, (size_t)(n - old_n) * 16, c->stream));
        R3_CUDA(c, cudaMemsetAsync(c->d_hot_sphere + old_n, 0, (size_t)(n - old_n) * 16, c->stream));
        R3_CUDA(c, cudaMemsetAsync(c->d_hot_radius + old_n, 0, (size_t)(n - old_n) * 4, c->stream));
    }
    const uint64_t whole = (old_n & 31u) ? first_word + 1 : first_word;   // first word that holds no kept slot
    if (new_words > whole) {
        R3_CUDA(c, cudaMemsetAsync(c->d_enabled_bits + whole, 0, (new_words - whole) * 4, c->stream));
        R3_CUDA(c, cudaMemsetAsync(c->d_affine_bits + whole, 0, (new_words - whole) * 4, c->stream));
        R3_CUDA(c, cudaMemsetAsync(c->d_centre_bits + whole, 0, (new_words - whole) * 4, c->stream));
    }
    if (old_n & 31u)
        R3_TRY(r3_launch_mask_word(c, c->d_enabled_bits + first_word, c->d_affine_bits + first_word, c->d_centre_bits + first_word, (1u << (old_n & 31u)) - 1u));
    c->hot_valid = true;
    return R3_OK;
}

// ------------------------------------------------------------------ multi-GPU exchange of the visible set (SURVEY 8e)
// One process per GPU.  Every rank owns flags + rows[2][n_ranks][words_per_rank]; rank r's compact kernel stores row r of the step's
// parity into the buffer of every rank through CUDA IPC peer mappings over NVLink / NVSwitch and publishes it with an epoch flag
// (st.release.sys).  Consumers (r3_exchange_merge, or any kernel of the host's) wait for the flag with ld.acquire.sys on the device.
// Protocol: the ranks call r3_object_uniform_upload(CULL) in lockstep (same number of steps); a rank consumes epoch e (or meets the
// others at a host barrier) before it issues epoch e + EX_SLOTS, which reuses the row set; consumers acknowledge their epoch to the producers
// (acks), which wait for the acknowledgements before they overwrite a row set — then no row is overwritten while it is read.
R3_EXPORT int r3_exchange_create(r3_ctx* c, uint32_t camera, uint32_t n_ranks, uint32_t my_rank, uint32_t max_objects_per_rank, uint8_t handle_out[R3_IPC_HANDLE_BYTES]) {
    if (!c || !handle_out) return r3_fail(c, R3_E_INVALID, "exchange_create: null");
    if (n_ranks == 0 || n_ranks > R3_MAX_EXCHANGE_RANKS || my_rank >= n_ranks || max_objects_per_rank == 0) return r3_fail(c, R3_E_INVALID, "exchange_create: bad rank layout");
    r3_camera* cam = r3_get_camera(c, camera);
    if (!cam) return r3_fail(c, R3_E_INVALID, "exchange_create: bad camera");
    static_assert(sizeof(cudaIpcMemHandle_t) == R3_IPC_HANDLE_BYTES, "IPC handle size");
    cudaSetDevice(c->device);
    if (cam->d_gathered) return r3_fail(c, R3_E_STATE, "exchange_create: already created for this camera");
    const uint32_t wpr = (((max_objects_per_rank + 31u) / 32u) + 63u) & ~63u;   // rows start 256-byte aligned
    const size_t total_words = EX_HEADER_WORDS + (size_t)EX_SLOTS * n_ranks * wpr;    // flags | EX_SLOTS sets of n_ranks rows
    R3_CUDA(c, cudaMalloc((void**)&cam->d_gathered, total_words * 4));
    R3_CUDA(c, cudaMemsetAsync(cam->d_gathered, 0, total_words * 4, c->stream));
    if (!cam->d_ex_done) R3_CUDA(c, cudaMalloc((void**)&cam->d_ex_done, 16));
    R3_CUDA(c, cudaMemsetAsync(cam->d_ex_done, 0, 16, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    cam->ex_epoch = 0; cam->ex_objects = 0;
    for (auto& e : cam->ex_consumed) e = 0;
    cudaIpcMemHandle_t h;
    R3_CUDA(c, cudaIpcGetMemHandle(&h, cam->d_gathered));
    memcpy(handle_out, &h, sizeof h);
    cam->ex_ranks = n_ranks; cam->ex_rank = my_rank; cam->ex_words_per_rank = wpr; cam->ex_connected = false;
    return R3_OK;
}
R3_EXPORT int r3_exchange_connect(r3_ctx* c, uint32_t camera, const uint8_t* handles) {
    if (!c || !handles) return r3_fail(c, R3_E_INVALID, "exchange_connect: null");
    r3_camera* cam = r3_get_camera(c, camera);
    if (!cam || !cam->d_gathered) return r3_fail(c, R3_E_STATE, "exchange_connect before exchange_create");
    cudaSetDevice(c->device);
    for (uint32_t r = 0; r < cam->ex_ranks; ++r) {
        if (r == cam->ex_rank) { cam->ex_peers[r] = cam->d_gathered; continue; }
        cudaIpcMemHandle_t h;
        memcpy(&h, handles + (size_t)r * R3_IPC_HANDLE_BYTES, sizeof h);
        void* p = nullptr;
        R3_CUDA(c, cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));   // maps the peer allocation and enables NVLink peer access
        cam->ex_peers[r] = (uint32_t*)p;
    }
    cam->ex_connected = true;
    return R3_OK;
}
R3_EXPORT int r3_exchange_words(r3_ctx* c, uint32_t camera, void** device_ptr, uint64_t* nbytes, uint32_t* words_per_rank) {
    if (!c || !device_ptr || !nbytes) return r3_fail(c, R3_E_INVALID, "exchange_words: null");
    r3_camera* cam = r3_get_camera(c, camera);
    if (!cam || !cam->d_gathered) return r3_fail(c, R3_E_STATE, "exchange_words before exchange_create");
    // the rows of the LAST step (epoch parity); complete once their flags carry the epoch — r3_exchange_merge waits for that on the device,
    // a host reader synchronises its stream and meets the other ranks at a barrier first
    *device_ptr = cam->d_gathered + EX_HEADER_WORDS + (size_t)(cam->ex_epoch % EX_SLOTS) * cam->ex_ranks * cam->ex_words_per_rank;
    *nbytes = (uint64_t)cam->ex_ranks * cam->ex_words_per_rank * 4;
    if (words_per_rank) *words_per_rank = cam->ex_words_per_rank;
    return R3_OK;
}
// Consumer of the exchange: the global visible list on this rank.  rank_objects[r] = slots of rank r's shard in the last step,
// rank_base[r] = global id of its slot 0 (NULL: r * max_objects_per_rank).  Chained on the epoch flags on the device; no host barrier.
static int r3_exchange_consume(r3_ctx* c, uint32_t camera, const uint32_t* rank_objects, const uint32_t* rank_base, bool expand);
R3_EXPORT int r3_exchange_merge(r3_ctx* c, uint32_t camera, const uint32_t* rank_objects, const uint32_t* rank_base) {
    return r3_exchange_consume(c, camera, rank_objects, rank_base, true);
}
static int r3_exchange_consume(r3_ctx* c, uint32_t camera, const uint32_t* rank_objects, const uint32_t* rank_base, bool expand) {
    if (!c || !rank_objects) return r3_fail(c, R3_E_INVALID, "exchange_merge: null");
    r3_camera* cam = r3_get_camera(c, camera);
    if (!cam || !cam->d_gathered || !cam->ex_connected) return r3_fail(c, R3_E_STATE, "exchange_merge before exchange_connect");
    if (cam->ex_epoch == 0) return r3_fail(c, R3_E_STATE, "exchange_merge before the first cull of the exchange");
    cudaSetDevice(c->device);
    MergeParams p{};
    uint64_t total = 0;
    for (uint32_t r = 0; r < cam->ex_ranks; ++r) {
        if ((rank_objects[r] + 31u) / 32u > cam->ex_words_per_rank) return r3_fail(c, R3_E_INVALID, "exchange_merge: a shard is larger than the exchange was created for");
        p.rank_objects[r] = rank_objects[r];
        p.rank_base[r] = rank_base ? rank_base[r] : r * cam->ex_words_per_rank * 32u;
        total += rank_objects[r];
    }
    if (total >= (1ull << 32)) return r3_fail(c, R3_E_INVALID, "exchange_merge: more than 2^32 objects");
    p.gathered = cam->d_gathered; p.n_ranks = cam->ex_ranks; p.words_per_rank = cam->ex_words_per_rank;
    p.epoch = cam->ex_epoch; p.parity = cam->ex_epoch % EX_SLOTS;
    p.tiles_per_rank = (cam->ex_words_per_rank + CP_THREADS - 1) / CP_THREADS;
    const uint32_t n_tiles = p.tiles_per_rank * cam->ex_ranks;
    if (expand) R3_TRY(r3_reserve_t(c, &cam->d_global_visible, &cam->global_visible_cap, total + 1));
    // scratch: [0] list length | [8 .. 8 + ranks] per-rank counts + total | [32 ..] tile counts
    R3_TRY(r3_reserve_t(c, &cam->d_merge_counts, &cam->merge_counts_cap, (uint64_t)n_tiles + 32));
    p.tile_counts = cam->d_merge_counts + 32; p.out = cam->d_global_visible; p.out_count = cam->d_merge_counts; p.out_cap = (uint32_t)total;
    // The consumer runs on the context's LOW-priority side stream, behind the cull that produced this rank's row: the NEXT cull + bake
    // (other parity) overlaps it and keeps the SMs — the merge CTAs fill the tail of the stream kernel and the small compaction kernel
    // (at high priority their 1024-thread CTAs displaced the stream kernel's).  The cull of epoch e + 2 — which overwrites this parity — waits for
    // this merge (r3_launch_cull_bake), and r3_exchange_merged / r3_sync wait for it before handing the list out.
    if (!c->side_stream) {
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);
        R3_CUDA(c, cudaStreamCreateWithPriority(&c->side_stream, cudaStreamNonBlocking, lo));
    }
    const int slot = (int)(cam->ex_epoch % EX_SLOTS);
    if (!cam->ex_cull_done[slot]) R3_CUDA(c, cudaEventCreateWithFlags(&cam->ex_cull_done[slot], cudaEventDisableTiming));
    if (!cam->ex_merge_done[slot]) R3_CUDA(c, cudaEventCreateWithFlags(&cam->ex_merge_done[slot], cudaEventDisableTiming));
    R3_CUDA(c, cudaEventRecord(cam->ex_cull_done[slot], c->stream));
    R3_CUDA(c, cudaStreamWaitEvent(c->side_stream, cam->ex_cull_done[slot], 0));
    exchange_wait_kernel<<<1, 32, 0, c->side_stream>>>(cam->d_gathered + p.parity * R3_MAX_EXCHANGE_RANKS, cam->ex_ranks, p.epoch);
    R3_CHECK_LAUNCH(c, "exchange_wait_kernel");
    if (!expand) {
        R3_CUDA(c, cudaMemsetAsync(cam->d_merge_counts + 8, 0, ((size_t)cam->ex_ranks + 1) * 4, c->side_stream));
        exchange_light_count_kernel<<<cam->ex_ranks * RC_SLICES, LC_THREADS, 0, c->side_stream>>>(p, cam->d_merge_counts + 8);
        R3_CHECK_LAUNCH(c, "exchange_light_count_kernel");
    } else {
        exchange_count_kernel<<<n_tiles, CP_THREADS, 0, c->side_stream>>>(p);
        R3_CHECK_LAUNCH(c, "exchange_count_kernel");
        exchange_rank_counts_kernel<<<1, 1024, 0, c->side_stream>>>(p.tile_counts, p.tiles_per_rank, cam->ex_ranks, cam->d_merge_counts + 8);
        R3_CHECK_LAUNCH(c, "exchange_rank_counts_kernel");
        exchange_expand_kernel<<<n_tiles, CP_THREADS, 0, c->side_stream>>>(p);
        R3_CHECK_LAUNCH(c, "exchange_expand_kernel");
    }
    {   // acknowledge the epoch to every producer (their next write into this slot waits for it)
        ExchangeParams ack{};
        for (uint32_t r = 0; r < cam->ex_ranks; ++r) ack.peers[r] = cam->ex_peers[r];
        ack.n_ranks = cam->ex_ranks; ack.flag_offset = cam->ex_rank;
        exchange_ack_kernel<<<1, 32, 0, c->side_stream>>>(ack, cam->ex_epoch);
        R3_CHECK_LAUNCH(c, "exchange_ack_kernel");
    }
    R3_CUDA(c, cudaEventRecord(cam->ex_merge_done[slot], c->side_stream));
    cam->ex_merge_pending[slot] = true;
    cam->ex_consumed[slot] = cam->ex_epoch;
    return R3_OK;
}
// Light consumer of the exchange: waits for every rank's epoch flag on the device (like r3_exchange_merge) and leaves the visible COUNT of
// every shard — counts[r], r < n_ranks, and their total in counts[n_ranks] — without expanding the list (whose size grows with the number
// of ranks: 4 B per visible object of the WHOLE world on every rank).  r3_exchange_counts reads them back (blocking).
R3_EXPORT int r3_exchange_count(r3_ctx* c, uint32_t camera, const uint32_t* rank_objects) {
    return r3_exchange_consume(c, camera, rank_objects, nullptr, false);
}
R3_EXPORT int r3_exchange_counts(r3_ctx* c, uint32_t camera, uint32_t* counts /* n_ranks + 1 */) {
    if (!c || !counts) return r3_fail(c, R3_E_INVALID, "exchange_counts: null");
    r3_camera* cam = r3_get_camera(c, camera);
    if (!cam || !cam->d_merge_counts) return r3_fail(c, R3_E_STATE, "exchange_counts before exchange_count / exchange_merge");
    cudaSetDevice(c->device);
    for (int k = 0; k < (int)EX_SLOTS; ++k)
        if (cam->ex_merge_pending[k]) { R3_CUDA(c, cudaStreamWaitEvent(c->stream, cam->ex_merge_done[k], 0)); cam->ex_merge_pending[k] = false; }
    R3_CUDA(c, cudaMemcpyAsync(counts, cam->d_merge_counts + 8, ((size_t)cam->ex_ranks + 1) * 4, cudaMemcpyDeviceToHost, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    return R3_OK;
}
R3_EXPORT int r3_exchange_merged(r3_ctx* c, uint32_t camera, void** device_list, void** device_count, uint64_t* capacity) {
    if (!c || !device_list || !device_count) return r3_fail(c, R3_E_INVALID, "exchange_merged: null");
    r3_camera* cam = r3_get_camera(c, camera);
    if (!cam || !cam->d_global_visible) return r3_fail(c, R3_E_STATE, "exchange_merged before exchange_merge");
    for (int k = 0; k < (int)EX_SLOTS; ++k)      // the main stream (and with it r3_sync) now waits for the merges in flight
        if (cam->ex_merge_pending[k]) { R3_CUDA(c, cudaStreamWaitEvent(c->stream, cam->ex_merge_done[k], 0)); cam->ex_merge_pending[k] = false; }
    *device_list = cam->d_global_visible; *device_count = cam->d_merge_counts;
    if (capacity) *capacity = cam->global_visible_cap;
    return R3_OK;
}
R3_EXPORT int r3_exchange_destroy(r3_ctx* c, uint32_t camera) {
    if (!c) return R3_E_INVALID;
    r3_camera* cam = r3_get_camera(c, camera);
    if (!cam) return r3_fail(c, R3_E_INVALID, "exchange_destroy: bad camera");
    cudaSetDevice(c->device);
    r3_stream_sync(c);
    for (uint32_t r = 0; r < cam->ex_ranks; ++r)
        if (cam->ex_connected && r != cam->ex_rank && cam->ex_peers[r]) cudaIpcCloseMemHandle(cam->ex_peers[r]);
    if (c->side_stream) cudaStreamSynchronize(c->side_stream);
    for (int k = 0; k < (int)EX_SLOTS; ++k) {
        if (cam->ex_cull_done[k]) cudaEventDestroy(cam->ex_cull_done[k]);
        if (cam->ex_merge_done[k]) cudaEventDestroy(cam->ex_merge_done[k]);
        cam->ex_cull_done[k] = cam->ex_merge_done[k] = nullptr; cam->ex_merge_pending[k] = false;
    }
    cudaFree(cam->d_gathered);
    cam->d_gathered = nullptr; cam->ex_connected = false; cam->ex_ranks = 0; cam->ex_epoch = 0;
    for (auto& p : cam->ex_peers) p = nullptr;
    return R3_OK;
}
