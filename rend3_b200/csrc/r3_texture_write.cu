// r3_texture_write.cu — rectangles of texels written into the bindless d2 table's blob and the skybox's faces from host or device memory
// (r3_write_texture_regions[_device]), and the blocking readback of either blob (r3_readback_texels).  rend3's textures are immutable
// (TextureManager::add uploads the levels once, rend3/src/managers/texture.rs:98-251), so there a texture that changes is added again every
// frame; here a video frame, a simulation's output, a painted decal or a streamed page is copied into the level it changes.
//
//   texture_region_plan_kernel  ONE CTA: checks every region against the device descriptors (the skybox's by value), writes its copy plan
//                               (destination, row bytes, pitches, copy width) and the exclusive scan of its work units, a unit being a row
//                               segment of at most SEG_BYTES bytes; a dropped region has no unit
//   texture_region_copy_kernel  persistent (one wave of resident CTAs): each warp takes units by grid stride, finds the unit's region by a
//                               binary search over the scan and copies the segment coalesced, 1 to 16 bytes per lane and step
// Both launch configurations depend on the SM count only, so frames whose region count stays above 0 keep the frame graph's topology.
// The host form runs the same two kernels on a staged copy of its arguments.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <vector>

#include "r3_common.cuh"
#include "r3_scan.cuh"

namespace {

constexpr uint32_t PLAN_THREADS = 256;
constexpr uint32_t COPY_THREADS = 256;
constexpr uint32_t SEG_BYTES = 2048;   // bytes of one unit: a warp moves it in 4 steps of 16 B per lane

struct texw_plan {
    uint8_t* dst;
    const uint8_t* src;
    uint64_t dst_pitch;       // bytes between rows (block rows) of the level
    uint32_t src_pitch, row_bytes;
    uint32_t segs;            // units per row
    uint32_t width_log2;      // copy width: 1 << width_log2 bytes
};
static_assert(sizeof(texw_plan) == 40, "texw_plan");

// where regions can land: the table (descriptors in device memory on the device, the host mirror on the host) and the skybox
struct texw_targets {
    const r3_texture_desc* descs; uint32_t n_textures;
    uint8_t* texels;
    r3_texture_desc sky; uint64_t sky_face_bytes; uint32_t has_sky;
    uint8_t* sky_texels;
};

struct texw_geom { uint64_t dst_offset, dst_pitch; uint32_t row_bytes, rows; };

__host__ __device__ inline uint64_t texw_level_bytes(uint32_t f, uint32_t w, uint32_t h) { return R3_TEXFMT_LEVEL_BYTES(f, w, h); }

// The rules of a valid region (include/rend3_b200.h) against the descriptor of its target (texw_target).  For a face, d->byte_offset
// already points at the face.
__host__ __device__ inline bool texw_check(const r3_texture_region& r, const r3_texture_desc* d, uint64_t nbytes, texw_geom* g) {
    if (r._reserved || r.level >= d->mip_count || !r.width || !r.height) return false;
    const uint32_t f = d->format;
    const uint32_t lw = (d->width >> r.level) ? (d->width >> r.level) : 1u, lh = (d->height >> r.level) ? (d->height >> r.level) : 1u;
    if ((uint64_t)r.x + r.width > lw || (uint64_t)r.y + r.height > lh) return false;
    const bool block = R3_TEXFMT_IS_BLOCK(f);
    const uint32_t elem = block ? R3_TEXFMT_BLOCK_BYTES(f) : R3_TEXFMT_BPP(f);
    uint32_t cols = r.width, rows = r.height, x = r.x, y = r.y, level_cols = lw;
    if (block) {
        if ((r.x & 3u) || (r.y & 3u)) return false;
        if (((r.width & 3u) && r.x + r.width != lw) || ((r.height & 3u) && r.y + r.height != lh)) return false;
        cols = (r.width + 3u) / 4u; rows = (r.height + 3u) / 4u; x = r.x / 4u; y = r.y / 4u; level_cols = (lw + 3u) / 4u;
    }
    const uint64_t row_bytes = (uint64_t)cols * elem;
    if (r.src_offset % elem || r.src_pitch % elem || r.src_pitch < row_bytes) return false;
    if (r.src_offset > nbytes) return false;
    const uint64_t room = nbytes - r.src_offset, span = (uint64_t)(rows - 1) * r.src_pitch;   // < 2^64: rows and pitch are 32-bit
    if (span > room || row_bytes > room - span) return false;
    uint64_t level_off = 0;
    for (uint32_t l = 0; l < r.level; ++l)
        level_off += texw_level_bytes(f, (d->width >> l) ? (d->width >> l) : 1u, (d->height >> l) ? (d->height >> l) : 1u);
    g->dst_pitch = (uint64_t)level_cols * elem;
    g->dst_offset = d->byte_offset + level_off + (uint64_t)y * g->dst_pitch + (uint64_t)x * elem;
    g->row_bytes = (uint32_t)row_bytes;   // <= src_pitch
    g->rows = rows;
    return true;
}

// false when a region's target does not exist; else its descriptor (copied, so that no pointer selects between two places) and blob.  A
// face's descriptor gets the face's byte offset and height = width.
__host__ __device__ inline bool texw_target(const texw_targets& t, uint32_t texture, r3_texture_desc* d, uint8_t** blob) {
    if (texture & 0x80000000u) {
        const uint32_t fi = texture & 0x7FFFFFFFu;
        if (!t.has_sky || fi >= 6u) return false;
        *d = t.sky;
        d->height = d->width;
        d->byte_offset += fi * t.sky_face_bytes;
        *blob = t.sky_texels;
        return true;
    }
    if (texture >= t.n_textures) return false;
    *d = t.descs[texture];
    *blob = t.texels;
    return true;
}

__global__ void __launch_bounds__(PLAN_THREADS) texture_region_plan_kernel(const r3_texture_region* __restrict__ regions, uint32_t n,
                                                                            const uint8_t* src, uint64_t nbytes, const texw_targets t,
                                                                            texw_plan* __restrict__ plans, unsigned long long* __restrict__ scan) {
    __shared__ unsigned long long s_warp[PLAN_THREADS / 32 + 1];
    const unsigned long long total = block_scan_excl_chunked<PLAN_THREADS, unsigned long long>(
        n, s_warp,
        [&](uint32_t i) -> unsigned long long {
            const r3_texture_region r = regions[i];
            r3_texture_desc d;
            uint8_t* blob = nullptr;
            texw_geom g;
            if (!texw_target(t, r.texture, &d, &blob) || !texw_check(r, &d, nbytes, &g)) return 0ull;   // dropped whole
            texw_plan p;
            p.dst = blob + g.dst_offset;
            p.src = src + r.src_offset;
            p.dst_pitch = g.dst_pitch;
            p.src_pitch = r.src_pitch;
            p.row_bytes = g.row_bytes;
            p.segs = (g.row_bytes + SEG_BYTES - 1) / SEG_BYTES;
            // the widest copy every row start of both sides and the row length are aligned to
            const uint64_t a = (uint64_t)(uintptr_t)p.dst | (uint64_t)(uintptr_t)p.src | p.dst_pitch | p.src_pitch | p.row_bytes | 16u;
            p.width_log2 = (uint32_t)(__ffsll((long long)a) - 1);
            plans[i] = p;
            return (unsigned long long)g.rows * p.segs;
        },
        [&](uint32_t i, unsigned long long v) { scan[i] = v; });
    if (threadIdx.x == 0) scan[n] = total;
}

template <typename T>
__device__ __forceinline__ void copy_span(uint8_t* dst, const uint8_t* src, uint32_t bytes, uint32_t lane) {
    T* d = reinterpret_cast<T*>(dst);
    const T* s = reinterpret_cast<const T*>(src);
    for (uint32_t i = lane; i < bytes / (uint32_t)sizeof(T); i += 32) d[i] = s[i];
}

__global__ void __launch_bounds__(COPY_THREADS) texture_region_copy_kernel(const texw_plan* __restrict__ plans,
                                                                           const unsigned long long* __restrict__ scan, uint32_t n) {
    const uint32_t lane = threadIdx.x & 31;
    const unsigned long long total = scan[n], warps = (unsigned long long)gridDim.x * (COPY_THREADS / 32);
    for (unsigned long long u = (unsigned long long)blockIdx.x * (COPY_THREADS / 32) + (threadIdx.x >> 5); u < total; u += warps) {
        uint32_t lo = 0, hi = n;   // scan[lo] <= u < scan[hi]: ends at the region that owns unit u (regions without units are skipped)
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (scan[mid] <= u) lo = mid; else hi = mid;
        }
        const texw_plan p = plans[lo];
        const unsigned long long local = u - scan[lo], row = local / p.segs;
        const uint32_t begin = (uint32_t)(local - row * p.segs) * SEG_BYTES, bytes = min(SEG_BYTES, p.row_bytes - begin);
        uint8_t* d = p.dst + row * p.dst_pitch + begin;
        const uint8_t* s = p.src + row * p.src_pitch + begin;
        switch (p.width_log2) {
            case 4: copy_span<uint4>(d, s, bytes, lane); break;
            case 3: copy_span<uint2>(d, s, bytes, lane); break;
            case 2: copy_span<uint32_t>(d, s, bytes, lane); break;
            case 1: copy_span<uint16_t>(d, s, bytes, lane); break;
            default: copy_span<uint8_t>(d, s, bytes, lane); break;
        }
    }
}

uint64_t sky_face_bytes(const r3_texture_desc& d) {
    uint64_t face = 0;
    for (uint32_t l = 0; l < d.mip_count; ++l) {
        const uint32_t w = (d.width >> l) ? (d.width >> l) : 1u;
        face += texw_level_bytes(d.format, w, w);
    }
    return face;
}

texw_targets targets(const r3_ctx* c, const r3_texture_desc* descs) {
    texw_targets t{};
    t.descs = descs; t.n_textures = c->n_textures; t.texels = c->d_texels;
    t.has_sky = c->has_skybox ? 1u : 0u;
    if (c->has_skybox) { t.sky = c->sky_desc; t.sky_face_bytes = sky_face_bytes(c->sky_desc); t.sky_texels = c->d_sky_texels; }
    return t;
}

// CTAs of the copy kernel resident at once on the whole GPU (a property of the binary: asked once)
int copy_grid(const r3_ctx* c) {
    static int per_sm = 0;
    if (!per_sm && (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, texture_region_copy_kernel, COPY_THREADS, 0) != cudaSuccess || per_sm < 1)) {
        cudaGetLastError();
        per_sm = 1;
    }
    return c->sm_count * per_sm;
}

int launch_regions(r3_ctx* c, const r3_texture_region* d_regions, uint32_t n, const uint8_t* d_src, uint64_t nbytes) {
    // plans then the scan's n + 1 entries; grow-only, so only a call with a larger n than every earlier one reallocates (and flushes a frame)
    const uint64_t need = (uint64_t)n * sizeof(texw_plan) + ((uint64_t)n + 1) * 8;
    R3_TRY(r3_reserve(c, &c->d_texw_plan, &c->texw_plan_cap, need, 1, false, false));
    texw_plan* plans = (texw_plan*)c->d_texw_plan;
    unsigned long long* scan = (unsigned long long*)(plans + n);
    texture_region_plan_kernel<<<1, PLAN_THREADS, 0, c->stream>>>(d_regions, n, d_src, nbytes, targets(c, c->d_tex_descs), plans, scan);
    R3_CHECK_LAUNCH(c, "texture_region_plan_kernel");
    texture_region_copy_kernel<<<copy_grid(c), COPY_THREADS, 0, c->stream>>>(plans, scan, n);
    R3_CHECK_LAUNCH(c, "texture_region_copy_kernel");
    return R3_OK;
}

}  // namespace

R3_EXPORT int r3_write_texture_regions(r3_ctx* c, const r3_texture_region* regions, uint32_t n, const void* texels, uint64_t nbytes) {
    if (!c) return R3_E_INVALID;
    if (n == 0) return R3_OK;
    if (!regions || (!texels && nbytes)) return r3_fail(c, R3_E_INVALID, "write_texture_regions: null");
    if (!c->n_textures && !c->has_skybox) return r3_fail(c, R3_E_STATE, "write_texture_regions: neither a texture table nor a skybox");
    // the whole call is checked against the host's copy of the descriptors before anything is enqueued
    const texw_targets t = targets(c, c->tex_desc_host.data());
    struct rect { uint32_t texture, level, x, y, x1, y1; };
    std::vector<rect> rects(n);
    for (uint32_t i = 0; i < n; ++i) {
        const r3_texture_region& r = regions[i];
        r3_texture_desc d;
        uint8_t* blob = nullptr;
        texw_geom g;
        if (!texw_target(t, r.texture, &d, &blob) || !texw_check(r, &d, nbytes, &g)) {
            char msg[96];
            snprintf(msg, sizeof msg, "write_texture_regions: region %u is invalid", i);
            return r3_fail(c, R3_E_INVALID, msg);
        }
        rects[i] = {r.texture, r.level, r.x, r.y, r.x + r.width, r.y + r.height};
    }
    // no two rectangles of one level may meet: sorted by (target, level, x), each is compared with the ones that start left of its end
    std::sort(rects.begin(), rects.end(), [](const rect& a, const rect& b) {
        return a.texture != b.texture ? a.texture < b.texture : a.level != b.level ? a.level < b.level : a.x < b.x;
    });
    for (uint32_t i = 0; i < n; ++i)
        for (uint32_t j = i + 1; j < n && rects[j].texture == rects[i].texture && rects[j].level == rects[i].level && rects[j].x < rects[i].x1; ++j)
            if (rects[j].y < rects[i].y1 && rects[i].y < rects[j].y1) return r3_fail(c, R3_E_INVALID, "write_texture_regions: two regions overlap");
    cudaSetDevice(c->device);
    // regions, then the texels from a 256-byte boundary, so a source's alignment on the device is its src_offset's
    const uint64_t region_bytes = (uint64_t)n * sizeof(r3_texture_region), texel_at = (region_bytes + 255) & ~255ull;
    R3_TRY(r3_reserve(c, &c->d_scratch, &c->scratch_cap, texel_at + nbytes, 1, false, false));
    uint8_t* s = (uint8_t*)c->d_scratch;
    R3_CUDA(c, cudaMemcpyAsync(s, regions, region_bytes, cudaMemcpyHostToDevice, c->stream));
    if (nbytes) R3_CUDA(c, cudaMemcpyAsync(s + texel_at, texels, nbytes, cudaMemcpyHostToDevice, c->stream));
    R3_TRY(launch_regions(c, (const r3_texture_region*)s, n, s + texel_at, nbytes));
    R3_CUDA(c, r3_stream_sync(c));   // host pointers are only borrowed for the call
    return R3_OK;
}

R3_EXPORT int r3_write_texture_regions_device(r3_ctx* c, const r3_texture_region* d_regions, uint32_t n, const void* d_texels, uint64_t nbytes) {
    if (!c) return R3_E_INVALID;
    if (n == 0) return R3_OK;
    if (!d_regions || ((uintptr_t)d_regions & 7u) || (!d_texels && nbytes))
        return r3_fail(c, R3_E_INVALID, "write_texture_regions_device: null or misaligned pointer (regions: 8 bytes)");
    if (!c->n_textures && !c->has_skybox) return r3_fail(c, R3_E_STATE, "write_texture_regions_device: neither a texture table nor a skybox");
    cudaSetDevice(c->device);
    return launch_regions(c, d_regions, n, (const uint8_t*)d_texels, nbytes);
}

R3_EXPORT int r3_readback_texels(r3_ctx* c, int skybox, uint64_t byte_offset, void* out, uint64_t nbytes) {
    if (!c) return R3_E_INVALID;
    if (!out && nbytes) return r3_fail(c, R3_E_INVALID, "readback_texels: null");
    const uint64_t size = skybox ? (c->has_skybox ? c->sky_desc.byte_offset + 6 * sky_face_bytes(c->sky_desc) : 0) : c->texel_bytes;
    if (byte_offset > size || nbytes > size - byte_offset) return r3_fail(c, R3_E_INVALID, "readback_texels: range outside the blob");
    if (nbytes == 0) return R3_OK;
    cudaSetDevice(c->device);
    R3_CUDA(c, r3_stream_sync(c));
    R3_CUDA(c, cudaMemcpy(out, (skybox ? c->d_sky_texels : c->d_texels) + byte_offset, nbytes, cudaMemcpyDeviceToHost));
    return R3_OK;
}
