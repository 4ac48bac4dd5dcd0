// r3_ctx.cu — context, uploads, readbacks and the C ABI glue of librend3_b200.so (include/rend3_b200.h).
// Host logic only; the kernels live in r3_cull_bake.cu, r3_tri_cull.cu, r3_raster.cu, r3_shade.cu.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>

#include "r3_common.cuh"

int r3_fail(r3_ctx* c, int code, const char* msg) {
    if (c) c->err = msg;
    return code;
}
int r3_cuda_fail(r3_ctx* c, cudaError_t e, const char* where) {
    if (c) {
        c->err = std::string(where) + ": " + cudaGetErrorString(e);
    }
    cudaGetLastError();   // clear the sticky-less error so later calls report their own
    return e == cudaErrorMemoryAllocation ? R3_E_OOM : R3_E_CUDA;
}
int r3_check_object_writer(r3_ctx* c, const char* who, uint32_t needs) {
    const bool no_objects = !c->d_objects || ((needs & R3_NEED_HOT) && !c->hot_valid);
    if ((needs & (R3_NEED_OBJECTS | R3_NEED_HOT)) && no_objects) return r3_fail(c, R3_E_STATE, (std::string(who) + " before set_objects").c_str());
    if ((needs & R3_NEED_OWNED) && c->objects_borrowed)
        return r3_fail(c, R3_E_STATE, (std::string(who) + ": the object buffer is borrowed (r3_set_objects_device)").c_str());
    if ((needs & R3_NEED_SPHERES) && c->n_mesh_spheres < c->n_slots)
        return r3_fail(c, R3_E_STATE, (std::string(who) + ": r3_set_object_mesh_spheres does not cover every slot").c_str());
    return R3_OK;
}

int r3_reserve(r3_ctx* c, void** ptr, uint64_t* cap, uint64_t need, size_t elem, bool keep, bool zero_new) {
    if (*ptr && *cap >= need) return R3_OK;
    uint64_t ncap = need < 16 ? 16 : need;
    void* n = nullptr;
    R3_CUDA(c, cudaMalloc(&n, ncap * elem));
    if (zero_new) R3_CUDA(c, cudaMemsetAsync(n, 0, ncap * elem, c->stream));
    if (*ptr) {
        if (keep && *cap) R3_CUDA(c, cudaMemcpyAsync(n, *ptr, *cap * elem, cudaMemcpyDeviceToDevice, c->stream));
        R3_CUDA(c, r3_stream_sync(c));
        cudaFree(*ptr);
    }
    *ptr = n;
    *cap = ncap;
    return R3_OK;
}

// ------------------------------------------------------------------ context
R3_EXPORT uint32_t r3_abi_version(void) { return R3_ABI_VERSION; }

R3_EXPORT int r3_ctx_create(int device, r3_ctx** out) {
    if (!out) return R3_E_INVALID;
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0 || device < 0 || device >= count) {
        cudaGetLastError();
        return R3_E_NO_DEVICE;   // there is no CPU fallback: the caller must fail (RendererInitializationError::MissingAdapter)
    }
    r3_ctx* c = new (std::nothrow) r3_ctx();
    if (!c) return R3_E_OOM;
    c->device = device;
    // the context's stream gets the greatest priority: the exchange consumer's side stream (least priority) then only fills the SMs it leaves idle
    int prio_least = 0, prio_greatest = 0;
    if (cudaSetDevice(device) == cudaSuccess) cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest);
    if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithPriority(&c->stream, cudaStreamNonBlocking, prio_greatest) != cudaSuccess) {
        delete c;
        cudaGetLastError();
        return R3_E_CUDA;
    }
    { int coop = 0; cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, device); c->coop_launch_ok = coop != 0; }
    if (cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || c->sm_count < 1) { cudaStreamDestroy(c->stream); delete c; cudaGetLastError(); return R3_E_CUDA; }
    if (cudaMalloc((void**)&c->d_stats, 8 * sizeof(unsigned long long)) != cudaSuccess) { delete c; return R3_E_OOM; }
    cudaMemsetAsync(c->d_stats, 0, 64, c->stream);
    // the shading reads the point-light count from this buffer in every frame: it exists from the start, holding no light
    c->point_bytes_cap = 16 + 16 * sizeof(r3_point_light);
    if (cudaMalloc((void**)&c->d_point, c->point_bytes_cap) != cudaSuccess) { cudaFree(c->d_stats); delete c; return R3_E_OOM; }
    cudaMemsetAsync(c->d_point, 0, c->point_bytes_cap, c->stream);
    *out = c;
    return R3_OK;
}

static void free_jobs(r3_jobs& j) { cudaFree(j.d_batches); cudaFree(j.d_regions); cudaFree(j.d_region_first_inv); cudaFree(j.d_header); }

R3_EXPORT int r3_ctx_destroy(r3_ctx* c) {
    if (!c) return R3_E_INVALID;
    cudaSetDevice(c->device);
    r3_stream_sync(c);
    if (c->side_stream) cudaStreamSynchronize(c->side_stream);
    r3_peer_destroy(c);
    r3_anim_destroy(c);
    r3_deform_destroy(c);
    r3_variants_destroy(c);
    if (!c->objects_borrowed) cudaFree(c->d_objects);
    cudaFree(c->d_hot_xyz); cudaFree(c->d_hot_w); cudaFree(c->d_hot_sphere); cudaFree(c->d_enabled_bits); cudaFree(c->d_affine_bits); cudaFree(c->d_hot_radius); cudaFree(c->d_centre_bits); cudaFree(c->d_tex_descs); cudaFree(c->d_texels); cudaFree(c->d_sky_texels);
    cudaFree(c->d_sort_key8); cudaFree(c->d_sort_loc); cudaFree(c->d_gsort_keys[0]); cudaFree(c->d_gsort_keys[1]); cudaFree(c->d_gsort_hist); cudaFree(c->d_gsort_header);
    cudaFree(c->d_mesh_spheres); cudaFree(c->d_live_bits); cudaFree(c->d_mesh); cudaFree(c->d_materials); cudaFree(c->d_dir); cudaFree(c->d_point);
    cudaFree(c->d_light_mats); cudaFree(c->d_atlas); cudaFree(c->d_light_src); cudaFree(c->d_shadow_cams); cudaFree(c->d_point_src); cudaFree(c->d_point_live);
    for (auto& k : c->cams) {
        cudaFree(k.d_matrices); cudaFree(k.d_visible); cudaFree(k.d_visible_count); cudaFree(k.d_tile_state);
        if (k.d_gathered) {   // visible-set exchange: unmap the peers' buffers, free ours
            for (uint32_t r = 0; r < k.ex_ranks; ++r)
                if (k.ex_connected && r != k.ex_rank && k.ex_peers[r]) cudaIpcCloseMemHandle(k.ex_peers[r]);
            cudaFree(k.d_gathered);
        }
        cudaFree(k.d_ex_done); cudaFree(k.d_global_visible); cudaFree(k.d_merge_counts);
        for (int q = 0; q < R3_EXCHANGE_SLOTS; ++q) { if (k.ex_cull_done[q]) cudaEventDestroy(k.ex_cull_done[q]); if (k.ex_merge_done[q]) cudaEventDestroy(k.ex_merge_done[q]); }
        free_jobs(k.jobs[0]); free_jobs(k.jobs[1]);
        cudaFree(k.index_buffer.d); cudaFree(k.draw_call_buffer.d); cudaFree(k.results_buffer.d);
        cudaFree(k.d_resid_bits); cudaFree(k.d_word_scan); cudaFree(k.d_block_sums);
        cudaFree(k.d_prev_inv[0]); cudaFree(k.d_prev_inv[1]); cudaFree(k.d_sort_keys[0]); cudaFree(k.d_sort_keys[1]); cudaFree(k.d_sort_hist); cudaFree(k.d_batch_tmp);
    }
    cudaFree(c->d_vis); cudaFree(c->d_hdr32); cudaFree(c->d_hdr16); cudaFree(c->d_depth); cudaFree(c->d_ldr);
    for (float* p : c->d_hiz) cudaFree(p);
    cudaFree(c->d_hiz_ptrs); cudaFree(c->d_hiz_dims);
    cudaFree(c->d_tris[0]); cudaFree(c->d_tris[1]); cudaFree(c->d_tris[2]); cudaFree(c->d_tris[3]); cudaFree(c->d_stats); cudaFree(c->d_scratch);
    cudaFree(c->d_texw_plan);
    cudaFree(c->d_frag_heads); cudaFree(c->d_frag_nodes);
    for (cudaEvent_t e : c->timer.pool) cudaEventDestroy(e);
    for (auto& x : c->frame_exec) if (x) cudaGraphExecDestroy(x);
    if (c->side_stream) cudaStreamDestroy(c->side_stream);
    cudaStreamDestroy(c->stream);
    delete c;
    return R3_OK;
}
R3_EXPORT const char* r3_last_error(const r3_ctx* c) { return c ? c->err.c_str() : "null context"; }
R3_EXPORT int r3_sync(r3_ctx* c) {
    if (!c) return R3_E_INVALID;
    cudaSetDevice(c->device);
    R3_CUDA(c, r3_stream_sync(c));
    if (c->side_stream) R3_CUDA(c, cudaStreamSynchronize(c->side_stream));   // exchange consumers in flight
    return R3_OK;
}
R3_EXPORT int r3_get_stream(r3_ctx* c, void** s) {
    if (!c || !s) return R3_E_INVALID;
    *s = (void*)c->stream;
    return R3_OK;
}
R3_EXPORT int r3_launch_count(r3_ctx* c, uint64_t* n) {
    if (!c || !n) return R3_E_INVALID;
    *n = c->launches;
    return R3_OK;
}

// ------------------------------------------------------------------ frame graph
// End the capture (if one is running) and submit what it recorded.  `slot` >= 0: keep the instantiated graph of that frame parity and
// update it in place next time (cudaGraphExecUpdate: same topology, new kernel arguments / pointers); slot < 0: one-off (an early flush).
static cudaError_t r3_submit_capture(r3_ctx* c, int slot) {
    if (!c->capturing) return cudaSuccess;
    c->capturing = false;
    cudaGraph_t g = nullptr;
    cudaError_t e = cudaStreamEndCapture(c->stream, &g);
    if (e != cudaSuccess || !g) return e != cudaSuccess ? e : cudaErrorUnknown;
    if (slot < 0) {
        cudaGraphExec_t x = nullptr;
        e = cudaGraphInstantiate(&x, g, 0);
        if (e == cudaSuccess) e = cudaGraphLaunch(x, c->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);   // the one-off exec is destroyed right away: wait for it
        if (x) cudaGraphExecDestroy(x);
        cudaGraphDestroy(g);
        return e;
    }
    cudaGraphExec_t& x = c->frame_exec[slot];
    if (x) {
        cudaGraphExecUpdateResultInfo info;
        if (cudaGraphExecUpdate(x, g, &info) != cudaSuccess) {   // another topology (new buffers sizes, another routine set): instantiate again
            cudaGetLastError();
            cudaGraphExecDestroy(x);
            x = nullptr;
        }
    }
    if (!x) {
        e = cudaGraphInstantiate(&x, g, 0);
        c->graph_reinstantiations++;
    }
    if (e == cudaSuccess) e = cudaGraphLaunch(x, c->stream);
    cudaGraphDestroy(g);
    return e;
}
cudaError_t r3_stream_sync(r3_ctx* c) {
    if (c->capturing) {
        // a stage needs the stream to drain in the middle of a recorded frame (a buffer grows, a host path reads back): submit what
        // was recorded, wait, and let the rest of the frame run eagerly
        const cudaError_t e = r3_submit_capture(c, -1);
        c->frames_flushed++;
        if (e != cudaSuccess) return e;
    }
    return cudaStreamSynchronize(c->stream);
}
R3_EXPORT int r3_frame_begin(r3_ctx* c) {
    if (!c) return R3_E_INVALID;
    cudaSetDevice(c->device);
    if (c->capturing) return r3_fail(c, R3_E_STATE, "frame_begin: a frame is already being recorded");
    if (c->timer.enabled) return R3_OK;       // per-kernel timing needs real event records: the frame runs eagerly
    // the invocation bounds of the device batching are read back once after the records changed: do it before the recording starts, so
    // that a frame after r3_update_objects / r3_set_objects does not have to flush in its middle for them
    if (c->gpu_batching_ok) R3_TRY(r3_compute_max_invocations(c));
    R3_CUDA(c, cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeRelaxed));
    c->capturing = true;
    return R3_OK;
}
R3_EXPORT int r3_frame_end(r3_ctx* c) {
    if (!c) return R3_E_INVALID;
    cudaSetDevice(c->device);
    const bool was = c->capturing;
    const cudaError_t e = r3_submit_capture(c, (int)(c->frame_index & 1u));
    c->frame_index++;
    if (was) c->frames_graphed++;
    if (e != cudaSuccess) return r3_cuda_fail(c, e, "frame_end (graph submission)");
    return R3_OK;
}
R3_EXPORT int r3_frame_graph_stats(r3_ctx* c, uint64_t stats[4]) {
    if (!c || !stats) return R3_E_INVALID;
    stats[0] = c->frame_index; stats[1] = c->frames_graphed; stats[2] = c->frames_flushed; stats[3] = c->graph_reinstantiations;
    return R3_OK;
}

// ------------------------------------------------------------------ stage timing
void r3_stage_begin(r3_ctx* c, int stage) {
    r3_stage_timer& t = c->timer;
    if (!t.enabled || c->capturing) return;
    if (t.pool.size() < 2 * (t.used + 1)) {
        cudaEvent_t a = nullptr, b = nullptr;
        if (cudaEventCreate(&a) != cudaSuccess || cudaEventCreate(&b) != cudaSuccess) { t.enabled = false; return; }
        t.pool.push_back(a); t.pool.push_back(b); t.stage_of.push_back(stage);
    }
    t.stage_of[t.used] = stage;
    cudaEventRecord(t.pool[2 * t.used], c->stream);
}
void r3_stage_end(r3_ctx* c) {
    r3_stage_timer& t = c->timer;
    if (!t.enabled || c->capturing) return;
    cudaEventRecord(t.pool[2 * t.used + 1], c->stream);
    t.used++;
}
R3_EXPORT int r3_set_stage_timing(r3_ctx* c, int enabled) {
    if (!c) return R3_E_INVALID;
    cudaSetDevice(c->device);
    c->timer.enabled = enabled != 0;
    c->timer.used = 0;
    return R3_OK;
}
R3_EXPORT int r3_stage_times(r3_ctx* c, double ms[8], uint32_t launches[8]) {
    if (!c || !ms || !launches) return R3_E_INVALID;
    cudaSetDevice(c->device);
    R3_CUDA(c, r3_stream_sync(c));
    for (int k = 0; k < 8; ++k) { ms[k] = 0.0; launches[k] = 0; }
    r3_stage_timer& t = c->timer;
    for (size_t k = 0; k < t.used; ++k) {
        float e = 0.f;
        if (cudaEventElapsedTime(&e, t.pool[2 * k], t.pool[2 * k + 1]) == cudaSuccess && t.stage_of[k] >= 0 && t.stage_of[k] < 8) { ms[t.stage_of[k]] += e; launches[t.stage_of[k]]++; }
    }
    t.used = 0;
    return R3_OK;
}

// ------------------------------------------------------------------ world data
R3_EXPORT int r3_set_objects(r3_ctx* c, const r3_object* recs, uint32_t n) {
    if (!c || (!recs && n)) return r3_fail(c, R3_E_INVALID, "set_objects: null records");
    cudaSetDevice(c->device);
    if (c->objects_borrowed) { c->d_objects = nullptr; c->objects_cap = 0; c->objects_borrowed = false; }
    R3_TRY(r3_reserve_t(c, &c->d_objects, &c->objects_cap, n));
    if (n) R3_CUDA(c, cudaMemcpyAsync(c->d_objects, recs, (size_t)n * sizeof(r3_object), cudaMemcpyHostToDevice, c->stream));
    c->n_slots = n;
    c->max_invocations_valid = false;
    R3_TRY(r3_split_objects(c));
    R3_CUDA(c, r3_stream_sync(c));   // host pointer is only borrowed for the call
    return R3_OK;
}
R3_EXPORT int r3_set_objects_device(r3_ctx* c, const void* dptr, uint32_t n) {
    if (!c || (!dptr && n)) return r3_fail(c, R3_E_INVALID, "set_objects_device: null pointer");
    if (!c->objects_borrowed) { cudaFree(c->d_objects); }
    c->d_objects = (r3_object*)dptr;
    c->objects_cap = n; c->n_slots = n; c->objects_borrowed = true;
    c->max_invocations_valid = false;
    cudaSetDevice(c->device);
    return r3_split_objects(c);   // snapshot of the hot fields: call again after changing the records
}

// ScatterCopy (rend3/shaders/scatter_copy.wgsl) of records of Q float4s (8: r3_object, 13: r3_material): entry i copies src record i
// to dst record idx[i], one 16-byte lane per float4.  blockDim.x must be a multiple of Q, so that a lane's float4 is threadIdx.x % Q.
template <uint32_t Q>
__global__ void scatter_records_kernel(float4* dst, const float4* src, const uint32_t* idx, uint32_t n, uint32_t count) {
    const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) / Q, k = threadIdx.x % Q;
    if (i >= n) return;
    const uint32_t s = idx[i];
    if (s >= count) return;   // out-of-range writes are dropped (robust buffer access)
    dst[(size_t)s * Q + k] = src[(size_t)i * Q + k];
}
constexpr uint32_t OBJECT_Q = sizeof(r3_object) / 16, MATERIAL_Q = sizeof(r3_material) / 16;
static_assert(sizeof(r3_object) == 16 * OBJECT_Q && sizeof(r3_material) == 16 * MATERIAL_Q, "records are whole float4s");
R3_EXPORT int r3_update_objects(r3_ctx* c, const uint32_t* slots, const r3_object* recs, uint32_t n) {
    if (!c || !slots || !recs) return r3_fail(c, R3_E_INVALID, "update_objects: null");
    if (n == 0) return R3_OK;
    cudaSetDevice(c->device);
    const uint64_t bytes = (uint64_t)n * (sizeof(r3_object) + 4);
    R3_TRY(r3_reserve(c, &c->d_scratch, &c->scratch_cap, bytes, 1, false, false));
    r3_object* d_recs = (r3_object*)c->d_scratch;
    uint32_t* d_slots = (uint32_t*)((uint8_t*)c->d_scratch + (size_t)n * sizeof(r3_object));
    R3_CUDA(c, cudaMemcpyAsync(d_recs, recs, (size_t)n * sizeof(r3_object), cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, cudaMemcpyAsync(d_slots, slots, (size_t)n * 4, cudaMemcpyHostToDevice, c->stream));
    scatter_records_kernel<OBJECT_Q><<<(n * 8 + 255) / 256, 256, 0, c->stream>>>((float4*)c->d_objects, (const float4*)d_recs, d_slots, n, c->n_slots);
    R3_CHECK_LAUNCH(c, "scatter_records_kernel<8>");
    R3_TRY(r3_split_slots(c, d_slots, n));
    c->max_invocations_valid = false;
    R3_CUDA(c, r3_stream_sync(c));
    return R3_OK;
}
// The sort facts of one slot as the device batching reads them: key8 = ((material_key << 1 | reason) << 1) | back_to_front, and the
// two counts the context derives any_blend and gpu_batching_ok from (r3_set_object_sort_info, r3_update_object_sort_info).
static inline uint8_t sort_key8(uint64_t key, uint8_t flags) {
    const uint32_t reason = (flags & 2) ? 0u : 1u;
    return (uint8_t)(((((uint32_t)key & 63u) << 1 | reason) << 1) | ((flags & 4) ? 1u : 0u));
}
static inline uint32_t sort_live_blend(uint64_t key, uint8_t flags) { return key == 2 && (flags & 1) ? 1u : 0u; }   // TransparencyType::Blend as u64 (pbr/material.rs:497-503)
static inline uint32_t sort_wide_key(uint64_t key) { return key >= 64 ? 1u : 0u; }                                 // only the host batching sorts such keys
static inline uint32_t sort_blend_slot(uint64_t key) { return key == 2 ? 1u : 0u; }                                  // live or not
static void sort_derive(r3_ctx* c) {
    // after r3_set_objects_enabled_device only the device knows which slots are live: then any slot with key 2 runs the blend routine
    // (over no fragments when none of them is present, which leaves the image as it is).  After r3_switch_object_variants_device only
    // the device knows the switched slots' keys: then any slot or variant with key 2 runs it, and a variant key >= 64 (which the device
    // batching's 6-bit keys cannot hold) keeps the batching on the host, which reads the current variants back.
    const bool conservative = c->presence_on_device || c->variants_on_device;
    c->any_blend = (conservative ? c->sort_blend_slots : c->sort_live_blend) != 0 || (c->variants_on_device && c->variant_key2);
    c->gpu_batching_ok = c->sort_wide_keys == 0 && c->sort_key.size() < (1u << 24) && !getenv("R3_HOST_BATCHING") &&
                         !(c->variants_on_device && c->variant_wide_key);
}
void r3_sort_set_key_flags(r3_ctx* c, uint32_t s, uint64_t key, uint8_t flags12) {
    const uint8_t was = c->sort_flags[s], now = (uint8_t)((was & 1u) | (flags12 & 6u));
    c->sort_wide_keys += sort_wide_key(key) - sort_wide_key(c->sort_key[s]);
    c->sort_blend_slots += sort_blend_slot(key) - sort_blend_slot(c->sort_key[s]);
    c->sort_live_blend += sort_live_blend(key, now) - sort_live_blend(c->sort_key[s], was);
    c->sort_key[s] = key; c->sort_flags[s] = now;
}

R3_EXPORT int r3_set_object_sort_info(r3_ctx* c, const uint64_t* key, const uint8_t* flags, const float* loc, uint32_t n) {
    if (!c || !key || !flags || !loc) return r3_fail(c, R3_E_INVALID, "set_object_sort_info: null");
    cudaSetDevice(c->device);
    R3_TRY(r3_variants_sync_host(c));   // device switches the host has not seen are settled before the mirrors are replaced
    c->sort_key.assign(key, key + n);
    c->sort_flags.assign(flags, flags + n);
    c->sort_loc.assign(loc, loc + 3 * (size_t)n);
    const uint32_t words = (n + 31) / 32;
    std::vector<uint32_t> bits(words ? words : 1, 0u);
    for (uint32_t i = 0; i < n; ++i)
        if (flags[i] & 1) bits[i >> 5] |= 1u << (i & 31);
    R3_TRY(r3_reserve_t(c, &c->d_live_bits, &c->live_bits_cap, words));
    R3_CUDA(c, cudaMemcpyAsync(c->d_live_bits, bits.data(), (size_t)words * 4, cudaMemcpyHostToDevice, c->stream));
    // device copies for the on-device batch_objects
    std::vector<uint8_t> key8(n ? n : 1, 0);
    c->sort_live_blend = 0; c->sort_wide_keys = 0; c->sort_blend_slots = 0;
    for (uint32_t i = 0; i < n; ++i) {
        c->sort_wide_keys += sort_wide_key(key[i]);
        c->sort_blend_slots += sort_blend_slot(key[i]);
        c->sort_live_blend += sort_live_blend(key[i], flags[i]);
        key8[i] = sort_key8(key[i], flags[i]);
    }
    uint32_t cap2 = c->sort_dev_cap;
    R3_TRY(r3_reserve_t(c, &c->d_sort_key8, &c->sort_dev_cap, n));
    if (!c->d_sort_loc || cap2 != c->sort_dev_cap) {
        cudaFree(c->d_sort_loc);
        c->d_sort_loc = nullptr;
        R3_CUDA(c, cudaMalloc((void**)&c->d_sort_loc, ((size_t)c->sort_dev_cap * 3 + 4) * 4));
    }
    if (n) {
        R3_CUDA(c, cudaMemcpyAsync(c->d_sort_key8, key8.data(), n, cudaMemcpyHostToDevice, c->stream));
        R3_CUDA(c, cudaMemcpyAsync(c->d_sort_loc, loc, (size_t)n * 12, cudaMemcpyHostToDevice, c->stream));
    }
    R3_CUDA(c, r3_stream_sync(c));
    r3_new_frame_epoch(c);
    c->have_live = true;
    c->presence_on_device = false;   // the flags say again which slots are live
    sort_derive(c);
    return R3_OK;
}
R3_EXPORT int r3_set_mesh_buffer(r3_ctx* c, const void* bytes, uint64_t nbytes) {
    if (!c || (!bytes && nbytes) || (nbytes & 3)) return r3_fail(c, R3_E_INVALID, "set_mesh_buffer: bad size");
    cudaSetDevice(c->device);
    r3_deform_note_mesh_write(c, true, 0, nbytes);   // the deformable set's indices are gone
    R3_TRY(r3_reserve_t(c, &c->d_mesh, &c->mesh_cap, nbytes / 4 + 4));
    if (nbytes) R3_CUDA(c, cudaMemcpyAsync(c->d_mesh, bytes, nbytes, cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    c->mesh_words = nbytes / 4;
    return R3_OK;
}
// any_frag_alpha (the raster's MODE_ALPHA kernels) follows three facts of each material: its flags, alpha_cutout > 0 and its albedo
// texture slot.  The host keeps that one bit per material, so that r3_update_materials can keep the count exact.
static inline uint8_t frag_alpha(const r3_material& m) {
    return (m.flags & R3_MAT_ALBEDO_ACTIVE) && m.alpha_cutout > 0.0f && (m.textures[R3_TEX_ALBEDO] || (m.flags & R3_MAT_ALBEDO_BLEND)) ? 1 : 0;
}
static void material_derive(r3_ctx* c) {
    // after r3_update_materials_device only the device knows the records: then the MODE_ALPHA kernels run, which give the same image
    // for materials that never discard (their triangles are not alpha-tested)
    c->any_frag_alpha = c->materials_on_device || c->n_frag_alpha != 0;
}
R3_EXPORT int r3_set_materials(r3_ctx* c, const r3_material* recs, uint32_t n) {
    if (!c || (!recs && n)) return r3_fail(c, R3_E_INVALID, "set_materials: null");
    cudaSetDevice(c->device);
    R3_TRY(r3_reserve_t(c, &c->d_materials, &c->materials_cap, n));
    if (n) R3_CUDA(c, cudaMemcpyAsync(c->d_materials, recs, (size_t)n * sizeof(r3_material), cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    c->n_materials = n;
    c->mat_frag_alpha.resize(n);
    c->n_frag_alpha = 0;
    for (uint32_t i = 0; i < n; ++i) c->n_frag_alpha += c->mat_frag_alpha[i] = frag_alpha(recs[i]);
    c->materials_on_device = false;   // the host sees every record again
    material_derive(c);
    return R3_OK;
}

// MaterialManager::update + evaluate's scatter of the stale records (material.rs:163-189, 202-227; util/freelist/buffer.rs)
static int launch_scatter_materials(r3_ctx* c, const uint32_t* d_idx, const r3_material* d_recs, uint32_t n, uint32_t count) {
    // 32 records per CTA: 13 full warps
    scatter_records_kernel<MATERIAL_Q><<<(uint32_t)(((uint64_t)n + 31) / 32), 32 * MATERIAL_Q, 0, c->stream>>>((float4*)c->d_materials, (const float4*)d_recs, d_idx, n, count);
    R3_CHECK_LAUNCH(c, "scatter_records_kernel<13>");
    return R3_OK;
}

R3_EXPORT int r3_update_materials(r3_ctx* c, const uint32_t* indices, const r3_material* recs, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (n == 0) return R3_OK;
    if (!recs) return r3_fail(c, R3_E_INVALID, "update_materials: null records");
    uint32_t count = c->n_materials;
    if (!indices) {
        if (n > count) return r3_fail(c, R3_E_INVALID, "update_materials: the dense form names materials past the table's count");
    } else {
        std::vector<uint32_t> sorted(indices, indices + n);
        std::sort(sorted.begin(), sorted.end());
        if (sorted.back() == 0xFFFFFFFFu) return r3_fail(c, R3_E_INVALID, "update_materials: index 0xFFFFFFFF");
        for (uint32_t i = 1; i < n; ++i)
            if (sorted[i] == sorted[i - 1]) return r3_fail(c, R3_E_INVALID, "update_materials: one index named twice");
        if (sorted.back() >= count) count = sorted.back() + 1;   // add_material's growth (material.rs:131-160)
    }
    cudaSetDevice(c->device);
    if (count > c->n_materials) {
        if (count > c->materials_cap || !c->d_materials) {
            uint64_t p = 16;
            while (p < count) p <<= 1;
            R3_TRY(r3_reserve_t(c, &c->d_materials, &c->materials_cap, p, true));
        }
        R3_CUDA(c, cudaMemsetAsync(c->d_materials + c->n_materials, 0, (size_t)(count - c->n_materials) * sizeof(r3_material), c->stream));
    }
    if (!indices) {
        R3_CUDA(c, cudaMemcpyAsync(c->d_materials, recs, (size_t)n * sizeof(r3_material), cudaMemcpyHostToDevice, c->stream));
    } else {
        // records then indices, staged on the host so that one copy carries both (the records stay 16-byte aligned on the device)
        const size_t rec_bytes = (size_t)n * sizeof(r3_material), bytes = rec_bytes + (size_t)n * 4;
        std::vector<uint8_t> staged(bytes);
        memcpy(staged.data(), recs, rec_bytes);
        memcpy(staged.data() + rec_bytes, indices, (size_t)n * 4);
        R3_TRY(r3_reserve(c, &c->d_scratch, &c->scratch_cap, bytes, 1, false, false));
        R3_CUDA(c, cudaMemcpyAsync(c->d_scratch, staged.data(), bytes, cudaMemcpyHostToDevice, c->stream));
        R3_TRY(launch_scatter_materials(c, (const uint32_t*)((uint8_t*)c->d_scratch + rec_bytes), (const r3_material*)c->d_scratch, n, count));
    }
    R3_CUDA(c, r3_stream_sync(c));   // host pointers are only borrowed for the call
    c->mat_frag_alpha.resize(count, 0);
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t m = indices ? indices[i] : i;
        const uint8_t now = frag_alpha(recs[i]);
        c->n_frag_alpha += now - c->mat_frag_alpha[m];
        c->mat_frag_alpha[m] = now;
    }
    c->n_materials = count;
    material_derive(c);
    return R3_OK;
}

R3_EXPORT int r3_update_materials_device(r3_ctx* c, const uint32_t* d_indices, const r3_material* d_recs, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (n == 0) return R3_OK;
    if (!d_recs || ((uintptr_t)d_recs & 15u) || ((uintptr_t)d_indices & 3u))
        return r3_fail(c, R3_E_INVALID, "update_materials_device: null or misaligned pointer (records: 16 bytes, indices: 4 bytes)");
    if (!c->n_materials) return r3_fail(c, R3_E_STATE, "update_materials_device: the material table is empty (r3_set_materials first)");
    if (!d_indices && n > c->n_materials) return r3_fail(c, R3_E_INVALID, "update_materials_device: the dense form names materials past the table's count");
    cudaSetDevice(c->device);
    if (!d_indices) R3_CUDA(c, cudaMemcpyAsync(c->d_materials, d_recs, (size_t)n * sizeof(r3_material), cudaMemcpyDeviceToDevice, c->stream));
    else R3_TRY(launch_scatter_materials(c, d_indices, d_recs, n, c->n_materials));
    c->materials_on_device = true;   // which materials discard per fragment is now known on the device only
    material_derive(c);
    return R3_OK;
}

R3_EXPORT int r3_readback_materials(r3_ctx* c, r3_material* out, uint32_t first, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (!out && n) return r3_fail(c, R3_E_INVALID, "readback_materials: null");
    if ((uint64_t)first + n > c->n_materials) return r3_fail(c, R3_E_INVALID, "readback_materials: range outside the material table");
    if (n == 0) return R3_OK;
    cudaSetDevice(c->device);
    R3_CUDA(c, r3_stream_sync(c));
    R3_CUDA(c, cudaMemcpy(out, c->d_materials + first, (size_t)n * sizeof(r3_material), cudaMemcpyDeviceToHost));
    return R3_OK;
}
R3_EXPORT int r3_set_textures(r3_ctx* c, const r3_texture_desc* descs, uint32_t n, const void* texels, uint64_t nbytes) {
    if (!c || (!descs && n) || (!texels && nbytes)) return r3_fail(c, R3_E_INVALID, "set_textures: null");
    for (uint32_t i = 0; i < n; ++i) {   // validated once here so the samplers index without checks
        const r3_texture_desc& d = descs[i];
        if (!d.width || !d.height || !d.mip_count || d.mip_count > 32 || d.format >= R3_TEXFMT_COUNT) return r3_fail(c, R3_E_INVALID, "set_textures: bad descriptor");
        uint64_t total = 0;
        for (uint32_t l = 0; l < d.mip_count; ++l) total += R3_TEXFMT_LEVEL_BYTES(d.format, (d.width >> l) ? (d.width >> l) : 1u, (d.height >> l) ? (d.height >> l) : 1u);
        if (d.byte_offset % 16 || d.byte_offset + total > nbytes) return r3_fail(c, R3_E_INVALID, "set_textures: mip chain outside the texel blob");
    }
    cudaSetDevice(c->device);
    R3_TRY(r3_reserve_t(c, &c->d_tex_descs, &c->tex_descs_cap, n));
    R3_TRY(r3_reserve_t(c, &c->d_texels, &c->texels_cap, nbytes + 16));
    if (n) R3_CUDA(c, cudaMemcpyAsync(c->d_tex_descs, descs, (size_t)n * sizeof(r3_texture_desc), cudaMemcpyHostToDevice, c->stream));
    if (nbytes) R3_CUDA(c, cudaMemcpyAsync(c->d_texels, texels, nbytes, cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    c->n_textures = n;
    c->texel_bytes = nbytes;
    c->tex_desc_host.assign(descs, descs + n);
    return R3_OK;
}

// ------------------------------------------------------------------ incremental world updates
// MeshManager::add / reallocate_buffers (managers/mesh.rs:123-184,264-308) for the mesh megabuffer and the texel blob: write
// `nbytes` at `offset` of a blob whose first `used` bytes are live.  A write past the capacity grows the allocation to the next power of
// two of end + slack, keeping its contents by a device copy (r3_reserve with keep); bytes between the old end and `offset` read 0; the
// `slack` bytes past the end stay allocated (the triangle test's bulk copies may read into them).  Returns the new live size in *used.
static int blob_write(r3_ctx* c, void** ptr, uint64_t* cap_bytes, uint64_t* used, uint64_t offset, const void* src, uint64_t nbytes, uint64_t slack) {
    const uint64_t end = offset + nbytes;
    if (end + slack > *cap_bytes || !*ptr) {
        uint64_t p = 16;
        while (p < end + slack) p <<= 1;
        R3_TRY(r3_reserve(c, ptr, cap_bytes, p, 1, true, false));
    }
    if (offset > *used) R3_CUDA(c, cudaMemsetAsync((uint8_t*)*ptr + *used, 0, offset - *used, c->stream));
    if (nbytes) R3_CUDA(c, cudaMemcpyAsync((uint8_t*)*ptr + offset, src, nbytes, cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, r3_stream_sync(c));   // the host bytes are only borrowed for the call
    if (end > *used) *used = end;
    return R3_OK;
}

R3_EXPORT int r3_update_mesh_buffer(r3_ctx* c, uint64_t byte_offset, const void* bytes, uint64_t nbytes) {
    if (!c) return R3_E_INVALID;
    if (nbytes == 0) return R3_OK;
    if (!bytes || (byte_offset & 3) || (nbytes & 3)) return r3_fail(c, R3_E_INVALID, "update_mesh_buffer: offset and size must be multiples of 4");
    if (byte_offset + nbytes < byte_offset || (byte_offset + nbytes) / 4 + 4 > (1ull << 62)) return r3_fail(c, R3_E_INVALID, "update_mesh_buffer: range overflows");
    cudaSetDevice(c->device);
    r3_deform_note_mesh_write(c, false, byte_offset, nbytes);   // new indices under the deformable set's corner lists
    uint64_t cap = c->d_mesh ? c->mesh_cap * 4 : 0, used = c->mesh_words * 4;
    void* p = c->d_mesh;
    const int rc = blob_write(c, &p, &cap, &used, byte_offset, bytes, nbytes, 16);   // >= 4 words of slack, as r3_set_mesh_buffer keeps
    c->d_mesh = (uint32_t*)p; c->mesh_cap = cap / 4;
    if (rc == R3_OK) c->mesh_words = used / 4;
    return rc;
}

static int check_texture_desc(r3_ctx* c, const r3_texture_desc& d, uint64_t blob_bytes, const char* who) {
    if (!d.width || !d.height || !d.mip_count || d.mip_count > 32 || d.format >= R3_TEXFMT_COUNT) return r3_fail(c, R3_E_INVALID, who);
    uint64_t total = 0;
    for (uint32_t l = 0; l < d.mip_count; ++l) total += R3_TEXFMT_LEVEL_BYTES(d.format, (d.width >> l) ? (d.width >> l) : 1u, (d.height >> l) ? (d.height >> l) : 1u);
    if (d.byte_offset % 16 || d.byte_offset + total > blob_bytes) return r3_fail(c, R3_E_INVALID, who);
    return R3_OK;
}

// TextureManager::add / fill (managers/texture.rs:98-251), a range of the table at a time
R3_EXPORT int r3_update_textures(r3_ctx* c, uint32_t first, const r3_texture_desc* descs, uint32_t n, uint64_t blob_offset, const void* texels, uint64_t nbytes) {
    if (!c) return R3_E_INVALID;
    if (n == 0 && nbytes == 0) return R3_OK;
    if ((!descs && n) || (!texels && nbytes)) return r3_fail(c, R3_E_INVALID, "update_textures: null");
    if (first > c->n_textures || (uint64_t)first + n > 0xFFFFFFFFull) return r3_fail(c, R3_E_INVALID, "update_textures: first entry past the end of the table");
    if (blob_offset % 16 || blob_offset + nbytes < blob_offset) return r3_fail(c, R3_E_INVALID, "update_textures: texel offset must be 16-aligned");
    const uint64_t blob = blob_offset + nbytes > c->texel_bytes ? blob_offset + nbytes : c->texel_bytes;
    for (uint32_t i = 0; i < n; ++i) R3_TRY(check_texture_desc(c, descs[i], blob, "update_textures: bad descriptor or mip chain outside the texel blob"));
    cudaSetDevice(c->device);
    if (nbytes) {
        void* p = c->d_texels;
        uint64_t used = c->texel_bytes;
        const int rc = blob_write(c, &p, &c->texels_cap, &used, blob_offset, texels, nbytes, 16);
        c->d_texels = (uint8_t*)p;
        R3_TRY(rc);
        c->texel_bytes = used;
    }
    if (n) {
        const uint64_t need = (uint64_t)first + n;
        if (need > c->tex_descs_cap || !c->d_tex_descs) {
            uint64_t p = 16;
            while (p < need) p <<= 1;
            R3_TRY(r3_reserve_t(c, &c->d_tex_descs, &c->tex_descs_cap, p, true));
        }
        R3_CUDA(c, cudaMemcpyAsync(c->d_tex_descs + first, descs, (size_t)n * sizeof(r3_texture_desc), cudaMemcpyHostToDevice, c->stream));
        R3_CUDA(c, r3_stream_sync(c));
        if (need > c->n_textures) c->n_textures = (uint32_t)need;
        c->tex_desc_host.resize(c->n_textures);
        std::copy(descs, descs + n, c->tex_desc_host.begin() + first);
    }
    return R3_OK;
}

// one thread per distinct slot: upd = slots[m] | key8 + live << 8 [m] | location bits [3 m]
__global__ void scatter_sort_info_kernel(const uint32_t* __restrict__ upd, uint32_t m, uint8_t* __restrict__ key8, float* __restrict__ loc, uint32_t* __restrict__ live_bits) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const uint32_t s = upd[i], kl = upd[m + i];
    key8[s] = (uint8_t)(kl & 255u);
    const uint32_t* l = upd + 2 * (size_t)m + 3 * (size_t)i;
    loc[3 * (size_t)s] = __uint_as_float(l[0]); loc[3 * (size_t)s + 1] = __uint_as_float(l[1]); loc[3 * (size_t)s + 2] = __uint_as_float(l[2]);
    slot_bit_assign(live_bits, s, kl & 256u);
}

// FreelistDerivedBuffer::apply's scatter of the stale entries (util/freelist/buffer.rs:85-97) for the facts batch_objects reads
R3_EXPORT int r3_update_object_sort_info(r3_ctx* c, const uint32_t* slots, const uint64_t* key, const uint8_t* flags, const float* loc, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (n == 0) return R3_OK;
    if (!slots || !key || !flags || !loc) return r3_fail(c, R3_E_INVALID, "update_object_sort_info: null");
    const size_t count = c->sort_key.size();
    if (!c->have_live) return r3_fail(c, R3_E_STATE, "update_object_sort_info before set_object_sort_info");
    for (uint32_t i = 0; i < n; ++i)
        if (slots[i] >= count) return r3_fail(c, R3_E_INVALID, "update_object_sort_info: slot beyond the sort info");
    cudaSetDevice(c->device);
    R3_TRY(r3_variants_sync_host(c));   // a device switch before this call must not be replayed over its entries later
    // the host mirrors (read by the host batching) take the entries in order: of a slot listed twice, the later entry wins
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t s = slots[i];
        c->sort_wide_keys += sort_wide_key(key[i]) - sort_wide_key(c->sort_key[s]);
        c->sort_blend_slots += sort_blend_slot(key[i]) - sort_blend_slot(c->sort_key[s]);
        c->sort_live_blend += sort_live_blend(key[i], flags[i]) - sort_live_blend(c->sort_key[s], c->sort_flags[s]);
        c->sort_key[s] = key[i]; c->sort_flags[s] = flags[i];
        memcpy(&c->sort_loc[3 * (size_t)s], loc + 3 * (size_t)i, 12);
    }
    // the device gets the final value of each distinct slot once
    std::vector<uint32_t> distinct;
    const uint32_t* list = slots;
    uint32_t m = n;
    for (uint32_t i = 1; i < n; ++i)
        if (slots[i] <= slots[i - 1]) {   // not strictly ascending: there may be repeats
            distinct.assign(slots, slots + n);
            std::sort(distinct.begin(), distinct.end());
            distinct.erase(std::unique(distinct.begin(), distinct.end()), distinct.end());
            list = distinct.data(); m = (uint32_t)distinct.size();
            break;
        }
    std::vector<uint32_t> upd((size_t)m * 5);
    for (uint32_t i = 0; i < m; ++i) {
        const uint32_t s = list[i];
        upd[i] = s;
        upd[(size_t)m + i] = sort_key8(c->sort_key[s], c->sort_flags[s]) | ((c->sort_flags[s] & 1u) << 8);
        memcpy(&upd[2 * (size_t)m + 3 * (size_t)i], &c->sort_loc[3 * (size_t)s], 12);
    }
    R3_TRY(r3_reserve(c, &c->d_scratch, &c->scratch_cap, upd.size() * 4, 1, false, false));
    R3_CUDA(c, cudaMemcpyAsync(c->d_scratch, upd.data(), upd.size() * 4, cudaMemcpyHostToDevice, c->stream));
    scatter_sort_info_kernel<<<(m + 255) / 256, 256, 0, c->stream>>>((const uint32_t*)c->d_scratch, m, c->d_sort_key8, c->d_sort_loc, c->d_live_bits);
    R3_CHECK_LAUNCH(c, "scatter_sort_info_kernel");
    R3_CUDA(c, r3_stream_sync(c));
    r3_new_frame_epoch(c);
    sort_derive(c);
    return R3_OK;
}

// r3_set_objects_enabled (r3_object_transforms.cu): the host form's entries, once on the device, go into the live bits of the host
// mirror and the live key-2 count (slots == nullptr: slots 0 .. n-1; slots without sort info have no live bit)
void r3_presence_set_host(r3_ctx* c, const uint32_t* slots, const uint8_t* enabled, uint32_t n) {
    if (!c->have_live) return;
    const size_t count = c->sort_flags.size();
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t s = slots ? slots[i] : i;
        if (s >= count) continue;
        const uint8_t was = c->sort_flags[s], now = (uint8_t)((was & ~1u) | (enabled[i] ? 1u : 0u));
        c->sort_live_blend += sort_live_blend(c->sort_key[s], now) - sort_live_blend(c->sort_key[s], was);
        c->sort_flags[s] = now;
    }
    sort_derive(c);
}
void r3_presence_derive(r3_ctx* c) { sort_derive(c); }

// FreelistDerivedBuffer::apply's growth (util/freelist/buffer.rs:66-83): a larger buffer that starts with a device copy of the old one
R3_EXPORT int r3_resize_objects(r3_ctx* c, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (n < c->n_slots) return r3_fail(c, R3_E_INVALID, "resize_objects: the object buffer only grows");
    if (c->objects_borrowed) return r3_fail(c, R3_E_STATE, "resize_objects: the object buffer is borrowed (r3_set_objects_device)");
    if (c->peer.connected) return r3_fail(c, R3_E_STATE, "resize_objects: peer buffers are sized for the current world");
    for (const r3_camera& k : c->cams)
        if (k.ex_connected) return r3_fail(c, R3_E_STATE, "resize_objects: a visible-set exchange is sized for the current world");
    if (n == c->n_slots) return R3_OK;
    cudaSetDevice(c->device);
    const uint32_t old_n = c->n_slots;
    if (n > c->objects_cap || !c->d_objects) R3_TRY(r3_reserve_t(c, &c->d_objects, &c->objects_cap, r3_hot_capacity(n), true));
    R3_CUDA(c, cudaMemsetAsync(c->d_objects + old_n, 0, (size_t)(n - old_n) * sizeof(r3_object), c->stream));
    R3_TRY(r3_grow_hot(c, old_n, n));
    R3_TRY(r3_grow_mesh_spheres(c, n));
    R3_TRY(r3_deform_grow_floors(c, n));
    R3_TRY(r3_variants_grow(c, n));
    c->n_slots = n;   // zero records have no triangles: the cached invocation bounds stay valid
    const size_t sorted = c->sort_key.size();
    if (c->have_live && sorted < n) {
        // the sort info grows with zeros as well: key 0, flags 0 (not live), location 0
        c->sort_key.resize(n, 0); c->sort_flags.resize(n, 0); c->sort_loc.resize(3 * (size_t)n, 0.0f);
        const uint32_t old_words = (uint32_t)((sorted + 31) / 32), words = (n + 31) / 32;
        R3_TRY(r3_reserve_t(c, &c->d_live_bits, &c->live_bits_cap, words, true));
        const uint32_t whole = (sorted & 31u) ? old_words : (uint32_t)(sorted / 32);
        if (words > whole) R3_CUDA(c, cudaMemsetAsync(c->d_live_bits + whole, 0, (size_t)(words - whole) * 4, c->stream));
        if (sorted & 31u) R3_TRY(r3_launch_mask_word(c, c->d_live_bits + sorted / 32, nullptr, nullptr, (1u << (sorted & 31u)) - 1u));
        if (n > c->sort_dev_cap || !c->d_sort_key8) {
            const uint32_t cap = (uint32_t)r3_hot_capacity(n);
            uint8_t* k8 = nullptr; float* l = nullptr;
            R3_CUDA(c, cudaMalloc((void**)&k8, cap));
            R3_CUDA(c, cudaMalloc((void**)&l, ((size_t)cap * 3 + 4) * 4));
            if (sorted) {
                R3_CUDA(c, cudaMemcpyAsync(k8, c->d_sort_key8, sorted, cudaMemcpyDeviceToDevice, c->stream));
                R3_CUDA(c, cudaMemcpyAsync(l, c->d_sort_loc, sorted * 12, cudaMemcpyDeviceToDevice, c->stream));
            }
            R3_CUDA(c, r3_stream_sync(c));
            cudaFree(c->d_sort_key8); cudaFree(c->d_sort_loc);
            c->d_sort_key8 = k8; c->d_sort_loc = l; c->sort_dev_cap = cap;
        }
        R3_CUDA(c, cudaMemsetAsync(c->d_sort_key8 + sorted, 0, n - sorted, c->stream));
        R3_CUDA(c, cudaMemsetAsync(c->d_sort_loc + 3 * sorted, 0, (n - sorted) * 12, c->stream));
        r3_new_frame_epoch(c);
        sort_derive(c);
    }
    R3_CUDA(c, r3_stream_sync(c));
    return R3_OK;
}
R3_EXPORT int r3_set_skybox(r3_ctx* c, const r3_texture_desc* desc, const void* texels, uint64_t nbytes) {
    if (!c) return R3_E_INVALID;
    c->has_skybox = false;
    if (!desc) return R3_OK;
    if (!texels || !desc->width || !desc->mip_count || desc->mip_count > 32 || desc->format > R3_TEXFMT_RGBA32_FLOAT) return r3_fail(c, R3_E_INVALID, "set_skybox: bad descriptor");
    const uint64_t bpp = desc->format == R3_TEXFMT_RGBA32_FLOAT ? 16 : 4;
    uint64_t face = 0;
    for (uint32_t l = 0; l < desc->mip_count; ++l) { const uint64_t w = (desc->width >> l) ? (desc->width >> l) : 1u; face += w * w * bpp; }
    if (desc->byte_offset % 16 || desc->byte_offset + 6 * face > nbytes) return r3_fail(c, R3_E_INVALID, "set_skybox: faces outside the texel blob");
    cudaSetDevice(c->device);
    R3_TRY(r3_reserve_t(c, &c->d_sky_texels, &c->sky_cap, nbytes + 16));
    R3_CUDA(c, cudaMemcpyAsync(c->d_sky_texels, texels, nbytes, cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    c->sky_desc = *desc; c->sky_desc.height = desc->width; c->has_skybox = true;
    return R3_OK;
}
R3_EXPORT int r3_set_directional_lights(r3_ctx* c, const void* bytes, uint64_t nbytes, uint32_t aw, uint32_t ah) {
    if (!c || !bytes || nbytes < 16) return r3_fail(c, R3_E_INVALID, "set_directional_lights: short buffer");
    cudaSetDevice(c->device);
    const uint32_t n = *(const uint32_t*)bytes;
    if (nbytes < 16 + (uint64_t)n * sizeof(r3_directional_light)) return r3_fail(c, R3_E_INVALID, "set_directional_lights: short buffer");
    R3_TRY(r3_reserve_t(c, &c->d_dir, &c->dir_cap, n));
    if (n) R3_CUDA(c, cudaMemcpyAsync(c->d_dir, (const uint8_t*)bytes + 16, (size_t)n * sizeof(r3_directional_light), cudaMemcpyHostToDevice, c->stream));
    c->n_dir = n;
    c->light_src_set = false;   // replaces r3_set_directional_light_sources
    c->dir_eval_pending = false;
    if (aw != c->atlas_w || ah != c->atlas_h || !c->d_atlas) {
        R3_CUDA(c, r3_stream_sync(c));
        cudaFree(c->d_atlas);
        c->d_atlas = nullptr;
        R3_CUDA(c, cudaMalloc((void**)&c->d_atlas, (size_t)aw * ah * 4 + 16));
        R3_CUDA(c, cudaMemsetAsync(c->d_atlas, 0, (size_t)aw * ah * 4, c->stream));
        c->atlas_w = aw; c->atlas_h = ah;
    }
    R3_CUDA(c, r3_stream_sync(c));
    return R3_OK;
}
R3_EXPORT int r3_set_point_lights(r3_ctx* c, const void* bytes, uint64_t nbytes) {
    if (!c || !bytes || nbytes < 16) return r3_fail(c, R3_E_INVALID, "set_point_lights: short buffer");
    cudaSetDevice(c->device);
    const uint32_t n = *(const uint32_t*)bytes;
    if (nbytes < 16 + (uint64_t)n * sizeof(r3_point_light)) return r3_fail(c, R3_E_INVALID, "set_point_lights: short buffer");
    R3_TRY(r3_reserve_point_buffer(c, n));
    // header and array together: the shading reads the count from the device, whichever call filled the buffer
    R3_CUDA(c, cudaMemcpyAsync(c->d_point, bytes, 16 + (size_t)n * sizeof(r3_point_light), cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    c->point_capacity = n;
    c->point_handles = 0;             // replaces the handle table of r3_set_point_light_sources
    c->point_eval_pending = false;
    return R3_OK;
}
void r3_new_frame_epoch(r3_ctx* c) {
    c->gsort_epoch++;
    c->gsort_valid = false;
    if (c->gsort_cameras_this_epoch) c->gsort_cameras_last_epoch = c->gsort_cameras_this_epoch;
    c->gsort_cameras_this_epoch = 0;
}
R3_EXPORT int r3_set_frame_uniforms(r3_ctx* c, const r3_frame_uniforms* u) {
    if (!c || !u) return r3_fail(c, R3_E_INVALID, "set_frame_uniforms: null");
    r3_new_frame_epoch(c);   // base.rs:142: once per frame, before any camera batches
    c->uniforms = *u;
    c->uniforms_set = true;
    return R3_OK;
}

// ------------------------------------------------------------------ cull + bake
R3_EXPORT int r3_object_uniform_upload(r3_ctx* c, uint32_t camera, const r3_camera_header* h, uint32_t mode) {
    R3_CAM_OR_FAIL(c, camera);
    if (!h) return r3_fail(c, R3_E_INVALID, "object_uniform_upload: null header");
    cudaSetDevice(c->device);
    if (h->object_count > c->n_slots) return r3_fail(c, R3_E_INVALID, "object_count exceeds the object buffer");
    cam->header = *h;
    cam->header_set = true;
    R3_TRY(r3_camera_buffers(c, cam, mode));
    return r3_launch_cull_bake(c, cam, mode);
}
int r3_camera_buffers(r3_ctx* c, r3_camera* cam, uint32_t mode) {
    const uint32_t n = cam->header.object_count;
    if (mode & R3_CB_BAKE) {
        // a resized per-camera buffer starts zeroed (culler.rs:459-476: new buffer when the size changes)
        if (cam->matrices_cap < n || !cam->d_matrices) {
            R3_CUDA(c, r3_stream_sync(c));
            cudaFree(cam->d_matrices);
            cam->d_matrices = nullptr;
            R3_CUDA(c, cudaMalloc((void**)&cam->d_matrices, ((size_t)n + 1) * sizeof(r3_object_matrices)));
            R3_CUDA(c, cudaMemsetAsync(cam->d_matrices, 0, ((size_t)n + 1) * sizeof(r3_object_matrices), c->stream));
            cam->matrices_cap = n;
        }
    }
    if (!cam->d_visible_count) {
        R3_CUDA(c, cudaMalloc((void**)&cam->d_visible_count, 16));
        R3_CUDA(c, cudaMemsetAsync(cam->d_visible_count, 0, 16, c->stream));
    }
    if (mode & R3_CB_CULL) R3_TRY(r3_reserve_t(c, &cam->d_visible, &cam->visible_cap, (uint64_t)n + 1));
    cam->visible_count_host = -1;
    return R3_OK;
}
R3_EXPORT int r3_visible_count(r3_ctx* c, uint32_t camera, uint32_t* count) {
    R3_CAM_OR_FAIL(c, camera);
    if (!count) return r3_fail(c, R3_E_INVALID, "null");
    cudaSetDevice(c->device);
    if (!cam->d_visible_count) { *count = 0; return R3_OK; }
    if (cam->visible_count_host < 0) {
        uint32_t v = 0;
        R3_CUDA(c, cudaMemcpyAsync(&v, cam->d_visible_count, 4, cudaMemcpyDeviceToHost, c->stream));
        R3_CUDA(c, r3_stream_sync(c));
        cam->visible_count_host = (int)v;
    }
    *count = (uint32_t)cam->visible_count_host;
    return R3_OK;
}
R3_EXPORT int r3_readback_visible(r3_ctx* c, uint32_t camera, uint32_t* out, uint32_t cap, uint32_t* count) {
    uint32_t n = 0;
    R3_TRY(r3_visible_count(c, camera, &n));
    r3_camera* cam = &c->cams[r3_cam_slot(camera)];
    if (count) *count = n;
    if (out && n) {
        if (cap < n) return r3_fail(c, R3_E_INVALID, "readback_visible: capacity too small");
        R3_CUDA(c, cudaMemcpyAsync(out, cam->d_visible, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream));
        R3_CUDA(c, r3_stream_sync(c));
    }
    return R3_OK;
}
R3_EXPORT int r3_readback_object_matrices(r3_ctx* c, uint32_t camera, r3_object_matrices* out, uint32_t first, uint32_t n) {
    R3_CAM_OR_FAIL(c, camera);
    if (!out || (uint64_t)first + n > cam->matrices_cap) return r3_fail(c, R3_E_INVALID, "readback_object_matrices: range");
    cudaSetDevice(c->device);
    if (n) R3_CUDA(c, cudaMemcpyAsync(out, cam->d_matrices + first, (size_t)n * sizeof *out, cudaMemcpyDeviceToHost, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    return R3_OK;
}

// ------------------------------------------------------------------ InputOutputBuffer (suballoc.rs:66-222)
static uint64_t next_pow2_u64(uint64_t v) { uint64_t p = 1; while (p < v) p <<= 1; return p; }
static uint64_t io_capacity(uint64_t in, uint64_t out) { return next_pow2_u64(in > out ? in : out) * 2; }

int r3_iobuf_new(r3_ctx* c, r3_iobuf* b, uint64_t elems, uint64_t elem_size, bool clear_on_swap) {
    b->capacity_elements = io_capacity(elems, elems);
    b->out_elems = b->in_elems = elems; b->flipped = false; b->clear_on_swap = clear_on_swap; b->elem_size = elem_size;
    R3_CUDA(c, cudaMalloc((void**)&b->d, b->capacity_elements * elem_size + 16));
    R3_CUDA(c, cudaMemsetAsync(b->d, 0, b->capacity_elements * elem_size, c->stream));   // wgpu buffers start zeroed
    b->created = true;
    return R3_OK;
}
int r3_iobuf_swap(r3_ctx* c, r3_iobuf* b, uint64_t new_elems) {
    const uint64_t old_out = b->out_off(), old_cap = b->capacity_elements;
    b->in_elems = b->out_elems; b->out_elems = new_elems; b->flipped = !b->flipped;
    const uint64_t ncap = io_capacity(b->in_elems, b->out_elems);
    if (ncap != b->capacity_elements) {
        uint8_t* nd = nullptr;
        R3_CUDA(c, cudaMalloc((void**)&nd, ncap * b->elem_size + 16));
        R3_CUDA(c, cudaMemsetAsync(nd, 0, ncap * b->elem_size, c->stream));
        b->capacity_elements = ncap;
        if (!b->clear_on_swap) {
            uint64_t bytes = b->in_elems * b->elem_size, room = (old_cap - old_out) * b->elem_size;
            if (bytes > room) bytes = room;
            if (bytes) R3_CUDA(c, cudaMemcpyAsync(nd + b->in_off() * b->elem_size, b->d + old_out * b->elem_size, bytes, cudaMemcpyDeviceToDevice, c->stream));
        }
        R3_CUDA(c, r3_stream_sync(c));
        cudaFree(b->d);
        b->d = nd;
    } else if (b->clear_on_swap) {
        R3_CUDA(c, cudaMemsetAsync(b->d, 0, b->capacity_elements * b->elem_size, c->stream));
    }
    return R3_OK;
}

static int io_read(r3_ctx* c, const r3_iobuf* b, int partition, void* out, uint64_t cap, uint64_t* count) {
    if (!b->created) { if (count) *count = 0; return R3_OK; }
    uint64_t elems = partition ? b->in_elems : b->out_elems, off = partition ? b->in_off() : b->out_off();
    const uint64_t room = b->capacity_elements / 2;
    if (elems > room) elems = room;
    if (count) *count = elems;
    if (out && elems) {
        if (cap < elems) return r3_fail(c, R3_E_INVALID, "readback: capacity too small");
        R3_CUDA(c, cudaMemcpyAsync(out, b->d + off * b->elem_size, elems * b->elem_size, cudaMemcpyDeviceToHost, c->stream));
        R3_CUDA(c, r3_stream_sync(c));
    }
    return R3_OK;
}
R3_EXPORT int r3_readback_indices(r3_ctx* c, uint32_t camera, int partition, uint32_t* out, uint64_t cap, uint64_t* count) {
    R3_CAM_OR_FAIL(c, camera);
    cudaSetDevice(c->device);
    return io_read(c, &cam->index_buffer, partition, out, cap, count);
}
R3_EXPORT int r3_readback_draw_calls(r3_ctx* c, uint32_t camera, int partition, r3_indirect_call* out, uint32_t cap, uint32_t* count) {
    R3_CAM_OR_FAIL(c, camera);
    cudaSetDevice(c->device);
    uint64_t n = 0;
    int rc = io_read(c, &cam->draw_call_buffer, partition, out, cap, &n);
    if (count) *count = (uint32_t)n;
    return rc;
}
R3_EXPORT int r3_readback_culling_results(r3_ctx* c, uint32_t camera, int partition, uint32_t* out, uint64_t cap, uint64_t* count) {
    R3_CAM_OR_FAIL(c, camera);
    cudaSetDevice(c->device);
    return io_read(c, &cam->results_buffer, partition, out, cap, count);
}

// ------------------------------------------------------------------ batching glue
R3_EXPORT int r3_batch_objects(r3_ctx* c, uint32_t camera, const float vp_loc[3], uint32_t max_dispatch_count) {
    R3_CAM_OR_FAIL(c, camera);
    if (!vp_loc) return r3_fail(c, R3_E_INVALID, "batch_objects: null location");
    cudaSetDevice(c->device);
    // Both paths split batches at the dispatch limit (batching.rs:196).  Material keys >= 64 and >= 2^24 slots (the sort key has no
    // room for them) or R3_HOST_BATCHING take the host path.  So does a world whose padded total reaches 2^31 when a batch can reach the
    // limit: the device path counts invocations in 32 bits and refuses it, and such a world always batched on the host.
    bool device = c->gpu_batching_ok && c->sort_key.size() >= cam->header.object_count;
    if (device) {
        R3_TRY(r3_compute_max_invocations(c));   // cached: one small reduction per object upload, never per frame
        device = !(c->max_total_invocations >= (1ull << 31) &&
                   c->max_object_invocations * R3_BATCH_SIZE >= (uint64_t)max_dispatch_count * R3_WORKGROUP_SIZE);
    }
    cam->batching_path = device ? 1 : 2;   // the device path raises it to 3 when it takes the frame-wide sort
    if (device) return r3_device_batch_objects(c, cam, vp_loc, max_dispatch_count);
    return r3_host_batch_objects(c, cam, vp_loc, max_dispatch_count);
}
R3_EXPORT int r3_batching_info(r3_ctx* c, uint32_t camera, uint32_t info[4]) {
    R3_CAM_OR_FAIL(c, camera);
    if (!info) return r3_fail(c, R3_E_INVALID, "batching_info: null");
    cudaSetDevice(c->device);
    info[0] = (uint32_t)cam->batching_path; info[1] = 0; info[2] = 0; info[3] = 0;
    const r3_jobs& j = cam->jobs[cam->cur];
    if ((cam->batching_path == 1 || cam->batching_path == 3) && j.d_header) {
        uint32_t hdr[8] = {0};
        R3_CUDA(c, cudaMemcpyAsync(hdr, j.d_header, 32, cudaMemcpyDeviceToHost, c->stream));
        R3_CUDA(c, r3_stream_sync(c));
        info[1] = hdr[4]; info[2] = hdr[1]; info[3] = hdr[2];
    } else if (cam->batching_path == 2) {
        info[2] = (uint32_t)j.batches.size(); info[3] = (uint32_t)j.regions.size();
    }
    return R3_OK;
}
R3_EXPORT int r3_batch_counts(r3_ctx* c, uint32_t camera, uint32_t* nb, uint32_t* nr, uint32_t* tot) {
    R3_CAM_OR_FAIL(c, camera);
    cudaSetDevice(c->device);
    R3_TRY(r3_download_jobs(c, cam));
    const r3_jobs& j = cam->jobs[cam->cur];
    if (nb) *nb = (uint32_t)j.batches.size();
    if (nr) *nr = (uint32_t)j.regions.size();
    if (tot) {
        uint64_t t = 0;
        for (const auto& b : j.batches) t += b.total_invocations;
        *tot = (uint32_t)t;
    }
    return R3_OK;
}
R3_EXPORT int r3_readback_batches(r3_ctx* c, uint32_t camera, r3_batch_data* b, r3_region* r) {
    R3_CAM_OR_FAIL(c, camera);
    cudaSetDevice(c->device);
    R3_TRY(r3_download_jobs(c, cam));
    const r3_jobs& j = cam->jobs[cam->cur];
    if (b && !j.batches.empty()) memcpy(b, j.batches.data(), j.batches.size() * sizeof *b);
    if (r && !j.regions.empty()) memcpy(r, j.regions.data(), j.regions.size() * sizeof *r);
    return R3_OK;
}

R3_EXPORT int r3_cull(r3_ctx* c, uint32_t camera, const r3_batch_data* batches, uint32_t n_batches, const r3_region* regions,
                      uint32_t n_regions) {
    R3_CAM_OR_FAIL(c, camera);
    cudaSetDevice(c->device);
    if (!cam->header_set) return r3_fail(c, R3_E_STATE, "cull before object_uniform_upload");
    if (batches) cam->cur = (cam->cache_idx == 0) ? 1 : 0;   // never overwrite the cached DrawCallSet
    r3_jobs& j = cam->jobs[cam->cur];
    if (batches) {
        if (!regions) return r3_fail(c, R3_E_INVALID, "cull: batches without regions");
        j.batches.assign(batches, batches + n_batches);
        j.regions.assign(regions, regions + n_regions);
        uint64_t tot = 0;
        for (const auto& b : j.batches) tot += b.total_invocations;
        j.total_invocations = (uint32_t)tot;
        j.device_built = false;
    }
    if (!j.device_built) {
        if (j.batches.empty()) { cam->has_draw_call_set = false; return R3_OK; }   // culler.rs:705-707
        R3_TRY(r3_upload_jobs(c, cam));
    }
    return r3_launch_triangle_cull(c, cam);
}

// ------------------------------------------------------------------ multi-GPU plumbing
R3_EXPORT int r3_device_ptr(r3_ctx* c, uint32_t camera, int which, void** p, uint64_t* nbytes) {
    R3_CAM_OR_FAIL(c, camera);
    if (!p || !nbytes) return r3_fail(c, R3_E_INVALID, "device_ptr: null");
    if (which == 0) { *p = cam->d_visible; *nbytes = (uint64_t)cam->visible_cap * 4; }
    else if (which == 1) { *p = c->d_hdr16; *nbytes = (uint64_t)c->width * c->height * 8; }
    else if (which == 2) { *p = cam->d_matrices; *nbytes = (uint64_t)cam->matrices_cap * 128; }
    else if (which == 3) { *p = cam->d_visible_count; *nbytes = 4; }
    else if (which == 4) { *p = cam->d_words; *nbytes = (((uint64_t)cam->header.object_count + 31) / 32) * 4; }   // 1 bit per object
    else if (which == 5) { *p = c->d_atlas; *nbytes = (uint64_t)c->atlas_w * c->atlas_h * 4; }   // shadow atlas (depth32f; reverse-Z depths order like their bits)
    else return r3_fail(c, R3_E_INVALID, "device_ptr: which");
    return R3_OK;
}
