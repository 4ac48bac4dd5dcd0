// r3_common.cuh — shared declarations of librend3_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/rend3_b200.h"

#define R3_EXPORT extern "C" __attribute__((visibility("default")))

constexpr int R3_MAX_CAMERAS = 64;          // slot 0 = viewport, 1+i = shadow i

struct r3_iobuf {                           // InputOutputBuffer, rend3-routine/src/culling/suballoc.rs:17-223
    uint8_t* d = nullptr;
    uint64_t capacity_elements = 0, out_elems = 0, in_elems = 0, elem_size = 0;
    bool flipped = false, clear_on_swap = false, created = false;
    uint64_t out_off() const { return flipped ? capacity_elements / 2 : 0; }
    uint64_t in_off() const { return flipped ? 0 : capacity_elements / 2; }
};

// device-side description of the draw calls of one camera/frame (what forward.rs:290-313 walks)
struct r3_jobs {
    r3_batch_data* d_batches = nullptr; uint32_t batches_cap = 0, n_batches = 0;
    r3_region* d_regions = nullptr; uint32_t regions_cap = 0, n_regions = 0;
    uint32_t* d_region_first_inv = nullptr;   // [n_regions+1] first global invocation of each region
    // device-side job header the downstream kernels read their counts from (so a frame needs no host sync):
    // [0] n_visible  [1] n_batches  [2] n_regions  [3] total_invocations  [4] overflow flag
    uint32_t* d_header = nullptr;
    uint32_t total_invocations = 0;           // exact (host batching) or an upper bound (device batching)
    bool device_built = false;                // host vectors are filled lazily by readbacks
    std::vector<r3_batch_data> batches;      // host copies (batch_objects builds these on the CPU)
    std::vector<r3_region> regions;
    bool valid = false;
};

// optional per-stage device timing (r3_set_stage_timing / r3_stage_times): CUDA event pairs around the kernels named below, so that
// bench.py can put a measured duration next to each kernel's algorithmic bytes / flops.  Off by default: no events are recorded.
enum { R3_STAGE_TRIANGLE_TEST = 0, R3_STAGE_RASTER_SETUP_COLOUR, R3_STAGE_RASTER_SETUP_DEPTH, R3_STAGE_RASTER_BANDS, R3_STAGE_RESOLVE, R3_STAGE_SORT,
       R3_STAGE_CULL_BAKE, R3_STAGE_TRIANGLE_COMPACT, R3_STAGE_COUNT };
struct r3_stage_timer {
    bool enabled = false;
    std::vector<cudaEvent_t> pool;            // recycled events: [2 k] start, [2 k + 1] stop
    std::vector<int> stage_of;                // stage of pair k
    size_t used = 0;
};
constexpr int R3_MAX_EXCHANGE_RANKS = 16;
constexpr int R3_EXCHANGE_SLOTS = 4;         // row sets of the visible-set exchange in flight (epoch % slots)
// peer-memory plumbing of the multi-GPU forward pass (r3_peer.cu): kinds of epoch flags
constexpr uint32_t R3_PEER_KINDS = 4;        // 0 shadow atlas rects, 1 colour rows, 2 frame done, 3 visibility words of the sharded triangle test
struct r3_peer_state {
    bool created = false, connected = false, has_atlas = false;
    uint32_t n_ranks = 0, rank = 0;
    uint32_t* d_flags = nullptr;              // this rank's flags[R3_PEER_KINDS][R3_MAX_EXCHANGE_RANKS]
    uint32_t* flags[R3_MAX_EXCHANGE_RANKS] = {}; float* atlas[R3_MAX_EXCHANGE_RANKS] = {}; uint16_t* hdr16[R3_MAX_EXCHANGE_RANKS] = {};   // peer mappings
    uint32_t sent[R3_PEER_KINDS] = {0, 0, 0, 0};
    uint32_t* d_tri_words = nullptr; uint64_t tri_cap_words = 0; uint32_t* tri_words[R3_MAX_EXCHANGE_RANKS] = {};   // staging arrays of the sharded triangle test
    const void* atlas_at_create = nullptr; const void* hdr_at_create = nullptr;
    cudaEvent_t side_event = nullptr; bool atlas_on_side = false;   // atlas copies run on the context's side stream
};
struct r3_camera {
    bool header_set = false;
    r3_camera_header header{};
    r3_object_matrices* d_matrices = nullptr; uint32_t matrices_cap = 0;
    uint32_t* d_visible = nullptr; uint32_t visible_cap = 0;
    uint32_t* d_visible_count = nullptr;      // device scalar
    unsigned long long* d_tile_state = nullptr; uint32_t tile_state_cap = 0;   // visibility words + per-CTA counts (two alternating sets)
    uint32_t* d_words = nullptr; uint32_t words_set = 0;                       // the set the last cull wrote
    // multi-GPU exchange of the visible set over NVLink peer memory (r3_exchange_*): gathered[n_ranks][words_per_rank]
    uint32_t* d_gathered = nullptr; uint32_t ex_ranks = 0, ex_rank = 0, ex_words_per_rank = 0; bool ex_connected = false;
    uint32_t* ex_peers[R3_MAX_EXCHANGE_RANKS] = {};   // peer-mapped gathered buffers (ex_peers[ex_rank] == d_gathered)
    uint32_t ex_epoch = 0, ex_objects = 0; uint32_t* d_ex_done = nullptr;       // step counter (parity = epoch & 1), CTA arrival counter of the publishing kernel
    cudaEvent_t ex_cull_done[R3_EXCHANGE_SLOTS] = {}, ex_merge_done[R3_EXCHANGE_SLOTS] = {}; bool ex_merge_pending[R3_EXCHANGE_SLOTS] = {}; uint32_t ex_consumed[R3_EXCHANGE_SLOTS] = {};   // consumers on the side stream; last epoch consumed per slot
    uint32_t* d_global_visible = nullptr; uint64_t global_visible_cap = 0; uint32_t* d_merge_counts = nullptr; uint64_t merge_counts_cap = 0;   // r3_exchange_merge
    int visible_count_host = -1;              // cached after a readback, -1 = unknown
    r3_jobs jobs[2]; int cur = 0;             // jobs[cur] = this frame, jobs[cur^1] = cached DrawCallSet (forward.rs:219)
    int batching_path = 0;                    // which batch_objects ran last for this camera: 0 none, 1 device, 2 host, 3 device with the frame-wide sort (r3_batching_info)
    uint64_t gsort_epoch_used = ~0ull;        // frame epoch in which this camera last batched (r3_gpu_batching.cu)
    bool has_draw_call_set = false; int cache_idx = -1;   // cache_idx: which jobs[] the forward routine cached, -1 = none
    std::vector<uint32_t> prev_invocation;    // PerCameraPreviousInvocationsMap (batching.rs:102-118), host batching
    uint32_t* d_prev_inv[2] = {nullptr, nullptr}; uint32_t prev_inv_cap = 0; int prev_inv_cur = 0;   // same map, device batching
    unsigned long long* d_sort_keys[2] = {nullptr, nullptr}; uint64_t sort_keys_cap = 0, sort_keys_cap2 = 0;
    uint32_t* d_sort_hist = nullptr; uint64_t sort_hist_cap = 0;
    uint32_t* d_batch_tmp = nullptr; uint64_t batch_tmp_cap = 0;
    r3_iobuf index_buffer, draw_call_buffer, results_buffer;   // CullingBuffers (culler.rs:88-125)
    // scratch of the ordered triangle compaction
    uint32_t* d_resid_bits = nullptr; uint64_t resid_bits_cap = 0;
    unsigned long long* d_word_scan = nullptr; uint64_t word_scan_cap = 0;
    unsigned long long* d_block_sums = nullptr; uint64_t block_sums_cap = 0;
};

struct r3_anim_state;                        // skeletal animation + resident skinning data (r3_animation.cu)
struct r3_deform_state;                      // the dynamic-mesh set: deformable or remeshable (r3_mesh_deform.cu)
struct r3_variant_state;                     // the object-variant set (r3_object_transforms.cu)

struct r3_tri_record { float xyw[3][3]; uint32_t object_id; uint32_t vid[3]; uint32_t _pad[3]; };   // 64 B
static_assert(sizeof(r3_tri_record) == 64, "triangle record");

struct r3_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t side_stream = nullptr;       // low-priority stream of the exchange consumer (r3_exchange_merge), created on first use
    std::string err;
    uint64_t launches = 0;
    bool coop_launch_ok = false;              // cudaDevAttrCooperativeLaunch (grid-wide barriers inside one launch)
    int sm_count = 1;                         // cudaDevAttrMultiProcessorCount: sizes the persistent grids
    // world
    r3_object* d_objects = nullptr; uint32_t n_slots = 0, objects_cap = 0; bool objects_borrowed = false;
    // dense copies of the fields the cull + bake stream reads (r3_cull_bake.cu): transform rows 0-2 (3 float4 per slot), transform row 3,
    // bounding spheres, enabled bits, affine bits (row 3 is exactly (+0, +0, +0, 1)), sphere radii, centre bits (the sphere's centre is
    // exactly the transform's translation column)
    float4* d_hot_xyz = nullptr; float4* d_hot_w = nullptr; float4* d_hot_sphere = nullptr; uint32_t* d_enabled_bits = nullptr; uint32_t* d_affine_bits = nullptr;
    float* d_hot_radius = nullptr; uint32_t* d_centre_bits = nullptr;
    uint64_t hot_cap = 0; bool hot_valid = false;
    std::vector<uint64_t> sort_key; std::vector<uint8_t> sort_flags; std::vector<float> sort_loc;
    uint32_t* d_live_bits = nullptr; uint32_t live_bits_cap = 0; bool have_live = false;
    uint8_t* d_sort_key8 = nullptr; float* d_sort_loc = nullptr; uint32_t sort_dev_cap = 0; bool gpu_batching_ok = false;
    // InternalObject::mesh_bounding_sphere per slot (r3_set_object_mesh_spheres): what r3_set_object_transforms moves to world space
    float4* d_mesh_spheres = nullptr; uint32_t n_mesh_spheres = 0, mesh_spheres_cap = 0;
    bool locations_moved = false;             // r3_set_object_transforms* ran since c->sort_loc last took the device's locations
    uint32_t sort_live_blend = 0, sort_wide_keys = 0;   // live slots with material key 2 (any_blend), slots with a key >= 64 (host batching)
    uint32_t sort_blend_slots = 0;            // slots with material key 2, live or not (any_blend while presence_on_device)
    bool presence_on_device = false;          // r3_set_objects_enabled_device ran since r3_set_object_sort_info: the host's live bits are stale
    // r3_switch_object_variants_device ran since the host last read the slots' current variants: its key and flag mirrors are stale.
    // variant_key2 / variant_wide_key: some variant of the set has material key 2 / a key >= 64
    bool variants_on_device = false, variant_key2 = false, variant_wide_key = false;
    // frame-wide sort shared by the cameras of one frame (r3_gpu_batching.cu)
    unsigned long long* d_gsort_keys[2] = {nullptr, nullptr}; uint64_t gsort_cap[2] = {0, 0}; uint32_t* d_gsort_hist = nullptr; uint64_t gsort_hist_cap = 0;
    uint32_t* d_gsort_header = nullptr; int gsort_src = 0; uint32_t gsort_n = 0; bool gsort_valid = false; float gsort_loc[3] = {0, 0, 0};
    uint64_t gsort_epoch = 0, gsort_sorted_epoch = ~0ull; uint32_t gsort_cameras_this_epoch = 0, gsort_cameras_last_epoch = 0;
    uint64_t max_total_invocations = 0, max_object_invocations = 0; bool max_invocations_valid = false;   // sum / max over all slots of round_up(tris, 256)
    // per-slot floor of the index_count those bounds take (a remeshable set's index_capacity; r3_mesh_deform.cu), only while such a set
    // exists: a remesh can grow a record's index_count back up to it without the host seeing the records
    uint32_t* d_invocation_floor = nullptr; uint32_t n_invocation_floor = 0, invocation_floor_cap = 0;
    uint32_t* d_mesh = nullptr; uint64_t mesh_words = 0, mesh_cap = 0;
    r3_material* d_materials = nullptr; uint32_t n_materials = 0, materials_cap = 0;
    bool has_skybox = false; r3_texture_desc sky_desc{}; uint8_t* d_sky_texels = nullptr; uint64_t sky_cap = 0;   // cube map of the skybox routine
    r3_texture_desc* d_tex_descs = nullptr; uint32_t n_textures = 0, tex_descs_cap = 0; uint8_t* d_texels = nullptr; uint64_t texels_cap = 0, texel_bytes = 0;
    // host copy of the table's n_textures descriptors (r3_set_textures, r3_update_textures): r3_write_texture_regions checks against it
    std::vector<r3_texture_desc> tex_desc_host;
    void* d_texw_plan = nullptr; uint64_t texw_plan_cap = 0;   // r3_texture_write.cu: per-region copy plans + unit scan, grow-only
    r3_directional_light* d_dir = nullptr; uint32_t n_dir = 0, dir_cap = 0;
    // shadow cameras evaluated on the device (r3_lights.cu): the sources of r3_set_directional_light_sources and one camera header per
    // light (view, view_proj, frustum written by the evaluation), both sized R3_MAX_SHADOWS; host copies of the placements
    r3_directional_light_source* d_light_src = nullptr; r3_camera_header* d_shadow_cams = nullptr;
    std::vector<r3_directional_light_source> light_src;
    bool light_src_set = false, shadow_cams_evaluated = false; uint32_t light_src_left_handed = 0;
    // r3_update_directional_light_sources[_device] ran since the last r3_evaluate_shadow_cameras: the cameras and view_proj are stale
    bool dir_eval_pending = false;
    // ShaderPointLightBuffer as the shading reads it: u32 count @0, r3_point_light array @16 (allocated at context creation, count 0).
    // The count is only known on the device; point_capacity (r3_set_point_lights' count, or the handle table's size) bounds it and sizes
    // the light prep.  point_handles: size of PointLightManager's handle table (r3_lights.cu), sources + live bytes on the device.
    uint8_t* d_point = nullptr; uint64_t point_bytes_cap = 0; uint32_t point_capacity = 0;
    r3_point_light_source* d_point_src = nullptr; uint8_t* d_point_live = nullptr; uint32_t point_handles = 0, point_src_cap = 0, point_live_cap = 0;
    bool point_eval_pending = false;          // sources set or updated since the last r3_evaluate_point_lights: the buffer is stale
    float* d_light_mats = nullptr; uint64_t light_mats_cap = 0;   // view-space light tables built by light_prep_kernel
    r3_frame_uniforms uniforms{}; bool uniforms_set = false;
    float* d_atlas = nullptr; uint32_t atlas_w = 0, atlas_h = 0;
    r3_camera cams[R3_MAX_CAMERAS];
    // render targets
    uint32_t width = 0, height = 0, samples = 1; float clear_color[4] = {0, 0, 0, 0};
    uint32_t row_begin = 0, row_end = 0;
    unsigned long long* d_vis = nullptr;      // (depth bits << 32) | (pass << 31) | record
    bool parity_target = false;               // also keep the f32 shading result before the rgba16f store (tests; off in production)
    float* d_hdr32 = nullptr; uint16_t* d_hdr16 = nullptr; float* d_depth = nullptr; uint8_t* d_ldr = nullptr;
    std::vector<float*> d_hiz; std::vector<uint32_t> hiz_w, hiz_h;
    float** d_hiz_ptrs = nullptr; uint32_t* d_hiz_dims = nullptr;
    r3_tri_record* d_tris[4] = {nullptr, nullptr, nullptr, nullptr}; uint64_t tris_cap[4] = {0, 0, 0, 0}; uint64_t n_tris[4] = {0, 0, 0, 0};   // predicted, residual, blend, shadow scratch
    bool any_frag_alpha = false;              // a material discards per fragment (cutout alpha from its albedo texture / vertex colour)
    std::vector<uint8_t> mat_frag_alpha;      // per material: it discards per fragment (r3_ctx.cu frag_alpha); n_frag_alpha of them set
    uint32_t n_frag_alpha = 0;
    bool materials_on_device = false;         // r3_update_materials_device ran since r3_set_materials: any_frag_alpha stays true
    unsigned long long* d_stats = nullptr;    // [8]: [0..3] forward statistics, [4] scratch of r3_compute_max_invocations
    // blend routine: per-sample fragment lists (head = node index + 1, 0 = empty; node = {record, depth bits, next, 0})
    bool any_blend = false;                   // some live object carries material key 2 (TransparencyType::Blend); see sort_blend_slots
    uint32_t* d_frag_heads = nullptr; uint64_t frag_heads_cap = 0;
    uint4* d_frag_nodes = nullptr; uint64_t frag_nodes_cap = 0;
    void* d_scratch = nullptr; uint64_t scratch_cap = 0;
    r3_stage_timer timer;
    r3_peer_state peer;
    uint32_t tri_shard_index = 0, tri_shard_count = 1;   // r3_set_cull_shard
    r3_anim_state* anim = nullptr;            // created by the first r3_set_animations / r3_set_skeletons
    r3_deform_state* deform = nullptr;        // created by the first r3_set_deformable_meshes or r3_set_remeshable_meshes
    r3_variant_state* variants = nullptr;     // created by the first r3_set_object_variants
    // frame graph
    bool capturing = false;                   // between r3_frame_begin and the submission (or an early flush)
    cudaGraphExec_t frame_exec[2] = {nullptr, nullptr};   // instantiated graphs of even / odd frames (the culling buffers ping-pong), updated in place
    uint64_t frame_index = 0, frames_graphed = 0, frames_flushed = 0, graph_reinstantiations = 0;
};

// ---- error plumbing (nothing throws across the C boundary)
int r3_fail(r3_ctx* c, int code, const char* msg);
int r3_cuda_fail(r3_ctx* c, cudaError_t e, const char* where);
#define R3_CUDA(c, call)                                                  \
    do {                                                                  \
        cudaError_t e__ = (call);                                         \
        if (e__ != cudaSuccess) return r3_cuda_fail((c), e__, #call);     \
    } while (0)
#define R3_CHECK_LAUNCH(c, name)                                          \
    do {                                                                  \
        (c)->launches++;                                                  \
        cudaError_t e__ = cudaGetLastError();                             \
        if (e__ != cudaSuccess) return r3_cuda_fail((c), e__, name);      \
    } while (0)
#define R3_TRY(expr)                                                      \
    do {                                                                  \
        int rc__ = (expr);                                                \
        if (rc__ != R3_OK) return rc__;                                   \
    } while (0)

// Frame graph (r3_frame_begin / r3_frame_end): the stream work of one frame is recorded by stream capture and submitted as ONE CUDA graph
// launch (the reference submits once per frame, graph.rs:510).  Anything that has to wait for the stream inside a frame first flushes what
// was recorded so far (r3_stream_sync does that), after which the rest of the frame runs eagerly.
cudaError_t r3_stream_sync(r3_ctx* c);
// stage timing: no-ops unless enabled
void r3_stage_begin(r3_ctx* c, int stage);
void r3_stage_end(r3_ctx* c);
static inline int r3_cam_slot(uint32_t camera) { return camera == R3_CAMERA_VIEWPORT ? 0 : (int)camera + 1; }
static inline r3_camera* r3_get_camera(r3_ctx* c, uint32_t camera) {
    if (!c || (camera != R3_CAMERA_VIEWPORT && camera >= R3_MAX_SHADOWS)) return nullptr;
    return &c->cams[r3_cam_slot(camera)];
}
#define R3_CAM_OR_FAIL(ctx, camera)                                                                              \
    if (!(ctx)) return R3_E_INVALID;                                                                             \
    if ((camera) != R3_CAMERA_VIEWPORT && (camera) >= R3_MAX_SHADOWS) return r3_fail((ctx), R3_E_INVALID, "bad camera"); \
    r3_camera* cam = &(ctx)->cams[r3_cam_slot(camera)]

// grow-only device allocation helper: keeps contents when `keep` is set
int r3_reserve(r3_ctx* c, void** ptr, uint64_t* cap_elems, uint64_t need_elems, size_t elem_size, bool keep, bool zero_new);
template <typename T, typename C>
int r3_reserve_t(r3_ctx* c, T** ptr, C* cap, uint64_t need, bool keep = false, bool zero_new = false) {
    uint64_t cap64 = *cap;
    int rc = r3_reserve(c, (void**)ptr, &cap64, need, sizeof(T), keep, zero_new);
    *cap = (C)cap64;
    return rc;
}

// stages implemented in the other translation units
int r3_launch_cull_bake(r3_ctx* c, r3_camera* cam, uint32_t mode);
// the same with view, view_proj and frustum read on the device from d_header (r3_shadow_uniform_upload); the rest from cam->header
int r3_launch_cull_bake_device_camera(r3_ctx* c, r3_camera* cam, uint32_t mode, const r3_camera_header* d_header);
int r3_camera_buffers(r3_ctx* c, r3_camera* cam, uint32_t mode);   // r3_object_uniform_upload's per-camera allocations
int r3_split_objects(r3_ctx* c);
int r3_split_slots(r3_ctx* c, const uint32_t* d_slots, uint32_t n);
int r3_grow_hot(r3_ctx* c, uint32_t old_n, uint32_t n);   // r3_resize_objects: keep the hot copies of slots < old_n, zero slots [old_n, n)
uint64_t r3_hot_capacity(uint64_t want);                    // slots the hot arrays (and a grown object buffer) are allocated for
int r3_launch_mask_word(r3_ctx* c, uint32_t* word_a, uint32_t* word_b, uint32_t* word_c, uint32_t keep_mask);   // *word &= keep_mask (any may be null)
int r3_launch_triangle_cull(r3_ctx* c, r3_camera* cam);
int r3_host_batch_objects(r3_ctx* c, r3_camera* cam, const float vp_loc[3], uint32_t max_dispatch_count);
int r3_upload_jobs(r3_ctx* c, r3_camera* cam);
int r3_device_batch_objects(r3_ctx* c, r3_camera* cam, const float vp_loc[3], uint32_t max_dispatch_count);
int r3_download_jobs(r3_ctx* c, r3_camera* cam);          // device-built jobs -> host vectors (readbacks / tests)
int r3_compute_max_invocations(r3_ctx* c);
void r3_new_frame_epoch(r3_ctx* c);          // the frame-wide sort of the previous frame is stale from here on
int r3_blend_collect(r3_ctx* c, bool* ran);   // r3_raster.cu: per-sample fragment lists of the blend routine
int r3_iobuf_new(r3_ctx* c, r3_iobuf* b, uint64_t elems, uint64_t elem_size, bool clear_on_swap);
int r3_iobuf_swap(r3_ctx* c, r3_iobuf* b, uint64_t new_elems);
// r3_skinning.cu: skinning_kernel over device-resident records, chunk prefix and joint matrices (r3_skin, r3_skin_posed)
int r3_launch_skinning(r3_ctx* c, const r3_skinning_input* d_inputs, const uint32_t* d_chunk_prefix, uint32_t n_skeletons, uint32_t total_chunks,
                       const float* d_joints, uint32_t n_joints);
void r3_anim_destroy(r3_ctx* c);             // r3_animation.cu: frees c->anim (r3_ctx_destroy)
// r3_object_transforms.cu: after device-side moves, poses and variant switches the host batching's sort mirrors (c->sort_loc, the key and
// flag mirrors) are behind the device's.  stage enqueues the copies that bring them up to date (*pending = true when it enqueued any);
// once the caller has drained the stream, apply writes what they brought into the mirrors.
int r3_stage_sort_mirrors(r3_ctx* c, bool* pending);
void r3_apply_sort_mirrors(r3_ctx* c);
int r3_grow_mesh_spheres(r3_ctx* c, uint32_t n);   // r3_resize_objects: zero spheres for the new slots, once spheres are set
// r3_ctx.cu: the host bookkeeping of r3_set_objects_enabled (exact: live bits of c->sort_flags, live key-2 count, any_blend) and, after
// the device form has set c->presence_on_device, any_blend's conservative rule
void r3_presence_set_host(r3_ctx* c, const uint32_t* slots, const uint8_t* enabled, uint32_t n);
void r3_presence_derive(r3_ctx* c);
int r3_reserve_point_buffer(r3_ctx* c, uint32_t n_lights);   // r3_lights.cu: room for n lights in c->d_point, contents kept
// r3_mesh_deform.cu: free c->deform (r3_ctx_destroy); a mesh-buffer write that invalidates the set's corner lists (r3_set_mesh_buffer:
// every byte; r3_update_mesh_buffer: [offset, offset + nbytes), which matters when it meets one of the set's index ranges)
void r3_deform_destroy(r3_ctx* c);
void r3_deform_note_mesh_write(r3_ctx* c, bool whole_buffer, uint64_t byte_offset, uint64_t nbytes);
int r3_deform_grow_floors(r3_ctx* c, uint32_t n);   // r3_resize_objects: zero invocation floors for the new slots, while they exist
// r3_mesh_deform.cu: c->d_invocation_floor from both of its sources, a remeshable set's index capacities and the object-variant set's
// group maxima (their slots are disjoint); freed when neither set exists.  Invalidates the cached invocation bound.
int r3_rebuild_invocation_floors(r3_ctx* c);
const std::vector<uint32_t>* r3_deform_listed_slots(r3_ctx* c);   // the current deformable / remeshable set's slots, nullptr without one
// r3_object_transforms.cu: the object-variant set (r3_set_object_variants)
void r3_variants_destroy(r3_ctx* c);
int r3_variants_grow(r3_ctx* c, uint32_t n);          // r3_resize_objects: the per-slot arrays grow, new slots unlisted
bool r3_variants_have_set(const r3_ctx* c);
bool r3_variants_list(const r3_ctx* c, uint32_t slot);   // the set lists the slot
int r3_variants_scatter_floors(r3_ctx* c);            // the listed slots' floors into c->d_invocation_floor (zeroed by the caller)
// after r3_switch_object_variants_device: bring the host's key / flag mirrors up to date, blocking
int r3_variants_sync_host(r3_ctx* c);
// r3_ctx.cu: slot s's material key and flags bits 1-2 into the host mirrors, with the counts any_blend and gpu_batching_ok follow (the
// caller re-derives them with r3_presence_derive)
void r3_sort_set_key_flags(r3_ctx* c, uint32_t s, uint64_t key, uint8_t flags12);
// slots with host sort facts (r3_set_object_sort_info): the device's key, location and live arrays cover [0, extent)
static inline uint32_t r3_sort_extent(const r3_ctx* c) { return c->have_live ? (uint32_t)c->sort_key.size() : 0u; }
// r3_ctx.cu: the preconditions of a call that writes object records.  Each failed one is R3_E_STATE with a message that starts with
// `who`; they are checked in the order of the flags.
enum : uint32_t {
    R3_NEED_OBJECTS = 1u,   // an object buffer exists: "<who> before set_objects"
    R3_NEED_HOT = 2u,       // ... and its cull + bake copies are valid (same message)
    R3_NEED_OWNED = 4u,     // the buffer is not borrowed (r3_set_objects_device)
    R3_NEED_SPHERES = 8u,   // r3_set_object_mesh_spheres covers every slot
};
int r3_check_object_writer(r3_ctx* c, const char* who, uint32_t needs);

#ifdef __CUDACC__
// Bit pattern of row 3 of an affine transform, column j: (+0, +0, +0, 1).  Bits, not floats: -0.0 and NaN are not affine
// (a product with -0.0 can carry its sign into MV / MVP).
__device__ __forceinline__ uint32_t affine_w_bits(uint32_t j) { return j == 3 ? 0x3f800000u : 0u; }
// The centre bit of a slot: its bounding sphere's centre has the bit patterns of the translation column (elements .w of rows 0-2), so
// the cull can take the centre from the transform it already holds.  Bits, not floats: -0.0 against +0.0 or two NaN payloads differ.
__device__ __forceinline__ bool centre_is_translation(float cx, float cy, float cz, float tx, float ty, float tz) {
    return __float_as_uint(cx) == __float_as_uint(tx) && __float_as_uint(cy) == __float_as_uint(ty) && __float_as_uint(cz) == __float_as_uint(tz);
}
// IEEE, never-contracted arithmetic for the bit-exact stages (SURVEY D7)
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float sqrt_rn(float a) { return __fsqrt_rn(a); }
// Slot s's bit of a bit-word array, set or cleared by an atomic: other slots of the word may be written by other threads
__device__ __forceinline__ void slot_bit_assign(uint32_t* words, uint32_t s, bool on) {
    const uint32_t bit = 1u << (s & 31u);
    if (on) atomicOr(&words[s >> 5], bit);
    else atomicAnd(&words[s >> 5], ~bit);
}
// *word = (*word & ~mask) | (bits & mask): a plain store when the warp owns the whole word, atomics when slots past the range share it
__device__ __forceinline__ void store_bits(uint32_t* word, uint32_t bits, uint32_t mask) {
    if (mask == 0xFFFFFFFFu) *word = bits;
    else if (mask) { atomicAnd(word, ~mask | bits); atomicOr(word, bits & mask); }
}
// BoundingSphere::apply_transform (util/frustum.rs:22-32), rule R12's object half: Vec3::length_squared of each axis, f32::max (fmaxf
// ignores a NaN operand as it does), sqrt; centre = matrix * (c, 1) in mul_vec4's order; radius = max_scale * r.  x, y, z: the xyz of the
// matrix's four columns; ms: the mesh sphere (centre, radius).  Every writer of a world sphere uses it: moves, poses, deforms, variants.
__device__ __forceinline__ float4 sphere_apply_transform_rn(const float (&x)[4], const float (&y)[4], const float (&z)[4], const float4& ms) {
    float ls[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) ls[c] = add_rn(add_rn(mul_rn(x[c], x[c]), mul_rn(y[c], y[c])), mul_rn(z[c], z[c]));
    const float max_scale = sqrt_rn(fmaxf(ls[0], fmaxf(ls[1], ls[2])));
    float4 sph;
    sph.x = add_rn(add_rn(add_rn(mul_rn(x[0], ms.x), mul_rn(x[1], ms.y)), mul_rn(x[2], ms.z)), mul_rn(x[3], 1.0f));
    sph.y = add_rn(add_rn(add_rn(mul_rn(y[0], ms.x), mul_rn(y[1], ms.y)), mul_rn(y[2], ms.z)), mul_rn(y[3], 1.0f));
    sph.z = add_rn(add_rn(add_rn(mul_rn(z[0], ms.x), mul_rn(z[1], ms.y)), mul_rn(z[2], ms.z)), mul_rn(z[3], 1.0f));
    sph.w = mul_rn(max_scale, ms.w);
    return sph;
}
// The sort location of a moved object, transform_point3a(Vec3A::ZERO), one component from one row r of the matrix (x, y or z as for
// sphere_apply_transform_rn): w + ((x * 0 + y * 0) + z * 0) — the translation for finite axes, NaN for an infinite one
__device__ __forceinline__ float sort_location_rn(const float (&r)[4]) {
    return add_rn(r[3], add_rn(add_rn(mul_rn(r[0], 0.0f), mul_rn(r[1], 0.0f)), mul_rn(r[2], 0.0f)));
}
// M * (x, y, z, w): column-major, accumulated x,y,z,w like WGSL's mat4x4*vec4
__device__ __forceinline__ float4 mat_vec_rn(const float* __restrict__ m, float x, float y, float z, float w) {
    float4 r;
    r.x = mul_rn(m[0], x); r.y = mul_rn(m[1], x); r.z = mul_rn(m[2], x); r.w = mul_rn(m[3], x);
    r.x = add_rn(r.x, mul_rn(m[4], y)); r.y = add_rn(r.y, mul_rn(m[5], y)); r.z = add_rn(r.z, mul_rn(m[6], y)); r.w = add_rn(r.w, mul_rn(m[7], y));
    r.x = add_rn(r.x, mul_rn(m[8], z)); r.y = add_rn(r.y, mul_rn(m[9], z)); r.z = add_rn(r.z, mul_rn(m[10], z)); r.w = add_rn(r.w, mul_rn(m[11], z));
    r.x = add_rn(r.x, mul_rn(m[12], w)); r.y = add_rn(r.y, mul_rn(m[13], w)); r.z = add_rn(r.z, mul_rn(m[14], w)); r.w = add_rn(r.w, mul_rn(m[15], w));
    return r;
}
// M * (x, y, z, 1)
__device__ __forceinline__ float4 mat_point_rn(const float* __restrict__ m, float x, float y, float z) {
    float4 r;
    r.x = mul_rn(m[0], x); r.y = mul_rn(m[1], x); r.z = mul_rn(m[2], x); r.w = mul_rn(m[3], x);
    r.x = add_rn(r.x, mul_rn(m[4], y)); r.y = add_rn(r.y, mul_rn(m[5], y)); r.z = add_rn(r.z, mul_rn(m[6], y)); r.w = add_rn(r.w, mul_rn(m[7], y));
    r.x = add_rn(r.x, mul_rn(m[8], z)); r.y = add_rn(r.y, mul_rn(m[9], z)); r.z = add_rn(r.z, mul_rn(m[10], z)); r.w = add_rn(r.w, mul_rn(m[11], z));
    r.x = add_rn(r.x, m[12]); r.y = add_rn(r.y, m[13]); r.z = add_rn(r.z, m[14]); r.w = add_rn(r.w, m[15]);
    return r;
}
#endif
