// r3_animation.cu — skeletal animation posed on the device, and skinning from the joint matrices it leaves in device memory.
//
// Replaces the joint half of rend3-anim's pose_animation_frame (rend3-anim/src/lib.rs:165-176, 190, 214-262) and the per-frame
// upload of the joint matrices that r3_skin makes.  Arithmetic: rule R12 (DESIGN.md §2), one IEEE f32 operation at a time in glam's
// order, never contracted (this unit is compiled with -fmad=false and uses the _rn intrinsics throughout).
//
// At upload the host checks everything (include/r3_anim_check.h) and sorts each skin's joints by level (level 0: the node has no parent
// joint; level l: the parent joint is at level l - 1).  A global matrix is one product of fixed operands, so any parent-first schedule
// gives the same bits; the levels let the threads of a CTA compute all joints of a level at once.  pose_kernel: one CTA per job —
// every joint's local matrix, then the globals level by level (in place over the locals, in shared memory, or in a global scratch for
// skins above R3_ANIM_SMEM_JOINTS joints), then global * inverse_bind stored into each target's range of the joint buffer.
//
// The object-transform half (lib.rs:192-212, set_object_transform of object.rs:302-316) is pose_objects_kernel: one thread per posed
// object samples its node's channel, builds the TRS matrix and writes the record's transform and world sphere and the slot's sort
// location.  The work is small and latency-bound; the cull + bake's dense copies of those slots are then refreshed by r3_split_slots.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/r3_anim_check.h"
#include "r3_common.cuh"

namespace {

constexpr uint32_t R3_ANIM_THREADS = 128;
constexpr uint32_t R3_ANIM_SMEM_JOINTS = 512;   // 512 x 17 floats = 34 KB of shared memory; larger skins use the global scratch
constexpr uint32_t R3_ANIM_STRIDE = 17;         // floats per matrix in the scratch (16 + 1: consecutive joints fall in different banks)

struct anim_skin_dev {                            // r3_anim_skin + its level table and its stretch of the level-ordered joint list
    uint32_t first_joint, joint_count, n_levels;
    uint64_t first_level, first_sched;
};

// sample_at_time (lib.rs:165-176): next = first key with time > t (the last key if none), prev = max(next - 1, 0),
// s = clamp((t - t_prev) / (t_next - t_prev), 0, 1) with f32::clamp's compares (NaN stays NaN)
__device__ __forceinline__ float key_factor(const float* __restrict__ keys, const r3_anim_track& tr, float t, uint32_t* prev, uint32_t* next) {
    const float* times = keys + tr.times;
    uint32_t lo = 0, hi = tr.count;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldg(times + mid) > t) hi = mid; else lo = mid + 1;
    }
    const uint32_t n = lo < tr.count ? lo : tr.count - 1, p = n ? n - 1 : 0;
    const float tp = __ldg(times + p), tn = __ldg(times + n);
    float s = div_rn(sub_rn(t, tp), sub_rn(tn, tp));
    if (s < 0.0f) s = 0.0f;
    if (s > 1.0f) s = 1.0f;
    *prev = p; *next = n;
    return s;
}

// Vec3::lerp: a + ((b - a) * s)
__device__ __forceinline__ float3 sample3(const float* __restrict__ keys, const r3_anim_track& tr, float t) {
    uint32_t p, n;
    const float s = key_factor(keys, tr, t, &p, &n);
    const float* a = keys + tr.values + 3ull * p;
    const float* b = keys + tr.values + 3ull * n;
    float r[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) { const float x = __ldg(a + i), y = __ldg(b + i); r[i] = add_rn(x, mul_rn(sub_rn(y, x), s)); }
    return make_float3(r[0], r[1], r[2]);
}

// glam's SSE2 dot4: (x x' + z z') + (y y' + w w')
__device__ __forceinline__ float dot4(const float* a, const float* b) {
    return add_rn(add_rn(mul_rn(a[0], b[0]), mul_rn(a[2], b[2])), add_rn(mul_rn(a[1], b[1]), mul_rn(a[3], b[3])));
}
// Quat::normalize as rule R12 fixes it: r * (1 / sqrt(dot(r, r))) (glam's SSE2 code may divide by the length instead: one rounding apart)
__device__ __forceinline__ void normalize4(float* r) {
    const float rcp = div_rn(1.0f, sqrt_rn(dot4(r, r)));
#pragma unroll
    for (int i = 0; i < 4; ++i) r[i] = mul_rn(r[i], rcp);
}

// <Quat as Lerp>::lerp (lib.rs:154-161): glam Quat::lerp — flip `end` by the SIGN BIT of the dot (a dot of -0.0 flips too),
// ((end ^ flip) - start) * s + start, normalize — and then rend3-anim's own .normalize()
__device__ __forceinline__ float4 sample_quat(const float* __restrict__ keys, const r3_anim_track& tr, float t) {
    uint32_t p, n;
    const float s = key_factor(keys, tr, t, &p, &n);
    const float* pa = keys + tr.values + 4ull * p;
    const float* pb = keys + tr.values + 4ull * n;
    float a[4], b[4], r[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { a[i] = __ldg(pa + i); b[i] = __ldg(pb + i); }
    const uint32_t flip = __float_as_uint(dot4(a, b)) & 0x80000000u;
#pragma unroll
    for (int i = 0; i < 4; ++i) r[i] = add_rn(mul_rn(sub_rn(__uint_as_float(__float_as_uint(b[i]) ^ flip), a[i]), s), a[i]);
    normalize4(r);
    normalize4(r);
    return make_float4(r[0], r[1], r[2], r[3]);
}

// Mat4::from_scale_rotation_translation: the axes of Mat3::from_quat (rend3_b200/glam.py::quat_to_axes), each Vec4 (w = 0) times its
// scale — so the w entry is 0 * s — and (t, 1)
__device__ __forceinline__ void from_srt(float3 sc, float4 q, float3 tr, float* m) {
    const float x2 = add_rn(q.x, q.x), y2 = add_rn(q.y, q.y), z2 = add_rn(q.z, q.z);
    const float xx = mul_rn(q.x, x2), xy = mul_rn(q.x, y2), xz = mul_rn(q.x, z2);
    const float yy = mul_rn(q.y, y2), yz = mul_rn(q.y, z2), zz = mul_rn(q.z, z2);
    const float wx = mul_rn(q.w, x2), wy = mul_rn(q.w, y2), wz = mul_rn(q.w, z2);
    const float ax[4] = {sub_rn(1.0f, add_rn(yy, zz)), add_rn(xy, wz), sub_rn(xz, wy), 0.0f};
    const float ay[4] = {sub_rn(xy, wz), sub_rn(1.0f, add_rn(xx, zz)), add_rn(yz, wx), 0.0f};
    const float az[4] = {add_rn(xz, wy), sub_rn(yz, wx), sub_rn(1.0f, add_rn(xx, yy)), 0.0f};
#pragma unroll
    for (int i = 0; i < 4; ++i) { m[i] = mul_rn(ax[i], sc.x); m[4 + i] = mul_rn(ay[i], sc.y); m[8 + i] = mul_rn(az[i], sc.z); }
    m[12] = tr.x; m[13] = tr.y; m[14] = tr.z; m[15] = 1.0f;
}

// Mat4 * Mat4 (glam mul_mat4): column j = a.mul_vec4(b.col(j))
__device__ __forceinline__ void mat_mul(const float* a, const float* b, float* out) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float4 c = mat_vec_rn(a, b[4 * j], b[4 * j + 1], b[4 * j + 2], b[4 * j + 3]);
        out[4 * j] = c.x; out[4 * j + 1] = c.y; out[4 * j + 2] = c.z; out[4 * j + 3] = c.w;
    }
}

__global__ void __launch_bounds__(R3_ANIM_THREADS) pose_kernel(const r3_pose_job* __restrict__ jobs, const r3_pose_target* __restrict__ targets,
                                                               const r3_anim_clip* __restrict__ clips, const anim_skin_dev* __restrict__ skins,
                                                               const r3_anim_joint* __restrict__ joints, const uint32_t* __restrict__ sched,
                                                               const uint32_t* __restrict__ levels, const r3_anim_channel* __restrict__ channels,
                                                               const float* __restrict__ keys, const uint64_t* __restrict__ spill_offset,
                                                               float* __restrict__ spill, float* __restrict__ joint_buf) {
    extern __shared__ float smem[];
    const r3_pose_job job = jobs[blockIdx.x];
    const r3_anim_clip clip = clips[job.clip];
    const anim_skin_dev sk = skins[clip.skin];
    const uint32_t n = sk.joint_count;
    float* buf = n <= R3_ANIM_SMEM_JOINTS ? smem : spill + spill_offset[blockIdx.x];
    const r3_anim_joint* skin_joints = joints + sk.first_joint;

    float t = job.time;                                              // time.clamp(0.0, duration) (lib.rs:190)
    if (t < 0.0f) t = 0.0f;
    if (t > clip.duration) t = clip.duration;

    // local matrices (lib.rs:219-238)
    for (uint32_t k = threadIdx.x; k < n; k += blockDim.x) {
        const r3_anim_channel* ch = channels + clip.first_channel + k;
        float m[16];
        if (!ch->animated) {
#pragma unroll
            for (int i = 0; i < 16; ++i) m[i] = (i % 5 == 0) ? 1.0f : 0.0f;   // Mat4::IDENTITY, not the bind pose (lib.rs:219)
        } else {
            const r3_anim_joint* jt = skin_joints + k;
            const r3_anim_track tt = ch->translation, rt = ch->rotation, st = ch->scale;
            const float3 tr = tt.times == R3_ANIM_ABSENT ? make_float3(jt->bind_translation[0], jt->bind_translation[1], jt->bind_translation[2]) : sample3(keys, tt, t);
            const float4 q = rt.times == R3_ANIM_ABSENT ? make_float4(jt->bind_rotation[0], jt->bind_rotation[1], jt->bind_rotation[2], jt->bind_rotation[3])
                                                        : sample_quat(keys, rt, t);
            const float3 sc = st.times == R3_ANIM_ABSENT ? make_float3(jt->bind_scale[0], jt->bind_scale[1], jt->bind_scale[2]) : sample3(keys, st, t);
            from_srt(sc, q, tr, m);
        }
        float* o = buf + (size_t)k * R3_ANIM_STRIDE;
#pragma unroll
        for (int i = 0; i < 16; ++i) o[i] = m[i];
    }
    __syncthreads();

    // global matrices level by level, in place (lib.rs:240-256)
    const float ident[16] = {1.0f, 0.0f, 0.0f, 0.0f, 0.0f, 1.0f, 0.0f, 0.0f, 0.0f, 0.0f, 1.0f, 0.0f, 0.0f, 0.0f, 0.0f, 1.0f};
    for (uint32_t l = 0; l < sk.n_levels; ++l) {
        const uint32_t end = levels[sk.first_level + l + 1];
        for (uint32_t i = levels[sk.first_level + l] + threadIdx.x; i < end; i += blockDim.x) {
            const uint32_t k = sched[sk.first_sched + i];
            const uint32_t parent = skin_joints[k].parent;
            if (parent == R3_ANIM_NO_PARENT) continue;                  // global = local
            float a[16], b[16], g[16];
            float* o = buf + (size_t)k * R3_ANIM_STRIDE;
#pragma unroll
            for (int e = 0; e < 16; ++e) b[e] = o[e];
            if (parent == R3_ANIM_PARENT_NOT_JOINT) {
#pragma unroll
                for (int e = 0; e < 16; ++e) a[e] = ident[e];              // IDENTITY * local: a real multiply
            } else {
                const float* pm = buf + (size_t)parent * R3_ANIM_STRIDE;
#pragma unroll
                for (int e = 0; e < 16; ++e) a[e] = pm[e];
            }
            mat_mul(a, b, g);
#pragma unroll
            for (int e = 0; e < 16; ++e) o[e] = g[e];
        }
        __syncthreads();
    }

    // joint matrices = global * inverse_bind (set_skeleton_joint_transforms), the first joint_count of them into every target
    uint32_t most = 0;
    for (uint32_t q = 0; q < job.target_count; ++q) most = max(most, targets[job.first_target + q].joint_count);
    for (uint32_t k = threadIdx.x; k < most; k += blockDim.x) {
        float g[16], ib[16], m[16];
        const float* o = buf + (size_t)k * R3_ANIM_STRIDE;
#pragma unroll
        for (int e = 0; e < 16; ++e) { g[e] = o[e]; ib[e] = __ldg(&skin_joints[k].inverse_bind[e]); }
        mat_mul(g, ib, m);
        for (uint32_t q = 0; q < job.target_count; ++q) {
            const r3_pose_target tg = targets[job.first_target + q];
            if (k >= tg.joint_count) continue;
            float4* dst = reinterpret_cast<float4*>(joint_buf + ((size_t)tg.joint_matrix_base_offset + k) * 16);
            dst[0] = make_float4(m[0], m[1], m[2], m[3]); dst[1] = make_float4(m[4], m[5], m[6], m[7]);
            dst[2] = make_float4(m[8], m[9], m[10], m[11]); dst[3] = make_float4(m[12], m[13], m[14], m[15]);
        }
    }
}

constexpr uint32_t R3_JOINT_WRITE_THREADS = 256;   // 8 writes per CTA

// set_skeleton_joint_matrices / set_skeleton_joint_transforms (renderer/mod.rs:302-337): one warp per write, lanes striding over its
// joints, each joint a 64-byte matrix read as four float4s (plus the inverse bind's 64 bytes) and stored as four float4s.  Without inverse
// binds the float4s are moved untouched, so every bit survives; with them the stored matrix is mat_mul(global, inverse_bind), pose_kernel's
// product.  A write whose destination or sources leave their arrays is dropped whole (64-bit sums): the host form checked them already,
// the device form cannot.
__global__ void __launch_bounds__(R3_JOINT_WRITE_THREADS) joint_write_kernel(const r3_joint_write* __restrict__ writes, uint32_t n_writes,
                                                                             const float4* __restrict__ mat4s, uint32_t n_mat4s,
                                                                             const float4* __restrict__ inverse_binds, uint32_t n_inverse_binds,
                                                                             float4* __restrict__ joint_buf, uint32_t n_joint_mats) {
    const uint32_t w = blockIdx.x * (R3_JOINT_WRITE_THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (w >= n_writes) return;
    const r3_joint_write jw = writes[w];
    const uint64_t n = jw.joint_count;
    if (jw.joint_matrix_base_offset + n > n_joint_mats || jw.first_matrix + n > n_mat4s) return;
    if (inverse_binds && jw.first_inverse_bind + n > n_inverse_binds) return;
    for (uint32_t k = lane; k < n; k += 32) {
        const float4* src = mat4s + ((size_t)jw.first_matrix + k) * 4;
        float4* dst = joint_buf + ((size_t)jw.joint_matrix_base_offset + k) * 4;
        float4 g[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) g[e] = __ldg(src + e);
        if (inverse_binds) {
            const float4* ibp = inverse_binds + ((size_t)jw.first_inverse_bind + k) * 4;
            float4 ib[4], m[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) ib[e] = __ldg(ibp + e);
            mat_mul(reinterpret_cast<const float*>(g), reinterpret_cast<const float*>(ib), reinterpret_cast<float*>(m));
#pragma unroll
            for (int e = 0; e < 4; ++e) dst[e] = m[e];
        } else {
#pragma unroll
            for (int e = 0; e < 4; ++e) dst[e] = g[e];
        }
    }
}

constexpr uint32_t R3_OBJ_POSE_THREADS = 128;

// The object-transform half of pose_animation_frame (lib.rs:190-212) + set_object_transform (object.rs:302-316), one thread per
// (job, target) item.  Rule R12: bind pose for an absent track, scale.z negated for a left-handed renderer, from_srt, then the record's
// transform and world sphere (float4 #0-4) and the sort location.  Slots at or past n_slots are skipped (ScatterCopy drops them).
__global__ void __launch_bounds__(R3_OBJ_POSE_THREADS) pose_objects_kernel(const uint2* __restrict__ items, uint32_t n_items, const r3_pose_job* __restrict__ jobs,
                                                                            const r3_object_pose_target* __restrict__ targets, const r3_anim_node_clip* __restrict__ clips,
                                                                            const r3_anim_node_channel* __restrict__ channels, const r3_anim_node* __restrict__ nodes,
                                                                            const float* __restrict__ keys, uint32_t left_handed, float4* __restrict__ objects,
                                                                            uint32_t n_slots, float* __restrict__ sort_loc, uint32_t sort_n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_items) return;
    const uint2 it = items[i];
    const r3_object_pose_target tg = targets[it.y];
    if (tg.slot >= n_slots) return;
    const r3_pose_job job = jobs[it.x];
    const r3_anim_node_clip clip = clips[job.clip];
    float t = job.time;                                                  // time.clamp(0.0, duration) (lib.rs:190)
    if (t < 0.0f) t = 0.0f;
    if (t > clip.duration) t = clip.duration;
    const r3_anim_node_channel* ch = channels + clip.first_channel + tg.channel;
    const r3_anim_node* nd = nodes + ch->node;
    // a missing property takes the node's bind pose (lib.rs:194-199)
    const r3_anim_track tt = ch->translation, rt = ch->rotation, st = ch->scale;
    const float3 tr = tt.times == R3_ANIM_ABSENT ? make_float3(nd->bind_translation[0], nd->bind_translation[1], nd->bind_translation[2]) : sample3(keys, tt, t);
    const float4 q = rt.times == R3_ANIM_ABSENT ? make_float4(nd->bind_rotation[0], nd->bind_rotation[1], nd->bind_rotation[2], nd->bind_rotation[3])
                                                : sample_quat(keys, rt, t);
    float3 sc = st.times == R3_ANIM_ABSENT ? make_float3(nd->bind_scale[0], nd->bind_scale[1], nd->bind_scale[2]) : sample3(keys, st, t);
    if (left_handed) sc.z = __uint_as_float(__float_as_uint(sc.z) ^ 0x80000000u);   // scale.z = -scale.z (lib.rs:201-203): a sign flip
    float m[16];
    from_srt(sc, q, tr, m);
    float x[4], y[4], z[4];   // xyz of the four columns
#pragma unroll
    for (int j = 0; j < 4; ++j) { x[j] = m[4 * j]; y[j] = m[4 * j + 1]; z[j] = m[4 * j + 2]; }
    const float4 sph = sphere_apply_transform_rn(x, y, z, make_float4(tg.mesh_sphere_center[0], tg.mesh_sphere_center[1], tg.mesh_sphere_center[2], tg.mesh_sphere_radius));
    float4* rec = objects + (size_t)tg.slot * 8;
    rec[0] = make_float4(m[0], m[1], m[2], m[3]); rec[1] = make_float4(m[4], m[5], m[6], m[7]);
    rec[2] = make_float4(m[8], m[9], m[10], m[11]); rec[3] = make_float4(m[12], m[13], m[14], m[15]);
    rec[4] = sph;
    if (sort_loc && tg.slot < sort_n) {
        float* l = sort_loc + 3 * (size_t)tg.slot;
        l[0] = sort_location_rn(x); l[1] = sort_location_rn(y); l[2] = sort_location_rn(z);
    }
}

// the sort locations of the posed slots, for the host mirror the host batching sorts by
__global__ void gather_locations_kernel(const uint32_t* __restrict__ slots, uint32_t n, const float* __restrict__ sort_loc, uint32_t sort_n, float* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = slots[i];
    if (s >= sort_n) return;
#pragma unroll
    for (int k = 0; k < 3; ++k) out[3 * (size_t)i + k] = sort_loc[3 * (size_t)s + k];
}

// a device array of n elements, a copy of src unless src is null (allocated even when empty, so that kernels always get a valid pointer)
template <typename T>
int upload_array(r3_ctx* c, T** out, const T* src, uint64_t n, std::vector<void*>& made) {
    void* p = nullptr;
    R3_CUDA(c, cudaMalloc(&p, (n ? n : 1) * sizeof(T)));
    made.push_back(p);
    if (n && src) R3_CUDA(c, cudaMemcpyAsync(p, src, n * sizeof(T), cudaMemcpyHostToDevice, c->stream));
    *out = (T*)p;
    return R3_OK;
}

// run `fill` (which allocates into `made`); on failure free what it made and leave the context as it was
template <typename F>
int transactional(r3_ctx* c, F fill) {
    std::vector<void*> made;
    int rc = fill(made);
    if (rc == R3_OK) {
        const cudaError_t e = r3_stream_sync(c);                      // host pointers are only borrowed for the call
        if (e != cudaSuccess) rc = r3_cuda_fail(c, e, "animation upload");
    }
    if (rc != R3_OK) {
        r3_stream_sync(c);
        for (void* p : made) cudaFree(p);
    }
    return rc;
}

}  // namespace

struct r3_anim_state {
    // r3_set_animations
    bool has_library = false;
    std::vector<r3_anim_skin> skins; std::vector<r3_anim_clip> clips;
    anim_skin_dev* d_skins = nullptr; r3_anim_joint* d_joints = nullptr; uint32_t* d_sched = nullptr; uint32_t* d_levels = nullptr;
    r3_anim_clip* d_clips = nullptr; r3_anim_channel* d_channels = nullptr; float* d_keys = nullptr;
    // r3_set_skeletons
    bool has_skeletons = false;
    r3_skinning_input* d_inputs = nullptr; uint32_t* d_prefix = nullptr; uint32_t n_skeletons = 0, total_chunks = 0;
    float* d_joint_buf = nullptr; uint32_t n_joint_mats = 0;
    // r3_set_pose_jobs
    bool has_jobs = false;
    r3_pose_job* d_jobs = nullptr; r3_pose_target* d_targets = nullptr; uint32_t n_jobs = 0;
    uint64_t* d_spill_offset = nullptr; float* d_spill = nullptr; uint32_t smem_bytes = 0;
    uint64_t jobs_cap = 0, targets_cap = 0, spill_offset_cap = 0, spill_cap = 0;   // grow-only (r3_set_pose_jobs runs every frame)
    // r3_set_joint_matrices' copies of its host arrays, grow-only (the call runs every frame)
    r3_joint_write* d_jw_writes = nullptr; float4* d_jw_mats = nullptr; float4* d_jw_ibs = nullptr;
    uint64_t jw_writes_cap = 0, jw_mats_cap = 0, jw_ibs_cap = 0;
    // r3_set_object_animations (independent of the skeletal state above)
    bool has_obj_library = false; uint32_t left_handed = 0;
    std::vector<r3_anim_node_clip> obj_clips;
    r3_anim_node* d_nodes = nullptr; r3_anim_node_clip* d_node_clips = nullptr; r3_anim_node_channel* d_node_channels = nullptr; float* d_obj_keys = nullptr;
    // r3_set_object_pose_jobs: the jobs and targets, and one item (job, target) per posed target with its slot
    bool has_obj_jobs = false; uint32_t n_obj_items = 0;
    r3_pose_job* d_obj_jobs = nullptr; r3_object_pose_target* d_obj_targets = nullptr; uint2* d_obj_items = nullptr; uint32_t* d_obj_slots = nullptr;
    float* d_loc_stage = nullptr;
    uint64_t obj_jobs_cap = 0, obj_targets_cap = 0, obj_items_cap = 0, obj_slots_cap = 0, loc_stage_cap = 0;   // grow-only
    std::vector<uint32_t> obj_slots;          // host copy of d_obj_slots
    std::vector<float> loc_stage;             // the posed slots' locations on their way to c->sort_loc
    bool locations_pending = false;           // r3_pose_objects ran since c->sort_loc last took the posed locations

    void free_library() { for (void* p : {(void*)d_skins, (void*)d_joints, (void*)d_sched, (void*)d_levels, (void*)d_clips, (void*)d_channels, (void*)d_keys}) cudaFree(p);
                          d_skins = nullptr; d_joints = nullptr; d_sched = nullptr; d_levels = nullptr; d_clips = nullptr; d_channels = nullptr; d_keys = nullptr;
                          has_library = false; skins.clear(); clips.clear(); }
    void free_skeletons() { for (void* p : {(void*)d_inputs, (void*)d_prefix, (void*)d_joint_buf}) cudaFree(p);
                            d_inputs = nullptr; d_prefix = nullptr; d_joint_buf = nullptr; has_skeletons = false; n_skeletons = total_chunks = n_joint_mats = 0; }
    void drop_jobs() { has_jobs = false; n_jobs = 0; smem_bytes = 0; }   // the buffers stay for the next r3_set_pose_jobs
    void free_jobs() { for (void* p : {(void*)d_jobs, (void*)d_targets, (void*)d_spill_offset, (void*)d_spill}) cudaFree(p);
                       d_jobs = nullptr; d_targets = nullptr; d_spill_offset = nullptr; d_spill = nullptr;
                       jobs_cap = targets_cap = spill_offset_cap = spill_cap = 0; drop_jobs(); }
    void free_joint_writes() { for (void* p : {(void*)d_jw_writes, (void*)d_jw_mats, (void*)d_jw_ibs}) cudaFree(p);
                               d_jw_writes = nullptr; d_jw_mats = nullptr; d_jw_ibs = nullptr; jw_writes_cap = jw_mats_cap = jw_ibs_cap = 0; }
    void free_obj_library() { for (void* p : {(void*)d_nodes, (void*)d_node_clips, (void*)d_node_channels, (void*)d_obj_keys}) cudaFree(p);
                              d_nodes = nullptr; d_node_clips = nullptr; d_node_channels = nullptr; d_obj_keys = nullptr;
                              has_obj_library = false; left_handed = 0; obj_clips.clear(); }
    void drop_obj_jobs() { has_obj_jobs = false; n_obj_items = 0; obj_slots.clear(); }   // the buffers stay for the next r3_set_object_pose_jobs
    void free_obj_jobs() { for (void* p : {(void*)d_obj_jobs, (void*)d_obj_targets, (void*)d_obj_items, (void*)d_obj_slots, (void*)d_loc_stage}) cudaFree(p);
                           d_obj_jobs = nullptr; d_obj_targets = nullptr; d_obj_items = nullptr; d_obj_slots = nullptr; d_loc_stage = nullptr;
                           obj_jobs_cap = obj_targets_cap = obj_items_cap = obj_slots_cap = loc_stage_cap = 0; drop_obj_jobs(); }
};

void r3_anim_destroy(r3_ctx* c) {
    if (!c->anim) return;
    c->anim->free_obj_jobs(); c->anim->free_obj_library();
    c->anim->free_joint_writes(); c->anim->free_jobs(); c->anim->free_skeletons(); c->anim->free_library();
    delete c->anim;
    c->anim = nullptr;
}

static int anim_state(r3_ctx* c) {
    if (!c->anim) c->anim = new (std::nothrow) r3_anim_state();
    return c->anim ? R3_OK : r3_fail(c, R3_E_OOM, "animation state");
}

R3_EXPORT int r3_set_animations(r3_ctx* c, const r3_anim_library* L) {
    if (!c) return R3_E_INVALID;
    const char* msg = "";
    if (r3_anim_check_library(L, &msg) != R3_OK) return r3_fail(c, R3_E_INVALID, msg);
    cudaSetDevice(c->device);
    R3_TRY(anim_state(c));
    // each skin's joints sorted by level into its own stretch of sched (skins may share joint records, so not the joint range);
    // levels[first_level + l] = first position of level l in that stretch
    std::vector<anim_skin_dev> dskins(L->n_skins);
    std::vector<uint32_t> sched, levels, level_of;
    for (uint32_t s = 0; s < L->n_skins; ++s) {
        const r3_anim_skin sk = L->skins[s];
        level_of.assign(sk.joint_count, 0u);
        uint32_t depth = 0;
        for (uint32_t i = 0; i < sk.joint_count; ++i) {             // order lists parents first (checked)
            const uint32_t k = L->order[sk.first_joint + i], p = L->joints[sk.first_joint + k].parent;
            level_of[k] = (p == R3_ANIM_NO_PARENT || p == R3_ANIM_PARENT_NOT_JOINT) ? 0u : level_of[p] + 1u;
            depth = std::max(depth, level_of[k] + 1u);
        }
        std::vector<uint32_t> start(depth + 1, 0u);
        for (uint32_t k = 0; k < sk.joint_count; ++k) start[level_of[k] + 1]++;
        for (uint32_t l = 0; l < depth; ++l) start[l + 1] += start[l];
        const size_t first_sched = sched.size();
        dskins[s] = {sk.first_joint, sk.joint_count, depth, (uint64_t)levels.size(), (uint64_t)first_sched};
        levels.insert(levels.end(), start.begin(), start.end());
        sched.resize(first_sched + sk.joint_count);
        for (uint32_t k = 0; k < sk.joint_count; ++k) sched[first_sched + start[level_of[k]]++] = k;
    }
    r3_anim_state* a = c->anim;
    r3_anim_state n;
    const int rc = transactional(c, [&](std::vector<void*>& made) {
        R3_TRY(upload_array(c, &n.d_skins, dskins.data(), dskins.size(), made));
        R3_TRY(upload_array(c, &n.d_joints, L->joints, L->n_joints, made));
        R3_TRY(upload_array(c, &n.d_sched, sched.data(), sched.size(), made));
        R3_TRY(upload_array(c, &n.d_levels, levels.data(), levels.size(), made));
        R3_TRY(upload_array(c, &n.d_clips, L->clips, L->n_clips, made));
        R3_TRY(upload_array(c, &n.d_channels, L->channels, L->n_channels, made));
        return upload_array(c, &n.d_keys, L->keys, L->n_keys, made);
    });
    if (rc != R3_OK) return rc;
    a->drop_jobs();
    a->free_library();
    a->d_skins = n.d_skins; a->d_joints = n.d_joints; a->d_sched = n.d_sched; a->d_levels = n.d_levels;
    a->d_clips = n.d_clips; a->d_channels = n.d_channels; a->d_keys = n.d_keys;
    n.d_skins = nullptr; n.d_joints = nullptr; n.d_sched = nullptr; n.d_levels = nullptr; n.d_clips = nullptr; n.d_channels = nullptr; n.d_keys = nullptr;
    a->skins.assign(L->skins, L->skins + L->n_skins);
    a->clips.assign(L->clips, L->clips + L->n_clips);
    a->has_library = true;
    return R3_OK;
}

R3_EXPORT int r3_set_skeletons(r3_ctx* c, const r3_skinning_input* inputs, uint32_t n_skeletons, const float* joint_matrices, uint32_t n_joints) {
    if (!c) return R3_E_INVALID;
    if ((!inputs && n_skeletons) || (!joint_matrices && n_joints)) return r3_fail(c, R3_E_INVALID, "set_skeletons: null");
    cudaSetDevice(c->device);
    R3_TRY(anim_state(c));
    std::vector<uint32_t> prefix(n_skeletons + 1, 0u);
    for (uint32_t s = 0; s < n_skeletons; ++s) prefix[s + 1] = prefix[s] + (inputs[s].vertex_count + 255u) / 256u;
    r3_anim_state* a = c->anim;
    r3_anim_state n;
    const int rc = transactional(c, [&](std::vector<void*>& made) {
        R3_TRY(upload_array(c, &n.d_inputs, inputs, n_skeletons, made));
        R3_TRY(upload_array(c, &n.d_prefix, prefix.data(), prefix.size(), made));
        return upload_array(c, &n.d_joint_buf, joint_matrices, (uint64_t)n_joints * 16, made);
    });
    if (rc != R3_OK) return rc;
    a->drop_jobs();
    a->free_skeletons();
    a->d_inputs = n.d_inputs; a->d_prefix = n.d_prefix; a->d_joint_buf = n.d_joint_buf;
    n.d_inputs = nullptr; n.d_prefix = nullptr; n.d_joint_buf = nullptr;
    a->n_skeletons = n_skeletons; a->total_chunks = prefix[n_skeletons]; a->n_joint_mats = n_joints;
    a->has_skeletons = true;
    return R3_OK;
}

R3_EXPORT int r3_set_pose_jobs(r3_ctx* c, const r3_pose_job* jobs, uint32_t n_jobs, const r3_pose_target* targets, uint32_t n_targets) {
    if (!c) return R3_E_INVALID;
    r3_anim_state* a = c->anim;
    if (!a || !a->has_library) return r3_fail(c, R3_E_STATE, "set_pose_jobs before set_animations");
    if (!a->has_skeletons) return r3_fail(c, R3_E_STATE, "set_pose_jobs before set_skeletons");
    const char* msg = "";
    if (r3_anim_check_jobs(a->skins.data(), a->clips.data(), (uint32_t)a->clips.size(), a->n_joint_mats, jobs, n_jobs, targets, n_targets, &msg) != R3_OK)
        return r3_fail(c, R3_E_INVALID, msg);
    cudaSetDevice(c->device);
    // scratch of the skins that do not fit in shared memory, sized here so that r3_pose_skeletons allocates nothing
    std::vector<uint64_t> spill_offset(n_jobs, 0u);
    uint64_t spill_floats = 0;
    uint32_t most = 0;
    for (uint32_t i = 0; i < n_jobs; ++i) {
        const uint32_t nj = a->skins[a->clips[jobs[i].clip].skin].joint_count;
        if (nj > R3_ANIM_SMEM_JOINTS) { spill_offset[i] = spill_floats; spill_floats += (uint64_t)nj * R3_ANIM_STRIDE; }
        else most = std::max(most, nj);
    }
    // the call is made every simulation frame: the buffers only grow, and a growth keeps the current jobs (a failed one leaves them)
    R3_TRY(r3_reserve_t(c, &a->d_jobs, &a->jobs_cap, std::max(n_jobs, 1u), true));
    R3_TRY(r3_reserve_t(c, &a->d_targets, &a->targets_cap, std::max(n_targets, 1u), true));
    R3_TRY(r3_reserve_t(c, &a->d_spill_offset, &a->spill_offset_cap, std::max(n_jobs, 1u), true));
    R3_TRY(r3_reserve_t(c, &a->d_spill, &a->spill_cap, std::max<uint64_t>(spill_floats, 1u), false));
    if (n_jobs) R3_CUDA(c, cudaMemcpyAsync(a->d_jobs, jobs, (size_t)n_jobs * sizeof(r3_pose_job), cudaMemcpyHostToDevice, c->stream));
    if (n_targets) R3_CUDA(c, cudaMemcpyAsync(a->d_targets, targets, (size_t)n_targets * sizeof(r3_pose_target), cudaMemcpyHostToDevice, c->stream));
    if (n_jobs) R3_CUDA(c, cudaMemcpyAsync(a->d_spill_offset, spill_offset.data(), (size_t)n_jobs * sizeof(uint64_t), cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, r3_stream_sync(c));                                    // host pointers are only borrowed for the call
    a->n_jobs = n_jobs;
    a->smem_bytes = most * R3_ANIM_STRIDE * (uint32_t)sizeof(float);
    a->has_jobs = true;
    return R3_OK;
}

R3_EXPORT int r3_pose_skeletons(r3_ctx* c) {
    if (!c) return R3_E_INVALID;
    r3_anim_state* a = c->anim;
    if (!a || !a->has_jobs) return r3_fail(c, R3_E_STATE, "pose_skeletons before set_animations + set_skeletons + set_pose_jobs");
    if (a->n_jobs == 0) return R3_OK;
    cudaSetDevice(c->device);
    pose_kernel<<<a->n_jobs, R3_ANIM_THREADS, a->smem_bytes, c->stream>>>(a->d_jobs, a->d_targets, a->d_clips, a->d_skins, a->d_joints, a->d_sched, a->d_levels,
                                                                         a->d_channels, a->d_keys, a->d_spill_offset, a->d_spill, a->d_joint_buf);
    R3_CHECK_LAUNCH(c, "pose_kernel");
    return R3_OK;
}

R3_EXPORT int r3_skin_posed(r3_ctx* c) {
    if (!c) return R3_E_INVALID;
    r3_anim_state* a = c->anim;
    if (!a || !a->has_skeletons) return r3_fail(c, R3_E_STATE, "skin_posed before set_skeletons");
    if (a->n_skeletons == 0) return R3_OK;
    if (!c->d_mesh) return r3_fail(c, R3_E_STATE, "skin_posed before set_mesh_buffer");
    cudaSetDevice(c->device);
    return r3_launch_skinning(c, a->d_inputs, a->d_prefix, a->n_skeletons, a->total_chunks, a->d_joint_buf, a->n_joint_mats);
}

R3_EXPORT int r3_readback_joint_matrices(r3_ctx* c, float* out, uint32_t first, uint32_t n) {
    if (!c) return R3_E_INVALID;
    r3_anim_state* a = c->anim;
    if (!a || !a->has_skeletons) return r3_fail(c, R3_E_STATE, "readback_joint_matrices before set_skeletons");
    if (!out && n) return r3_fail(c, R3_E_INVALID, "readback_joint_matrices: null");
    if ((uint64_t)first + n > a->n_joint_mats) return r3_fail(c, R3_E_INVALID, "readback_joint_matrices: range outside the joint buffer");
    if (n == 0) return R3_OK;
    cudaSetDevice(c->device);
    R3_CUDA(c, r3_stream_sync(c));
    R3_CUDA(c, cudaMemcpy(out, a->d_joint_buf + (size_t)first * 16, (size_t)n * 64, cudaMemcpyDeviceToHost));
    return R3_OK;
}

// ------------------------------------------------------------------ joint matrices set by the application (set_skeleton_joint_*)
static int launch_joint_writes(r3_ctx* c, const r3_joint_write* d_writes, uint32_t n_writes, const float* d_mat4s, uint32_t n_mat4s,
                               const float* d_inverse_binds, uint32_t n_inverse_binds) {
    constexpr uint32_t per_cta = R3_JOINT_WRITE_THREADS / 32;
    r3_anim_state* a = c->anim;
    joint_write_kernel<<<(uint32_t)(((uint64_t)n_writes + per_cta - 1) / per_cta), R3_JOINT_WRITE_THREADS, 0, c->stream>>>(
        d_writes, n_writes, reinterpret_cast<const float4*>(d_mat4s), n_mat4s, reinterpret_cast<const float4*>(d_inverse_binds), n_inverse_binds,
        reinterpret_cast<float4*>(a->d_joint_buf), a->n_joint_mats);
    R3_CHECK_LAUNCH(c, "joint_write_kernel");
    return R3_OK;
}

R3_EXPORT int r3_set_joint_matrices(r3_ctx* c, const r3_joint_write* writes, uint32_t n_writes, const float* mat4s, uint32_t n_mat4s,
                                    const float* inverse_binds, uint32_t n_inverse_binds) {
    if (!c) return R3_E_INVALID;
    r3_anim_state* a = c->anim;
    if (!a || !a->has_skeletons) return r3_fail(c, R3_E_STATE, "set_joint_matrices before set_skeletons");
    if ((!writes && n_writes) || (!mat4s && n_mat4s) || (!inverse_binds && n_inverse_binds)) return r3_fail(c, R3_E_INVALID, "set_joint_matrices: null");
    const char* msg = "";
    if (r3_anim_check_joint_writes(a->n_joint_mats, writes, n_writes, n_mat4s, inverse_binds != nullptr, n_inverse_binds, &msg) != R3_OK)
        return r3_fail(c, R3_E_INVALID, msg);
    if (n_writes == 0) return R3_OK;
    cudaSetDevice(c->device);
    R3_TRY(r3_reserve_t(c, &a->d_jw_writes, &a->jw_writes_cap, n_writes));
    R3_TRY(r3_reserve_t(c, &a->d_jw_mats, &a->jw_mats_cap, std::max<uint64_t>(4ull * n_mat4s, 1u)));
    if (inverse_binds) R3_TRY(r3_reserve_t(c, &a->d_jw_ibs, &a->jw_ibs_cap, std::max<uint64_t>(4ull * n_inverse_binds, 1u)));
    R3_CUDA(c, cudaMemcpyAsync(a->d_jw_writes, writes, (size_t)n_writes * sizeof(r3_joint_write), cudaMemcpyHostToDevice, c->stream));
    if (n_mat4s) R3_CUDA(c, cudaMemcpyAsync(a->d_jw_mats, mat4s, (size_t)n_mat4s * 64, cudaMemcpyHostToDevice, c->stream));
    if (inverse_binds && n_inverse_binds) R3_CUDA(c, cudaMemcpyAsync(a->d_jw_ibs, inverse_binds, (size_t)n_inverse_binds * 64, cudaMemcpyHostToDevice, c->stream));
    R3_TRY(launch_joint_writes(c, a->d_jw_writes, n_writes, (const float*)a->d_jw_mats, n_mat4s, inverse_binds ? (const float*)a->d_jw_ibs : nullptr,
                               n_inverse_binds));
    R3_CUDA(c, r3_stream_sync(c));                                    // host pointers are only borrowed for the call
    return R3_OK;
}

R3_EXPORT int r3_set_joint_matrices_device(r3_ctx* c, const r3_joint_write* d_writes, uint32_t n_writes, const float* d_mat4s, uint32_t n_mat4s,
                                           const float* d_inverse_binds, uint32_t n_inverse_binds) {
    if (!c) return R3_E_INVALID;
    r3_anim_state* a = c->anim;
    if (!a || !a->has_skeletons) return r3_fail(c, R3_E_STATE, "set_joint_matrices_device before set_skeletons");
    if (n_writes == 0) return R3_OK;
    if (!d_writes || (!d_mat4s && n_mat4s) || (!d_inverse_binds && n_inverse_binds) || ((uintptr_t)d_writes & 3u) || ((uintptr_t)d_mat4s & 15u) ||
        ((uintptr_t)d_inverse_binds & 15u))
        return r3_fail(c, R3_E_INVALID, "set_joint_matrices_device: null or misaligned pointer (matrices: 16 bytes, writes: 4 bytes)");
    cudaSetDevice(c->device);
    return launch_joint_writes(c, d_writes, n_writes, d_mat4s, n_mat4s, d_inverse_binds, n_inverse_binds);
}

// ------------------------------------------------------------------ object animation (the object-transform half of pose_animation_frame)
// Host batching sorts by the host mirror c->sort_loc: after r3_pose_objects it takes the posed slots' locations from the device.  The
// stage half enqueues a gather and its copy to the host (the caller drains the stream, which the host batching does anyway for the
// visible list); the apply half writes them into the mirror.
int r3_anim_stage_posed_locations(r3_ctx* c, bool* staged) {
    *staged = false;
    r3_anim_state* a = c->anim;
    if (!a || !a->locations_pending) return R3_OK;
    const uint32_t n = a->n_obj_items, sort_n = r3_sort_extent(c);
    if (n == 0 || sort_n == 0 || !c->d_sort_loc) { a->locations_pending = false; return R3_OK; }
    gather_locations_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>(a->d_obj_slots, n, c->d_sort_loc, sort_n, a->d_loc_stage);
    R3_CHECK_LAUNCH(c, "gather_locations_kernel");
    a->loc_stage.resize(3 * (size_t)n);
    R3_CUDA(c, cudaMemcpyAsync(a->loc_stage.data(), a->d_loc_stage, (size_t)n * 12, cudaMemcpyDeviceToHost, c->stream));
    *staged = true;
    return R3_OK;
}
void r3_anim_apply_posed_locations(r3_ctx* c) {
    r3_anim_state* a = c->anim;
    if (!a || !a->locations_pending) return;   // stage enqueued nothing: it clears the flag unless it did
    const size_t sort_n = c->sort_key.size();
    for (size_t i = 0; i < a->obj_slots.size(); ++i)
        if (a->obj_slots[i] < sort_n) memcpy(&c->sort_loc[3 * (size_t)a->obj_slots[i]], &a->loc_stage[3 * i], 12);
    a->locations_pending = false;
}
// the same, blocking: before the posed slots' list is replaced
static int refresh_posed_locations(r3_ctx* c) {
    bool staged = false;
    R3_TRY(r3_anim_stage_posed_locations(c, &staged));
    if (!staged) return R3_OK;
    R3_CUDA(c, r3_stream_sync(c));
    r3_anim_apply_posed_locations(c);
    return R3_OK;
}

R3_EXPORT int r3_set_object_animations(r3_ctx* c, const r3_anim_object_library* L) {
    if (!c) return R3_E_INVALID;
    const char* msg = "";
    if (r3_anim_check_object_library(L, &msg) != R3_OK) return r3_fail(c, R3_E_INVALID, msg);
    R3_TRY(r3_check_object_writer(c, "set_object_animations", R3_NEED_OWNED));
    cudaSetDevice(c->device);
    R3_TRY(anim_state(c));
    r3_anim_state* a = c->anim;
    r3_anim_state n;
    const int rc = transactional(c, [&](std::vector<void*>& made) {
        R3_TRY(upload_array(c, &n.d_nodes, L->nodes, L->n_nodes, made));
        R3_TRY(upload_array(c, &n.d_node_clips, L->clips, L->n_clips, made));
        R3_TRY(upload_array(c, &n.d_node_channels, L->channels, L->n_channels, made));
        return upload_array(c, &n.d_obj_keys, L->keys, L->n_keys, made);
    });
    if (rc != R3_OK) return rc;
    R3_TRY(refresh_posed_locations(c));
    a->drop_obj_jobs();
    a->free_obj_library();
    a->d_nodes = n.d_nodes; a->d_node_clips = n.d_node_clips; a->d_node_channels = n.d_node_channels; a->d_obj_keys = n.d_obj_keys;
    n.d_nodes = nullptr; n.d_node_clips = nullptr; n.d_node_channels = nullptr; n.d_obj_keys = nullptr;
    a->obj_clips.assign(L->clips, L->clips + L->n_clips);
    a->left_handed = L->left_handed ? 1u : 0u;
    a->has_obj_library = true;
    return R3_OK;
}

R3_EXPORT int r3_set_object_pose_jobs(r3_ctx* c, const r3_pose_job* jobs, uint32_t n_jobs, const r3_object_pose_target* targets, uint32_t n_targets) {
    if (!c) return R3_E_INVALID;
    r3_anim_state* a = c->anim;
    if (!a || !a->has_obj_library) return r3_fail(c, R3_E_STATE, "set_object_pose_jobs before set_object_animations");
    R3_TRY(r3_check_object_writer(c, "set_object_pose_jobs", R3_NEED_OWNED));
    const char* msg = "";
    uint32_t* listed = nullptr;
    uint64_t n_items = 0;
    if (r3_anim_check_object_jobs(a->obj_clips.data(), (uint32_t)a->obj_clips.size(), c->n_slots, jobs, n_jobs, targets, n_targets, &listed, &n_items, &msg) != R3_OK)
        return r3_fail(c, R3_E_INVALID, msg);
    std::vector<uint32_t> slots(listed, listed + n_items);
    free(listed);
    std::vector<uint2> items;
    items.reserve(n_items);
    for (uint32_t i = 0; i < n_jobs; ++i)
        for (uint32_t t = 0; t < jobs[i].target_count; ++t) items.push_back(make_uint2(i, jobs[i].first_target + t));
    const uint32_t n = (uint32_t)n_items;   // distinct slots below n_slots
    cudaSetDevice(c->device);
    R3_TRY(refresh_posed_locations(c));
    // the call is made every simulation frame: the buffers only grow, and a growth keeps the current jobs (a failed one leaves them)
    R3_TRY(r3_reserve_t(c, &a->d_obj_jobs, &a->obj_jobs_cap, std::max(n_jobs, 1u), true));
    R3_TRY(r3_reserve_t(c, &a->d_obj_targets, &a->obj_targets_cap, std::max(n_targets, 1u), true));
    R3_TRY(r3_reserve_t(c, &a->d_obj_items, &a->obj_items_cap, std::max(n, 1u), true));
    R3_TRY(r3_reserve_t(c, &a->d_obj_slots, &a->obj_slots_cap, std::max(n, 1u), true));
    R3_TRY(r3_reserve_t(c, &a->d_loc_stage, &a->loc_stage_cap, 3 * (uint64_t)std::max(n, 1u), false));
    if (n_jobs) R3_CUDA(c, cudaMemcpyAsync(a->d_obj_jobs, jobs, (size_t)n_jobs * sizeof(r3_pose_job), cudaMemcpyHostToDevice, c->stream));
    if (n_targets) R3_CUDA(c, cudaMemcpyAsync(a->d_obj_targets, targets, (size_t)n_targets * sizeof(r3_object_pose_target), cudaMemcpyHostToDevice, c->stream));
    if (n) {
        R3_CUDA(c, cudaMemcpyAsync(a->d_obj_items, items.data(), (size_t)n * sizeof(uint2), cudaMemcpyHostToDevice, c->stream));
        R3_CUDA(c, cudaMemcpyAsync(a->d_obj_slots, slots.data(), (size_t)n * 4, cudaMemcpyHostToDevice, c->stream));
    }
    R3_CUDA(c, r3_stream_sync(c));                                    // host pointers are only borrowed for the call
    a->n_obj_items = n;
    a->obj_slots.swap(slots);
    a->has_obj_jobs = true;
    return R3_OK;
}

R3_EXPORT int r3_pose_objects(r3_ctx* c) {
    if (!c) return R3_E_INVALID;
    r3_anim_state* a = c->anim;
    if (!a || !a->has_obj_jobs) return r3_fail(c, R3_E_STATE, "pose_objects before set_object_animations + set_object_pose_jobs");
    R3_TRY(r3_check_object_writer(c, "pose_objects", R3_NEED_OBJECTS | R3_NEED_OWNED));
    if (a->n_obj_items == 0) return R3_OK;
    cudaSetDevice(c->device);
    const uint32_t n = a->n_obj_items, sort_n = r3_sort_extent(c);
    pose_objects_kernel<<<(n + R3_OBJ_POSE_THREADS - 1) / R3_OBJ_POSE_THREADS, R3_OBJ_POSE_THREADS, 0, c->stream>>>(
        a->d_obj_items, n, a->d_obj_jobs, a->d_obj_targets, a->d_node_clips, a->d_node_channels, a->d_nodes, a->d_obj_keys, a->left_handed,
        reinterpret_cast<float4*>(c->d_objects), c->n_slots, c->d_sort_loc, sort_n);
    R3_CHECK_LAUNCH(c, "pose_objects_kernel");
    R3_TRY(r3_split_slots(c, a->d_obj_slots, n));                     // rows_xyz / rows_w / spheres and the affine bit of the posed slots
    r3_new_frame_epoch(c);                                            // a frame-wide sort made before the pose is stale
    a->locations_pending = true;
    return R3_OK;
}

R3_EXPORT int r3_readback_objects(r3_ctx* c, r3_object* out, float* locations, uint32_t first, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (!out && n) return r3_fail(c, R3_E_INVALID, "readback_objects: null");
    if ((uint64_t)first + n > c->n_slots) return r3_fail(c, R3_E_INVALID, "readback_objects: range outside the object buffer");
    if (locations && (uint64_t)first + n > r3_sort_extent(c))
        return r3_fail(c, R3_E_INVALID, "readback_objects: range outside the sort info");
    if (n == 0) return R3_OK;
    cudaSetDevice(c->device);
    R3_CUDA(c, r3_stream_sync(c));
    R3_CUDA(c, cudaMemcpy(out, c->d_objects + first, (size_t)n * sizeof(r3_object), cudaMemcpyDeviceToHost));
    if (locations) R3_CUDA(c, cudaMemcpy(locations, c->d_sort_loc + 3 * (size_t)first, (size_t)n * 12, cudaMemcpyDeviceToHost));
    return R3_OK;
}
