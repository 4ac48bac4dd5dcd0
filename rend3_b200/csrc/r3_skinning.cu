// r3_skinning.cu — GPU skinning: 4-joint linear blend of position / normal / tangent into the mesh megabuffer.
//
// Replaces GpuSkinner::execute_pass + skinning.wgsl::main (rend3-routine/src/skinning.rs:54-199,
// rend3-routine/shaders/src/skinning.wgsl:37-94).  The reference issues one dispatch per skeleton; here one launch
// covers every skeleton: a CTA handles 256 vertices of one skeleton (found through a prefix table of 256-vertex
// chunks), joint matrices are read through the read-only path (they are shared by all vertices of a skeleton).
// The skinned positions feed the bit-exact cull / raster stages, so the arithmetic is IEEE f32 in WGSL source order
// without FMA contraction (same rule as the bake kernel); normalize = v / sqrt(dot(v, v)).
#include <vector>

#include "r3_common.cuh"

namespace {

__device__ __forceinline__ float3 load3(const uint32_t* __restrict__ mesh, uint64_t words, uint32_t byte_off, uint32_t idx) {
    const uint64_t f = (uint64_t)(byte_off >> 2) + (uint64_t)idx * 3u;
    if (f + 2 >= words) return make_float3(0.f, 0.f, 0.f);
    return make_float3(__uint_as_float(mesh[f]), __uint_as_float(mesh[f + 1]), __uint_as_float(mesh[f + 2]));
}
__device__ __forceinline__ void store3(uint32_t* __restrict__ mesh, uint64_t words, uint32_t byte_off, uint32_t idx, float3 v) {
    const uint64_t f = (uint64_t)(byte_off >> 2) + (uint64_t)idx * 3u;
    if (f + 2 >= words) return;   // out-of-range stores are dropped (robust buffer access)
    mesh[f] = __float_as_uint(v.x); mesh[f + 1] = __float_as_uint(v.y); mesh[f + 2] = __float_as_uint(v.z);
}
__device__ __forceinline__ float dot3_rn(float3 a, float3 b) { return add_rn(add_rn(mul_rn(a.x, b.x), mul_rn(a.y, b.y)), mul_rn(a.z, b.z)); }
// mat3 * v with WGSL's column accumulation
__device__ __forceinline__ float3 mat3_vec_rn(const float* __restrict__ m, float3 v) {
    return make_float3(add_rn(add_rn(mul_rn(m[0], v.x), mul_rn(m[4], v.y)), mul_rn(m[8], v.z)), add_rn(add_rn(mul_rn(m[1], v.x), mul_rn(m[5], v.y)), mul_rn(m[9], v.z)),
                       add_rn(add_rn(mul_rn(m[2], v.x), mul_rn(m[6], v.y)), mul_rn(m[10], v.z)));
}
__device__ __forceinline__ float3 normalize_rn(float3 v) {
    const float l = __fsqrt_rn(dot3_rn(v, v));
    return make_float3(div_rn(v.x, l), div_rn(v.y, l), div_rn(v.z, l));
}

__global__ void __launch_bounds__(256) skinning_kernel(uint32_t* __restrict__ mesh, uint64_t mesh_words, const r3_skinning_input* __restrict__ inputs,
                                                       const uint32_t* __restrict__ chunk_prefix, uint32_t n_skeletons, const float* __restrict__ joints,
                                                       uint32_t n_joints) {
    // skeleton of this CTA: last s with chunk_prefix[s] <= blockIdx.x
    uint32_t lo = 0, hi = n_skeletons;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (chunk_prefix[mid] <= blockIdx.x) lo = mid; else hi = mid;
    }
    const r3_skinning_input in = inputs[lo];
    const uint32_t idx = (blockIdx.x - chunk_prefix[lo]) * 256u + threadIdx.x;
    if (idx >= in.vertex_count) return;

    // extract_attribute_vec4_u16 / vec4_f32 (rend3/shaders/vertex_attributes.wgsl:68-85)
    const uint64_t ji = (uint64_t)(in.joint_indices_offset >> 2) + (uint64_t)idx * 2u, jw = (uint64_t)(in.joint_weight_offset >> 2) + (uint64_t)idx * 4u;
    const uint32_t v0 = ji + 1 < mesh_words ? mesh[ji] : 0u, v1 = ji + 1 < mesh_words ? mesh[ji + 1] : 0u;
    const uint32_t joint_index[4] = {v0 & 0xFFFFu, v0 >> 16, v1 & 0xFFFFu, v1 >> 16};
    float weight[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) weight[k] = jw + 3 < mesh_words ? __uint_as_float(mesh[jw + k]) : 0.0f;

    float3 pos = make_float3(0.f, 0.f, 0.f), normal = pos, tangent = pos;
    if (in.base_position_offset != R3_ATTR_ABSENT) pos = load3(mesh, mesh_words, in.base_position_offset, idx);
    if (in.base_normal_offset != R3_ATTR_ABSENT) normal = load3(mesh, mesh_words, in.base_normal_offset, idx);
    if (in.base_tangent_offset != R3_ATTR_ABSENT) tangent = load3(mesh, mesh_words, in.base_tangent_offset, idx);

    float3 pos_acc = make_float3(0.f, 0.f, 0.f), norm_acc = pos_acc, tang_acc = pos_acc;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float w = weight[i];
        if (w > 0.0f) {                                                             // skinning.wgsl:68
            const uint32_t j = in.joint_matrix_base_offset + joint_index[i];
            float m[16];
#pragma unroll
            for (int k = 0; k < 16; ++k) m[k] = j < n_joints ? __ldg(&joints[(size_t)j * 16 + k]) : 0.0f;
            const float4 tp = mat_point_rn(m, pos.x, pos.y, pos.z);
            pos_acc = make_float3(add_rn(pos_acc.x, mul_rn(tp.x, w)), add_rn(pos_acc.y, mul_rn(tp.y, w)), add_rn(pos_acc.z, mul_rn(tp.z, w)));
            const float3 c0 = make_float3(m[0], m[1], m[2]), c1 = make_float3(m[4], m[5], m[6]), c2 = make_float3(m[8], m[9], m[10]);
            const float3 iss = make_float3(div_rn(1.0f, dot3_rn(c0, c0)), div_rn(1.0f, dot3_rn(c1, c1)), div_rn(1.0f, dot3_rn(c2, c2)));   // math/matrix.wgsl:1-7
            const float3 tn = mat3_vec_rn(m, make_float3(mul_rn(iss.x, normal.x), mul_rn(iss.y, normal.y), mul_rn(iss.z, normal.z)));
            const float3 tt = mat3_vec_rn(m, make_float3(mul_rn(iss.x, tangent.x), mul_rn(iss.y, tangent.y), mul_rn(iss.z, tangent.z)));
            norm_acc = make_float3(add_rn(norm_acc.x, mul_rn(tn.x, w)), add_rn(norm_acc.y, mul_rn(tn.y, w)), add_rn(norm_acc.z, mul_rn(tn.z, w)));
            tang_acc = make_float3(add_rn(tang_acc.x, mul_rn(tt.x, w)), add_rn(tang_acc.y, mul_rn(tt.y, w)), add_rn(tang_acc.z, mul_rn(tt.z, w)));
        }
    }
    norm_acc = normalize_rn(norm_acc);
    tang_acc = normalize_rn(tang_acc);
    if (in.updated_position_offset != R3_ATTR_ABSENT) store3(mesh, mesh_words, in.updated_position_offset, idx, pos_acc);
    if (in.updated_normal_offset != R3_ATTR_ABSENT) store3(mesh, mesh_words, in.updated_normal_offset, idx, norm_acc);
    if (in.updated_tangent_offset != R3_ATTR_ABSENT) store3(mesh, mesh_words, in.updated_tangent_offset, idx, tang_acc);
}

}  // namespace

R3_EXPORT int r3_skin(r3_ctx* c, const r3_skinning_input* inputs, uint32_t n_skeletons, const float* joint_matrices, uint32_t n_joints) {
    if (!c || (!inputs && n_skeletons) || (!joint_matrices && n_joints)) return r3_fail(c, R3_E_INVALID, "skin: null");
    if (n_skeletons == 0) return R3_OK;
    if (!c->d_mesh) return r3_fail(c, R3_E_STATE, "skin before set_mesh_buffer");
    cudaSetDevice(c->device);
    std::vector<uint32_t> prefix(n_skeletons + 1, 0u);
    for (uint32_t s = 0; s < n_skeletons; ++s) prefix[s + 1] = prefix[s] + (inputs[s].vertex_count + 255u) / 256u;
    const uint32_t total_chunks = prefix[n_skeletons];
    if (total_chunks == 0) return R3_OK;
    // staging: inputs | chunk prefix | joint matrices
    const uint64_t b_in = (uint64_t)n_skeletons * sizeof(r3_skinning_input), b_pre = ((uint64_t)n_skeletons + 1) * 4, b_j = (uint64_t)n_joints * 64;
    const uint64_t off_pre = (b_in + 15) & ~15ull, off_j = (off_pre + b_pre + 15) & ~15ull;
    R3_TRY(r3_reserve(c, &c->d_scratch, &c->scratch_cap, off_j + b_j + 64, 1, false, false));
    uint8_t* base = (uint8_t*)c->d_scratch;
    R3_CUDA(c, cudaMemcpyAsync(base, inputs, b_in, cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, cudaMemcpyAsync(base + off_pre, prefix.data(), b_pre, cudaMemcpyHostToDevice, c->stream));
    if (n_joints) R3_CUDA(c, cudaMemcpyAsync(base + off_j, joint_matrices, b_j, cudaMemcpyHostToDevice, c->stream));
    R3_TRY(r3_launch_skinning(c, (const r3_skinning_input*)base, (const uint32_t*)(base + off_pre), n_skeletons, total_chunks, (const float*)(base + off_j), n_joints));
    R3_CUDA(c, r3_stream_sync(c));   // host pointers are only borrowed for the call
    return R3_OK;
}

int r3_launch_skinning(r3_ctx* c, const r3_skinning_input* d_inputs, const uint32_t* d_chunk_prefix, uint32_t n_skeletons, uint32_t total_chunks,
                       const float* d_joints, uint32_t n_joints) {
    if (total_chunks == 0) return R3_OK;
    skinning_kernel<<<total_chunks, 256, 0, c->stream>>>(c->d_mesh, c->mesh_words, d_inputs, d_chunk_prefix, n_skeletons, d_joints, n_joints);
    R3_CHECK_LAUNCH(c, "skinning_kernel");
    return R3_OK;
}

R3_EXPORT int r3_readback_mesh_buffer(r3_ctx* c, void* bytes, uint64_t cap) {
    if (!c || !bytes) return r3_fail(c, R3_E_INVALID, "readback_mesh_buffer: null");
    if (cap < c->mesh_words * 4) return r3_fail(c, R3_E_INVALID, "readback_mesh_buffer: capacity too small");
    cudaSetDevice(c->device);
    if (c->mesh_words) R3_CUDA(c, cudaMemcpyAsync(bytes, c->d_mesh, c->mesh_words * 4, cudaMemcpyDeviceToHost, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    return R3_OK;
}
