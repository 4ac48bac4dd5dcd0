// r3_lights.cu — DirectionalLightManager::evaluate (rend3/src/managers/directional.rs:99-157) on the device: every directional light's
// texel-snapped orthographic shadow camera around the viewer (directional/shadow_camera.rs:6-33), so that a frame whose camera moves needs
// no light upload.  The arithmetic is rule R13 (DESIGN.md §2): one IEEE f32 operation at a time in the order written, never contracted
// (this unit is compiled with -fmad=false and every operation is an explicit _rn intrinsic).
//
//   r3_set_directional_light_sources  blocking: static light fields into the light buffer (through r3_set_directional_lights, which also
//                                     allocates the atlas), the sources into device memory
//   r3_evaluate_shadow_cameras        one thread per light writes the light's view_proj and its camera header (view, view_proj, frustum)
//   r3_shadow_uniform_upload          the cull + bake of Shadow(i) reading that header on the device
//   r3_readback_shadow_cameras        blocking readback of the headers and light records
//   r3_update_directional_light_sources[_device]  DirectionalLightChanges applied to the sources and the light records' static fields
// and PointLightManager's handle table with its evaluate (second half of the file).
#include <algorithm>
#include <cmath>
#include <cstring>

#include "r3_common.cuh"
#include "r3_scan.cuh"

namespace {

struct v3 { float x, y, z; };

__device__ __forceinline__ v3 sub3(v3 a, v3 b) { return {sub_rn(a.x, b.x), sub_rn(a.y, b.y), sub_rn(a.z, b.z)}; }
__device__ __forceinline__ v3 add3(v3 a, v3 b) { return {add_rn(a.x, b.x), add_rn(a.y, b.y), add_rn(a.z, b.z)}; }
// glam's scalar dot: (x x' + y y') + z z'
__device__ __forceinline__ float dot3(v3 a, v3 b) { return add_rn(add_rn(mul_rn(a.x, b.x), mul_rn(a.y, b.y)), mul_rn(a.z, b.z)); }
// glam.py::cross: (a.y b.z - b.y a.z, a.z b.x - b.z a.x, a.x b.y - b.x a.y)
__device__ __forceinline__ v3 cross3(v3 a, v3 b) {
    return {sub_rn(mul_rn(a.y, b.z), mul_rn(b.y, a.z)), sub_rn(mul_rn(a.z, b.x), mul_rn(b.z, a.x)), sub_rn(mul_rn(a.x, b.y), mul_rn(b.x, a.y))};
}
// normalize = v * (1 / sqrt(dot3))
__device__ __forceinline__ v3 normalize3(v3 a) {
    const float r = div_rn(1.0f, __fsqrt_rn(dot3(a, a)));
    return {mul_rn(a.x, r), mul_rn(a.y, r), mul_rn(a.z, r)};
}

// glam.py::look_to_lh into m[16] (column-major)
__device__ void look_to_lh(v3 eye, v3 dir, float* m) {
    const v3 up = {0.0f, 1.0f, 0.0f};
    const v3 f = normalize3(dir);
    const v3 s = normalize3(cross3(up, f));
    const v3 u = cross3(f, s);
    m[0] = s.x; m[1] = u.x; m[2] = f.x; m[3] = 0.0f;
    m[4] = s.y; m[5] = u.y; m[6] = f.y; m[7] = 0.0f;
    m[8] = s.z; m[9] = u.z; m[10] = f.z; m[11] = 0.0f;
    m[12] = -dot3(eye, s); m[13] = -dot3(eye, u); m[14] = -dot3(eye, f); m[15] = 1.0f;
}
// look_at_lh(eye, center) = look_to_lh(eye, center - eye); look_at_rh(eye, center) = look_to_lh(eye, eye - center)
__device__ void look_at(v3 eye, v3 center, bool lh, float* m) { look_to_lh(eye, lh ? sub3(center, eye) : sub3(eye, center), m); }

// transform_point3: ((x_axis px + y_axis py) + z_axis pz) + w_axis
__device__ __forceinline__ v3 transform_point3(const float* m, v3 p) {
    float r[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) r[k] = add_rn(add_rn(add_rn(mul_rn(m[k], p.x), mul_rn(m[4 + k], p.y)), mul_rn(m[8 + k], p.z)), m[12 + k]);
    return {r[0], r[1], r[2]};
}

// Mat4::inverse: the GLM cofactor expansion glam's SSE2 build uses.  m[4 c + r] = column c, row r.  Coefficients a*b - c*d; the
// cofactor columns ((v1 f0 - v2 f1) + v3 f2) times the sign vectors; det = SSE2 dot4 of column 0 with the first cofactor row,
// (d.x + d.z) + (d.y + d.w); every element times (1 / det).
__device__ void inverse4(const float* m, float* out) {
#define M(c, r) m[4 * (c) + (r)]
#define COEF(a, b, c, d) sub_rn(mul_rn(a, b), mul_rn(c, d))
    float fac[6][4];
    const int rr[6][2] = {{2, 3}, {1, 3}, {1, 2}, {0, 3}, {0, 2}, {0, 1}};   // (row i, row j) of Fac0..Fac5
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        const int i = rr[k][0], j = rr[k][1];
        const float c0 = COEF(M(2, i), M(3, j), M(3, i), M(2, j));
        const float c2 = COEF(M(1, i), M(3, j), M(3, i), M(1, j));
        const float c3 = COEF(M(1, i), M(2, j), M(2, i), M(1, j));
        fac[k][0] = c0; fac[k][1] = c0; fac[k][2] = c2; fac[k][3] = c3;
    }
    float vec[4][4];   // vec[r] = (m[1][r], m[0][r], m[0][r], m[0][r])
#pragma unroll
    for (int r = 0; r < 4; ++r) { vec[r][0] = M(1, r); vec[r][1] = M(0, r); vec[r][2] = M(0, r); vec[r][3] = M(0, r); }
    // inv_c = (vec[a] fac[p] - vec[b] fac[q]) + vec[e] fac[t]
    const int terms[4][6] = {{1, 0, 2, 1, 3, 2}, {0, 0, 2, 3, 3, 4}, {0, 1, 1, 3, 3, 5}, {0, 2, 1, 4, 2, 5}};
    const float sign_a[4] = {1.0f, -1.0f, 1.0f, -1.0f}, sign_b[4] = {-1.0f, 1.0f, -1.0f, 1.0f};
    float inv[16];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const int* t = terms[c];
        const float* sg = (c & 1) ? sign_b : sign_a;
#pragma unroll
        for (int k = 0; k < 4; ++k)
            inv[4 * c + k] = mul_rn(add_rn(sub_rn(mul_rn(vec[t[0]][k], fac[t[1]][k]), mul_rn(vec[t[2]][k], fac[t[3]][k])), mul_rn(vec[t[4]][k], fac[t[5]][k])), sg[k]);
    }
    const float d0 = mul_rn(M(0, 0), inv[0]), d1 = mul_rn(M(0, 1), inv[4]), d2 = mul_rn(M(0, 2), inv[8]), d3 = mul_rn(M(0, 3), inv[12]);
    const float rcp = div_rn(1.0f, add_rn(add_rn(d0, d2), add_rn(d1, d3)));
#pragma unroll
    for (int k = 0; k < 16; ++k) out[k] = mul_rn(inv[k], rcp);
#undef COEF
#undef M
}

// one thread per light: R13
__global__ void __launch_bounds__(64) shadow_camera_kernel(const r3_directional_light_source* __restrict__ src, uint32_t n, uint32_t left_handed,
                                                            float lx, float ly, float lz, r3_directional_light* __restrict__ lights,
                                                            r3_camera_header* __restrict__ cams) {
    const uint32_t i = threadIdx.x;
    if (i >= n) return;
    const r3_directional_light_source s = src[i];
    const bool lh = left_handed != 0;
    const v3 dir = {s.direction[0], s.direction[1], s.direction[2]}, zero = {0.0f, 0.0f, 0.0f}, loc = {lx, ly, lz};
    const float texel = div_rn(s.distance, (float)s.resolution);
    float origin_view[16], inv[16], view[16], vp[16];
    look_at(zero, dir, lh, origin_view);
    const v3 cov = transform_point3(origin_view, loc);
    // Rust's f32 % (fmodf): exact, with the sign of the dividend
    const v3 shadow_loc = {sub_rn(cov.x, fmodf(cov.x, texel)), sub_rn(cov.y, fmodf(cov.y, texel)), sub_rn(cov.z, 0.0f)};
    inverse4(origin_view, inv);
    const v3 new_loc = transform_point3(inv, shadow_loc);
    look_at(new_loc, add3(new_loc, dir), lh, view);
    // orthographic_{lh,rh}(-h, h, -h, h, h, -h), h = distance * 0.5 (camera.rs:90-96)
    const float half = mul_rn(s.distance, 0.5f), left = -half, right = half, bottom = -half, top = half, near = half, far = -half;
    const float rcp_w = div_rn(1.0f, sub_rn(right, left)), rcp_h = div_rn(1.0f, sub_rn(top, bottom));
    const float r = div_rn(1.0f, lh ? sub_rn(far, near) : sub_rn(near, far));
    float proj[16] = {add_rn(rcp_w, rcp_w), 0.0f, 0.0f, 0.0f, 0.0f, add_rn(rcp_h, rcp_h), 0.0f, 0.0f, 0.0f, 0.0f, r, 0.0f,
                      mul_rn(-add_rn(left, right), rcp_w), mul_rn(-add_rn(top, bottom), rcp_h), lh ? mul_rn(-r, near) : mul_rn(r, near), 1.0f};
    // view_proj = proj * view: column j = ((p0 v.x + p1 v.y) + p2 v.z) + p3 v.w
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float4 col = mat_vec_rn(proj, view[4 * j], view[4 * j + 1], view[4 * j + 2], view[4 * j + 3]);
        vp[4 * j] = col.x; vp[4 * j + 1] = col.y; vp[4 * j + 2] = col.z; vp[4 * j + 3] = col.w;
    }
    r3_camera_header h;
    memset(&h, 0, sizeof h);
#pragma unroll
    for (int k = 0; k < 16; ++k) { h.view[k] = view[k]; h.view_proj[k] = vp[k]; lights[i].view_proj[k] = vp[k]; }
    // Frustum::from_matrix (util/frustum.rs:96-145): left = r3 + r0, right = r3 - r0, top = r3 - r1, bottom = r3 + r1, near = r3 - r2,
    // each divided by |abc|
    const int row[5] = {0, 0, 1, 1, 2};
    const bool plus[5] = {true, false, false, true, false};
#pragma unroll
    for (int pl = 0; pl < 5; ++pl) {
        float q[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) q[c] = plus[pl] ? add_rn(vp[4 * c + 3], vp[4 * c + row[pl]]) : sub_rn(vp[4 * c + 3], vp[4 * c + row[pl]]);
        const float mag = __fsqrt_rn(dot3({q[0], q[1], q[2]}, {q[0], q[1], q[2]}));
#pragma unroll
        for (int c = 0; c < 4; ++c) h.frustum[pl][c] = div_rn(q[c], mag);
    }
    h.shadow_index = i;
    h.resolution[0] = (float)s.size; h.resolution[1] = (float)s.size;
    h.flags = lh ? R3_PCU_POSITIVE_AREA_VISIBLE : 0u;   // TriangleVisibility::from_winding_and_face: Cw (Left) + Front culled
    cams[i] = h;
}

// ---- DirectionalLightManager::update (directional.rs:91-93): update_from_changes of the masked fields
constexpr uint32_t DIR_CHANGE_BITS = R3_DIR_CHANGE_COLOR | R3_DIR_CHANGE_INTENSITY | R3_DIR_CHANGE_DIRECTION | R3_DIR_CHANGE_DISTANCE;
constexpr uint32_t DIR_CHANGE_BATCH = 64;   // entries per launch of the host form: 3 KB of kernel parameters, under the 4 KB limit

// the host mirror and the kernel apply an entry through this one function
__host__ __device__ __forceinline__ void apply_directional_change(r3_directional_light_source& s, const r3_directional_light_change& e) {
    const uint32_t m = e.mask;
    if (m & R3_DIR_CHANGE_COLOR) { s.color[0] = e.color[0]; s.color[1] = e.color[1]; s.color[2] = e.color[2]; }
    if (m & R3_DIR_CHANGE_INTENSITY) s.intensity = e.intensity;
    if (m & R3_DIR_CHANGE_DIRECTION) { s.direction[0] = e.direction[0]; s.direction[1] = e.direction[1]; s.direction[2] = e.direction[2]; }
    if (m & R3_DIR_CHANGE_DISTANCE) s.distance = e.distance;
}

// where the entries come from: a batch passed by value as kernel parameters (host form) or an array in device memory (device form)
struct DirChangeParams {
    r3_directional_light_change e[DIR_CHANGE_BATCH];
    __device__ const r3_directional_light_change& operator[](uint32_t k) const { return e[k]; }
};
struct DirChangeDevice {
    const r3_directional_light_change* p;
    __device__ const r3_directional_light_change& operator[](uint32_t k) const { return p[k]; }
};

// thread i owns light i and walks the entries in array order, so a later entry's fields override an earlier one's.  An entry naming
// no light of the set or carrying an unknown bit is dropped whole (the host form has rejected those already).  A light that some
// non-empty mask touched gets its source and the light record's static fields rewritten: colour * intensity with the single multiply of
// r3_set_directional_light_sources, direction copied.  view_proj and the camera header are the next r3_evaluate_shadow_cameras'.
template <class Changes>
__global__ void __launch_bounds__(64) directional_light_change_kernel(const __grid_constant__ Changes changes, uint32_t n, uint32_t n_lights,
                                                                      r3_directional_light_source* __restrict__ src,
                                                                      r3_directional_light* __restrict__ lights) {
    const uint32_t i = threadIdx.x;
    if (i >= n_lights) return;
    r3_directional_light_source s = src[i];
    bool changed = false;
    for (uint32_t k = 0; k < n; ++k) {
        const r3_directional_light_change& e = changes[k];
        if (e.index != i || (e.mask & ~DIR_CHANGE_BITS)) continue;
        apply_directional_change(s, e);
        changed |= e.mask != 0;
    }
    if (!changed) return;
    src[i] = s;
#pragma unroll
    for (int k = 0; k < 3; ++k) { lights[i].color[k] = __fmul_rn(s.color[k], s.intensity); lights[i].direction[k] = s.direction[k]; }
}

template <class Changes>
int launch_directional_light_change(r3_ctx* c, const Changes& changes, uint32_t n) {
    static_assert(R3_MAX_SHADOWS <= 64, "one thread per light");
    directional_light_change_kernel<Changes><<<1, 64, 0, c->stream>>>(changes, n, (uint32_t)c->light_src.size(), c->d_light_src, c->d_dir);
    R3_CHECK_LAUNCH(c, "directional_light_change_kernel");
    return R3_OK;
}

}  // namespace

R3_EXPORT int r3_set_directional_light_sources(r3_ctx* c, const r3_directional_light_source* lights, uint32_t n, uint32_t aw, uint32_t ah,
                                               uint32_t left_handed) {
    if (!c) return R3_E_INVALID;
    if (!lights && n) return r3_fail(c, R3_E_INVALID, "set_directional_light_sources: null lights");
    if (n > R3_MAX_SHADOWS) return r3_fail(c, R3_E_INVALID, "set_directional_light_sources: more lights than R3_MAX_SHADOWS");
    for (uint32_t i = 0; i < n; ++i) {
        const r3_directional_light_source& s = lights[i];
        if (s.size == 0 || (uint64_t)s.offset[0] + s.size > aw || (uint64_t)s.offset[1] + s.size > ah)
            return r3_fail(c, R3_E_INVALID, "set_directional_light_sources: empty map or placement outside the atlas");
    }
    cudaSetDevice(c->device);
    if (!c->d_light_src) R3_CUDA(c, cudaMalloc((void**)&c->d_light_src, R3_MAX_SHADOWS * sizeof(r3_directional_light_source)));
    if (!c->d_shadow_cams) R3_CUDA(c, cudaMalloc((void**)&c->d_shadow_cams, R3_MAX_SHADOWS * sizeof(r3_camera_header)));
    // the static fields as directional.rs:135-156 writes them; view_proj stays 0 until the first evaluation
    std::vector<uint8_t> bytes(16 + (size_t)n * sizeof(r3_directional_light), 0);
    *reinterpret_cast<uint32_t*>(bytes.data()) = n;
    r3_directional_light* dl = reinterpret_cast<r3_directional_light*>(bytes.data() + 16);
    const float w = (float)aw, h = (float)ah;
    for (uint32_t i = 0; i < n; ++i) {
        const r3_directional_light_source& s = lights[i];
        for (int k = 0; k < 3; ++k) { dl[i].color[k] = s.color[k] * s.intensity; dl[i].direction[k] = s.direction[k]; }
        dl[i].inv_resolution[0] = 1.0f / w; dl[i].inv_resolution[1] = 1.0f / h;
        dl[i].atlas_offset[0] = (float)s.offset[0] / w; dl[i].atlas_offset[1] = (float)s.offset[1] / h;
        dl[i].atlas_size[0] = (float)s.size / w; dl[i].atlas_size[1] = (float)s.size / h;
    }
    if (n) R3_CUDA(c, cudaMemcpyAsync(c->d_light_src, lights, (size_t)n * sizeof(r3_directional_light_source), cudaMemcpyHostToDevice, c->stream));
    R3_TRY(r3_set_directional_lights(c, bytes.data(), bytes.size(), aw, ah));   // drains the stream: `lights` is only borrowed
    c->light_src.assign(lights, lights + n);
    c->light_src_left_handed = left_handed ? 1u : 0u;
    c->light_src_set = true;
    c->shadow_cams_evaluated = false;
    c->dir_eval_pending = false;
    return R3_OK;
}

R3_EXPORT int r3_update_directional_light_sources(r3_ctx* c, const r3_directional_light_change* changes, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (!c->light_src_set) return r3_fail(c, R3_E_STATE, "update_directional_light_sources before set_directional_light_sources");
    if (!changes && n) return r3_fail(c, R3_E_INVALID, "update_directional_light_sources: null changes");
    for (uint32_t k = 0; k < n; ++k) {
        if (changes[k].index >= c->light_src.size()) return r3_fail(c, R3_E_INVALID, "update_directional_light_sources: no such light");
        if (changes[k].mask & ~DIR_CHANGE_BITS) return r3_fail(c, R3_E_INVALID, "update_directional_light_sources: unknown mask bit");
    }
    if (n == 0) return R3_OK;
    cudaSetDevice(c->device);
    // the entries travel by value: nothing is copied to the device and nothing waits, so `changes` is free on return
    for (uint32_t first = 0; first < n; first += DIR_CHANGE_BATCH) {
        DirChangeParams batch;
        memset(&batch, 0, sizeof batch);
        const uint32_t m = std::min(n - first, DIR_CHANGE_BATCH);
        memcpy(batch.e, changes + first, (size_t)m * sizeof *changes);
        R3_TRY(launch_directional_light_change(c, batch, m));
    }
    for (uint32_t k = 0; k < n; ++k) apply_directional_change(c->light_src[changes[k].index], changes[k]);
    c->dir_eval_pending = true;
    return R3_OK;
}

R3_EXPORT int r3_update_directional_light_sources_device(r3_ctx* c, const r3_directional_light_change* d_changes, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (!c->light_src_set) return r3_fail(c, R3_E_STATE, "update_directional_light_sources_device before set_directional_light_sources");
    if (n == 0) return R3_OK;
    if (!d_changes) return r3_fail(c, R3_E_INVALID, "update_directional_light_sources_device: null changes");
    cudaSetDevice(c->device);
    R3_TRY(launch_directional_light_change(c, DirChangeDevice{d_changes}, n));
    c->dir_eval_pending = true;
    return R3_OK;
}

R3_EXPORT int r3_evaluate_shadow_cameras(r3_ctx* c, const float loc[3]) {
    if (!c) return R3_E_INVALID;
    if (!loc) return r3_fail(c, R3_E_INVALID, "evaluate_shadow_cameras: null location");
    if (!c->light_src_set) return r3_fail(c, R3_E_STATE, "evaluate_shadow_cameras before set_directional_light_sources");
    cudaSetDevice(c->device);
    const uint32_t n = (uint32_t)c->light_src.size();
    if (n) {
        shadow_camera_kernel<<<1, 64, 0, c->stream>>>(c->d_light_src, n, c->light_src_left_handed, loc[0], loc[1], loc[2], c->d_dir, c->d_shadow_cams);
        R3_CHECK_LAUNCH(c, "shadow_camera_kernel");
    }
    c->shadow_cams_evaluated = true;
    c->dir_eval_pending = false;
    return R3_OK;
}

R3_EXPORT int r3_shadow_uniform_upload(r3_ctx* c, uint32_t shadow_index, uint32_t object_count, uint32_t mode) {
    if (!c) return R3_E_INVALID;
    if (!c->light_src_set || !c->shadow_cams_evaluated) return r3_fail(c, R3_E_STATE, "shadow_uniform_upload before set_directional_light_sources + evaluate_shadow_cameras");
    if (c->dir_eval_pending) return r3_fail(c, R3_E_STATE, "shadow_uniform_upload: directional lights updated since the last evaluate_shadow_cameras");
    if (shadow_index >= c->light_src.size()) return r3_fail(c, R3_E_INVALID, "shadow_uniform_upload: no such light");
    if (object_count > c->n_slots) return r3_fail(c, R3_E_INVALID, "object_count exceeds the object buffer");
    cudaSetDevice(c->device);
    r3_camera* cam = &c->cams[r3_cam_slot(shadow_index)];
    // the fields the host knows; view, view_proj and frustum stay on the device (the triangle cull reads none of them)
    r3_camera_header h;
    memset(&h, 0, sizeof h);
    const float size = (float)c->light_src[shadow_index].size;
    h.shadow_index = shadow_index;
    h.resolution[0] = size; h.resolution[1] = size;
    h.flags = c->light_src_left_handed ? R3_PCU_POSITIVE_AREA_VISIBLE : 0u;
    h.object_count = object_count;
    cam->header = h;
    cam->header_set = true;
    R3_TRY(r3_camera_buffers(c, cam, mode));
    return r3_launch_cull_bake_device_camera(c, cam, mode, c->d_shadow_cams + shadow_index);
}

R3_EXPORT int r3_readback_shadow_cameras(r3_ctx* c, r3_camera_header* out, r3_directional_light* lights, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (!out && n) return r3_fail(c, R3_E_INVALID, "readback_shadow_cameras: null");
    if (!c->light_src_set || !c->shadow_cams_evaluated) return r3_fail(c, R3_E_STATE, "readback_shadow_cameras before evaluate_shadow_cameras");
    if (c->dir_eval_pending) return r3_fail(c, R3_E_STATE, "readback_shadow_cameras: directional lights updated since the last evaluate_shadow_cameras");
    if (n > c->light_src.size()) return r3_fail(c, R3_E_INVALID, "readback_shadow_cameras: more cameras than lights");
    cudaSetDevice(c->device);
    if (n) R3_CUDA(c, cudaMemcpyAsync(out, c->d_shadow_cams, (size_t)n * sizeof *out, cudaMemcpyDeviceToHost, c->stream));
    if (n && lights) R3_CUDA(c, cudaMemcpyAsync(lights, c->d_dir, (size_t)n * sizeof *lights, cudaMemcpyDeviceToHost, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    return R3_OK;
}

// ------------------------------------------------------------------ point lights
// PointLightManager (rend3/src/managers/point.rs) on the device: the handle table `data: Vec<Option<PointLight>>` as sources + live
// bytes, add / update / remove as one scatter kernel (from host or device memory) and evaluate (point.rs:58-74) as one CTA that compacts
// the live handles in ascending order into ShaderPointLightBuffer — rule R14 (DESIGN.md §2): position (x, y, z, 1), colour = three
// __fmul_rn(c, intensity), radius copied; nothing is clamped, so NaN, inf, negative and zero values reach the shading unchanged.
namespace {

constexpr int POINT_EVAL_THREADS = 256;

// one thread per listed handle; out-of-range handles are dropped (the device form cannot grow the table)
__global__ void point_light_scatter_kernel(const uint32_t* __restrict__ handles, const r3_point_light_source* __restrict__ lights,
                                           const uint8_t* __restrict__ live, uint32_t n, uint32_t n_handles,
                                           r3_point_light_source* __restrict__ table, uint8_t* __restrict__ table_live) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t h = handles[i];
    if (h >= n_handles) return;
    const uint8_t l = live ? (live[i] != 0 ? 1 : 0) : 1;
    if (l) table[h] = lights[i];   // a removed handle keeps its record: evaluate skips it, the next add overwrites it
    table_live[h] = l;
}

// data.iter().flatten() in handle order: one CTA walks the table a block at a time, the running count carried across the chunks
__global__ void __launch_bounds__(POINT_EVAL_THREADS) point_light_evaluate_kernel(const r3_point_light_source* __restrict__ table,
                                                                                   const uint8_t* __restrict__ table_live, uint32_t n_handles,
                                                                                   uint8_t* __restrict__ out) {
    __shared__ uint32_t s_warp[POINT_EVAL_THREADS / 32 + 1];
    float4* dst = reinterpret_cast<float4*>(out + 16);
    const uint32_t count = block_scan_excl_chunked<POINT_EVAL_THREADS, uint32_t>(
        n_handles, s_warp, [&](uint32_t h) { return table_live[h] ? 1u : 0u; },
        [&](uint32_t h, uint32_t pos) {
            if (!table_live[h]) return;
            const r3_point_light_source s = table[h];
            dst[2 * (size_t)pos] = make_float4(s.position[0], s.position[1], s.position[2], 1.0f);
            dst[2 * (size_t)pos + 1] = make_float4(__fmul_rn(s.color[0], s.intensity), __fmul_rn(s.color[1], s.intensity),
                                                   __fmul_rn(s.color[2], s.intensity), s.radius);
        });
    if (threadIdx.x == 0) *reinterpret_cast<uint4*>(out) = make_uint4(count, 0u, 0u, 0u);
}

// the table's device arrays hold at least n handles, contents kept; the handles in [c->point_handles, n) start dead
int grow_point_table(r3_ctx* c, uint32_t n) {
    if (n <= c->point_handles) return R3_OK;
    R3_TRY(r3_reserve_t(c, &c->d_point_src, &c->point_src_cap, n, true));
    R3_TRY(r3_reserve_t(c, &c->d_point_live, &c->point_live_cap, n, true));
    R3_TRY(r3_reserve_point_buffer(c, n));
    R3_CUDA(c, cudaMemsetAsync(c->d_point_live + c->point_handles, 0, n - c->point_handles, c->stream));
    return R3_OK;
}

int launch_point_scatter(r3_ctx* c, const uint32_t* handles, const r3_point_light_source* lights, const uint8_t* live, uint32_t n) {
    point_light_scatter_kernel<<<(n + 255) / 256, 256, 0, c->stream>>>(handles, lights, live, n, c->point_handles, c->d_point_src, c->d_point_live);
    R3_CHECK_LAUNCH(c, "point_light_scatter_kernel");
    return R3_OK;
}

}  // namespace

int r3_reserve_point_buffer(r3_ctx* c, uint32_t n_lights) {
    uint64_t cap = c->point_bytes_cap;
    void* p = c->d_point;
    const int rc = r3_reserve(c, &p, &cap, 16 + (uint64_t)n_lights * sizeof(r3_point_light), 1, true, false);
    c->d_point = (uint8_t*)p; c->point_bytes_cap = cap;
    return rc;
}

R3_EXPORT int r3_set_point_light_sources(r3_ctx* c, const r3_point_light_source* lights, const uint8_t* live, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (!lights && n) return r3_fail(c, R3_E_INVALID, "set_point_light_sources: null lights");
    cudaSetDevice(c->device);
    R3_TRY(r3_reserve_t(c, &c->d_point_src, &c->point_src_cap, n, true));   // kept: a failed allocation leaves the old table
    R3_TRY(r3_reserve_t(c, &c->d_point_live, &c->point_live_cap, n, true));
    R3_TRY(r3_reserve_point_buffer(c, n));
    if (n) {
        R3_CUDA(c, cudaMemcpyAsync(c->d_point_src, lights, (size_t)n * sizeof *lights, cudaMemcpyHostToDevice, c->stream));
        if (live) R3_CUDA(c, cudaMemcpyAsync(c->d_point_live, live, n, cudaMemcpyHostToDevice, c->stream));
        else R3_CUDA(c, cudaMemsetAsync(c->d_point_live, 1, n, c->stream));
    }
    R3_CUDA(c, r3_stream_sync(c));   // `lights` and `live` are only borrowed
    c->point_handles = n;
    c->point_capacity = n;
    c->point_eval_pending = true;
    return R3_OK;
}

R3_EXPORT int r3_update_point_light_sources(r3_ctx* c, const uint32_t* handles, const r3_point_light_source* lights, const uint8_t* live, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (!handles || !lights || !live) return r3_fail(c, R3_E_INVALID, "update_point_light_sources: null");
    if (n == 0) return R3_OK;
    std::vector<uint32_t> sorted(handles, handles + n);
    std::sort(sorted.begin(), sorted.end());
    for (uint32_t i = 1; i < n; ++i)
        if (sorted[i] == sorted[i - 1]) return r3_fail(c, R3_E_INVALID, "update_point_light_sources: a handle is named twice");
    if (sorted.back() == 0xFFFFFFFFu) return r3_fail(c, R3_E_INVALID, "update_point_light_sources: handle 0xFFFFFFFF (the table size would not fit 32 bits)");
    cudaSetDevice(c->device);
    const uint32_t size = std::max(c->point_handles, sorted.back() + 1u);
    R3_TRY(grow_point_table(c, size));
    const size_t bytes = (size_t)n * (sizeof(r3_point_light_source) + 4 + 1);
    R3_TRY(r3_reserve(c, &c->d_scratch, &c->scratch_cap, bytes, 1, false, false));
    r3_point_light_source* d_lights = (r3_point_light_source*)c->d_scratch;
    uint32_t* d_handles = (uint32_t*)(d_lights + n);
    uint8_t* d_live = (uint8_t*)(d_handles + n);
    R3_CUDA(c, cudaMemcpyAsync(d_lights, lights, (size_t)n * sizeof *lights, cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, cudaMemcpyAsync(d_handles, handles, (size_t)n * 4, cudaMemcpyHostToDevice, c->stream));
    R3_CUDA(c, cudaMemcpyAsync(d_live, live, n, cudaMemcpyHostToDevice, c->stream));
    c->point_handles = size;
    c->point_capacity = size;
    R3_TRY(launch_point_scatter(c, d_handles, d_lights, d_live, n));
    R3_CUDA(c, r3_stream_sync(c));
    c->point_eval_pending = true;
    return R3_OK;
}

R3_EXPORT int r3_update_point_light_sources_device(r3_ctx* c, const uint32_t* d_handles, const r3_point_light_source* d_lights, const uint8_t* d_live, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (n == 0) return R3_OK;
    if (!d_handles || !d_lights) return r3_fail(c, R3_E_INVALID, "update_point_light_sources_device: null");
    cudaSetDevice(c->device);
    R3_TRY(launch_point_scatter(c, d_handles, d_lights, d_live, n));
    c->point_eval_pending = true;
    return R3_OK;
}

R3_EXPORT int r3_evaluate_point_lights(r3_ctx* c) {
    if (!c) return R3_E_INVALID;
    cudaSetDevice(c->device);
    point_light_evaluate_kernel<<<1, POINT_EVAL_THREADS, 0, c->stream>>>(c->d_point_src, c->d_point_live, c->point_handles, c->d_point);
    R3_CHECK_LAUNCH(c, "point_light_evaluate_kernel");
    c->point_capacity = c->point_handles;
    c->point_eval_pending = false;
    return R3_OK;
}

R3_EXPORT int r3_readback_point_lights(r3_ctx* c, void* bytes, uint64_t capacity) {
    if (!c) return R3_E_INVALID;
    if (!bytes || capacity < 16) return r3_fail(c, R3_E_INVALID, "readback_point_lights: room for the 16-byte header needed");
    cudaSetDevice(c->device);
    R3_CUDA(c, cudaMemcpyAsync(bytes, c->d_point, 16, cudaMemcpyDeviceToHost, c->stream));
    R3_CUDA(c, r3_stream_sync(c));
    const uint64_t held = (c->point_bytes_cap - 16) / sizeof(r3_point_light);
    const uint64_t count = std::min<uint64_t>(*(const uint32_t*)bytes, held);
    const uint64_t n = std::min<uint64_t>(count * sizeof(r3_point_light), capacity - 16);
    if (n) {
        R3_CUDA(c, cudaMemcpyAsync((uint8_t*)bytes + 16, c->d_point + 16, n, cudaMemcpyDeviceToHost, c->stream));
        R3_CUDA(c, r3_stream_sync(c));
    }
    return R3_OK;
}
