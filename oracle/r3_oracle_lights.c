/* r3_oracle_lights.c — CPU ORACLE of the device-evaluated shadow cameras (test infrastructure; never linked into the product).
 *
 * Plain-C restatement of DirectionalLightManager::evaluate (rend3/src/managers/directional.rs:99-157) and of the shadow camera
 * (directional/shadow_camera.rs:6-33) with the arithmetic of rule R13 (DESIGN.md §2): strict IEEE f32, one operation at a time in source
 * order, no contraction (-ffp-contract=off).  It exports the r3o_ twins of r3_set_directional_light_sources, r3_evaluate_shadow_cameras,
 * r3_shadow_uniform_upload and r3_readback_shadow_cameras with the same argument checks; they drive the base oracle through
 * r3o_set_directional_lights and r3o_object_uniform_upload.
 *
 * Its state lives in a table keyed by the context.  r3o_lights_release drops it (before the context is destroyed) and r3o_lights_forget
 * marks the sources unset; oracle/lights.py calls the latter before every r3o_set_directional_lights, which replaces the sources.
 */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../include/rend3_b200.h"
#include "r3_oracle.h"

#define API __attribute__((visibility("default")))

int r3o_set_directional_lights(r3o_ctx* c, const void* bytes, uint64_t nbytes, uint32_t aw, uint32_t ah);
int r3o_object_uniform_upload(r3o_ctx* c, uint32_t camera, const r3_camera_header* h, uint32_t mode);

typedef struct lights_state {
    const r3o_ctx* ctx;
    struct lights_state* next;
    int set, evaluated;
    uint32_t n, left_handed;
    r3_directional_light_source src[R3_MAX_SHADOWS];
    r3_camera_header cams[R3_MAX_SHADOWS];
} lights_state;

static lights_state* g_states;
static pthread_mutex_t g_lights_lock = PTHREAD_MUTEX_INITIALIZER;

static int fail(r3o_ctx* c, int code, const char* msg) {
    if (c) snprintf(c->err, sizeof c->err, "%s", msg);
    return code;
}

static lights_state* find(const r3o_ctx* c, int create) {
    pthread_mutex_lock(&g_lights_lock);
    lights_state* s = g_states;
    while (s && s->ctx != c) s = s->next;
    if (!s && create) {
        s = (lights_state*)calloc(1, sizeof *s);
        if (s) { s->ctx = c; s->next = g_states; g_states = s; }
    }
    pthread_mutex_unlock(&g_lights_lock);
    return s;
}

API void r3o_lights_release(const r3o_ctx* c) {
    pthread_mutex_lock(&g_lights_lock);
    lights_state** p = &g_states;
    while (*p && (*p)->ctx != c) p = &(*p)->next;
    lights_state* s = *p;
    if (s) *p = s->next;
    pthread_mutex_unlock(&g_lights_lock);
    free(s);
}
API void r3o_lights_forget(const r3o_ctx* c) {
    lights_state* s = find(c, 0);
    if (s) { s->set = 0; s->evaluated = 0; }
}

/* ------------------------------------------------------------------ R13, one f32 operation per statement */
typedef struct { float x, y, z; } f3;

static float dot3(f3 a, f3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
static f3 cross3(f3 a, f3 b) { f3 r = {a.y * b.z - b.y * a.z, a.z * b.x - b.z * a.x, a.x * b.y - b.x * a.y}; return r; }
static f3 normalize3(f3 a) {
    const float r = 1.0f / sqrtf(dot3(a, a));
    f3 o = {a.x * r, a.y * r, a.z * r};
    return o;
}
/* glam.py::look_to_lh, up = Y; m[4 c + r] */
static void look_to_lh(f3 eye, f3 dir, float* m) {
    const f3 up = {0.0f, 1.0f, 0.0f};
    const f3 f = normalize3(dir);
    const f3 s = normalize3(cross3(up, f));
    const f3 u = cross3(f, s);
    const float c[16] = {s.x, u.x, f.x, 0.0f, s.y, u.y, f.y, 0.0f, s.z, u.z, f.z, 0.0f, -dot3(eye, s), -dot3(eye, u), -dot3(eye, f), 1.0f};
    memcpy(m, c, sizeof c);
}
static void look_at(f3 eye, f3 center, int lh, float* m) {
    f3 d;
    if (lh) { d.x = center.x - eye.x; d.y = center.y - eye.y; d.z = center.z - eye.z; }
    else { d.x = eye.x - center.x; d.y = eye.y - center.y; d.z = eye.z - center.z; }
    look_to_lh(eye, d, m);
}
static f3 transform_point3(const float* m, f3 p) {
    f3 r;
    r.x = ((m[0] * p.x + m[4] * p.y) + m[8] * p.z) + m[12];
    r.y = ((m[1] * p.x + m[5] * p.y) + m[9] * p.z) + m[13];
    r.z = ((m[2] * p.x + m[6] * p.y) + m[10] * p.z) + m[14];
    return r;
}
/* glam's SSE2 Mat4::inverse (GLM cofactor expansion), written out element by element */
static void inverse4(const float* m, float* out) {
#define M(c, r) m[4 * (c) + (r)]
    float fac[6][4];
    static const int rows[6][2] = {{2, 3}, {1, 3}, {1, 2}, {0, 3}, {0, 2}, {0, 1}};
    for (int k = 0; k < 6; ++k) {
        const int i = rows[k][0], j = rows[k][1];
        const float c0 = M(2, i) * M(3, j) - M(3, i) * M(2, j);
        const float c2 = M(1, i) * M(3, j) - M(3, i) * M(1, j);
        const float c3 = M(1, i) * M(2, j) - M(2, i) * M(1, j);
        fac[k][0] = c0; fac[k][1] = c0; fac[k][2] = c2; fac[k][3] = c3;
    }
    float vec[4][4];
    for (int r = 0; r < 4; ++r) { vec[r][0] = M(1, r); vec[r][1] = M(0, r); vec[r][2] = M(0, r); vec[r][3] = M(0, r); }
    static const int terms[4][6] = {{1, 0, 2, 1, 3, 2}, {0, 0, 2, 3, 3, 4}, {0, 1, 1, 3, 3, 5}, {0, 2, 1, 4, 2, 5}};
    static const float sign_a[4] = {1.0f, -1.0f, 1.0f, -1.0f}, sign_b[4] = {-1.0f, 1.0f, -1.0f, 1.0f};
    float inv[16];
    for (int c = 0; c < 4; ++c) {
        const int* t = terms[c];
        const float* sg = (c & 1) ? sign_b : sign_a;
        for (int k = 0; k < 4; ++k) {
            const float a = vec[t[0]][k] * fac[t[1]][k], b = vec[t[2]][k] * fac[t[3]][k], e = vec[t[4]][k] * fac[t[5]][k];
            inv[4 * c + k] = ((a - b) + e) * sg[k];
        }
    }
    const float d0 = M(0, 0) * inv[0], d1 = M(0, 1) * inv[4], d2 = M(0, 2) * inv[8], d3 = M(0, 3) * inv[12];
    const float rcp = 1.0f / ((d0 + d2) + (d1 + d3));
    for (int k = 0; k < 16; ++k) out[k] = inv[k] * rcp;
#undef M
}

static void shadow_camera(const r3_directional_light_source* s, int lh, const float* loc, r3_camera_header* h) {
    const f3 dir = {s->direction[0], s->direction[1], s->direction[2]}, zero = {0.0f, 0.0f, 0.0f}, l = {loc[0], loc[1], loc[2]};
    const float texel = s->distance / (float)s->resolution;
    float origin_view[16], inv[16], view[16], vp[16];
    look_at(zero, dir, lh, origin_view);
    const f3 cov = transform_point3(origin_view, l);
    f3 shadow_loc;
    shadow_loc.x = cov.x - fmodf(cov.x, texel);
    shadow_loc.y = cov.y - fmodf(cov.y, texel);
    shadow_loc.z = cov.z - 0.0f;
    inverse4(origin_view, inv);
    const f3 nl = transform_point3(inv, shadow_loc);
    const f3 center = {nl.x + dir.x, nl.y + dir.y, nl.z + dir.z};
    look_at(nl, center, lh, view);
    const float half = s->distance * 0.5f, left = -half, right = half, bottom = -half, top = half, near = half, far = -half;
    const float rcp_w = 1.0f / (right - left), rcp_h = 1.0f / (top - bottom);
    const float r = lh ? 1.0f / (far - near) : 1.0f / (near - far);
    const float proj[16] = {rcp_w + rcp_w, 0.0f, 0.0f, 0.0f, 0.0f, rcp_h + rcp_h, 0.0f, 0.0f, 0.0f, 0.0f, r, 0.0f,
                            -(left + right) * rcp_w, -(top + bottom) * rcp_h, lh ? (-r) * near : r * near, 1.0f};
    for (int j = 0; j < 4; ++j)
        for (int k = 0; k < 4; ++k)
            vp[4 * j + k] = ((proj[k] * view[4 * j] + proj[4 + k] * view[4 * j + 1]) + proj[8 + k] * view[4 * j + 2]) + proj[12 + k] * view[4 * j + 3];
    memset(h, 0, sizeof *h);
    memcpy(h->view, view, 64);
    memcpy(h->view_proj, vp, 64);
    static const int prow[5] = {0, 0, 1, 1, 2};
    static const int plus[5] = {1, 0, 0, 1, 0};
    for (int p = 0; p < 5; ++p) {
        float q[4];
        for (int c = 0; c < 4; ++c) q[c] = plus[p] ? vp[4 * c + 3] + vp[4 * c + prow[p]] : vp[4 * c + 3] - vp[4 * c + prow[p]];
        const float mag = sqrtf((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]);
        for (int c = 0; c < 4; ++c) h->frustum[p][c] = q[c] / mag;
    }
    h->resolution[0] = (float)s->size;
    h->resolution[1] = (float)s->size;
    h->flags = lh ? R3_PCU_POSITIVE_AREA_VISIBLE : 0u;
}

/* ------------------------------------------------------------------ entry points */
API int r3o_set_directional_light_sources(r3o_ctx* c, const r3_directional_light_source* lights, uint32_t n, uint32_t aw, uint32_t ah, uint32_t left_handed) {
    if (!c) return R3_E_INVALID;
    if (!lights && n) return fail(c, R3_E_INVALID, "set_directional_light_sources: null lights");
    if (n > R3_MAX_SHADOWS) return fail(c, R3_E_INVALID, "set_directional_light_sources: more lights than R3_MAX_SHADOWS");
    for (uint32_t i = 0; i < n; ++i)
        if (lights[i].size == 0 || (uint64_t)lights[i].offset[0] + lights[i].size > aw || (uint64_t)lights[i].offset[1] + lights[i].size > ah)
            return fail(c, R3_E_INVALID, "set_directional_light_sources: empty map or placement outside the atlas");
    lights_state* s = find(c, 1);
    if (!s) return fail(c, R3_E_OOM, "lights state");
    uint8_t* bytes = (uint8_t*)calloc(1, 16 + (size_t)n * sizeof(r3_directional_light));
    if (!bytes) return fail(c, R3_E_OOM, "set_directional_light_sources: out of memory");
    *(uint32_t*)bytes = n;
    r3_directional_light* dl = (r3_directional_light*)(bytes + 16);
    const float w = (float)aw, h = (float)ah;
    for (uint32_t i = 0; i < n; ++i) {
        for (int k = 0; k < 3; ++k) { dl[i].color[k] = lights[i].color[k] * lights[i].intensity; dl[i].direction[k] = lights[i].direction[k]; }
        dl[i].inv_resolution[0] = 1.0f / w; dl[i].inv_resolution[1] = 1.0f / h;
        dl[i].atlas_offset[0] = (float)lights[i].offset[0] / w; dl[i].atlas_offset[1] = (float)lights[i].offset[1] / h;
        dl[i].atlas_size[0] = (float)lights[i].size / w; dl[i].atlas_size[1] = (float)lights[i].size / h;
    }
    const int rc = r3o_set_directional_lights(c, bytes, 16 + (uint64_t)n * sizeof(r3_directional_light), aw, ah);
    free(bytes);
    if (rc != R3_OK) return rc;
    if (n) memcpy(s->src, lights, (size_t)n * sizeof *lights);
    s->n = n; s->left_handed = left_handed ? 1u : 0u; s->set = 1; s->evaluated = 0;
    return R3_OK;
}

API int r3o_evaluate_shadow_cameras(r3o_ctx* c, const float loc[3]) {
    if (!c) return R3_E_INVALID;
    if (!loc) return fail(c, R3_E_INVALID, "evaluate_shadow_cameras: null location");
    lights_state* s = find(c, 0);
    if (!s || !s->set) return fail(c, R3_E_STATE, "evaluate_shadow_cameras before set_directional_light_sources");
    for (uint32_t i = 0; i < s->n; ++i) {
        shadow_camera(&s->src[i], (int)s->left_handed, loc, &s->cams[i]);
        s->cams[i].shadow_index = i;
        memcpy(c->dir_lights[i].view_proj, s->cams[i].view_proj, 64);
    }
    s->evaluated = 1;
    return R3_OK;
}

API int r3o_shadow_uniform_upload(r3o_ctx* c, uint32_t shadow_index, uint32_t object_count, uint32_t mode) {
    if (!c) return R3_E_INVALID;
    lights_state* s = find(c, 0);
    if (!s || !s->set || !s->evaluated) return fail(c, R3_E_STATE, "shadow_uniform_upload before set_directional_light_sources + evaluate_shadow_cameras");
    if (shadow_index >= s->n) return fail(c, R3_E_INVALID, "shadow_uniform_upload: no such light");
    if (object_count > c->n_slots) return fail(c, R3_E_INVALID, "object_count exceeds the object buffer");
    r3_camera_header h = s->cams[shadow_index];
    h.object_count = object_count;
    return r3o_object_uniform_upload(c, shadow_index, &h, mode);
}

API int r3o_readback_shadow_cameras(r3o_ctx* c, r3_camera_header* out, r3_directional_light* lights, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (!out && n) return fail(c, R3_E_INVALID, "readback_shadow_cameras: null");
    lights_state* s = find(c, 0);
    if (!s || !s->set || !s->evaluated) return fail(c, R3_E_STATE, "readback_shadow_cameras before evaluate_shadow_cameras");
    if (n > s->n) return fail(c, R3_E_INVALID, "readback_shadow_cameras: more cameras than lights");
    if (n) memcpy(out, s->cams, (size_t)n * sizeof *out);
    if (n && lights) memcpy(lights, c->dir_lights, (size_t)n * sizeof *lights);
    return R3_OK;
}
