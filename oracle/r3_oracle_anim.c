/* r3_oracle_anim.c — CPU ORACLE of the skeletal-animation entry points (test infrastructure; never linked into the product).
 *
 * Plain-C restatement of the joint half of rend3-anim's pose_animation_frame (rend3-anim/src/lib.rs:165-176, 190, 214-262) with the
 * glam arithmetic of rule R12 (DESIGN.md §2): strict IEEE f32, one operation at a time in source order, no contraction
 * (-ffp-contract=off).  It exports the r3o_ twins of r3_set_animations, r3_set_skeletons, r3_set_pose_jobs, r3_pose_skeletons,
 * r3_skin_posed and r3_readback_joint_matrices with the same argument checks (include/r3_anim_check.h).
 *
 * It is a library of its own that links libr3_oracle.so (r3o_skin, the context's error text and mesh buffer): the animation state of a
 * context lives in a table keyed by the context, dropped by r3o_anim_release before the context is destroyed (oracle/anim.py does it).
 * Unlike the CUDA path, which schedules joints by level, this one computes the globals in the skin's topological order, as the
 * reference does: the two schedules must give the same bits.
 */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../include/r3_anim_check.h"
#include "r3_oracle.h"

#define API __attribute__((visibility("default")))

int r3o_skin(r3o_ctx* c, const r3_skinning_input* inputs, uint32_t n_skeletons, const float* joints, uint32_t n_joints);

typedef struct anim_state {
    const r3o_ctx* ctx;
    struct anim_state* next;
    int has_library, has_skeletons, has_jobs;
    r3_anim_skin* skins; uint32_t n_skins;
    r3_anim_joint* joints; uint32_t n_joints;
    uint32_t* order;
    r3_anim_clip* clips; uint32_t n_clips;
    r3_anim_channel* channels; uint32_t n_channels;
    float* keys; uint64_t n_keys;
    r3_skinning_input* inputs; uint32_t n_skeletons;
    float* joint_buf; uint32_t n_joint_mats;
    r3_pose_job* jobs; uint32_t n_jobs;
    r3_pose_target* targets; uint32_t n_targets;
} anim_state;

static anim_state* g_states;
static pthread_mutex_t g_lock = PTHREAD_MUTEX_INITIALIZER;

static int fail(r3o_ctx* c, int code, const char* msg) {
    if (c) snprintf(c->err, sizeof c->err, "%s", msg);
    return code;
}

static anim_state* find(const r3o_ctx* c, int create) {
    pthread_mutex_lock(&g_lock);
    anim_state* s = g_states;
    while (s && s->ctx != c) s = s->next;
    if (!s && create) {
        s = (anim_state*)calloc(1, sizeof *s);
        if (s) { s->ctx = c; s->next = g_states; g_states = s; }
    }
    pthread_mutex_unlock(&g_lock);
    return s;
}

static void free_library(anim_state* s) {
    free(s->skins); free(s->joints); free(s->order); free(s->clips); free(s->channels); free(s->keys);
    s->skins = NULL; s->joints = NULL; s->order = NULL; s->clips = NULL; s->channels = NULL; s->keys = NULL;
    s->n_skins = s->n_joints = s->n_clips = s->n_channels = 0; s->n_keys = 0; s->has_library = 0;
}
static void free_skeletons(anim_state* s) {
    free(s->inputs); free(s->joint_buf);
    s->inputs = NULL; s->joint_buf = NULL; s->n_skeletons = s->n_joint_mats = 0; s->has_skeletons = 0;
}
static void free_jobs(anim_state* s) {
    free(s->jobs); free(s->targets);
    s->jobs = NULL; s->targets = NULL; s->n_jobs = s->n_targets = 0; s->has_jobs = 0;
}

/* forget the animation state of a context (call before r3o_ctx_destroy) */
API void r3o_anim_release(const r3o_ctx* c) {
    pthread_mutex_lock(&g_lock);
    anim_state** p = &g_states;
    while (*p && (*p)->ctx != c) p = &(*p)->next;
    anim_state* s = *p;
    if (s) *p = s->next;
    pthread_mutex_unlock(&g_lock);
    if (s) { free_jobs(s); free_skeletons(s); free_library(s); free(s); }
}

static void* dup_array(const void* src, uint64_t n, size_t elem, int* ok) {
    void* p = malloc(n ? n * elem : 1);
    if (!p) { *ok = 0; return NULL; }
    if (n) memcpy(p, src, n * elem);
    return p;
}

API int r3o_set_animations(r3o_ctx* c, const r3_anim_library* L) {
    if (!c) return R3_E_INVALID;
    const char* msg = "";
    if (r3_anim_check_library(L, &msg) != R3_OK) return fail(c, R3_E_INVALID, msg);
    anim_state* s = find(c, 1);
    if (!s) return fail(c, R3_E_OOM, "animation state");
    anim_state n;
    memset(&n, 0, sizeof n);
    int ok = 1;
    n.skins = dup_array(L->skins, L->n_skins, sizeof *L->skins, &ok);
    n.joints = dup_array(L->joints, L->n_joints, sizeof *L->joints, &ok);
    n.order = dup_array(L->order, L->n_joints, sizeof *L->order, &ok);
    n.clips = dup_array(L->clips, L->n_clips, sizeof *L->clips, &ok);
    n.channels = dup_array(L->channels, L->n_channels, sizeof *L->channels, &ok);
    n.keys = dup_array(L->keys, L->n_keys, sizeof *L->keys, &ok);
    if (!ok) { free_library(&n); return fail(c, R3_E_OOM, "set_animations: out of memory"); }
    free_jobs(s);
    free_library(s);
    s->skins = n.skins; s->joints = n.joints; s->order = n.order; s->clips = n.clips; s->channels = n.channels; s->keys = n.keys;
    s->n_skins = L->n_skins; s->n_joints = L->n_joints; s->n_clips = L->n_clips; s->n_channels = L->n_channels; s->n_keys = L->n_keys;
    s->has_library = 1;
    return R3_OK;
}

API int r3o_set_skeletons(r3o_ctx* c, const r3_skinning_input* inputs, uint32_t n_skeletons, const float* joint_matrices, uint32_t n_joints) {
    if (!c) return R3_E_INVALID;
    if ((!inputs && n_skeletons) || (!joint_matrices && n_joints)) return fail(c, R3_E_INVALID, "set_skeletons: null");
    anim_state* s = find(c, 1);
    if (!s) return fail(c, R3_E_OOM, "animation state");
    int ok = 1;
    r3_skinning_input* in = dup_array(inputs, n_skeletons, sizeof *inputs, &ok);
    float* jb = dup_array(joint_matrices, (uint64_t)n_joints * 16, sizeof(float), &ok);
    if (!ok) { free(in); free(jb); return fail(c, R3_E_OOM, "set_skeletons: out of memory"); }
    free_jobs(s);
    free_skeletons(s);
    s->inputs = in; s->n_skeletons = n_skeletons; s->joint_buf = jb; s->n_joint_mats = n_joints;
    s->has_skeletons = 1;
    return R3_OK;
}

API int r3o_set_pose_jobs(r3o_ctx* c, const r3_pose_job* jobs, uint32_t n_jobs, const r3_pose_target* targets, uint32_t n_targets) {
    if (!c) return R3_E_INVALID;
    anim_state* s = find(c, 0);
    if (!s || !s->has_library) return fail(c, R3_E_STATE, "set_pose_jobs before set_animations");
    if (!s->has_skeletons) return fail(c, R3_E_STATE, "set_pose_jobs before set_skeletons");
    const char* msg = "";
    if (r3_anim_check_jobs(s->skins, s->clips, s->n_clips, s->n_joint_mats, jobs, n_jobs, targets, n_targets, &msg) != R3_OK)
        return fail(c, R3_E_INVALID, msg);
    int ok = 1;
    r3_pose_job* j = dup_array(jobs, n_jobs, sizeof *jobs, &ok);
    r3_pose_target* t = dup_array(targets, n_targets, sizeof *targets, &ok);
    if (!ok) { free(j); free(t); return fail(c, R3_E_OOM, "set_pose_jobs: out of memory"); }
    free_jobs(s);
    s->jobs = j; s->n_jobs = n_jobs; s->targets = t; s->n_targets = n_targets;
    s->has_jobs = 1;
    return R3_OK;
}

/* ---- R12 arithmetic */
typedef struct { float x, y, z; } f3;

/* sample_at_time (lib.rs:165-176): the reference's linear search for the first key with time > t */
static float key_factor(const float* keys, const r3_anim_track* tr, float t, uint32_t* prev, uint32_t* next) {
    const float* times = keys + tr->times;
    uint32_t n = tr->count - 1;
    for (uint32_t i = 0; i < tr->count; ++i)
        if (times[i] > t) { n = i; break; }
    const uint32_t p = n ? n - 1 : 0;
    float s = (t - times[p]) / (times[n] - times[p]);
    if (s < 0.0f) s = 0.0f;   /* f32::clamp: NaN passes through */
    if (s > 1.0f) s = 1.0f;
    *prev = p; *next = n;
    return s;
}
static f3 sample3(const float* keys, const r3_anim_track* tr, float t) {
    uint32_t p, n;
    const float s = key_factor(keys, tr, t, &p, &n);
    const float* a = keys + tr->values + 3ull * p;
    const float* b = keys + tr->values + 3ull * n;
    f3 r = {a[0] + ((b[0] - a[0]) * s), a[1] + ((b[1] - a[1]) * s), a[2] + ((b[2] - a[2]) * s)};   /* Vec3::lerp */
    return r;
}
static float dot4(const float* a, const float* b) { return (a[0] * b[0] + a[2] * b[2]) + (a[1] * b[1] + a[3] * b[3]); }   /* SSE2 dot4 */
static void normalize4(float* r) {
    const float rcp = 1.0f / sqrtf(dot4(r, r));
    for (int i = 0; i < 4; ++i) r[i] = r[i] * rcp;
}
static void sample_quat(const float* keys, const r3_anim_track* tr, float t, float* r) {
    uint32_t p, n;
    const float s = key_factor(keys, tr, t, &p, &n);
    const float* a = keys + tr->values + 4ull * p;
    const float* b = keys + tr->values + 4ull * n;
    const float d = dot4(a, b);
    uint32_t flip;
    memcpy(&flip, &d, 4);
    flip &= 0x80000000u;   /* _mm_and_ps(dot, -0.0): the sign bit, so a dot of -0.0 flips as well */
    for (int i = 0; i < 4; ++i) {
        uint32_t u;
        memcpy(&u, &b[i], 4);
        u ^= flip;
        float e;
        memcpy(&e, &u, 4);
        r[i] = ((e - a[i]) * s) + a[i];
    }
    normalize4(r);   /* inside glam's Quat::lerp */
    normalize4(r);   /* rend3-anim's .normalize() (lib.rs:159) */
}
static void from_srt(f3 sc, const float* q, f3 tr, float* m) {
    const float x = q[0], y = q[1], z = q[2], w = q[3];
    const float x2 = x + x, y2 = y + y, z2 = z + z;
    const float xx = x * x2, xy = x * y2, xz = x * z2, yy = y * y2, yz = y * z2, zz = z * z2, wx = w * x2, wy = w * y2, wz = w * z2;
    const float ax[4] = {1.0f - (yy + zz), xy + wz, xz - wy, 0.0f};
    const float ay[4] = {xy - wz, 1.0f - (xx + zz), yz + wx, 0.0f};
    const float az[4] = {xz + wy, yz - wx, 1.0f - (xx + yy), 0.0f};
    for (int i = 0; i < 4; ++i) { m[i] = ax[i] * sc.x; m[4 + i] = ay[i] * sc.y; m[8 + i] = az[i] * sc.z; }
    m[12] = tr.x; m[13] = tr.y; m[14] = tr.z; m[15] = 1.0f;
}
static void mat_mul(const float* a, const float* b, float* out) {   /* column j = ((a0 bj.x + a1 bj.y) + a2 bj.z) + a3 bj.w */
    for (int j = 0; j < 4; ++j)
        for (int r = 0; r < 4; ++r) {
            float v = a[r] * b[4 * j];
            v = v + a[4 + r] * b[4 * j + 1];
            v = v + a[8 + r] * b[4 * j + 2];
            v = v + a[12 + r] * b[4 * j + 3];
            out[4 * j + r] = v;
        }
}
static const float IDENTITY[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};

static void pose_job(anim_state* s, const r3_pose_job* job, float* local, float* global) {
    const r3_anim_clip clip = s->clips[job->clip];
    const r3_anim_skin sk = s->skins[clip.skin];
    const r3_anim_joint* joints = s->joints + sk.first_joint;
    float t = job->time;
    if (t < 0.0f) t = 0.0f;
    if (t > clip.duration) t = clip.duration;
    for (uint32_t k = 0; k < sk.joint_count; ++k) {
        const r3_anim_channel* ch = &s->channels[clip.first_channel + k];
        float* m = local + 16ull * k;
        if (!ch->animated) { memcpy(m, IDENTITY, sizeof IDENTITY); continue; }
        const r3_anim_joint* jt = &joints[k];
        f3 tr = {jt->bind_translation[0], jt->bind_translation[1], jt->bind_translation[2]};
        f3 sc = {jt->bind_scale[0], jt->bind_scale[1], jt->bind_scale[2]};
        float q[4] = {jt->bind_rotation[0], jt->bind_rotation[1], jt->bind_rotation[2], jt->bind_rotation[3]};
        if (ch->translation.times != R3_ANIM_ABSENT) tr = sample3(s->keys, &ch->translation, t);
        if (ch->rotation.times != R3_ANIM_ABSENT) sample_quat(s->keys, &ch->rotation, t, q);
        if (ch->scale.times != R3_ANIM_ABSENT) sc = sample3(s->keys, &ch->scale, t);
        from_srt(sc, q, tr, m);
    }
    for (uint32_t i = 0; i < sk.joint_count; ++i) {   /* joint_nodes_topological_order (lib.rs:243-256) */
        const uint32_t k = s->order[sk.first_joint + i], p = joints[k].parent;
        if (p == R3_ANIM_NO_PARENT) memcpy(global + 16ull * k, local + 16ull * k, 64);
        else mat_mul(p == R3_ANIM_PARENT_NOT_JOINT ? IDENTITY : global + 16ull * p, local + 16ull * k, global + 16ull * k);
    }
    for (uint32_t q = 0; q < job->target_count; ++q) {   /* set_skeleton_joint_transforms, truncated to the skeleton's joints */
        const r3_pose_target tg = s->targets[job->first_target + q];
        for (uint32_t k = 0; k < tg.joint_count; ++k)
            mat_mul(global + 16ull * k, joints[k].inverse_bind, s->joint_buf + ((uint64_t)tg.joint_matrix_base_offset + k) * 16);
    }
}

API int r3o_pose_skeletons(r3o_ctx* c) {
    if (!c) return R3_E_INVALID;
    anim_state* s = find(c, 0);
    if (!s || !s->has_jobs) return fail(c, R3_E_STATE, "pose_skeletons before set_animations + set_skeletons + set_pose_jobs");
    uint32_t most = 1;
    for (uint32_t i = 0; i < s->n_skins; ++i) if (s->skins[i].joint_count > most) most = s->skins[i].joint_count;
    int ok = 1;
#pragma omp parallel
    {
        float* scratch = (float*)malloc(2ull * 16 * most * sizeof(float));
        if (!scratch) {
#pragma omp atomic write
            ok = 0;
        }
#pragma omp for schedule(dynamic, 16)
        for (uint32_t i = 0; i < s->n_jobs; ++i)
            if (scratch) pose_job(s, &s->jobs[i], scratch, scratch + 16ull * most);
        free(scratch);
    }
    return ok ? R3_OK : fail(c, R3_E_OOM, "pose_skeletons: out of memory");
}

API int r3o_skin_posed(r3o_ctx* c) {
    if (!c) return R3_E_INVALID;
    anim_state* s = find(c, 0);
    if (!s || !s->has_skeletons) return fail(c, R3_E_STATE, "skin_posed before set_skeletons");
    if (s->n_skeletons && !c->mesh) return fail(c, R3_E_STATE, "skin_posed before set_mesh_buffer");
    return r3o_skin(c, s->inputs, s->n_skeletons, s->joint_buf, s->n_joint_mats);
}

API int r3o_readback_joint_matrices(r3o_ctx* c, float* out, uint32_t first, uint32_t n) {
    if (!c) return R3_E_INVALID;
    anim_state* s = find(c, 0);
    if (!s || !s->has_skeletons) return fail(c, R3_E_STATE, "readback_joint_matrices before set_skeletons");
    if (!out && n) return fail(c, R3_E_INVALID, "readback_joint_matrices: null");
    if ((uint64_t)first + n > s->n_joint_mats) return fail(c, R3_E_INVALID, "readback_joint_matrices: range outside the joint buffer");
    if (n) memcpy(out, s->joint_buf + (uint64_t)first * 16, (size_t)n * 64);
    return R3_OK;
}
