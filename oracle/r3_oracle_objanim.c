/* r3_oracle_objanim.c — CPU ORACLE of the object-animation entry points (test infrastructure; never linked into the product).
 *
 * Plain-C restatement of the object-transform half of rend3-anim's pose_animation_frame (rend3-anim/src/lib.rs:181-212) and of
 * Renderer::set_object_transform (rend3/src/managers/object.rs:302-316, util/frustum.rs:22-32) with the arithmetic of rule R12
 * (DESIGN.md §2): strict IEEE f32, one operation at a time in source order, no contraction (-ffp-contract=off).  It exports the r3o_
 * twins of r3_set_object_animations, r3_set_object_pose_jobs, r3_pose_objects and r3_readback_objects with the same argument checks
 * (include/r3_anim_check.h); they write the oracle context's `objects` and `sort_loc`.
 *
 * This unit includes the skeletal oracle (r3_oracle_anim.c), so one library exports both halves and the object half samples its
 * tracks with the very same key search, lerp, nlerp and TRS compose.  Its own state lives in a table keyed by the context, dropped by
 * r3o_objanim_release before the context is destroyed (oracle/objanim.py does it, with r3o_anim_release).
 */
#include "r3_oracle_anim.c"

typedef struct objanim_state {
    const r3o_ctx* ctx;
    struct objanim_state* next;
    int has_library, has_jobs;
    uint32_t left_handed;
    r3_anim_node* nodes; uint32_t n_nodes;
    r3_anim_node_clip* clips; uint32_t n_clips;
    r3_anim_node_channel* channels; uint32_t n_channels;
    float* keys; uint64_t n_keys;
    r3_pose_job* jobs; uint32_t n_jobs;
    r3_object_pose_target* targets; uint32_t n_targets;
} objanim_state;

static objanim_state* g_obj_states;

static objanim_state* obj_find(const r3o_ctx* c, int create) {
    pthread_mutex_lock(&g_lock);
    objanim_state* s = g_obj_states;
    while (s && s->ctx != c) s = s->next;
    if (!s && create) {
        s = (objanim_state*)calloc(1, sizeof *s);
        if (s) { s->ctx = c; s->next = g_obj_states; g_obj_states = s; }
    }
    pthread_mutex_unlock(&g_lock);
    return s;
}

static void obj_free_library(objanim_state* s) {
    free(s->nodes); free(s->clips); free(s->channels); free(s->keys);
    s->nodes = NULL; s->clips = NULL; s->channels = NULL; s->keys = NULL;
    s->n_nodes = s->n_clips = s->n_channels = 0; s->n_keys = 0; s->has_library = 0; s->left_handed = 0;
}
static void obj_free_jobs(objanim_state* s) {
    free(s->jobs); free(s->targets);
    s->jobs = NULL; s->targets = NULL; s->n_jobs = s->n_targets = 0; s->has_jobs = 0;
}

/* forget the object-animation state of a context (call before r3o_ctx_destroy) */
API void r3o_objanim_release(const r3o_ctx* c) {
    pthread_mutex_lock(&g_lock);
    objanim_state** p = &g_obj_states;
    while (*p && (*p)->ctx != c) p = &(*p)->next;
    objanim_state* s = *p;
    if (s) *p = s->next;
    pthread_mutex_unlock(&g_lock);
    if (s) { obj_free_jobs(s); obj_free_library(s); free(s); }
}

API int r3o_set_object_animations(r3o_ctx* c, const r3_anim_object_library* L) {
    if (!c) return R3_E_INVALID;
    const char* msg = "";
    if (r3_anim_check_object_library(L, &msg) != R3_OK) return fail(c, R3_E_INVALID, msg);
    objanim_state* s = obj_find(c, 1);
    if (!s) return fail(c, R3_E_OOM, "object animation state");
    objanim_state n;
    memset(&n, 0, sizeof n);
    int ok = 1;
    n.nodes = dup_array(L->nodes, L->n_nodes, sizeof *L->nodes, &ok);
    n.clips = dup_array(L->clips, L->n_clips, sizeof *L->clips, &ok);
    n.channels = dup_array(L->channels, L->n_channels, sizeof *L->channels, &ok);
    n.keys = dup_array(L->keys, L->n_keys, sizeof *L->keys, &ok);
    if (!ok) { obj_free_library(&n); return fail(c, R3_E_OOM, "set_object_animations: out of memory"); }
    obj_free_jobs(s);
    obj_free_library(s);
    s->nodes = n.nodes; s->clips = n.clips; s->channels = n.channels; s->keys = n.keys;
    s->n_nodes = L->n_nodes; s->n_clips = L->n_clips; s->n_channels = L->n_channels; s->n_keys = L->n_keys;
    s->left_handed = L->left_handed ? 1u : 0u;
    s->has_library = 1;
    return R3_OK;
}

API int r3o_set_object_pose_jobs(r3o_ctx* c, const r3_pose_job* jobs, uint32_t n_jobs, const r3_object_pose_target* targets, uint32_t n_targets) {
    if (!c) return R3_E_INVALID;
    objanim_state* s = obj_find(c, 0);
    if (!s || !s->has_library) return fail(c, R3_E_STATE, "set_object_pose_jobs before set_object_animations");
    const char* msg = "";
    if (r3_anim_check_object_jobs(s->clips, s->n_clips, c->n_slots, jobs, n_jobs, targets, n_targets, NULL, NULL, &msg) != R3_OK)
        return fail(c, R3_E_INVALID, msg);
    int ok = 1;
    r3_pose_job* j = dup_array(jobs, n_jobs, sizeof *jobs, &ok);
    r3_object_pose_target* t = dup_array(targets, n_targets, sizeof *targets, &ok);
    if (!ok) { free(j); free(t); return fail(c, R3_E_OOM, "set_object_pose_jobs: out of memory"); }
    obj_free_jobs(s);
    s->jobs = j; s->n_jobs = n_jobs; s->targets = t; s->n_targets = n_targets;
    s->has_jobs = 1;
    return R3_OK;
}

/* f32::max: a NaN operand is ignored (the other one is returned) */
static float f32_max(float a, float b) { return a != a ? b : b != b ? a : (a > b ? a : b); }

static void pose_object(const objanim_state* s, r3o_ctx* c, const r3_pose_job* job, const r3_object_pose_target* tg) {
    if (tg->slot >= c->n_slots) return;   /* ScatterCopy drops out-of-range writes */
    const r3_anim_node_clip clip = s->clips[job->clip];
    float t = job->time;                  /* time.clamp(0.0, duration) (lib.rs:190) */
    if (t < 0.0f) t = 0.0f;
    if (t > clip.duration) t = clip.duration;
    const r3_anim_node_channel* ch = &s->channels[clip.first_channel + tg->channel];
    const r3_anim_node* nd = &s->nodes[ch->node];
    /* a missing property takes the node's bind pose (lib.rs:194-199) */
    f3 tr = {nd->bind_translation[0], nd->bind_translation[1], nd->bind_translation[2]};
    f3 sc = {nd->bind_scale[0], nd->bind_scale[1], nd->bind_scale[2]};
    float q[4] = {nd->bind_rotation[0], nd->bind_rotation[1], nd->bind_rotation[2], nd->bind_rotation[3]};
    if (ch->translation.times != R3_ANIM_ABSENT) tr = sample3(s->keys, &ch->translation, t);
    if (ch->rotation.times != R3_ANIM_ABSENT) sample_quat(s->keys, &ch->rotation, t, q);
    if (ch->scale.times != R3_ANIM_ABSENT) sc = sample3(s->keys, &ch->scale, t);
    if (s->left_handed) sc.z = -sc.z;     /* lib.rs:201-203: a sign flip */
    float m[16];
    from_srt(sc, q, tr, m);
    /* set_object_transform (object.rs:311-314): the transform, BoundingSphere::apply_transform (util/frustum.rs:22-32), the location */
    r3_object* o = &c->objects[tg->slot];
    memcpy(o->transform, m, sizeof m);
    float ls[3];
    for (int a = 0; a < 3; ++a) ls[a] = (m[4 * a] * m[4 * a] + m[4 * a + 1] * m[4 * a + 1]) + m[4 * a + 2] * m[4 * a + 2];
    const float max_scale = sqrtf(f32_max(ls[0], f32_max(ls[1], ls[2])));
    const float* cc = tg->mesh_sphere_center;
    for (int r = 0; r < 3; ++r) {         /* mul_vec4(matrix, (c, 1)): ((x cx + y cy) + z cz) + w 1 */
        float v = m[r] * cc[0];
        v = v + m[4 + r] * cc[1];
        v = v + m[8 + r] * cc[2];
        v = v + m[12 + r] * 1.0f;
        o->sphere_center[r] = v;
    }
    o->sphere_radius = max_scale * tg->mesh_sphere_radius;
    if (c->sort_loc && tg->slot < c->sort_n)   /* transform_point3a(ZERO): w + ((x 0 + y 0) + z 0) */
        for (int r = 0; r < 3; ++r) c->sort_loc[3 * (size_t)tg->slot + r] = m[12 + r] + ((m[r] * 0.0f + m[4 + r] * 0.0f) + m[8 + r] * 0.0f);
}

API int r3o_pose_objects(r3o_ctx* c) {
    if (!c) return R3_E_INVALID;
    objanim_state* s = obj_find(c, 0);
    if (!s || !s->has_jobs) return fail(c, R3_E_STATE, "pose_objects before set_object_animations + set_object_pose_jobs");
    if (!c->objects) return fail(c, R3_E_STATE, "pose_objects before set_objects");
    for (uint32_t i = 0; i < s->n_jobs; ++i)
        for (uint32_t k = 0; k < s->jobs[i].target_count; ++k) pose_object(s, c, &s->jobs[i], &s->targets[s->jobs[i].first_target + k]);
    return R3_OK;
}

API int r3o_readback_objects(r3o_ctx* c, r3_object* out, float* locations, uint32_t first, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (!out && n) return fail(c, R3_E_INVALID, "readback_objects: null");
    if ((uint64_t)first + n > c->n_slots) return fail(c, R3_E_INVALID, "readback_objects: range outside the object buffer");
    if (locations && (uint64_t)first + n > (c->sort_loc ? c->sort_n : 0u)) return fail(c, R3_E_INVALID, "readback_objects: range outside the sort info");
    if (n) memcpy(out, c->objects + first, (size_t)n * sizeof(r3_object));
    if (n && locations) memcpy(locations, c->sort_loc + 3 * (size_t)first, (size_t)n * 12);
    return R3_OK;
}
