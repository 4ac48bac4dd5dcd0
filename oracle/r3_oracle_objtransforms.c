/* r3_oracle_objtransforms.c — CPU ORACLE of the bulk object-transform entry points (test infrastructure; never linked into the product).
 *
 * Plain-C restatement of Renderer::set_object_transform (rend3/src/managers/object.rs:302-316, util/frustum.rs:22-32) for many objects,
 * with the arithmetic of rule R12's object half (DESIGN.md §2): strict IEEE f32, one operation at a time in source order, no
 * contraction (-ffp-contract=off).  It exports the r3o_ twins of r3_set_object_mesh_spheres and r3_set_object_transforms with the same
 * argument checks in the same order; they write the oracle context's `objects` and `sort_loc`.
 *
 * This unit includes the object-animation oracle (r3_oracle_objanim.c, and through it the skeletal one), so one library exports all
 * three and the transform here uses the very f32_max the pose uses.  The mesh spheres live in a table keyed by the context, dropped by
 * r3o_objtransforms_release before the context is destroyed (oracle/objtransforms.py does it, with the other two releases).  Like the
 * sort info they belong to no record: r3o_set_objects keeps them, and a world that outgrew them is R3_E_STATE.
 */
#include "r3_oracle_objanim.c"

typedef struct objtr_state {
    const r3o_ctx* ctx;
    struct objtr_state* next;
    float* spheres; uint32_t n_spheres;      /* (centre, radius) per slot */
} objtr_state;

static objtr_state* g_objtr_states;

static objtr_state* objtr_find(const r3o_ctx* c, int create) {
    pthread_mutex_lock(&g_lock);
    objtr_state* s = g_objtr_states;
    while (s && s->ctx != c) s = s->next;
    if (!s && create) {
        s = (objtr_state*)calloc(1, sizeof *s);
        if (s) { s->ctx = c; s->next = g_objtr_states; g_objtr_states = s; }
    }
    pthread_mutex_unlock(&g_lock);
    return s;
}

/* forget the mesh spheres of a context (call before r3o_ctx_destroy) */
API void r3o_objtransforms_release(const r3o_ctx* c) {
    pthread_mutex_lock(&g_lock);
    objtr_state** p = &g_objtr_states;
    while (*p && (*p)->ctx != c) p = &(*p)->next;
    objtr_state* s = *p;
    if (s) *p = s->next;
    pthread_mutex_unlock(&g_lock);
    if (s) { free(s->spheres); free(s); }
}

/* every slot below `limit` and no slot named twice */
static int check_slots(r3o_ctx* c, const uint32_t* slots, uint32_t n, uint32_t limit, const char* beyond, const char* twice) {
    uint8_t* seen = (uint8_t*)calloc((size_t)limit + 1, 1);
    if (!seen) return fail(c, R3_E_OOM, "slot check: out of memory");
    int rc = R3_OK;
    for (uint32_t i = 0; i < n && rc == R3_OK; ++i) {
        if (slots[i] >= limit) rc = fail(c, R3_E_INVALID, beyond);
        else if (seen[slots[i]]++) rc = fail(c, R3_E_INVALID, twice);
    }
    free(seen);
    return rc;
}

API int r3o_set_object_mesh_spheres(r3o_ctx* c, const uint32_t* slots, const float* center_radius, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (!center_radius && n) return fail(c, R3_E_INVALID, "set_object_mesh_spheres: null");
    objtr_state* s = objtr_find(c, 1);
    if (!s) return fail(c, R3_E_OOM, "object transform state");
    if (!slots) {
        int ok = 1;
        float* sp = dup_array(center_radius, (uint64_t)n * 4, sizeof(float), &ok);
        if (!ok) return fail(c, R3_E_OOM, "set_object_mesh_spheres: out of memory");
        free(s->spheres);
        s->spheres = sp; s->n_spheres = n;
        return R3_OK;
    }
    if (n == 0) return R3_OK;
    int rc = check_slots(c, slots, n, s->n_spheres, "set_object_mesh_spheres: slot beyond the mesh spheres", "set_object_mesh_spheres: one slot named twice");
    if (rc != R3_OK) return rc;
    for (uint32_t i = 0; i < n; ++i) memcpy(s->spheres + 4 * (size_t)slots[i], center_radius + 4 * (size_t)i, 16);
    return R3_OK;
}

/* set_object_transform (object.rs:311-314): the transform, BoundingSphere::apply_transform (util/frustum.rs:22-32), the location */
static void move_object(r3o_ctx* c, uint32_t slot, const float* m, const float* ms) {
    r3_object* o = &c->objects[slot];
    memcpy(o->transform, m, 64);
    float ls[3];
    for (int a = 0; a < 3; ++a) ls[a] = (m[4 * a] * m[4 * a] + m[4 * a + 1] * m[4 * a + 1]) + m[4 * a + 2] * m[4 * a + 2];
    const float max_scale = sqrtf(f32_max(ls[0], f32_max(ls[1], ls[2])));
    for (int r = 0; r < 3; ++r) {         /* mul_vec4(matrix, (c, 1)): ((x cx + y cy) + z cz) + w 1 */
        float v = m[r] * ms[0];
        v = v + m[4 + r] * ms[1];
        v = v + m[8 + r] * ms[2];
        v = v + m[12 + r] * 1.0f;
        o->sphere_center[r] = v;
    }
    o->sphere_radius = max_scale * ms[3];
    if (c->sort_loc && slot < c->sort_n)   /* transform_point3a(ZERO): w + ((x 0 + y 0) + z 0) */
        for (int r = 0; r < 3; ++r) c->sort_loc[3 * (size_t)slot + r] = m[12 + r] + ((m[r] * 0.0f + m[4 + r] * 0.0f) + m[8 + r] * 0.0f);
}

API int r3o_set_object_transforms(r3o_ctx* c, const uint32_t* slots, const float* mat4s, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (n == 0) return R3_OK;
    if (!mat4s) return fail(c, R3_E_INVALID, "set_object_transforms: null");
    if (!c->objects) return fail(c, R3_E_STATE, "set_object_transforms before set_objects");
    objtr_state* s = objtr_find(c, 0);
    if ((s ? s->n_spheres : 0u) < c->n_slots) return fail(c, R3_E_STATE, "set_object_transforms: r3_set_object_mesh_spheres does not cover every slot");
    if (!slots && n > c->n_slots) return fail(c, R3_E_INVALID, "set_object_transforms: more matrices than slots");
    if (slots) {
        int rc = check_slots(c, slots, n, c->n_slots, "set_object_transforms: slot beyond the object buffer", "set_object_transforms: one slot named twice");
        if (rc != R3_OK) return rc;
    }
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t slot = slots ? slots[i] : i;
        move_object(c, slot, mat4s + 16 * (size_t)i, s->spheres + 4 * (size_t)slot);
    }
    return R3_OK;
}
