/* r3_oracle_points.c — CPU ORACLE of the device-evaluated point lights (test infrastructure; never linked into the product).
 *
 * Plain-C restatement of PointLightManager (rend3/src/managers/point.rs): the handle table `data: Vec<Option<PointLight>>` and its
 * evaluate (point.rs:58-74) by rule R14 (DESIGN.md §2) — the live handles in ascending order, position (x, y, z, 1), colour * intensity
 * as three f32 multiplies (-ffp-contract=off), radius as given.  It exports the r3o_ twins of r3_set_point_light_sources,
 * r3_update_point_light_sources, r3_evaluate_point_lights and r3_readback_point_lights with the same argument checks; the evaluation
 * feeds the base oracle's point_lights through r3o_set_point_lights.
 *
 * This unit includes the shadow-camera oracle (r3_oracle_lights.c), so one library exports the twins of both light paths.  The handle
 * tables live in a table keyed by the context: r3o_points_release drops a context's (before the context is destroyed) and
 * r3o_points_forget empties it; oracle/points.py calls the latter after every r3o_set_point_lights, which replaces the table.
 */
#include "r3_oracle_lights.c"

typedef struct points_state {
    const r3o_ctx* ctx;
    struct points_state* next;
    r3_point_light_source* src;   /* records + live bytes, n_handles entries */
    uint8_t* live;
    uint32_t n_handles;
} points_state;

static points_state* g_points_states;

static points_state* points_find(const r3o_ctx* c, int create) {
    pthread_mutex_lock(&g_lights_lock);
    points_state* s = g_points_states;
    while (s && s->ctx != c) s = s->next;
    if (!s && create) {
        s = (points_state*)calloc(1, sizeof *s);
        if (s) { s->ctx = c; s->next = g_points_states; g_points_states = s; }
    }
    pthread_mutex_unlock(&g_lights_lock);
    return s;
}

API void r3o_points_release(const r3o_ctx* c) {
    pthread_mutex_lock(&g_lights_lock);
    points_state** p = &g_points_states;
    while (*p && (*p)->ctx != c) p = &(*p)->next;
    points_state* s = *p;
    if (s) *p = s->next;
    pthread_mutex_unlock(&g_lights_lock);
    if (s) { free(s->src); free(s->live); }
    free(s);
}
API void r3o_points_forget(const r3o_ctx* c) {
    points_state* s = points_find(c, 0);
    if (s) s->n_handles = 0;
}

/* the table holds n handles; the new ones start dead.  R3_OK or R3_E_OOM */
static int point_table_resize(points_state* s, uint32_t n) {
    r3_point_light_source* src = (r3_point_light_source*)realloc(s->src, ((size_t)n + 1) * sizeof *src);
    if (!src) return R3_E_OOM;
    s->src = src;
    uint8_t* live = (uint8_t*)realloc(s->live, (size_t)n + 1);
    if (!live) return R3_E_OOM;
    s->live = live;
    if (n > s->n_handles) {
        memset(s->src + s->n_handles, 0, (size_t)(n - s->n_handles) * sizeof *src);
        memset(s->live + s->n_handles, 0, n - s->n_handles);
    }
    s->n_handles = n;
    return R3_OK;
}

API int r3o_set_point_light_sources(r3o_ctx* c, const r3_point_light_source* lights, const uint8_t* live, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (!lights && n) return fail(c, R3_E_INVALID, "set_point_light_sources: null lights");
    points_state* s = points_find(c, 1);
    if (!s) return fail(c, R3_E_OOM, "point lights state");
    s->n_handles = 0;
    if (point_table_resize(s, n) != R3_OK) return fail(c, R3_E_OOM, "set_point_light_sources: out of memory");
    for (uint32_t h = 0; h < n; ++h) {
        s->src[h] = lights[h];
        s->live[h] = live ? (live[h] != 0) : 1;
    }
    return R3_OK;
}

API int r3o_update_point_light_sources(r3o_ctx* c, const uint32_t* handles, const r3_point_light_source* lights, const uint8_t* live, uint32_t n) {
    if (!c) return R3_E_INVALID;
    if (!handles || !lights || !live) return fail(c, R3_E_INVALID, "update_point_light_sources: null");
    uint32_t top = 0;
    for (uint32_t i = 0; i < n; ++i) {   /* quadratic: the oracle's lists are short */
        if (handles[i] == 0xFFFFFFFFu) return fail(c, R3_E_INVALID, "update_point_light_sources: handle 0xFFFFFFFF");
        for (uint32_t j = 0; j < i; ++j)
            if (handles[j] == handles[i]) return fail(c, R3_E_INVALID, "update_point_light_sources: a handle is named twice");
        if (handles[i] + 1u > top) top = handles[i] + 1u;
    }
    if (n == 0) return R3_OK;
    points_state* s = points_find(c, 1);
    if (!s) return fail(c, R3_E_OOM, "point lights state");
    if (top > s->n_handles && point_table_resize(s, top) != R3_OK) return fail(c, R3_E_OOM, "update_point_light_sources: out of memory");
    for (uint32_t i = 0; i < n; ++i) {   /* add's resize, then data[handle] = Some(light) or None */
        if (live[i]) s->src[handles[i]] = lights[i];
        s->live[handles[i]] = live[i] != 0;
    }
    return R3_OK;
}

/* evaluate (point.rs:58-74): the live handles in ascending order, position (x, y, z, 1), colour * intensity (three f32 multiplies),
 * radius as given */
API int r3o_evaluate_point_lights(r3o_ctx* c) {
    if (!c) return R3_E_INVALID;
    points_state* s = points_find(c, 1);
    if (!s) return fail(c, R3_E_OOM, "point lights state");
    uint32_t count = 0;
    for (uint32_t h = 0; h < s->n_handles; ++h) count += s->live[h] ? 1u : 0u;
    uint8_t* bytes = (uint8_t*)calloc(1, 16 + (size_t)count * sizeof(r3_point_light));
    if (!bytes) return fail(c, R3_E_OOM, "evaluate_point_lights: out of memory");
    *(uint32_t*)bytes = count;
    r3_point_light* out = (r3_point_light*)(bytes + 16);
    uint32_t k = 0;
    for (uint32_t h = 0; h < s->n_handles; ++h) {
        if (!s->live[h]) continue;
        const r3_point_light_source* l = &s->src[h];
        for (int a = 0; a < 3; ++a) { out[k].position[a] = l->position[a]; out[k].color[a] = l->color[a] * l->intensity; }
        out[k].position[3] = 1.0f;
        out[k].radius = l->radius;
        ++k;
    }
    const int rc = r3o_set_point_lights(c, bytes, 16 + (uint64_t)count * sizeof(r3_point_light));
    free(bytes);
    return rc;
}

API int r3o_readback_point_lights(r3o_ctx* c, void* bytes, uint64_t capacity) {
    if (!c) return R3_E_INVALID;
    if (!bytes || capacity < 16) return fail(c, R3_E_INVALID, "readback_point_lights: room for the 16-byte header needed");
    memset(bytes, 0, 16);
    *(uint32_t*)bytes = c->n_point;
    uint64_t n = (uint64_t)c->n_point * sizeof(r3_point_light);
    if (n > capacity - 16) n = capacity - 16;
    if (n) memcpy((uint8_t*)bytes + 16, c->point_lights, n);
    return R3_OK;
}
