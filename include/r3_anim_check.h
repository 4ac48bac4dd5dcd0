/* r3_anim_check.h — argument checks of r3_set_animations / r3_set_pose_jobs and r3_set_object_animations / r3_set_object_pose_jobs,
 * shared by the library and its CPU oracle so that both reject exactly the same inputs, and of r3_set_joint_matrices.  Plain C99 / C++,
 * header only.
 *
 * The checks turn the reference's panic sites into errors (rend3-anim/src/lib.rs:166-175, 190; skeleton.rs:151-162):
 *   an empty key channel (`times.len() - 1` underflow), fewer values than key times, a NaN or negative duration (f32::clamp's assert),
 *   a target joint count above the skin's (set_joint_matrices' assert), a target outside the joint buffer, an index out of range, an
 *   order that is not a permutation listing parents first.
 * One departure: key times must be finite, >= 0 and strictly increasing (glTF 2.0 §3.11 requires it).  That is what lets a binary
 * search return the reference's linear "first key with time > t" for every t, NaN included (no key compares greater: the last key).
 * Two jobs may not write overlapping joint ranges (the order in which they land would be unspecified). */
#ifndef R3_ANIM_CHECK_H
#define R3_ANIM_CHECK_H

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "rend3_b200.h"

/* returns R3_OK, or R3_E_INVALID with *msg set; allocates nothing that outlives the call */
static inline int r3_anim_check_track(const r3_anim_track* t, uint32_t stride, const float* keys, uint64_t n_keys, const char** msg) {
    if (t->times == R3_ANIM_ABSENT) return R3_OK;
    if (t->count == 0) { *msg = "animation: empty key channel"; return R3_E_INVALID; }
    if (t->value_count < t->count) { *msg = "animation: fewer values than key times"; return R3_E_INVALID; }
    if ((uint64_t)t->times + t->count > n_keys || (uint64_t)t->values + (uint64_t)t->value_count * stride > n_keys) {
        *msg = "animation: key range outside the key blob"; return R3_E_INVALID;
    }
    for (uint32_t i = 0; i < t->count; ++i) {
        const float v = keys[(uint64_t)t->times + i];
        if (!(v >= 0.0f) || !isfinite(v) || (i > 0 && !(v > keys[(uint64_t)t->times + i - 1]))) {
            *msg = "animation: key times must be finite, >= 0 and strictly increasing"; return R3_E_INVALID;
        }
    }
    return R3_OK;
}

static inline int r3_anim_check_library(const r3_anim_library* L, const char** msg) {
    *msg = "";
    if (!L) { *msg = "set_animations: null library"; return R3_E_INVALID; }
    if ((!L->skins && L->n_skins) || (!L->joints && L->n_joints) || (!L->order && L->n_joints) || (!L->clips && L->n_clips) ||
        (!L->channels && L->n_channels) || (!L->keys && L->n_keys)) {
        *msg = "set_animations: null array"; return R3_E_INVALID;
    }
    uint8_t* seen = (uint8_t*)malloc(L->n_joints ? L->n_joints : 1);
    if (!seen) { *msg = "set_animations: out of host memory"; return R3_E_INVALID; }
    int rc = R3_OK;
    for (uint32_t s = 0; s < L->n_skins && rc == R3_OK; ++s) {
        const r3_anim_skin sk = L->skins[s];
        if ((uint64_t)sk.first_joint + sk.joint_count > L->n_joints) { *msg = "set_animations: skin joint range out of range"; rc = R3_E_INVALID; break; }
        memset(seen, 0, sk.joint_count ? sk.joint_count : 1);
        for (uint32_t i = 0; i < sk.joint_count; ++i) {
            const uint32_t j = L->order[sk.first_joint + i];
            if (j >= sk.joint_count || seen[j]) { *msg = "set_animations: order is not a permutation of the skin's joints"; rc = R3_E_INVALID; break; }
            const uint32_t p = L->joints[sk.first_joint + j].parent;
            if (p != R3_ANIM_NO_PARENT && p != R3_ANIM_PARENT_NOT_JOINT) {
                if (p >= sk.joint_count) { *msg = "set_animations: parent joint index out of range"; rc = R3_E_INVALID; break; }
                if (!seen[p]) { *msg = "set_animations: order lists a joint before its parent"; rc = R3_E_INVALID; break; }
            }
            seen[j] = 1;
        }
    }
    free(seen);
    if (rc != R3_OK) return rc;
    for (uint32_t c = 0; c < L->n_clips; ++c) {
        const r3_anim_clip cl = L->clips[c];
        if (cl.skin >= L->n_skins) { *msg = "set_animations: clip skin out of range"; return R3_E_INVALID; }
        if (!(cl.duration >= 0.0f)) { *msg = "set_animations: clip duration is NaN or negative"; return R3_E_INVALID; }
        const r3_anim_skin sk = L->skins[cl.skin];
        if ((uint64_t)cl.first_channel + sk.joint_count > L->n_channels) { *msg = "set_animations: clip channel range out of range"; return R3_E_INVALID; }
        for (uint32_t k = 0; k < sk.joint_count; ++k) {
            const r3_anim_channel* ch = &L->channels[cl.first_channel + k];
            if (!ch->animated) continue;
            if (r3_anim_check_track(&ch->translation, 3, L->keys, L->n_keys, msg) != R3_OK) return R3_E_INVALID;
            if (r3_anim_check_track(&ch->rotation, 4, L->keys, L->n_keys, msg) != R3_OK) return R3_E_INVALID;
            if (r3_anim_check_track(&ch->scale, 3, L->keys, L->n_keys, msg) != R3_OK) return R3_E_INVALID;
        }
    }
    return R3_OK;
}

static inline int r3_anim_range_cmp(const void* a, const void* b) {
    const uint64_t x = ((const uint64_t*)a)[0], y = ((const uint64_t*)b)[0];
    return x < y ? -1 : x > y ? 1 : 0;
}

/* n ranges [r[2i], r[2i + 1]) of the joint buffer, sorted in place by their start: R3_E_INVALID with *msg = overlap_msg when two overlap */
static inline int r3_anim_check_disjoint(uint64_t* r, uint64_t n, const char* overlap_msg, const char** msg) {
    qsort(r, n, 2 * sizeof(uint64_t), r3_anim_range_cmp);
    for (uint64_t i = 1; i < n; ++i)
        if (r[2 * i] < r[2 * (i - 1) + 1]) { *msg = overlap_msg; return R3_E_INVALID; }
    return R3_OK;
}

/* jobs against the skins / clips of the library that is set and a joint buffer of n_joint_matrices matrices */
static inline int r3_anim_check_jobs(const r3_anim_skin* skins, const r3_anim_clip* clips, uint32_t n_clips, uint32_t n_joint_matrices,
                                     const r3_pose_job* jobs, uint32_t n_jobs, const r3_pose_target* targets, uint32_t n_targets,
                                     const char** msg) {
    *msg = "";
    if ((!jobs && n_jobs) || (!targets && n_targets)) { *msg = "set_pose_jobs: null array"; return R3_E_INVALID; }
    uint64_t n_ranges = 0;
    for (uint32_t i = 0; i < n_jobs; ++i) {
        const r3_pose_job j = jobs[i];
        if (j.clip >= n_clips) { *msg = "set_pose_jobs: clip out of range"; return R3_E_INVALID; }
        if ((uint64_t)j.first_target + j.target_count > n_targets) { *msg = "set_pose_jobs: target range out of range"; return R3_E_INVALID; }
        const uint32_t skin_joints = skins[clips[j.clip].skin].joint_count;
        for (uint32_t t = 0; t < j.target_count; ++t) {
            const r3_pose_target tg = targets[j.first_target + t];
            if (tg.joint_count > skin_joints) { *msg = "set_pose_jobs: target joint count above the skin's"; return R3_E_INVALID; }
            if ((uint64_t)tg.joint_matrix_base_offset + tg.joint_count > n_joint_matrices) { *msg = "set_pose_jobs: target outside the joint buffer"; return R3_E_INVALID; }
            n_ranges += tg.joint_count != 0;
        }
    }
    uint64_t* r = (uint64_t*)malloc(n_ranges ? n_ranges * 2 * sizeof(uint64_t) : 16);
    if (!r) { *msg = "set_pose_jobs: out of host memory"; return R3_E_INVALID; }
    uint64_t n = 0;
    for (uint32_t i = 0; i < n_jobs; ++i)
        for (uint32_t t = 0; t < jobs[i].target_count; ++t) {
            const r3_pose_target tg = targets[jobs[i].first_target + t];
            if (tg.joint_count) { r[2 * n] = tg.joint_matrix_base_offset; r[2 * n + 1] = (uint64_t)tg.joint_matrix_base_offset + tg.joint_count; ++n; }
        }
    const int rc = r3_anim_check_disjoint(r, n, "set_pose_jobs: two targets write overlapping joint ranges", msg);
    free(r);
    return rc;
}

/* r3_set_joint_matrices' writes against a joint buffer of n_joint_matrices matrices, n_mat4s source matrices and, when with_inverse_binds,
 * n_inverse_binds inverse binds: every range inside its array (64-bit sums), the destinations of the writes with joint_count > 0 disjoint */
static inline int r3_anim_check_joint_writes(uint32_t n_joint_matrices, const r3_joint_write* writes, uint32_t n_writes, uint32_t n_mat4s,
                                             int with_inverse_binds, uint32_t n_inverse_binds, const char** msg) {
    *msg = "";
    uint64_t n_ranges = 0;
    for (uint32_t i = 0; i < n_writes; ++i) {
        const r3_joint_write w = writes[i];
        if (w.joint_count == 0) continue;   /* does nothing, wherever it points */
        if ((uint64_t)w.joint_matrix_base_offset + w.joint_count > n_joint_matrices) { *msg = "set_joint_matrices: destination outside the joint buffer"; return R3_E_INVALID; }
        if ((uint64_t)w.first_matrix + w.joint_count > n_mat4s) { *msg = "set_joint_matrices: source outside the matrices"; return R3_E_INVALID; }
        if (with_inverse_binds && (uint64_t)w.first_inverse_bind + w.joint_count > n_inverse_binds) {
            *msg = "set_joint_matrices: source outside the inverse binds"; return R3_E_INVALID;
        }
        n_ranges++;
    }
    uint64_t* r = (uint64_t*)malloc(n_ranges ? n_ranges * 2 * sizeof(uint64_t) : 16);
    if (!r) { *msg = "set_joint_matrices: out of host memory"; return R3_E_INVALID; }
    uint64_t n = 0;
    for (uint32_t i = 0; i < n_writes; ++i)
        if (writes[i].joint_count) { r[2 * n] = writes[i].joint_matrix_base_offset; r[2 * n + 1] = (uint64_t)writes[i].joint_matrix_base_offset + writes[i].joint_count; ++n; }
    const int rc = r3_anim_check_disjoint(r, n, "set_joint_matrices: two writes' destinations overlap", msg);
    free(r);
    return rc;
}

/* ---- object animation (r3_set_object_animations / r3_set_object_pose_jobs): the same track rules, the same duration rule */
static inline int r3_anim_check_object_library(const r3_anim_object_library* L, const char** msg) {
    *msg = "";
    if (!L) { *msg = "set_object_animations: null library"; return R3_E_INVALID; }
    if ((!L->nodes && L->n_nodes) || (!L->clips && L->n_clips) || (!L->channels && L->n_channels) || (!L->keys && L->n_keys)) {
        *msg = "set_object_animations: null array"; return R3_E_INVALID;
    }
    for (uint32_t c = 0; c < L->n_clips; ++c) {
        const r3_anim_node_clip cl = L->clips[c];
        if (!(cl.duration >= 0.0f)) { *msg = "set_object_animations: clip duration is NaN or negative"; return R3_E_INVALID; }
        if ((uint64_t)cl.first_channel + cl.channel_count > L->n_channels) { *msg = "set_object_animations: clip channel range out of range"; return R3_E_INVALID; }
    }
    for (uint32_t k = 0; k < L->n_channels; ++k) {
        const r3_anim_node_channel* ch = &L->channels[k];
        if (ch->node >= L->n_nodes) { *msg = "set_object_animations: channel node out of range"; return R3_E_INVALID; }
        if (r3_anim_check_track(&ch->translation, 3, L->keys, L->n_keys, msg) != R3_OK) return R3_E_INVALID;
        if (r3_anim_check_track(&ch->rotation, 4, L->keys, L->n_keys, msg) != R3_OK) return R3_E_INVALID;
        if (r3_anim_check_track(&ch->scale, 3, L->keys, L->n_keys, msg) != R3_OK) return R3_E_INVALID;
    }
    return R3_OK;
}

static inline int r3_anim_slot_cmp(const void* a, const void* b) {
    const uint32_t x = *(const uint32_t*)a, y = *(const uint32_t*)b;
    return x < y ? -1 : x > y ? 1 : 0;
}

/* jobs against the clips of the object library that is set and an object buffer of n_slots slots.  On success, when `slots_out` is
 * not null, *slots_out is a malloc'd list of the slot of every (job, target) pair in job order (*n_out entries; the caller frees it). */
static inline int r3_anim_check_object_jobs(const r3_anim_node_clip* clips, uint32_t n_clips, uint32_t n_slots, const r3_pose_job* jobs,
                                            uint32_t n_jobs, const r3_object_pose_target* targets, uint32_t n_targets,
                                            uint32_t** slots_out, uint64_t* n_out, const char** msg) {
    *msg = "";
    if ((!jobs && n_jobs) || (!targets && n_targets)) { *msg = "set_object_pose_jobs: null array"; return R3_E_INVALID; }
    uint64_t n = 0;
    for (uint32_t i = 0; i < n_jobs; ++i) {
        const r3_pose_job j = jobs[i];
        if (j.clip >= n_clips) { *msg = "set_object_pose_jobs: clip out of range"; return R3_E_INVALID; }
        if ((uint64_t)j.first_target + j.target_count > n_targets) { *msg = "set_object_pose_jobs: target range out of range"; return R3_E_INVALID; }
        for (uint32_t t = 0; t < j.target_count; ++t) {
            const r3_object_pose_target tg = targets[j.first_target + t];
            if (tg.channel >= clips[j.clip].channel_count) { *msg = "set_object_pose_jobs: target channel out of the clip's range"; return R3_E_INVALID; }
            if (tg.slot >= n_slots) { *msg = "set_object_pose_jobs: target slot beyond the object buffer"; return R3_E_INVALID; }
        }
        n += j.target_count;
    }
    uint32_t* s = (uint32_t*)malloc(n ? n * sizeof(uint32_t) : 4);
    uint32_t* sorted = (uint32_t*)malloc(n ? n * sizeof(uint32_t) : 4);
    if (!s || !sorted) { free(s); free(sorted); *msg = "set_object_pose_jobs: out of host memory"; return R3_E_INVALID; }
    uint64_t k = 0;
    for (uint32_t i = 0; i < n_jobs; ++i)
        for (uint32_t t = 0; t < jobs[i].target_count; ++t) s[k++] = targets[jobs[i].first_target + t].slot;
    if (n) memcpy(sorted, s, n * sizeof(uint32_t));
    qsort(sorted, n, sizeof(uint32_t), r3_anim_slot_cmp);
    int rc = R3_OK;
    for (uint64_t i = 1; i < n; ++i)
        if (sorted[i] == sorted[i - 1]) { *msg = "set_object_pose_jobs: two targets name the same slot"; rc = R3_E_INVALID; break; }
    free(sorted);
    if (rc != R3_OK || !slots_out) { free(s); return rc; }
    *slots_out = s;
    *n_out = n;
    return R3_OK;
}

#endif /* R3_ANIM_CHECK_H */
