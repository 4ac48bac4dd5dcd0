"""Restatement of the object-transform half of rend3-anim's pose_animation_frame (rend3-anim/src/lib.rs:181-212) and of
Renderer::set_object_transform (rend3/src/managers/object.rs:302-316, util/frustum.rs:22-32) over the arrays of r3_set_object_animations /
r3_set_object_pose_jobs.

`pose_objects` follows rule R12 (DESIGN.md §2) one IEEE f32 operation at a time — numpy float32 scalars and element-wise ufuncs, never
contracted — with the key search, lerp, nlerp and TRS compose of tests/anim_reference.py; the oracle and the CUDA kernel must equal it
bit for bit.  With F = float64 it is the same algorithm in float64."""
import numpy as np

from anim_reference import _from_srt, _sample3, _sample_quat
from rend3_b200.layouts import ANIM_ABSENT

f32 = np.float32


def f32_max(a, b):
    """f32::max: a NaN operand is ignored (Python's max and np.maximum do not ignore it)."""
    if np.isnan(a):
        return b
    if np.isnan(b):
        return a
    return a if a > b else b


def node_matrix(library, clip, channel, t, F=f32):
    """Steps 1-4 of the rule: the TRS matrix (M[col, row]) of the clip's channel at time t."""
    nodes, clips, channels, keys, left_handed = library.arrays()
    cl = clips[int(clip)]
    t = F(t)
    if t < F(0):                                                          # time.clamp(0.0, duration)
        t = F(0)
    if t > F(cl["duration"]):
        t = F(cl["duration"])
    ch = channels[int(cl["first_channel"]) + int(channel)]
    nd = nodes[int(ch["node"])]
    # a missing property takes the bind pose, not IDENTITY's
    tr = nd["bind_translation"].astype(F) if ch["translation"]["times"] == ANIM_ABSENT else _sample3(keys, ch["translation"], t, F)
    q = nd["bind_rotation"].astype(F) if ch["rotation"]["times"] == ANIM_ABSENT else _sample_quat(keys, ch["rotation"], t, F)
    sc = (nd["bind_scale"].astype(F) if ch["scale"]["times"] == ANIM_ABSENT else _sample3(keys, ch["scale"], t, F)).copy()
    if left_handed:
        sc[2] = -sc[2]                                                    # a sign flip
    return _from_srt(sc, q, tr, F)


def set_object_transform(m, center, radius, F=f32):
    """Step 5: (transform (16,), world sphere centre (3,), radius, location (3,)) of a record whose mesh sphere is (center, radius)."""
    ls = [F(F(F(m[a][0] * m[a][0]) + F(m[a][1] * m[a][1])) + F(m[a][2] * m[a][2])) for a in range(3)]   # Vec3::length_squared
    max_scale = F(np.sqrt(f32_max(ls[0], f32_max(ls[1], ls[2]))))
    c = np.asarray(center, dtype=F)
    ctr = ((m[0] * c[0] + m[1] * c[1]) + m[2] * c[2]) + m[3] * F(1)      # Mat4 * (c, 1), mul_vec4's order
    zero = F(0)
    loc = m[3] + ((m[0] * zero + m[1] * zero) + m[2] * zero)             # transform_point3a(ZERO)
    return np.asarray(m, dtype=F).reshape(16), ctr[:3].astype(F), F(max_scale * F(radius)), loc[:3].astype(F)


def pose_objects(library, jobs, targets, records, locations, F=f32):
    """(transforms (n, 16), spheres (n, 4), locations (n, 3)) in dtype F: the given records' and locations' values with every job's
    targets posed.  Slots at or past len(records) are skipped; locations only exist for slots below len(locations)."""
    tf = np.array(records["transform"], dtype=F).reshape(-1, 16).copy()
    sph = np.concatenate([records["sphere_center"], records["sphere_radius"][:, None]], axis=1).astype(F)
    loc = np.array(locations, dtype=F).reshape(-1, 3).copy()
    with np.errstate(all="ignore"):
        for job in jobs:
            for k in range(int(job["target_count"])):
                tg = targets[int(job["first_target"]) + k]
                s = int(tg["slot"])
                if s >= len(tf):
                    continue
                m = node_matrix(library, job["clip"], tg["channel"], job["time"], F)
                tf[s], c, r, l = set_object_transform(m, tg["mesh_sphere_center"], tg["mesh_sphere_radius"], F)
                sph[s, :3], sph[s, 3] = c, r
                if s < len(loc):
                    loc[s] = l
    return tf, sph, loc


def posed_records(library, jobs, targets, records, locations):
    """The float32 rule applied to a copy of the records: (records, locations)."""
    tf, sph, loc = pose_objects(library, jobs, targets, records, locations)
    out = records.copy()
    out["transform"], out["sphere_center"], out["sphere_radius"] = tf, sph[:, :3], sph[:, 3]
    return out, loc
