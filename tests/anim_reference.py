"""Restatements of the joint half of rend3-anim's pose_animation_frame (rend3-anim/src/lib.rs:165-176, 190, 214-262) over the arrays of
r3_set_animations / r3_set_pose_jobs.

`pose_f32` follows rule R12 (DESIGN.md §2) one IEEE f32 operation at a time in source order — numpy float32 scalars and element-wise
ufuncs, never contracted — with the reference's linear key search and its topological order; the oracle and the CUDA kernel must
equal it bit for bit.  `pose_f64` is the same algorithm in float64: the distance between the two is the rounding of the f32 path."""
import numpy as np

from rend3_b200 import glam
from rend3_b200.layouts import ANIM_ABSENT, ANIM_NO_PARENT, ANIM_PARENT_NOT_JOINT

f32 = np.float32


def _factor(keys, tr, t, F):
    times = keys[int(tr["times"]): int(tr["times"]) + int(tr["count"])].astype(F)
    nxt = next((i for i, x in enumerate(times) if x > t), len(times) - 1)   # position(|time| time > t).unwrap_or(len - 1)
    prv = max(nxt - 1, 0)
    s = F(F(t - times[prv]) / F(times[nxt] - times[prv]))
    if s < F(0):                                                          # f32::clamp: NaN passes through
        s = F(0)
    if s > F(1):
        s = F(1)
    return s, prv, nxt


def _sample3(keys, tr, t, F):
    s, p, n = _factor(keys, tr, t, F)
    v = int(tr["values"])
    a, b = keys[v + 3 * p: v + 3 * p + 3].astype(F), keys[v + 3 * n: v + 3 * n + 3].astype(F)
    return a + ((b - a) * s)                                              # Vec3::lerp


def _dot4(a, b, F):
    return F(F(F(a[0] * b[0]) + F(a[2] * b[2])) + F(F(a[1] * b[1]) + F(a[3] * b[3])))   # SSE2 dot4


def _normalize4(r, F):
    return r * F(F(1) / F(np.sqrt(_dot4(r, r, F))))


def _sample_quat(keys, tr, t, F):
    s, p, n = _factor(keys, tr, t, F)
    v = int(tr["values"])
    a, b = keys[v + 4 * p: v + 4 * p + 4].astype(F), keys[v + 4 * n: v + 4 * n + 4].astype(F)
    if np.signbit(_dot4(a, b, F)):                                       # _mm_and_ps(dot, -0.0): the sign BIT
        b = -b                                                            # the xor with the sign bit is a negation, NaN included
    r = ((b - a) * s) + a
    return _normalize4(_normalize4(r, F), F)                              # Quat::lerp's normalize, then rend3-anim's (lib.rs:159)


def _axes(q, F):
    if F is f32:
        return glam.quat_to_axes(q)
    x, y, z, w = [F(v) for v in q]
    x2, y2, z2 = x + x, y + y, z + z
    xx, xy, xz, yy, yz, zz, wx, wy, wz = x * x2, x * y2, x * z2, y * y2, y * z2, z * z2, w * x2, w * y2, w * z2
    return (np.array([1 - (yy + zz), xy + wz, xz - wy]), np.array([xy - wz, 1 - (xx + zz), yz + wx]), np.array([xz + wy, yz - wx, 1 - (xx + yy)]))


def _from_srt(sc, q, tr, F):
    """Mat4::from_scale_rotation_translation: each axis is a Vec4 with w = 0 multiplied by its scale (w = 0 * s)."""
    ax = _axes(q, F)
    cols = [np.append(ax[i].astype(F), F(0)) * F(sc[i]) for i in range(3)]
    cols.append(np.array([tr[0], tr[1], tr[2], 1], dtype=F))
    return np.array(cols, dtype=F)                                        # M[col, row]


def _mul(a, b, F):
    if F is f32:
        return glam.mul(a, b)
    return np.array([((a[0] * b[j][0] + a[1] * b[j][1]) + a[2] * b[j][2]) + a[3] * b[j][3] for j in range(4)])


def pose(library, jobs, targets, joint_buf, F=f32):
    """Returns a copy of joint_buf ((n, 16), column major) with every job's matrices written, in dtype F."""
    skins, joints, order, clips, channels, keys = library.arrays()
    out = np.array(joint_buf, dtype=F).reshape(-1, 16).copy()
    ident = np.eye(4, dtype=F)
    with np.errstate(all="ignore"):
        for job in jobs:
            clip = clips[int(job["clip"])]
            sk = skins[int(clip["skin"])]
            first, n = int(sk["first_joint"]), int(sk["joint_count"])
            t = F(job["time"])
            if t < F(0):                                                  # time.clamp(0.0, duration)
                t = F(0)
            if t > F(clip["duration"]):
                t = F(clip["duration"])
            local = []
            for k in range(n):
                ch = channels[int(clip["first_channel"]) + k]
                jt = joints[first + k]
                if not ch["animated"]:
                    local.append(ident.copy())                            # IDENTITY, not the bind pose (lib.rs:219)
                    continue
                tr = jt["bind_translation"].astype(F) if ch["translation"]["times"] == ANIM_ABSENT else _sample3(keys, ch["translation"], t, F)
                q = jt["bind_rotation"].astype(F) if ch["rotation"]["times"] == ANIM_ABSENT else _sample_quat(keys, ch["rotation"], t, F)
                sc = jt["bind_scale"].astype(F) if ch["scale"]["times"] == ANIM_ABSENT else _sample3(keys, ch["scale"], t, F)
                local.append(_from_srt(sc, q, tr, F))
            glob = [None] * n
            for i in range(n):
                k = int(order[first + i])
                p = int(joints[first + k]["parent"])
                if p == ANIM_NO_PARENT:
                    glob[k] = local[k]
                elif p == ANIM_PARENT_NOT_JOINT:
                    glob[k] = _mul(ident, local[k], F)                    # a real multiply: its bits can differ from local
                else:
                    glob[k] = _mul(glob[p], local[k], F)
            for q in range(int(job["target_count"])):
                tg = targets[int(job["first_target"]) + q]
                base = int(tg["joint_matrix_base_offset"])
                for k in range(int(tg["joint_count"])):
                    ib = joints[first + k]["inverse_bind"].astype(F).reshape(4, 4)
                    out[base + k] = _mul(glob[k], ib, F).reshape(16)
    return out


def pose_f64(library, jobs, targets, joint_buf):
    return pose(library, jobs, targets, joint_buf, np.float64)


def same_bits(a, b):
    """Bit equality, any NaN equal to any NaN (the sign and payload of a NaN are not part of rule R12)."""
    a, b = np.asarray(a, dtype=f32), np.asarray(b, dtype=f32)
    return a.shape == b.shape and bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))
