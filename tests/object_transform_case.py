"""Cases for r3_set_object_mesh_spheres / r3_set_object_transforms and a numpy float32 restatement of what they compute.

`move_objects` is rule R12's object half (DESIGN.md §2) for whole arrays: every step one IEEE f32 operation on float32 arrays — numpy's
element-wise ufuncs never contract — in the order of tests/object_anim_reference.py::set_object_transform, which it must equal bit for
bit; so must the oracle and the CUDA kernel."""
import numpy as np

from harness import to_device
from rend3_b200.scenes import object_cloud_records, random_unit_quaternions, trs_matrices

f32 = np.float32


def move_objects(matrices, mesh_spheres):
    """(spheres (n, 4), locations (n, 3)) of objects with transforms `matrices` (n, 16) column-major and mesh spheres (n, 4)."""
    m = np.asarray(matrices, dtype=f32).reshape(-1, 4, 4)            # m[:, column, row]
    ms = np.asarray(mesh_spheres, dtype=f32).reshape(-1, 4)
    with np.errstate(all="ignore"):
        ls = [(m[:, a, 0] * m[:, a, 0] + m[:, a, 1] * m[:, a, 1]) + m[:, a, 2] * m[:, a, 2] for a in range(3)]   # Vec3::length_squared
        max_scale = np.sqrt(np.fmax(ls[0], np.fmax(ls[1], ls[2])))   # f32::max ignores a NaN operand, as np.fmax does
        out = np.empty((len(m), 4), dtype=f32)
        for r in range(3):                                           # mul_vec4(matrix, (c, 1)): ((x cx + y cy) + z cz) + w 1
            out[:, r] = ((m[:, 0, r] * ms[:, 0] + m[:, 1, r] * ms[:, 1]) + m[:, 2, r] * ms[:, 2]) + m[:, 3, r] * f32(1)
        out[:, 3] = max_scale * ms[:, 3]
        zero = f32(0)
        loc = np.stack([m[:, 3, r] + ((m[:, 0, r] * zero + m[:, 1, r] * zero) + m[:, 2, r] * zero) for r in range(3)], axis=1)
    return out, loc.astype(f32)


def moved_records(records, locations, mesh_spheres, matrices, slots=None):
    """Copies of (records, locations) with `matrices` applied to `slots` (None: slots 0 .. n-1).  Slots at or past len(records) are
    dropped; locations exist only below len(locations)."""
    rec, loc = records.copy(), np.array(locations, dtype=f32).reshape(-1, 3).copy()
    mats = np.asarray(matrices, dtype=f32).reshape(-1, 16)
    s = np.arange(len(mats)) if slots is None else np.asarray(slots, dtype=np.int64)
    keep = s < len(rec)
    s, mats = s[keep], mats[keep]
    sph, l = move_objects(mats, np.asarray(mesh_spheres, dtype=f32).reshape(-1, 4)[s])
    rec["transform"][s], rec["sphere_center"][s], rec["sphere_radius"][s] = mats, sph[:, :3], sph[:, 3]
    in_loc = s < len(loc)
    loc[s[in_loc]] = l[in_loc]
    return rec, loc


def same_bits(a, b):
    """Equal bit for bit, except that any NaN equals any NaN."""
    a, b = np.ascontiguousarray(a, dtype=f32), np.ascontiguousarray(b, dtype=f32)
    return a.shape == b.shape and bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


def same_records(a, b):
    """Records equal: the float fields by same_bits, every other field exactly (field by field: the record has padding, which numpy's
    structured copies do not carry)."""
    floats = ("transform", "sphere_center", "sphere_radius")
    return len(a) == len(b) and all(same_bits(a[f], b[f]) if f in floats else a[f].tobytes() == b[f].tobytes() for f in a.dtype.names)


def world(n, seed=3, extent=60.0):
    """(records, key, flags, locations, mesh spheres) of an object cloud whose mesh spheres are off-centre and of varied radius."""
    rec = object_cloud_records(n, seed=seed, extent=extent)
    rng = np.random.default_rng(seed + 100)
    key = rng.integers(0, 3, n).astype(np.uint64)
    flags = (1 | 2 * rng.integers(0, 2, n) | 4 * (key == 2)).astype(np.uint8)
    ms = np.concatenate([rng.uniform(-0.5, 0.5, (n, 3)), rng.uniform(0.2, 2.0, (n, 1))], axis=1).astype(f32)
    return rec, key, flags, rec["sphere_center"].copy(), ms


def seeded_matrices(n, seed=5, extent=60.0):
    """TRS matrices with non-uniform, sometimes negative scale."""
    rng = np.random.default_rng(seed)
    t = trs_matrices(rng.uniform(-extent, extent, (n, 3)).astype(f32), random_unit_quaternions(rng, n), np.ones((n, 1), f32)).reshape(n, 4, 4)
    sc = (rng.uniform(0.2, 3.0, (n, 3)) * rng.choice([-1.0, 1.0], (n, 3), p=[0.15, 0.85])).astype(f32)
    t[:, :3, :] *= sc[:, :, None]
    return np.ascontiguousarray(t.reshape(n, 16), dtype=f32)


def edge_matrices():
    """(matrices (k, 16), mesh spheres (k, 4), names): the rule's edges."""
    ident = np.eye(4, dtype=f32)
    inf, nan = f32(np.inf), f32(np.nan)
    cases = []

    def add(name, m, sphere=(0.25, -0.5, 0.75, 1.5)):
        cases.append((name, np.asarray(m, dtype=f32).reshape(16), np.asarray(sphere, dtype=f32)))
    m = ident.copy(); m[3, :3] = (1, 2, 3)
    add("affine", m)
    m = m.copy(); m[2, 3] = f32(-0.0)
    add("row 3 (+0, +0, -0, 1)", m)
    m = m.copy(); m[:, 3] = (0.1, -0.2, 0.3, 0.9)
    add("row 3 arbitrary", m)
    m = ident.copy(); m[0, 0], m[1, 1] = -2.0, 0.5
    add("negative scale", m)
    m = ident.copy(); m[0, 0] = m[1, 1] = m[2, 2] = 0.0; m[3, :3] = (4, 5, 6)
    add("zero scale", m)
    m = ident.copy(); m[1, 2] = inf; m[3, :3] = (1, 1, 1)
    add("inf in an axis: NaN location", m)
    m = ident.copy(); m[0, 1] = nan; m[1, 1] = 3.0
    add("NaN in one axis: f32::max ignores it", m)
    m = ident.copy(); m[:3, :3] = nan
    add("NaN in every axis", m)
    m = ident.copy(); m[3, 0] = nan
    add("NaN translation", m)
    m = ident.copy(); m[0, 0] = 2.0; m[3, :3] = (7, 8, 9)
    add("zero-radius mesh sphere", m, (1.0, 2.0, 3.0, 0.0))
    add("zero mesh sphere", m, (0.0, 0.0, 0.0, 0.0))
    m = ident.copy(); m[0, 0] = f32(1e20); m[1, 1] = f32(1e-30)
    add("overflowing length squared", m)
    names, mats, spheres = zip(*cases)
    return np.stack(mats), np.stack(spheres), list(names)


def apply(b, form, mats, slots):
    """One move through the host or the device form; returns what must stay alive until the stream has drained."""
    if form == "host":
        b.set_object_transforms(mats, slots)
        return None
    keep = (to_device(b, mats.reshape(-1, 16)), None if slots is None else to_device(b, np.asarray(slots, dtype=np.uint32).view(np.int32)))
    b.set_object_transforms_device(keep[0], keep[1])
    return keep
