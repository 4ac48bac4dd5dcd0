"""Rule R15 (DESIGN.md §2) restated in numpy: what rebuilding a mesh from new positions (MeshBuilder::build, rend3-types/src/lib.rs:
477-512, 662-702, 784-836; BoundingSphere::from_mesh, util/frustum.rs:15-56) and re-adding its objects (ObjectManager::add,
object.rs:267-284) produce.  Every step is one float32 operation in the reference's order; the sums run in triangle order through
np.add.at, which applies its updates one at a time in the order of the index array.  This is the expected value of r3_deform_meshes."""
import numpy as np

f32 = np.float32


def _cross(a, b):
    """glam.py::cross, row-wise: (a.y b.z - b.y a.z, a.z b.x - b.z a.x, a.x b.y - b.x a.y)"""
    return np.stack([a[:, 1] * b[:, 2] - b[:, 1] * a[:, 2], a[:, 2] * b[:, 0] - b[:, 2] * a[:, 0],
                     a[:, 0] * b[:, 1] - b[:, 0] * a[:, 1]], axis=1).astype(f32)


def _dot(a, b):
    return ((a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]).astype(f32)


def normalize_or_zero(v):
    """Vec3::normalize_or_zero row-wise: rcp = 1 / sqrt(dot(v, v)); v * rcp when rcp is finite and > 0, else zero"""
    with np.errstate(all="ignore"):
        rcp = (f32(1.0) / np.sqrt(_dot(v, v))).astype(f32)
        ok = np.isfinite(rcp) & (rcp > 0)
        return np.where(ok[:, None], (v * rcp[:, None]).astype(f32), f32(0)).astype(f32)


def _edges(pos, tri):
    p1, p2, p3 = pos[tri[:, 0]], pos[tri[:, 1]], pos[tri[:, 2]]
    return (p2 - p1).astype(f32), (p3 - p1).astype(f32)


def normals(pos, indices, left_handed):
    """calculate_normals_for_buffers: face normals summed per vertex from +0.0 in triangle order, then normalize_or_zero"""
    pos = np.asarray(pos, dtype=f32).reshape(-1, 3)
    tri = np.asarray(indices, dtype=np.int64).reshape(-1, 3)
    acc = np.zeros_like(pos)
    with np.errstate(all="ignore"):
        e1, e2 = _edges(pos, tri)
        fn = _cross(e1, e2) if left_handed else _cross(e2, e1)
        np.add.at(acc, tri.reshape(-1), np.repeat(fn, 3, axis=0))
    return normalize_or_zero(acc)


def tangents(pos, nrm, uv, indices):
    """calculate_tangents_for_buffers: r = 1 / (uv1.x uv2.y - uv1.y uv2.x), t = e1 * uv2.y - (e2 * uv1.y) * r summed in triangle order,
    then Gram-Schmidt against the normal and normalize_or_zero.  No nan_to_num: that is world.py's departure."""
    pos = np.asarray(pos, dtype=f32).reshape(-1, 3)
    uv = np.asarray(uv, dtype=f32).reshape(-1, 2)
    tri = np.asarray(indices, dtype=np.int64).reshape(-1, 3)
    acc = np.zeros_like(pos)
    with np.errstate(all="ignore"):
        e1, e2 = _edges(pos, tri)
        uv1 = (uv[tri[:, 1]] - uv[tri[:, 0]]).astype(f32)
        uv2 = (uv[tri[:, 2]] - uv[tri[:, 0]]).astype(f32)
        r = (f32(1.0) / (uv1[:, 0] * uv2[:, 1] - uv1[:, 1] * uv2[:, 0]).astype(f32)).astype(f32)
        t = ((e1 * uv2[:, 1:2]).astype(f32) - ((e2 * uv1[:, 1:2]).astype(f32) * r[:, None]).astype(f32)).astype(f32)
        np.add.at(acc, tri.reshape(-1), np.repeat(t, 3, axis=0))
        n = np.asarray(nrm, dtype=f32).reshape(-1, 3)
        gs = (acc - (n * _dot(n, acc)[:, None]).astype(f32)).astype(f32)
    return normalize_or_zero(gs)


def bbox_sequential(pos):
    """find_mesh_center's fold, literally: acc = first; acc = _mm_max_ps(acc, p) = acc > p ? acc : p (min alike), per component"""
    pos = np.asarray(pos, dtype=f32).reshape(-1, 3)
    mx, mn = [pos[0, c] for c in range(3)], [pos[0, c] for c in range(3)]
    for i in range(1, len(pos)):
        for c in range(3):
            p = pos[i, c]
            mx[c] = mx[c] if mx[c] > p else p
            mn[c] = mn[c] if mn[c] < p else p
    return np.array(mx, dtype=f32), np.array(mn, dtype=f32)


def bbox_r15(pos):
    """R15's parallel form of the same fold, per component: the NaN if the last vertex is NaN; else the largest (smallest) vertex after
    the last NaN, a tie (-0.0 == +0.0 included) going to the later vertex"""
    pos = np.asarray(pos, dtype=f32).reshape(-1, 3)
    n = len(pos)
    mx, mn = np.zeros(3, f32), np.zeros(3, f32)
    for c in range(3):
        x = pos[:, c]
        nan = np.flatnonzero(np.isnan(x))
        start = int(nan[-1]) + 1 if len(nan) else 0
        if start == n:
            mx[c] = mn[c] = x[n - 1]
            continue
        tail = x[start:]
        mx[c] = x[start + np.flatnonzero(tail == tail.max())[-1]]
        mn[c] = x[start + np.flatnonzero(tail == tail.min())[-1]]
    return mx, mn


def mesh_sphere(pos):
    """BoundingSphere::from_mesh under R15: centre = (max + min) / 2, radius = fold of f32::max(0, |p - centre|) (NaN lengths ignored);
    an empty mesh gives zeros.  Returns float32 (cx, cy, cz, r)."""
    pos = np.asarray(pos, dtype=f32).reshape(-1, 3)
    if len(pos) == 0:
        return np.zeros(4, dtype=f32)
    mx, mn = bbox_r15(pos)
    with np.errstate(all="ignore"):
        centre = ((mx + mn).astype(f32) / f32(2.0)).astype(f32)
        d = (pos - centre).astype(f32)
        ln = np.sqrt(_dot(d, d)).astype(f32)
        radius = np.fmax.reduce(ln, initial=f32(0.0))
    return np.array([centre[0], centre[1], centre[2], radius], dtype=f32)


def apply_transform(transforms, spheres):
    """BoundingSphere::apply_transform (rule R12's object half) for records' column-major transforms (n, 16) and spheres (n, 4)"""
    m = np.asarray(transforms, dtype=f32).reshape(-1, 4, 4)   # m[:, j] = column j
    s = np.asarray(spheres, dtype=f32).reshape(-1, 4)
    with np.errstate(all="ignore"):
        ls = [((m[:, j, 0] * m[:, j, 0] + m[:, j, 1] * m[:, j, 1]) + m[:, j, 2] * m[:, j, 2]).astype(f32) for j in range(3)]
        max_scale = np.sqrt(np.fmax(ls[0], np.fmax(ls[1], ls[2]))).astype(f32)
        out = np.zeros((len(m), 4), dtype=f32)
        for r in range(3):
            out[:, r] = (((m[:, 0, r] * s[:, 0] + m[:, 1, r] * s[:, 1]) + m[:, 2, r] * s[:, 2]) + m[:, 3, r] * f32(1.0)).astype(f32)
        out[:, 3] = (max_scale * s[:, 3]).astype(f32)
    return out


def deform_expected(mesh_words, objects, locations, mesh_spheres, meshes, positions, slots, object_meshes):
    """The mesh buffer (u32 words), object records, sort locations and per-slot mesh spheres after a deform, and the per-mesh spheres.
    `meshes`: DEFORMABLE_MESH_DTYPE records; `positions`: (sum vertex_count, 3) in set order; the rest as r3_set_deformable_meshes takes
    them.  Inputs are not modified."""
    from rend3_b200.layouts import DEFORM_LEFT_HANDED, DEFORM_NORMALS, DEFORM_TANGENTS

    words = np.array(mesh_words, dtype=np.uint32).copy()
    # a byte copy: numpy's copy of a structured array need not keep the bytes between its fields
    objs = np.frombuffer(bytearray(np.ascontiguousarray(objects).tobytes()), dtype=objects.dtype)
    loc, ms = np.array(locations, dtype=f32).copy(), np.array(mesh_spheres, dtype=f32).copy()
    pos_all = np.asarray(positions, dtype=f32).reshape(-1, 3)
    spheres, base = np.zeros((len(meshes), 4), dtype=f32), 0
    for i, m in enumerate(meshes):
        vc = int(m["vertex_count"])
        pos = pos_all[base:base + vc]
        base += vc
        idx = words[int(m["first_index"]):int(m["first_index"]) + int(m["index_count"])]
        flags = int(m["flags"])

        def put(off, arr):
            words[int(off) // 4:int(off) // 4 + arr.size] = np.ascontiguousarray(arr, dtype=f32).reshape(-1).view(np.uint32)

        def get(off, k):
            return words[int(off) // 4:int(off) // 4 + k * vc].view(f32).reshape(-1, k).copy()
        uv = get(m["uv0_offset"], 2) if flags & DEFORM_TANGENTS else None
        own_n = get(m["normal_offset"], 3) if (flags & DEFORM_TANGENTS) and not (flags & DEFORM_NORMALS) else None
        put(m["position_offset"], pos)
        n = own_n
        if flags & DEFORM_NORMALS:
            n = normals(pos, idx, bool(flags & DEFORM_LEFT_HANDED))
            put(m["normal_offset"], n)
        if flags & DEFORM_TANGENTS:
            put(m["tangent_offset"], tangents(pos, n, uv, idx))
        spheres[i] = mesh_sphere(pos)
    if len(slots):
        s = np.asarray(slots, dtype=np.int64)
        sph = spheres[np.asarray(object_meshes, dtype=np.int64)]
        ms[s] = sph
        world = apply_transform(objs["transform"][s], sph)
        objs["sphere_center"][s] = world[:, :3]
        objs["sphere_radius"][s] = world[:, 3]
        loc[s] = world[:, :3]
    return words, objs, loc, ms, spheres
