"""Worlds for r3_set_remeshable_meshes / r3_remesh_meshes: meshes added at their capacity by world.py (so every range in the mesh buffer
is capacity-sized), their remeshable-set records, and frames of new vertices and indices for them: quads of a grid kept by a moving mask
with the vertices compacted, prefixes of a 4096-triangle fan, random triangles with repeated corners and unreferenced vertices, NaN
positions, supplied normals and tangents, colour0.  The expected state of a remesh is R15's restatement (mesh_deform_reference.py) of
rebuilding each mesh from the new vertices and indices and re-adding its objects."""
from dataclasses import dataclass
from typing import List, Optional

import numpy as np

import mesh_deform_case as dcase
import mesh_deform_reference as ref
from rend3_b200.layouts import (ATTR_ABSENT, DEFORM_LEFT_HANDED, DEFORM_NORMALS, DEFORM_TANGENTS, DEFORMABLE_MESH_DTYPE,
                                REMESHABLE_MESH_DTYPE)
from rend3_b200.scenes import cube_example_camera, random_unit_quaternions, trs_matrices
from rend3_b200.world import LEFT, DirectionalLight, Mesh, MeshBuilder, Object, PbrMaterial, Renderer

f32 = np.float32


@dataclass
class Frame:
    """one mesh's new vertices and indices; normals / tangents only where the mesh takes them from its streams"""
    positions: np.ndarray
    indices: np.ndarray
    uv: Optional[np.ndarray] = None
    normals: Optional[np.ndarray] = None
    tangents: Optional[np.ndarray] = None
    color: Optional[np.ndarray] = None   # (n, 4) uint8


@dataclass
class Kind:
    """one mesh of the set: `capacity` is the Frame it is added with (its ranges' sizes), and which attributes it has"""
    name: str
    capacity: Frame
    uv: bool
    color: bool
    own_normals: bool
    own_tangents: bool


def masked_grid(nx, ny, keep, t=0.0, uv=True, color=False, size=2.0):
    """the quads of an nx x ny grid where keep (ny-1, nx-1) is set, its vertices compacted in grid order by a cumsum over the used ones"""
    s = dcase.grid(nx, ny, uv=uv, size=size)
    pos = dcase.wave(s.positions, t)
    quads = s.indices.reshape(-1, 6)[np.asarray(keep, bool).reshape(-1)]
    used = np.zeros(len(pos), bool)
    used[quads.reshape(-1)] = True
    remap = (np.cumsum(used) - 1).astype(np.uint32)
    f = Frame(pos[used].astype(f32), remap[quads.reshape(-1)].astype(np.uint32), s.uv[used] if uv else None)
    if color:
        f.color = (np.arange(4 * len(pos)).reshape(-1, 4) * 37 % 251).astype(np.uint8)[used]
    return f


def kinds() -> List[Kind]:
    rng = np.random.default_rng(7)
    full = np.ones((11, 15), bool)
    fan = dcase.fan()
    rc = dcase.repeated_corners()
    an = dcase.grid(9, 6)
    return [
        Kind("grid", masked_grid(16, 12, full), True, False, False, False),
        Kind("grid-colour-no-uv", masked_grid(10, 9, np.ones((8, 9), bool), uv=False, color=True), False, True, False, False),
        Kind("fan", Frame(fan.positions, fan.indices, fan.uv), True, False, False, False),
        Kind("repeated", Frame(rc.positions, rc.indices, rc.uv), True, False, False, False),
        Kind("own-normals", Frame(an.positions, an.indices, an.uv, rng.standard_normal((len(an.positions), 3)).astype(f32)),
             True, False, True, False),
        Kind("own-normals-tangents", Frame(an.positions, an.indices, an.uv, rng.standard_normal((len(an.positions), 3)).astype(f32),
                                           rng.standard_normal((len(an.positions), 3)).astype(f32)), True, False, True, True),
    ]


def frame_for(k: Kind, step: int, seed: int = 0, nan: bool = False) -> Frame:
    """step 0: the capacity itself; then shrinking, empty (step 2), growing and varying topologies within the capacity"""
    rng = np.random.default_rng(1000 * seed + step)
    c = k.capacity
    if step == 0:
        f = Frame(c.positions.copy(), c.indices.copy(), c.uv, c.normals, c.tangents, c.color)
    elif step == 2:
        f = Frame(np.zeros((0, 3), f32), np.zeros(0, np.uint32), None if c.uv is None else np.zeros((0, 2), f32),
                  None if c.normals is None else np.zeros((0, 3), f32), None if c.tangents is None else np.zeros((0, 3), f32),
                  None if c.color is None else np.zeros((0, 4), np.uint8))
    elif k.name.startswith("grid"):
        ny, nx = (11, 15) if k.name == "grid" else (8, 9)
        keep = rng.random((ny, nx)) < (0.3 if step == 1 else 0.8)
        src = masked_grid(16 if k.name == "grid" else 10, 12 if k.name == "grid" else 9, keep, t=0.3 * step, uv=c.uv is not None,
                          color=c.color is not None)
        f = src
    else:
        tris = c.indices.reshape(-1, 3)
        n_t = max(1, int(len(tris) * (0.25 if step == 1 else 0.9)))
        pick = np.sort(rng.choice(len(tris), n_t, replace=False))
        idx = tris[pick].reshape(-1).astype(np.uint32)
        n_v = int(min(len(c.positions), idx.max() + 1 + 5))   # a few vertices past the last one named: unreferenced
        f = Frame(dcase.wave(c.positions[:n_v], 0.4 * step), idx, None if c.uv is None else c.uv[:n_v],
                  None if c.normals is None else c.normals[:n_v][::-1].copy(), None if c.tangents is None else c.tangents[:n_v] * f32(0.5),
                  None if c.color is None else c.color[:n_v])
    if nan and len(f.positions):
        f.positions = dcase.wave(f.positions, 0.0, seed=seed, specials=True)
    return f


@dataclass
class RemeshWorld:
    renderer: Renderer
    ev: object
    kinds: List[Kind]
    records: np.ndarray        # REMESHABLE_MESH_DTYPE
    slots: np.ndarray
    object_meshes: np.ndarray


def add_capacity_mesh(r: Renderer, k: Kind, handedness) -> int:
    c = k.capacity
    if k.own_tangents:   # world.py's MeshBuilder always computes tangents from uv0: a mesh with its own is made directly
        attrs = [(0, c.positions), (1, c.normals), (3, c.uv), (2, c.tangents)]
        return r.add_mesh(Mesh(attrs, len(c.positions), c.indices, left_handed=handedness == LEFT))
    mb = MeshBuilder.new(c.positions, handedness).with_indices(c.indices)
    if k.own_normals:
        mb = mb.with_vertex_normals(c.normals)
    if k.uv:
        mb = mb.with_vertex_texture_coordinates_0(c.uv)
    if k.color:
        mb = mb.with_vertex_color_0(c.color)
    return r.add_mesh(mb.build())


def remeshable_records(r: Renderer, mesh_ids) -> np.ndarray:
    out = np.zeros(len(mesh_ids), dtype=REMESHABLE_MESH_DTYPE)
    for i, mid in enumerate(mesh_ids):
        m = r.meshes[mid]
        rg = m["ranges"]
        flags = (DEFORM_LEFT_HANDED if m["left_handed"] else 0) | (DEFORM_NORMALS if m["normals_calculated"] else 0) \
            | (DEFORM_TANGENTS if m["tangents_calculated"] else 0)
        out[i] = (rg[0], rg.get(1, ATTR_ABSENT), rg.get(2, ATTR_ABSENT), rg.get(3, ATTR_ABSENT), rg.get(5, ATTR_ABSENT),
                  m["index_start"] // 4, m["index_count"], m["vertex_count"], flags)
    return out


def build_world(ks: List[Kind], handedness=LEFT, objects_per_mesh=2, seed=0, extent=6.0, undeformed_objects=3) -> RemeshWorld:
    rng = np.random.default_rng(seed)
    r = Renderer(handedness, aspect_ratio=16 / 9)
    r.add_material(PbrMaterial(albedo_value=(0.6, 0.5, 0.4, 1.0), roughness_factor=0.5))
    r.add_material(PbrMaterial(albedo_value=(0.3, 0.6, 0.8, 1.0), roughness_factor=0.3))
    r.set_camera_data(cube_example_camera(2.0))
    r.add_directional_light(DirectionalLight(color=(1, 1, 1), intensity=1.0, direction=(-1.0, -4.0, 2.0), distance=40.0, resolution=256))
    mesh_ids = [add_capacity_mesh(r, k, handedness) for k in ks]
    other = r.add_mesh(MeshBuilder.new(dcase.grid(3, 3).positions, handedness).with_indices(dcase.grid(3, 3).indices).build())
    n = len(ks) * objects_per_mesh + undeformed_objects
    t = trs_matrices(rng.uniform(-extent, extent, (n, 3)).astype(f32), random_unit_quaternions(rng, n), rng.uniform(0.5, 1.5, (n, 1)).astype(f32))
    slots, object_meshes, j = [], [], 0
    for _ in range(undeformed_objects // 2):   # an unrelated slot in front of the set's
        r.add_object(Object(other, 0, t[j])); j += 1
    for i, mid in enumerate(mesh_ids):
        for _ in range(objects_per_mesh):
            slots.append(r.add_object(Object(mid, j % 2, t[j]))); object_meshes.append(i); j += 1
    while j < n:
        r.add_object(Object(other, 0, t[j])); j += 1
    ev = r.evaluate()
    return RemeshWorld(r, ev, ks, remeshable_records(r, mesh_ids), np.asarray(slots, np.uint32), np.asarray(object_meshes, np.uint32))


def streams(w: RemeshWorld, frames: List[Frame], counts=None):
    """the r3_remesh_meshes streams at capacity strides, as keyword arguments of Backend.remesh_meshes; `counts` overrides the frames'"""
    rec = w.records
    vcap, icap = rec["vertex_capacity"].astype(np.int64), rec["index_capacity"].astype(np.int64)
    nv, ni = int(vcap.sum()), int(icap.sum())
    vb, ib = np.r_[0, np.cumsum(vcap)], np.r_[0, np.cumsum(icap)]
    out = dict(counts=np.zeros((len(rec), 2), np.uint32), positions=np.zeros((nv, 3), f32), indices=np.zeros(ni, np.uint32))
    want = dict(normals=(3, f32), tangents=(3, f32), uv0=(2, f32), color0=(1, np.uint32))
    for i, (m, f) in enumerate(zip(rec, frames)):
        v, k = len(f.positions), len(f.indices)
        out["counts"][i] = (v, k)
        out["positions"][vb[i]:vb[i] + v] = f.positions
        out["indices"][ib[i]:ib[i] + k] = f.indices
        for name, a in (("normals", f.normals if not m["flags"] & DEFORM_NORMALS and m["normal_offset"] != ATTR_ABSENT else None),
                        ("tangents", f.tangents if not m["flags"] & DEFORM_TANGENTS and m["tangent_offset"] != ATTR_ABSENT else None),
                        ("uv0", f.uv if m["uv0_offset"] != ATTR_ABSENT else None),
                        ("color0", None if f.color is None or m["color0_offset"] == ATTR_ABSENT else np.ascontiguousarray(f.color).view(np.uint32))):
            if a is None:
                continue
            cols, dt = want[name]
            if name not in out:
                out[name] = np.zeros((nv, cols) if cols > 1 else nv, dt)
            out[name][vb[i]:vb[i] + v] = a.reshape(v, cols) if cols > 1 else a.reshape(v)
    if counts is not None:
        out["counts"] = np.asarray(counts, np.uint32)
    return out


def expected(words, objs, loc, ms, w: RemeshWorld, frames: List[Frame], applied=None):
    """R15's restatement of a remesh from the state (words, objs, loc, ms): every applied mesh (all when `applied` is None) gets its new
    indices and supplied attributes written, then deform_expected rebuilds positions, normals, tangents, spheres and its objects, whose
    index_count becomes the new one.  Returns (words, objs, loc, ms, spheres of the applied meshes)."""
    rec = w.records
    idx = [i for i in range(len(rec)) if applied is None or applied[i]]
    words = np.array(words, dtype=np.uint32).copy()
    dm = np.zeros(len(idx), DEFORMABLE_MESH_DTYPE)
    for j, i in enumerate(idx):
        m, f = rec[i], frames[i]
        v = len(f.positions)
        fi = int(m["first_index"])
        words[fi:fi + len(f.indices)] = f.indices
        for off, a, own in ((m["normal_offset"], f.normals, not m["flags"] & DEFORM_NORMALS),
                            (m["tangent_offset"], f.tangents, not m["flags"] & DEFORM_TANGENTS), (m["uv0_offset"], f.uv, True),
                            (m["color0_offset"], None if f.color is None else np.ascontiguousarray(f.color).view(np.uint32), True)):
            if off != ATTR_ABSENT and own and v:
                flat = np.ascontiguousarray(a).reshape(-1)
                words[int(off) // 4:int(off) // 4 + flat.size] = flat.view(np.uint32)
        dm[j] = (m["position_offset"], m["normal_offset"], m["tangent_offset"], m["uv0_offset"], fi, len(f.indices), v, m["flags"])
    sel = np.isin(w.object_meshes, idx)
    remap = {i: j for j, i in enumerate(idx)}
    om = np.array([remap[int(x)] for x in w.object_meshes[sel]], np.uint32)
    pos = np.concatenate([frames[i].positions for i in idx]) if idx else np.zeros((0, 3), f32)
    words, objs, loc, ms, spheres = ref.deform_expected(words, objs, loc, ms, dm, pos, w.slots[sel], om)
    for s, j in zip(w.slots[sel], om):
        objs["index_count"][int(s)] = dm[j]["index_count"]
    return words, objs, loc, ms, spheres


def upload(b, ev):
    dcase.upload(b, ev)
