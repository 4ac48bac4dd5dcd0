"""Worlds for r3_set_deformable_meshes / r3_deform_meshes: meshes built by MeshBuilder (world.py), their deformable-set records, the
objects that draw them, and new positions for a deform — every edge R15 names (handedness, cancelling faces, a 4096-triangle fan,
repeated corners, unreferenced vertices, r = inf, NaN / inf / ±0 positions, authored normals, no uv0, an empty mesh, a 1 M-vertex grid)."""
from dataclasses import dataclass
from typing import List, Optional

import numpy as np

from rend3_b200.layouts import ATTR_ABSENT, DEFORM_LEFT_HANDED, DEFORM_NORMALS, DEFORM_TANGENTS, DEFORMABLE_MESH_DTYPE
from rend3_b200.scenes import cube_example_camera, random_unit_quaternions, trs_matrices
from rend3_b200.world import LEFT, DirectionalLight, EvalOutput, Mesh, MeshBuilder, Object, PbrMaterial, Renderer

import mesh_deform_reference as ref

f32 = np.float32


@dataclass
class MeshSpec:
    positions: np.ndarray
    indices: np.ndarray
    uv: Optional[np.ndarray] = None
    normals: Optional[np.ndarray] = None


def grid(nx, ny, uv=True, size=2.0):
    """nx x ny vertices in the xz plane, two triangles per quad; uv0 [0, 1]^2"""
    u, v = np.meshgrid(np.linspace(0, 1, nx, dtype=f32), np.linspace(0, 1, ny, dtype=f32))
    pos = np.stack([(u - f32(0.5)) * f32(size), np.zeros_like(u), (v - f32(0.5)) * f32(size)], -1).reshape(-1, 3).astype(f32)
    a = (np.arange(ny - 1)[:, None] * nx + np.arange(nx - 1)[None, :]).reshape(-1)
    idx = np.stack([a, a + nx, a + nx + 1, a + nx + 1, a + 1, a], -1).reshape(-1).astype(np.uint32)
    return MeshSpec(pos, idx, np.stack([u, v], -1).reshape(-1, 2).astype(f32) if uv else None)


def double_sided(spec):
    """every triangle twice, the second reversed: the face normals of the two copies nearly cancel"""
    t = spec.indices.reshape(-1, 3)
    return MeshSpec(spec.positions, np.concatenate([t, t[:, ::-1]]).reshape(-1).astype(np.uint32), spec.uv)


def fan(n_tris=4096):
    """vertex 0 at the centre of a closed ring: its corner list holds all n_tris triangles"""
    a = np.linspace(0, 2 * np.pi, n_tris, endpoint=False)
    pos = np.concatenate([[[0, 0.1, 0]], np.stack([np.cos(a), np.zeros_like(a), np.sin(a)], -1)]).astype(f32)
    i = np.arange(n_tris)
    idx = np.stack([np.zeros_like(i), 1 + i, 1 + (i + 1) % n_tris], -1).reshape(-1).astype(np.uint32)
    uv = np.concatenate([[[0.5, 0.5]], np.stack([0.5 + 0.5 * np.cos(a), 0.5 + 0.5 * np.sin(a)], -1)]).astype(f32)
    return MeshSpec(pos, idx, uv)


def repeated_corners(seed=3, n=300, tris=900):
    """random triangles, some naming a vertex twice or three times, and vertices no triangle names"""
    rng = np.random.default_rng(seed)
    pos = rng.standard_normal((n, 3)).astype(f32)
    t = rng.integers(0, n - 20, (tris, 3))
    t[::7, 1] = t[::7, 0]
    t[::11, 2] = t[::11, 0]
    t[::29, 1:] = t[::29, :1]
    return MeshSpec(pos, t.reshape(-1).astype(np.uint32), rng.uniform(0, 1, (n, 2)).astype(f32))


def uv_degenerate():
    """a grid whose uv0 is constant on one half: uv1.x uv2.y - uv1.y uv2.x = 0, so r = 1 / 0 = inf there"""
    s = grid(9, 9)
    s.uv[s.positions[:, 0] < 0] = f32(0.25)
    return s


def authored_normals():
    """a grid built with its own normals and uv0: only tangents are recomputed, against those normals"""
    s = grid(12, 7)
    rng = np.random.default_rng(5)
    s.normals = rng.standard_normal((len(s.positions), 3)).astype(f32)
    return s


def empty():
    return MeshSpec(np.zeros((0, 3), f32), np.zeros(0, np.uint32))


def edge_specs() -> List[MeshSpec]:
    return [grid(17, 9), double_sided(grid(6, 5)), fan(), repeated_corners(), uv_degenerate(), grid(8, 8, uv=False), authored_normals(),
            empty(), grid(5, 5)]


SPECIAL = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0], dtype=f32)


def wave(pos, t, seed=0, specials=False):
    """new positions: a travelling wave over the rest pose; with `specials`, NaN, inf and ±0 written into some components"""
    p = np.asarray(pos, dtype=f32).copy()
    if len(p) == 0:
        return p
    p[:, 1] += (f32(0.3) * np.sin(f32(3.0) * p[:, 0] + f32(t)) * np.cos(f32(2.0) * p[:, 2] - f32(t))).astype(f32)
    p[:, 0] += (f32(0.05) * np.cos(f32(5.0) * p[:, 2] + f32(t))).astype(f32)
    if specials:
        rng = np.random.default_rng(seed)
        at = rng.integers(0, p.size, max(4, p.size // 30))
        p.reshape(-1)[at] = SPECIAL[np.arange(len(at)) % len(SPECIAL)]
        p[-1, 0] = np.nan    # the last vertex NaN: that component's box is NaN
        p[0, 2] = f32(-0.0)
    return p.astype(f32)


@dataclass
class DeformWorld:
    renderer: Renderer
    ev: EvalOutput
    mesh_ids: List[int]
    meshes: np.ndarray           # DEFORMABLE_MESH_DTYPE, one per mesh id
    slots: np.ndarray            # uint32: the objects that draw the meshes
    object_meshes: np.ndarray    # uint32: their index into `meshes`
    rest: List[np.ndarray]       # each mesh's build positions


def deformable_records(r: Renderer, mesh_ids) -> np.ndarray:
    """the r3_deformable_mesh of meshes added with Renderer.add_mesh"""
    out = np.zeros(len(mesh_ids), dtype=DEFORMABLE_MESH_DTYPE)
    for i, mid in enumerate(mesh_ids):
        m = r.meshes[mid]
        rg = m["ranges"]
        flags = (DEFORM_LEFT_HANDED if m["left_handed"] else 0) | (DEFORM_NORMALS if m["normals_calculated"] else 0) \
            | (DEFORM_TANGENTS if m["tangents_calculated"] else 0)
        out[i] = (rg[0], rg.get(1, ATTR_ABSENT), rg.get(2, ATTR_ABSENT), rg.get(3, ATTR_ABSENT), m["index_start"] // 4, m["index_count"],
                  m["vertex_count"], flags)
    return out


def vectorised_mesh(s: MeshSpec, handedness=LEFT) -> Mesh:
    """MeshBuilder::build of a spec without authored normals, its attributes in build's order, with the restatement's vectorised
    normals and tangents (equal to world.py's loops on finite meshes, and fast enough for a million vertices)"""
    n = len(s.positions)
    nrm = ref.normals(s.positions, s.indices, handedness == LEFT)
    attrs = [(0, s.positions)] + ([(3, s.uv)] if s.uv is not None else []) + [(1, nrm)]
    if s.uv is not None:
        attrs.append((2, ref.tangents(s.positions, nrm, s.uv, s.indices)))
    return Mesh(attrs, n, s.indices, left_handed=handedness == LEFT, normals_calculated=True, tangents_calculated=s.uv is not None)


def build_world(specs: List[MeshSpec], handedness=LEFT, objects_per_mesh=2, seed=0, extent=6.0, undeformed_objects=3,
                vectorised=False) -> DeformWorld:
    """every spec as a mesh (MeshBuilder without normals unless the spec has them; `vectorised`: vectorised_mesh), objects_per_mesh
    objects of each at random transforms, and a few objects of a mesh outside the set; the camera of the cube example, one shadowed
    light"""
    rng = np.random.default_rng(seed)
    r = Renderer(handedness, aspect_ratio=16 / 9)
    r.add_material(PbrMaterial(albedo_value=(0.6, 0.5, 0.4, 1.0), roughness_factor=0.5))
    r.add_material(PbrMaterial(albedo_value=(0.3, 0.6, 0.8, 1.0), roughness_factor=0.3))
    r.set_camera_data(cube_example_camera(2.0))
    r.add_directional_light(DirectionalLight(color=(1, 1, 1), intensity=1.0, direction=(-1.0, -4.0, 2.0), distance=40.0, resolution=256))
    mesh_ids = []
    for s in specs:
        if vectorised:
            mesh_ids.append(r.add_mesh(vectorised_mesh(s, handedness)))
            continue
        mb = MeshBuilder.new(s.positions, handedness).with_indices(s.indices)
        if s.normals is not None:
            mb = mb.with_vertex_normals(s.normals)
        if s.uv is not None:
            mb = mb.with_vertex_texture_coordinates_0(s.uv)
        mesh_ids.append(r.add_mesh(mb.build()))
    other = r.add_mesh(MeshBuilder.new(grid(3, 3).positions, handedness).with_indices(grid(3, 3).indices).build())
    slots, object_meshes = [], []
    n = len(specs) * objects_per_mesh + undeformed_objects
    t = trs_matrices(rng.uniform(-extent, extent, (n, 3)).astype(f32), random_unit_quaternions(rng, n),
                     rng.uniform(0.5, 1.5, (n, 1)).astype(f32))
    k = 0
    for i, mid in enumerate(mesh_ids):
        for _ in range(objects_per_mesh):
            slots.append(r.add_object(Object(mid, k % 2, t[k])))
            object_meshes.append(i)
            k += 1
    for _ in range(undeformed_objects):
        r.add_object(Object(other, 0, t[k]))
        k += 1
    ev = r.evaluate()
    return DeformWorld(r, ev, mesh_ids, deformable_records(r, mesh_ids), np.asarray(slots, np.uint32), np.asarray(object_meshes, np.uint32),
                       [np.asarray(s.positions, f32) for s in specs])


def rebuilt_world(specs: List[MeshSpec], new_positions: List[np.ndarray], **kw) -> DeformWorld:
    """the same world with every mesh built from its new positions (the reference's path: build + add_mesh + add of the objects)"""
    moved = [MeshSpec(p, s.indices, s.uv, s.normals) for s, p in zip(specs, new_positions)]
    return build_world(moved, **kw)


def upload(b, ev: EvalOutput):
    """what upload_world sends for the state a deform reads and writes"""
    b.set_objects(ev.object_buffer)
    flags = (ev.object_live & 1) | ((ev.object_atomic & 1) << 1) | ((ev.object_back_to_front & 1) << 2)
    b.set_object_sort_info(ev.object_material_key, flags.astype(np.uint8), np.ascontiguousarray(ev.object_location, dtype=f32))
    b.set_object_mesh_spheres(ev.object_mesh_sphere)
    b.set_mesh_buffer(ev.mesh_buffer)


def bits(a):
    return np.ascontiguousarray(a, dtype=f32).view(np.uint32)


def canon(a):
    """float32 bits with every NaN as 0x7FC00000: the bits of a NaN that arithmetic makes are not part of R15 (x86 and the GPU make
    different default NaNs); copied values keep theirs and are compared as they are"""
    a = np.array(a, dtype=f32)
    a[np.isnan(a)] = np.float32(np.nan)
    return a.view(np.uint32)


def canon_records(r):
    out = np.frombuffer(bytearray(np.ascontiguousarray(r).tobytes()), dtype=r.dtype)
    for f in ("transform", "sphere_center", "sphere_radius"):
        v = out[f]
        v[np.isnan(v)] = np.float32(np.nan)
    return out.tobytes()
