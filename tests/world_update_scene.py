"""A world that changes from frame to frame, for the incremental-update tests.

`ChangingWorld` holds an `EvalOutput` and mutates it in place.  Each step returns a `Delta` naming what changed: object slots,
sort-info entries, a growth of the object buffer, mesh ranges, texture-table entries with their texels, and whether the material
table changed.  One context can then be fed the full arrays (`BaseRenderGraph.upload_world`) and another only the changes (`upload_delta`).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Tuple

import numpy as np

from rend3_b200.layouts import MATERIAL_DTYPE, TEXTURE_DESC_DTYPE
from rend3_b200.scenes import (bulk_object_records, cube_example_camera, eval_with_bulk_objects, random_unit_quaternions,
                               subdivided_cube_mesh, trs_matrices)
from rend3_b200.world import BLEND, CUTOUT, LEFT, DirectionalLight, PbrMaterial, PointLight, Renderer, Texture

f32 = np.float32


@dataclass
class Delta:
    objects: np.ndarray = field(default_factory=lambda: np.zeros(0, dtype=np.uint32))   # distinct slots whose records changed
    sort: Optional[Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]] = None       # (slots, key, flags, location) entries, in order
    resize: Optional[int] = None                                                       # new slot count, applied first
    mesh: List[Tuple[int, np.ndarray]] = field(default_factory=list)                   # (byte offset, u32 words)
    textures: Optional[Tuple[int, np.ndarray, int, np.ndarray]] = None                 # (first entry, descs, texel offset, texel bytes)
    materials: bool = False


def sort_flags(ev) -> np.ndarray:
    return ((ev.object_live & 1) | ((ev.object_atomic & 1) << 1) | ((ev.object_back_to_front & 1) << 2)).astype(np.uint8)


def texture_blob(tex: Texture):
    raw = np.concatenate([np.ascontiguousarray(l).view(np.uint8).reshape(-1) for l in tex.stored_levels()])
    raw = np.concatenate([raw, np.zeros((-len(raw)) % 16, dtype=np.uint8)])
    d = np.zeros(1, dtype=TEXTURE_DESC_DTYPE)
    d["width"], d["height"], d["mip_count"], d["format"] = tex.data.shape[1], tex.data.shape[0], len(tex.stored_levels()), tex.format()
    return d, raw


class ChangingWorld:
    """A textured cube field: two shadowed directional lights, point lights, opaque / cutout / blend materials."""

    def __init__(self, n_objects: int = 3000, seed: int = 7, resolution=(256, 160), blend: bool = True):
        self.rng = rng = np.random.default_rng(seed)
        r = self.r = Renderer(LEFT, aspect_ratio=resolution[0] / resolution[1])
        self.meshes = [r.add_mesh(subdivided_cube_mesh(k, with_uv=True)) for k in (1, 2)]
        img = rng.integers(0, 256, (32, 32, 4), dtype=np.uint8)
        alpha = rng.integers(0, 256, (16, 16, 4), dtype=np.uint8)
        t0, t1 = r.add_texture_2d(Texture(img, srgb=True)), r.add_texture_2d(Texture(alpha, srgb=True))
        self.mats = [r.add_material(PbrMaterial(albedo_texture=t0, roughness_factor=0.5)),
                     r.add_material(PbrMaterial(albedo_texture=t1, roughness_factor=0.6, transparency=CUTOUT, alpha_cutout=0.5)),
                     r.add_material(PbrMaterial(albedo_value=(0.3, 0.6, 0.9, 0.5), roughness_factor=0.4, transparency=BLEND)),
                     r.add_material(PbrMaterial(albedo_value=(0.7, 0.7, 0.7, 1.0), roughness_factor=0.8))]
        r.set_camera_data(cube_example_camera(8.0))
        for d in ((-1.0, -4.0, 2.0), (2.0, -3.0, -1.0)):
            r.add_directional_light(DirectionalLight(color=(1, 1, 1), intensity=0.6, direction=d, distance=80.0, resolution=256))
        for _ in range(3):
            r.add_point_light(PointLight(position=tuple(rng.uniform(-12, 12, 3)), color=tuple(rng.uniform(0.3, 1.0, 3)), radius=15.0, intensity=3.0))
        self.n = n_objects
        self.translation = rng.uniform(-14.0, 14.0, (n_objects, 3)).astype(f32)
        self.quat = random_unit_quaternions(rng, n_objects)
        self.scale = rng.uniform(0.5, 1.4, (n_objects, 1)).astype(f32)
        self.mesh_ids = np.asarray(self.meshes)[rng.integers(0, 2, n_objects)]
        choice = rng.random(n_objects)
        self.mat_ids = np.where(choice < 0.7, 0, np.where(choice < 0.85, 3, 1)).astype(np.uint32)
        if blend:
            self.mat_ids[choice > 0.97] = 2
        self.enabled = np.ones(n_objects, dtype=bool)
        rec, loc = bulk_object_records(r, self._transforms(np.arange(n_objects)), self.mesh_ids, self.mat_ids, capacity=n_objects)
        self.ev = eval_with_bulk_objects(r, rec, loc, n_objects)

    # ---- state -> EvalOutput
    def _transforms(self, slots):
        return trs_matrices(self.translation[slots], self.quat[slots], self.scale[slots])

    def _refresh(self, slots) -> Delta:
        """Rebuild the records and sort info of `slots` from the state; a delta naming them."""
        slots = np.unique(np.asarray(slots, dtype=np.int64))
        if len(slots) == 0:
            return Delta()
        rec, loc = bulk_object_records(self.r, self._transforms(slots), self.mesh_ids[slots], self.mat_ids[slots], enabled=self.enabled[slots],
                                       capacity=len(slots))
        ev, mats = self.ev, self.r.materials
        ev.object_buffer[slots] = rec
        ev.object_location[slots] = loc
        ev.object_material_key[slots] = [mats[m].key() for m in self.mat_ids[slots]]
        ev.object_atomic[slots] = [mats[m].atomic_capable() for m in self.mat_ids[slots]]
        ev.object_back_to_front[slots] = [mats[m].back_to_front() for m in self.mat_ids[slots]]
        ev.object_live[slots] = self.enabled[slots]
        return Delta(objects=slots.astype(np.uint32), sort=self.sort_entries(slots))

    def sort_entries(self, slots):
        ev = self.ev
        slots = np.asarray(slots, dtype=np.int64)
        return (slots.astype(np.uint32), ev.object_material_key[slots].copy(), sort_flags(ev)[slots], ev.object_location[slots].copy())

    def live_slots(self, frac: float) -> np.ndarray:
        live = np.flatnonzero(self.enabled)
        return np.sort(self.rng.choice(live, max(1, int(frac * self.n)), replace=False))

    # ---- changes
    def move(self, frac: float) -> Delta:
        s = self.live_slots(frac)
        self.translation[s] += self.rng.uniform(-1.0, 1.0, (len(s), 3)).astype(f32)
        return self._refresh(s)

    def kill(self, slots) -> Delta:
        self.enabled[slots] = False
        return self._refresh(slots)

    def revive(self, slots) -> Delta:
        self.enabled[slots] = True
        return self._refresh(slots)

    def set_material(self, slots, mat) -> Delta:
        self.mat_ids[slots] = mat
        return self._refresh(slots)

    def wide_key(self, slot: int, key: int) -> Delta:
        """A material key >= 64 on one slot (the host batching sorts it), record unchanged."""
        self.ev.object_material_key[slot] = key
        return Delta(sort=self.sort_entries([slot]))

    def grow(self, extra: int, used: int, texture_size: int = 24) -> Delta:
        """Append a mesh and a texture with a material that uses them, grow the object buffer by `extra` slots and fill the first
        `used` of them with objects of that mesh and material."""
        r, ev = self.r, self.ev
        old_words = len(r.mesh_words)
        mesh = r.add_mesh(subdivided_cube_mesh(3, with_uv=True))
        words = r.mesh_words[old_words:].copy()
        ev.mesh_buffer = r.mesh_words.copy()
        tex = Texture(self.rng.integers(0, 256, (texture_size, texture_size, 4), dtype=np.uint8), srgb=True)
        first, off = len(ev.texture_descs), len(ev.texture_texels)
        desc, raw = texture_blob(tex)
        desc["byte_offset"] = off
        table = np.zeros(first + 1, dtype=TEXTURE_DESC_DTYPE)   # np.concatenate would promote the padded dtype to a packed one
        table[:first], table[first] = ev.texture_descs, desc[0]
        ev.texture_descs = table
        ev.texture_texels = np.concatenate([ev.texture_texels, raw])
        mat = r.add_material(PbrMaterial(albedo_texture=first, roughness_factor=0.3))
        ev.material_buffer = np.zeros(len(r.materials), dtype=MATERIAL_DTYPE)
        for i, m in enumerate(r.materials):
            ev.material_buffer[i] = m.to_record()
        # the object buffer and the sort arrays grow with zeros
        n0, n1 = self.n, self.n + extra
        def grow(a):   # np.concatenate would promote the padded record dtype to a packed one
            out = np.zeros((len(a) + extra,) + a.shape[1:], dtype=a.dtype)
            out[:len(a)] = a
            return out
        ev.object_buffer = grow(ev.object_buffer)
        for f in ("object_material_key", "object_atomic", "object_back_to_front", "object_live", "object_location"):
            setattr(ev, f, grow(getattr(ev, f)))
        self.translation = grow(self.translation); self.quat = grow(self.quat); self.scale = grow(self.scale)
        self.mesh_ids = grow(self.mesh_ids); self.mat_ids = grow(self.mat_ids); self.enabled = grow(self.enabled)
        new = np.arange(n0, n0 + used)
        self.translation[new] = self.rng.uniform(-10.0, 10.0, (used, 3)).astype(f32)
        self.quat[new] = random_unit_quaternions(self.rng, used)
        self.scale[new] = 0.8
        self.mesh_ids[new], self.mat_ids[new], self.enabled[new] = mesh, mat, True
        self.n = n1
        d = self._refresh(new)
        d.resize, d.mesh, d.materials = (n1 if extra else None), [(old_words * 4, words)], True
        d.textures = (first, desc, off, raw)
        return d

    def replace_texture(self, entry: int, texture_size: int = 40) -> Delta:
        """TextureManager::fill of an existing entry with another image (another size): its texels go to the end of the blob."""
        ev = self.ev
        tex = Texture(self.rng.integers(0, 256, (texture_size, texture_size, 4), dtype=np.uint8), srgb=True)
        desc, raw = texture_blob(tex)
        off = len(ev.texture_texels)
        desc["byte_offset"] = off
        ev.texture_descs[entry] = desc[0]
        ev.texture_texels = np.concatenate([ev.texture_texels, raw])
        return Delta(textures=(entry, desc, off, raw))


def merge(*deltas: Delta) -> Delta:
    out = Delta()
    objs = [d.objects for d in deltas if len(d.objects)]
    out.objects = np.unique(np.concatenate(objs)).astype(np.uint32) if objs else out.objects
    sorts = [d.sort for d in deltas if d.sort is not None]
    if sorts:
        out.sort = tuple(np.concatenate([s[k] for s in sorts]) for k in range(4))
    for d in deltas:
        out.resize = d.resize or out.resize
        out.mesh += d.mesh
        out.textures = d.textures or out.textures
        out.materials |= d.materials
    return out


def upload_delta(b, ev, d: Delta):
    """Only the changes, through the incremental entry points (materials keep their full call)."""
    if d.resize is not None:
        b.resize_objects(d.resize)
    if len(d.objects):
        b.update_objects(d.objects, ev.object_buffer[d.objects.astype(np.int64)])
    if d.sort is not None:
        b.update_object_sort_info(*d.sort)
    for off, words in d.mesh:
        b.update_mesh_buffer(off, words)
    if d.textures is not None:
        first, descs, off, raw = d.textures
        b.update_textures(first, descs, off, raw)
    if d.materials:
        b.set_materials(ev.material_buffer)
