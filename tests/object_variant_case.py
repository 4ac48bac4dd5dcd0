"""A world whose objects switch between prepared mesh and material variants (r3_set_object_variants, r3_switch_object_variants,
r3_switch_object_variants_device), and the state they must leave.

The variants of `VariantWorld` are ChangingWorld's two cube meshes (LOD0: 48 triangles, LOD1: 12) with each material; the group of a
slot whose first material is m holds, in this order, (LOD0, m), (LOD1, m), (LOD0, partner[m]), (LOD1, partner[m]), so a choice is
lod + 2 * swapped.  `choose` re-adds the switched objects in the world's own state (ChangingWorld._refresh: the vectorised
ObjectManager::add at the current transform), which gives the records and sort entries the update path uploads and the oracle renders.
"""
import numpy as np

from rend3_b200.layouts import ATTR_ABSENT, OBJECT_VARIANT_DTYPE, VARIANT_GROUP_DTYPE
from world_update_scene import ChangingWorld, Delta, upload_delta

f32 = np.float32
PARTNER_BLEND = {0: 2, 1: 3, 2: 0, 3: 1}     # opaque <-> blend, cutout <-> opaque
PARTNER_OPAQUE = {0: 3, 1: 0, 2: 0, 3: 1}    # never a key-2 material


def variant_record(r, mesh: int, material: int) -> np.ndarray:
    """What ObjectManager::add takes from a mesh and a material (object.rs:267-284), as one OBJECT_VARIANT_DTYPE record."""
    m, mat = r.meshes[mesh], r.materials[material]
    v = np.zeros((), dtype=OBJECT_VARIANT_DTYPE)
    v["first_index"], v["index_count"], v["material_index"] = m["index_start"] // 4, m["index_count"], material
    v["attr_offset"] = [m["ranges"].get(s, ATTR_ABSENT) for s in range(6)]
    v["sort_flags"] = (int(mat.atomic_capable()) << 1) | (int(mat.back_to_front()) << 2)
    v["material_key"] = mat.key()
    v["mesh_sphere"][:3], v["mesh_sphere"][3] = m["center"], m["radius"]
    return v


class VariantWorld(ChangingWorld):
    def __init__(self, n_objects=2000, seed=7, blend=True, partner=None):
        super().__init__(n_objects=n_objects, seed=seed, blend=blend)
        self.partner = partner or (PARTNER_BLEND if blend else PARTNER_OPAQUE)
        lod0, lod1 = self.meshes[1], self.meshes[0]
        self.lod_mesh = (lod0, lod1)
        table = []
        for m in range(len(self.mats)):
            own = m if blend or m != 2 else 0       # without blend no variant carries the key-2 material
            for mat in (own, self.partner[m]):
                table += [variant_record(self.r, lod0, mat), variant_record(self.r, lod1, mat)]
        self.variants = np.array(table, dtype=OBJECT_VARIANT_DTYPE)
        self.groups = np.zeros(len(self.mats), dtype=VARIANT_GROUP_DTYPE)
        self.groups["first"], self.groups["count"] = 4 * np.arange(len(self.mats)), 4
        self.first_mat = self.mat_ids.copy()
        self.slot_groups = self.first_mat.astype(np.uint32)
        self.choice = np.where(self.mesh_ids == lod0, 0, 1).astype(np.uint32)   # what the slots draw now (not yet a switch)
        ms = np.array([[*self.r.meshes[k]["center"], self.r.meshes[k]["radius"]] for k in self.mesh_ids], dtype=f32)
        self.mesh_spheres = ms

    def variant_of(self, slots, choices):
        return 4 * self.slot_groups[slots] + choices

    def choose(self, choices) -> Delta:
        """Every slot takes variant group.first + choices[slot]: the re-add of the changed slots in the world's state.  The delta names them."""
        choices = np.asarray(choices, dtype=np.uint32)
        changed = np.flatnonzero(choices != self.choice)
        self.choice = choices.copy()
        lod, swapped = choices[changed] & 1, choices[changed] >> 1
        self.mesh_ids[changed] = np.asarray(self.lod_mesh)[lod]
        partner = np.array([self.partner[m] for m in range(len(self.mats))])
        self.mat_ids[changed] = np.where(swapped == 1, partner[self.first_mat[changed]], self.first_mat[changed])
        ms = np.array([[*self.r.meshes[k]["center"], self.r.meshes[k]["radius"]] for k in self.mesh_ids[changed]], dtype=f32).reshape(-1, 4)
        self.mesh_spheres[changed] = ms
        return self._refresh(changed)

    def lod_choices(self, camera_location, threshold, swap):
        """LOD by distance from the camera (LOD1 beyond `threshold`), plus the material swap of the slots in `swap` (bool per slot)."""
        d = np.linalg.norm(self.translation - np.asarray(camera_location, dtype=f32), axis=1)
        return ((d > threshold).astype(np.uint32) + 2 * np.asarray(swap, dtype=np.uint32)).astype(np.uint32)


def update_path(b, w: VariantWorld, d: Delta):
    """The changed slots through r3_update_objects + r3_update_object_sort_info + r3_set_object_mesh_spheres (the way in before the
    variant calls)."""
    if d.objects is None or len(d.objects) == 0:
        return
    upload_delta(b, w.ev, d)
    b.set_object_mesh_spheres(w.mesh_spheres[d.objects.astype(np.int64)], d.objects)


def expected_bound(index_counts, floors):
    """r3_debug_invocation_bound's (sum, largest) of round_up(max(index_count, floor) / 3, 256)."""
    t = ((np.maximum(np.asarray(index_counts, np.int64), np.asarray(floors, np.int64)) // 3 + 255) // 256) * 256
    return int(t.sum()), int(t.max(initial=0))
