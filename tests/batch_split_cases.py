"""Tiny worlds for the dispatch-limit split of batch_objects (batching.rs:194-209), with their batch tables worked out by hand.

A batch closes before object e when (invocations so far) + triangles(e) >= max_dispatch_count x 256, or when it already holds 256
objects; a region closes at a batch boundary or a material-key change.  Every object is visible and the sort order is the slot order
(keys non-decreasing, distances increasing), so a case is its triangle counts, its keys, the limit and the expected partition.
"""
import numpy as np

from rend3_b200.backend import CAMERA_VIEWPORT
from rend3_b200.layouts import BATCH_DTYPE, REGION_DTYPE
from rend3_b200.routines import per_camera_header
from rend3_b200.scenes import cloud_camera, object_cloud_records

NO_PREVIOUS = 0xFFFFFFFF


def case(tris, max_dispatch, batches, keys=None):
    """batches: the slots of each batch, in order ([] is the leading empty batch)."""
    n = len(tris)
    return {"tris": np.asarray(tris, dtype=np.uint32), "keys": np.zeros(n, dtype=np.uint64) if keys is None else np.asarray(keys, dtype=np.uint64),
            "max_dispatch": max_dispatch, "batches": batches}


CASES = {
    # L = 0: every object opens a batch, the first one behind an empty batch
    "limit0": case([1, 2, 3], 0, [[], [0], [1], [2]]),
    # L = 256: any object after a non-empty one splits, unless it has no triangles
    "limit256": case([10, 0, 100, 300, 5], 1, [[0], [1, 2], [3], [4]]),
    # cur + T lands exactly on L = 768, and one below it
    "exactly_at_limit": case([256, 256, 256], 3, [[0, 1], [2]]),
    "one_below_limit": case([256, 256, 255], 3, [[0, 1, 2]]),
    # T_0 >= L: the reference closes an empty batch first
    "first_alone_at_limit": case([512, 1], 2, [[], [0], [1]]),
    "first_below_limit": case([511, 1], 2, [[0], [1]]),
    # one object alone over L, then small ones share a batch again
    "alone_over_limit": case([10, 1000, 10, 10], 2, [[0], [1], [2, 3]]),
    # object 256 hits the 256-object limit and the dispatch limit (256 x 256 invocations) at once: one split
    "object_and_dispatch_limit": case([1] * 257, 256, [list(range(256)), [256]]),
    # 76,800-triangle meshes at the default limit (65535 x 256): 218 of them fit in a batch
    "big_meshes_default_limit": case([76_800] * 300, 65535, [list(range(218)), list(range(218, 300))]),
    # a material-key change at the split object (one region closes), and one inside a batch (a new region in the same batch)
    "key_change_at_split": case([300, 300, 10], 2, [[0], [1], [2]], keys=[0, 1, 1]),
    "key_change_inside": case([300, 10, 10], 2, [[0], [1, 2]], keys=[0, 0, 1]),
}


def load(backend, c, n_extra_dead=0):
    """Upload the case's world (every slot live, atomic capable, visible) and run batch_objects at the origin."""
    tris = c["tris"]
    n = len(tris)
    rec = object_cloud_records(n, seed=31, extent=50.0, disabled_fraction=0.0)
    rec["sphere_radius"][:] = 1.0e6
    rec["index_count"] = tris * 3
    loc = np.zeros((n, 3), dtype=np.float32)
    loc[:, 0] = np.arange(1, n + 1, dtype=np.float32)       # distance grows with the slot: the sort order is the slot order
    backend.set_objects(rec)
    backend.set_object_sort_info(c["keys"], np.full(n, 3, dtype=np.uint8), loc)
    backend.object_uniform_upload(CAMERA_VIEWPORT, per_camera_header(cloud_camera(), CAMERA_VIEWPORT, (640, 480), 1, n))
    backend.batch_objects(CAMERA_VIEWPORT, np.zeros(3, dtype=np.float32), c["max_dispatch"])


def expected_tables(c):
    """The batch and region tables of a first frame (no previous invocations) from the hand-made partition."""
    tris, keys = c["tris"], c["keys"]
    batches = np.zeros(len(c["batches"]), dtype=BATCH_DTYPE)
    regions = []
    base = 0
    for b, slots in enumerate(c["batches"]):
        cur = 0
        region_inv = region_obj = 0
        for o, s in enumerate(slots):
            if o > 0 and keys[s] != keys[slots[o - 1]]:
                regions.append((b, int(keys[slots[o - 1]])))
                region_inv, region_obj = cur, 0
            info = batches[b]["object_culling_information"][o]
            info["invocation_start"], info["invocation_end"] = cur, cur + tris[s]
            info["object_id"], info["region_id"] = s, len(regions)
            info["base_region_invocation"], info["local_region_id"] = region_inv, region_obj
            info["previous_global_invocation"], info["atomic_capable"] = NO_PREVIOUS, 1
            region_obj += 1
            cur += (int(tris[s]) + 255) // 256 * 256
        last = slots[-1] if slots else 0                      # the empty batch's region carries the first object's key
        regions.append((b, int(keys[last])))
        batches[b]["total_objects"], batches[b]["total_invocations"], batches[b]["batch_base_invocation"] = len(slots), cur, base
        base += cur
    reg = np.zeros(len(regions), dtype=REGION_DTYPE)
    for r, (job, key) in enumerate(regions):
        reg[r]["job_index"], reg[r]["material_key"] = job, key
    return batches, reg


def assert_same_tables(got_b, got_r, want_b, want_r, what=""):
    """Batches, regions and object_culling_information[:total_objects]; the records past that are unspecified (batching.rs:186)."""
    assert len(got_b) == len(want_b), f"{what}: {len(got_b)} batches, expected {len(want_b)}"
    assert got_r.tobytes() == want_r.tobytes(), f"{what}: region tables differ"
    for f in ("total_objects", "total_invocations", "batch_base_invocation"):
        bad = np.flatnonzero(got_b[f] != want_b[f])
        assert not len(bad), f"{what}: batch {bad[0]} {f}: {got_b[f][bad[0]]} != {want_b[f][bad[0]]}"
    used = np.arange(got_b.dtype["object_culling_information"].shape[0])[None, :] < want_b["total_objects"].astype(np.int64)[:, None]
    g, w = (np.ascontiguousarray(t["object_culling_information"]).view(np.uint32).reshape(len(t), used.shape[1], -1) for t in (got_b, want_b))
    same = (g == w).all(axis=-1) | ~used
    bad = np.argwhere(~same)
    assert not len(bad), f"{what}: batch {bad[0][0]} object {bad[0][1]} differs"
