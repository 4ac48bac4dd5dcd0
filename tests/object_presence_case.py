"""A pool world for r3_set_objects_enabled / r3_set_objects_enabled_device and the state they must leave.

The host prepares every slot once (mesh, material, transform, sort key); each frame switches slots on and off.  `pool_state` is what a
slot's presence means for the uploaded arrays: the record's `enabled` word and the live bit (bit 0) of the sort flags follow it, nothing
else changes.  The same state fed through r3_update_objects + r3_update_object_sort_info (`update_path`) is the reference the two new
calls are held to bit for bit."""
import numpy as np

from world_update_scene import ChangingWorld, sort_flags

f32 = np.float32


def pool_world(n_objects=2000, seed=7, blend=True):
    """ChangingWorld's textured cube field as a pool: opaque, cutout (texture alpha) and, with `blend`, key-2 slots; two shadowed
    directional lights and three point lights.  Every slot starts present."""
    return ChangingWorld(n_objects=n_objects, seed=seed, blend=blend)


def pool_state(ev, present):
    """(records, sort flags) of the pool `ev` with `present` (bool per slot) applied."""
    present = np.asarray(present, dtype=bool)
    rec = ev.object_buffer.copy()
    rec["enabled"] = present.astype(rec["enabled"].dtype)
    flags = (sort_flags(ev) & np.uint8(0xFE)) | present.astype(np.uint8)
    return rec, flags.astype(np.uint8)


def state_eval(ev, present):
    """A copy of `ev` whose records and live bits say `present` (for full uploads, e.g. to the oracle)."""
    import copy

    out = copy.copy(ev)
    out.object_buffer, _ = pool_state(ev, present)
    out.object_live = np.asarray(present, dtype=np.uint8).copy()
    return out


def update_path(b, ev, present, slots):
    """`slots` set to `present` through the record and sort-info scatter calls (the way in before r3_set_objects_enabled)."""
    slots = np.asarray(slots, dtype=np.int64)
    if len(slots) == 0:
        return
    rec, flags = pool_state(ev, present)
    b.update_objects(slots.astype(np.uint32), rec[slots])
    b.update_object_sort_info(slots.astype(np.uint32), ev.object_material_key[slots], flags[slots], ev.object_location[slots])


def switch_script(n, rng, watch):
    """Presence per frame (bool (n,)) with the slots that changed: random subsets, all off, all on, the bit-word edges 0, 31, 32, 33 and
    n - 1, and slot `watch` switched off, on and off in successive frames."""
    cur = np.ones(n, dtype=bool)
    frames = []

    def step(new):
        nonlocal cur
        changed = np.flatnonzero(new != cur)
        cur = new.copy()
        frames.append((cur.copy(), changed))
    new = cur.copy(); new[rng.choice(n, n // 3, replace=False)] = False; step(new)
    new = cur.copy(); flip = rng.choice(n, n // 10, replace=False); new[flip] = ~new[flip]; step(new)
    step(np.zeros(n, dtype=bool))
    step(np.ones(n, dtype=bool))
    new = cur.copy(); new[[0, 31, 32, 33, n - 1]] = False; step(new)
    new = cur.copy(); new[[31, 33]] = True; new[watch] = False; step(new)
    new = cur.copy(); new[watch] = True; step(new)
    flip = rng.choice(n, 40, replace=False)
    new = cur.copy(); new[flip[flip != watch]] ^= True; new[watch] = False; step(new)
    return frames
