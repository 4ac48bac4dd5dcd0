"""Seeded scenes for the object-animation tests: nodes that carry objects, bound with rend3_b200.animation's ObjectAnimationData, and
pose jobs at awkward times.

Covered on purpose: both handednesses; tracks absent per property (the bind pose fills in) and a node in the clip with all three
absent; single-key tracks; times before 0, beyond the duration, exactly on keys, NaN and +-inf; negative and zero scales, in the keys
and in the bind pose; several objects on one node; nodes with objects the clip does not animate; many jobs (scene instances)."""
import numpy as np

from animation_case import _track, _unit_quat, times_for
from rend3_b200.animation import Animation, Node, NodeChannels, ObjectAnimationData, Track
from rend3_b200.layouts import OBJECT_DTYPE

f32 = np.float32


def _records(n, rng):
    """n object records with random transforms, spheres and cold fields (the pose must leave the cold fields and `enabled` alone)."""
    rec = np.zeros(n, dtype=OBJECT_DTYPE)
    rec["transform"] = rng.uniform(-2, 2, (n, 16)).astype(f32)
    rec["sphere_center"] = rng.uniform(-5, 5, (n, 3)).astype(f32)
    rec["sphere_radius"] = rng.uniform(0.1, 2, n).astype(f32)
    rec["first_index"] = rng.integers(0, 1000, n)
    rec["index_count"] = 3 * rng.integers(1, 100, n)
    rec["material_index"] = rng.integers(0, 3, n)
    rec["attr_offset"] = rng.integers(0, 1 << 20, (n, 6))
    rec["enabled"] = rng.integers(0, 2, n)
    return rec


def scene(seed, n_nodes=24, n_animations=2, per_node=(1, 3)):
    """Nodes (about 2/3 of them carry 1..3 objects of an instance of `slots_per_instance` slots) and animations over them."""
    rng = np.random.default_rng(seed)
    nodes, slot = [], 0
    for i in range(n_nodes):
        scale = rng.uniform(0.5, 1.5, 3).astype(f32)
        if i % 7 == 5:
            scale[int(rng.integers(0, 3))] = -scale[0]                  # a negative bind scale
        if i % 11 == 9:
            scale[int(rng.integers(0, 3))] = 0.0                        # a zero bind scale
        objs = []
        if rng.random() < 0.67:
            for _ in range(int(rng.integers(per_node[0], per_node[1] + 1))):
                objs.append((slot, rng.uniform(-1, 1, 3).astype(f32), f32(rng.uniform(0.2, 2.0))))
                slot += 1
        nodes.append(Node(None, rng.uniform(-3, 3, 3).astype(f32), _unit_quat(rng), scale, objs))
    animations = []
    for a in range(n_animations):
        duration = float(rng.uniform(1.0, 3.0))
        channels = {}
        for n in range(n_nodes):
            if rng.random() < 0.15:                                     # a node the clip does not animate: its objects stay put
                continue
            has = rng.random(3) < 0.6
            if n % 9 == 4:
                has[:] = False                                          # all three tracks absent: the bind pose
            n_keys = int(rng.choice([1, 2, 5, 30]))
            sc = _track(rng, n_keys, 3, duration) if has[2] else None
            if sc is not None and n % 5 == 1:
                sc.values[len(sc.values) // 2] = (0.0, -1.0, 2.0)       # zero and negative scale keys
            channels[n] = NodeChannels(_track(rng, n_keys, 3, duration) if has[0] else None,
                                       _track(rng, 2 if n % 6 == 3 else n_keys, 4, duration, "negative_dot" if n % 6 == 3 else None) if has[1] else None,
                                       sc)
        animations.append(Animation(channels, duration))
    return nodes, animations, slot


def case(seed=0, left_handed=False, n_nodes=24, instances=None):
    """(data, jobs, targets, records, sort locations): every animation at every time of times_for, one instance of the scene per
    job, instances laid out one after another, plus untouched slots at the end (and in between, when objects of a node go unanimated)."""
    rng = np.random.default_rng(seed + 500)
    nodes, animations, per_instance = scene(seed, n_nodes)
    data = ObjectAnimationData(nodes, animations, left_handed)
    frames = []
    for a, anim in enumerate(animations):
        for t in times_for(anim, rng):
            frames.append((a, t, len(frames) * per_instance))
    if instances is not None:
        frames = [(i % len(animations), float(rng.uniform(-0.2, 3.2)), i * per_instance) for i in range(instances)]
    jobs, targets = data.pose_jobs(frames)
    n = len(frames) * per_instance + 5
    return data, jobs, targets, _records(n, rng), rng.uniform(-9, 9, (n, 3)).astype(f32)


def single_node(channels=None, translation=(1.0, 2.0, 3.0), rotation=(0.0, 0.0, 0.0, 1.0), scale=(1.0, 1.0, 1.0), center=(0.0, 0.0, 0.0),
                radius=1.0, left_handed=False, duration=1.0):
    """One node carrying one object in slot 0 (of 2 slots), animated by `channels` (NodeChannels, default: all tracks absent)."""
    node = Node(None, np.array(translation, f32), np.array(rotation, f32), np.array(scale, f32), [(0, np.array(center, f32), f32(radius))])
    data = ObjectAnimationData([node], [Animation({0: channels or NodeChannels()}, duration)], left_handed)
    return data


def key_track(times, values):
    return Track(np.array(times, f32), np.array(values, f32))


def sort_info(n):
    return np.zeros(n, np.uint64), np.ones(n, np.uint8)


def run(b, data, jobs, targets, records, loc):
    b.set_objects(records)
    b.set_object_sort_info(*sort_info(len(records)), loc)
    data.upload(b)
    b.set_object_pose_jobs(jobs, targets)
    b.pose_objects()
    return b.readback_objects(0, len(records))
