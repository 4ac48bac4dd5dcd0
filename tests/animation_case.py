"""Seeded glTF-shaped scenes for the skeletal-animation tests: skins of many shapes and sizes, bound with rend3_b200.animation's
AnimationData, and pose jobs at awkward times.

Covered on purpose: a chain of 200 levels, a star, a humanoid tree, random trees of 1 / 31 / 32 / 33 / 255 / 1024 joints; joints whose
parent node is not a joint and joints the clip does not animate; channels with only some of T / R / S, single-key channels, consecutive
quaternion keys with a negative dot and with a dot of exactly -0.0; times on keys, before the first key, at the last key, beyond the
duration, NaN and +-inf; several targets per job and targets that keep fewer joints than the skin has."""
import numpy as np

from rend3_b200 import glam
from rend3_b200.animation import Animation, AnimationData, Node, NodeChannels, Skin, Track

f32 = np.float32


def _unit_quat(rng):
    q = rng.standard_normal(4)
    return (q / np.linalg.norm(q)).astype(f32)


def _random_node(rng, parent):
    return Node(parent, rng.uniform(-1, 1, 3).astype(f32), _unit_quat(rng), rng.uniform(0.5, 1.5, 3).astype(f32))


def _parents(shape, n, rng):
    """Parent joint index (or -1) of joints 0..n-1 of one skin."""
    if shape == "chain":
        return [-1] + list(range(n - 1))
    if shape == "star":
        return [-1] + [0] * (n - 1)
    if shape == "humanoid":   # spine of 6, head of 3, two arms of 5 + two hands of 15, two legs of 6
        p = [-1, 0, 1, 2, 3, 4, 5, 6, 7]
        for _side in range(2):
            base = len(p)
            p += [3, base, base + 1, base + 2, base + 3]
            wrist = base + 4
            for _finger in range(5):
                f = len(p)
                p += [wrist, f, f + 1]
        for _side in range(2):
            base = len(p)
            p += [0, base, base + 1, base + 2, base + 3, base + 4]
        return p[:n] if n <= len(p) else p + [int(rng.integers(0, len(p) + i)) for i in range(n - len(p))]
    return [-1] + [int(rng.integers(0, i)) for i in range(1, n)]


def _track(rng, n_keys, width, t_end, special=None):
    times = np.sort(rng.uniform(0, t_end, n_keys)).astype(f32)
    times = np.unique(times)
    if width == 4:
        vals = np.array([_unit_quat(rng) for _ in times], dtype=f32)
        if special == "negative_dot" and len(vals) >= 2:
            vals[1] = -vals[0] + f32(0.05) * _unit_quat(rng)
            vals[1] /= np.linalg.norm(vals[1])
        if special == "negzero_dot" and len(vals) >= 2:
            vals[0] = (1, 0, 0, 0)
            vals[1] = (-0.0, -1.0, -0.0, -0.0)
    else:
        vals = rng.uniform(-1.5, 1.5, (len(times), 3)).astype(f32) if width == 3 else None
    return Track(times, vals)


def skin_scene(shape, n_joints, seed, n_animations=2, outside_parent=True):
    """One skin of n_joints over a scene whose root node is not a joint (so the skin's root joints have a non-joint parent when
    `outside_parent`), with n_animations clips."""
    rng = np.random.default_rng(seed)
    par = _parents(shape, n_joints, rng)
    nodes = [_random_node(rng, None)]                                   # node 0: a non-joint parent
    for k in range(n_joints):
        root_parent = 0 if outside_parent and k % 2 == 0 else None
        nodes.append(_random_node(rng, root_parent if par[k] < 0 else par[k] + 1))
    joints = list(range(1, n_joints + 1))
    inv_bind = np.array([glam.from_scale_rotation_translation(rng.uniform(0.5, 1.5, 3), _unit_quat(rng), rng.uniform(-1, 1, 3)).reshape(16)
                         for _ in joints], dtype=f32)
    animations = []
    for a in range(n_animations):
        duration = float(rng.uniform(1.0, 3.0))
        channels = {}
        for k, node in enumerate(joints):
            if rng.random() < 0.15:                                     # unanimated joint: IDENTITY local
                continue
            n_keys = int(rng.choice([1, 2, 5, 30, 120]))
            special = "negzero_dot" if k == 1 else "negative_dot" if k % 7 == 3 else None
            has = rng.random(3) < 0.7
            if not has.any():
                has[int(rng.integers(0, 3))] = True
            channels[node] = NodeChannels(
                _track(rng, n_keys, 3, duration) if has[0] else None,
                _track(rng, 2 if special else n_keys, 4, duration, special) if has[1] or special else None,
                _track(rng, n_keys, 3, duration) if has[2] else None)
        animations.append(Animation(channels, duration))
    return nodes, [Skin(joints, inv_bind)], animations


def times_for(animation, rng):
    """Key times, before / at / beyond the ends, NaN and infinities."""
    tracks = [t for c in animation.channels.values() for t in (c.translation, c.rotation, c.scale) if t is not None]
    some = tracks[0] if tracks else Track(np.array([0.5 * animation.duration], dtype=f32), None)
    on_key = float(some.times[len(some.times) // 2])
    return [on_key, float(some.times[0]), float(some.times[-1]), -0.5, 0.0, float(animation.duration), float(animation.duration) + 1.0,
            float("nan"), float("inf"), float("-inf"), float(rng.uniform(0, animation.duration))]


def case(shape, n_joints, seed=0):
    """(library, jobs, targets, initial joint buffer): every clip at every time of times_for, two skeletons per job, the second keeping
    fewer joints than the skin when it has more than one, plus an untouched range at the end of the buffer."""
    rng = np.random.default_rng(seed + 1000)
    nodes, skins, animations = skin_scene(shape, n_joints, seed)
    data = AnimationData(nodes, skins, animations)
    frames, base = [], 0
    for a, anim in enumerate(animations):
        for t in times_for(anim, rng):
            short = max(n_joints - 1 - int(rng.integers(0, max(n_joints // 4, 1))), 1) if n_joints > 1 else 1
            frames.append((a, t, {0: [(base, n_joints), (base + n_joints, short)]}))
            base += n_joints + short
    jobs, targets = data.pose_jobs(frames)
    buf = rng.uniform(-2, 2, (base + 3, 16)).astype(f32)                # 3 trailing matrices no job writes
    return data.library, jobs, targets, buf


SHAPES = [("chain", 200), ("star", 32), ("humanoid", 65), ("random", 1), ("random", 31), ("random", 32), ("random", 33), ("random", 255),
          ("random", 1024)]


def overlap_case(seed=0, n_a=30, n_b=40, small_only=False):
    """Two skins over ONE joint range: skin A = joints [0, n_a) (a chain), skin B = [0, n_b) (A's chain plus a second chain rooted at
    joint n_a), one shared topological order, both animated by clips over the same channel records — built directly as library arrays
    (AnimationData gives every skin joint records of its own).  `small_only` poses only skin A."""
    from rend3_b200.animation import Library
    from rend3_b200.layouts import (ANIM_ABSENT, ANIM_CHANNEL_DTYPE, ANIM_CLIP_DTYPE, ANIM_JOINT_DTYPE, ANIM_NO_PARENT, ANIM_SKIN_DTYPE,
                                    POSE_JOB_DTYPE, POSE_TARGET_DTYPE)

    rng = np.random.default_rng(seed)
    joints = np.zeros(n_b, dtype=ANIM_JOINT_DTYPE)
    for k in range(n_b):
        joints[k]["parent"] = ANIM_NO_PARENT if k in (0, n_a) else k - 1
        joints[k]["bind_translation"], joints[k]["bind_rotation"], joints[k]["bind_scale"] = rng.uniform(-1, 1, 3), _unit_quat(rng), rng.uniform(0.5, 1.5, 3)
        joints[k]["inverse_bind"] = glam.from_scale_rotation_translation(rng.uniform(0.5, 1.5, 3), _unit_quat(rng), rng.uniform(-1, 1, 3)).reshape(16)
    keys, channels, duration = [], np.zeros(n_b, dtype=ANIM_CHANNEL_DTYPE), 2.0
    n_keys = 0
    for k in range(n_b):
        channels[k]["animated"] = k % 5 != 4
        for prop, width in (("translation", 3), ("rotation", 4), ("scale", 3)):
            if rng.random() < 0.25:
                channels[k][prop]["times"] = ANIM_ABSENT
                continue
            tr = _track(rng, int(rng.integers(1, 12)), width, duration)
            channels[k][prop]["times"], channels[k][prop]["count"] = n_keys, len(tr.times)
            keys.append(tr.times)
            n_keys += len(tr.times)
            channels[k][prop]["values"], channels[k][prop]["value_count"] = n_keys, len(tr.times)
            keys.append(tr.values.reshape(-1))
            n_keys += tr.values.size
    library = Library(np.array([(0, n_a), (0, n_b)], dtype=ANIM_SKIN_DTYPE), joints, np.arange(n_b, dtype=np.uint32),
                      np.array([(0, 0, duration), (1, 0, duration)], dtype=ANIM_CLIP_DTYPE), channels, np.concatenate(keys).astype(f32))
    jobs, targets, base = [], [], 0
    for t in (0.0, 0.37, 1.2, 2.0, 5.0):
        for clip, n in ((0, n_a),) if small_only else ((0, n_a), (1, n_b)):
            jobs.append((clip, t, len(targets), 1))
            targets.append((base, n))
            base += n
    buf = rng.uniform(-2, 2, (base + 2, 16)).astype(f32)
    return library, np.array(jobs, dtype=POSE_JOB_DTYPE), np.array(targets, dtype=POSE_TARGET_DTYPE), buf


def mixed_case(seed=0):
    """One launch mixing skins that fit in shared memory (65 joints) with one that spills to the global scratch (1024 joints)."""
    na, sa, aa = skin_scene("humanoid", 65, seed, n_animations=1)
    nb, sb, ab = skin_scene("random", 1024, seed + 1, n_animations=1)
    off = len(na)
    nodes = na + [Node(None if n.parent is None else n.parent + off, n.translation, n.rotation, n.scale) for n in nb]
    skins = sa + [Skin([j + off for j in s.joints], s.inverse_bind) for s in sb]
    channels = dict(aa[0].channels)
    channels.update({k + off: v for k, v in ab[0].channels.items()})
    data = AnimationData(nodes, skins, [Animation(channels, max(aa[0].duration, ab[0].duration))])
    frames, base = [], 0
    for t in (0.1, 0.9, 1.7, float("nan")):
        frames.append((0, t, {0: [(base, 65), (base + 65, 40)], 1: [(base + 105, 1024)]}))
        base += 105 + 1024
    jobs, targets = data.pose_jobs(frames)
    buf = np.random.default_rng(seed).uniform(-2, 2, (base + 1, 16)).astype(f32)
    return data.library, jobs, targets, buf


def crowd(n_instances=4096, seed=0, n_keys=60):
    """n_instances of a humanoid-shaped skin (65 joints, depth 10), two skeletons each, one clip with T / R / S on every joint."""
    rng = np.random.default_rng(seed)
    nodes, skins, _ = skin_scene("humanoid", 65, seed, n_animations=0, outside_parent=False)
    duration = 2.0
    channels = {}
    for node in skins[0].joints:
        channels[node] = NodeChannels(_track(rng, n_keys, 3, duration), _track(rng, n_keys, 4, duration), _track(rng, n_keys, 3, duration))
    data = AnimationData(nodes, skins, [Animation(channels, duration)])
    frames = [(0, float(rng.uniform(0, duration)), {0: [(130 * i, 65), (130 * i + 65, 65)]}) for i in range(n_instances)]
    jobs, targets = data.pose_jobs(frames)
    return data, jobs, targets, np.zeros((130 * n_instances, 16), dtype=f32)


def _posed_cube_world():
    """The smoke scene whose cube mesh is skinned in place: its position range is overwritten by r3_skin_posed from a copy appended to
    the mesh buffer, so every rendered cube shows the pose."""
    from rend3_b200.layouts import ATTR_ABSENT, SKINNING_INPUT_DTYPE
    from rend3_b200.scenes import cube_field_scene

    ev = cube_field_scene(n_objects=300, seed=7, resolution=(256, 144))
    pos_off, nrm_off = (int(x) for x in ev.object_buffer["attr_offset"][0][:2])
    nv = (nrm_off - pos_off) // 12
    assert nv > 0
    rng = np.random.default_rng(11)
    words = ev.mesh_buffer
    base = len(words)
    idx = rng.integers(0, 4, (nv, 4)).astype(np.uint16)
    w = rng.random((nv, 4)).astype(f32)
    w = (w / w.sum(axis=1, keepdims=True)).astype(f32)
    extra = [words[pos_off // 4: pos_off // 4 + 3 * nv], idx.view(np.uint32).reshape(-1), w.view(np.uint32).reshape(-1)]
    rec = np.zeros(1, dtype=SKINNING_INPUT_DTYPE)
    rec["base_position_offset"] = 4 * base
    rec["joint_indices_offset"] = 4 * (base + 3 * nv)
    rec["joint_weight_offset"] = 4 * (base + 5 * nv)
    rec["updated_position_offset"] = pos_off
    for f in ("base_normal_offset", "base_tangent_offset", "updated_normal_offset", "updated_tangent_offset"):
        rec[f] = ATTR_ABSENT
    rec["vertex_count"] = nv
    ev.mesh_buffer = np.concatenate([words] + extra)
    # a small 4-joint chain whose poses stay near the bind pose
    nodes = [Node(None)] + [Node(k, (0.0, 0.1, 0.0)) for k in range(3)]
    tracks = {n: NodeChannels(Track(np.array([0, 1, 2], f32), np.array([[0, 0, 0], [0.1, 0, 0], [0, 0.1, 0]], f32)),
                              Track(np.array([0, 2], f32), np.array([[0, 0, 0, 1], [0, 0.2, 0, 0.98]], f32) / np.float32(np.linalg.norm([0, 0.2, 0, 0.98]))))
              for n in range(4)}
    data = AnimationData(nodes, [Skin([0, 1, 2, 3], np.tile(glam.identity().reshape(16), (4, 1)))], [Animation(tracks, 2.0)])
    return ev, rec, data
