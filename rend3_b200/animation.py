"""Host mirror of rend3-anim's AnimationData (rend3-anim/src/lib.rs:37-143): turns a glTF-shaped scene — nodes with a parent and a
bind pose, skins, animations with per-node key channels — into the arrays of r3_set_animations, and pose_animation_frame calls into
r3_set_pose_jobs records.

Binding follows AnimationData::from_gltf_scene: a skin's joints are looked up through node_to_joint_idx, its processing order is the
scene's topological order filtered to the skin's joint nodes, and every animation gets one clip per skin (pose_animation_frame poses
every skin of the scene, lib.rs:214; a skin the animation does not touch has no animated joint and comes out as IDENTITY * inverse
bind).  Channels of nodes that are not joints of a skin are left out of that skin's clip: the reference indexes node_to_joint_idx with
them (lib.rs:236) and would panic.

ObjectAnimationData is the object-transform half (lib.rs:192-212): the channels of nodes that carry objects, for
r3_set_object_animations, and r3_set_object_pose_jobs records.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from .layouts import (ANIM_ABSENT, ANIM_CHANNEL_DTYPE, ANIM_CLIP_DTYPE, ANIM_JOINT_DTYPE, ANIM_NO_PARENT, ANIM_NODE_CHANNEL_DTYPE,
                      ANIM_NODE_CLIP_DTYPE, ANIM_NODE_DTYPE, ANIM_PARENT_NOT_JOINT, ANIM_SKIN_DTYPE, OBJECT_POSE_TARGET_DTYPE, POSE_JOB_DTYPE,
                      POSE_TARGET_DTYPE)

f32 = np.float32


@dataclass
class Track:
    """AnimationChannel<T>: key times and one value (Vec3, or Quat x, y, z, w) per key."""
    times: np.ndarray
    values: np.ndarray


@dataclass
class NodeChannels:
    translation: Optional[Track] = None
    rotation: Optional[Track] = None
    scale: Optional[Track] = None


@dataclass
class Node:
    """A scene node: its parent node and local_transform.to_scale_rotation_translation(); `objects` are the primitives of the node's
    object, each (object slot, mesh bounding-sphere centre, radius) — InternalObject::mesh_bounding_sphere."""
    parent: Optional[int] = None
    translation: Sequence[float] = (0.0, 0.0, 0.0)
    rotation: Sequence[float] = (0.0, 0.0, 0.0, 1.0)
    scale: Sequence[float] = (1.0, 1.0, 1.0)
    objects: List[Tuple[int, Sequence[float], float]] = field(default_factory=list)


@dataclass
class Skin:
    joints: List[int]                      # node index of joint k
    inverse_bind: np.ndarray               # (joint count, 16) column major


@dataclass
class Animation:
    channels: Dict[int, NodeChannels]      # keyed by node
    duration: float


@dataclass
class Library:
    """The arrays of r3_anim_library."""
    skins: np.ndarray
    joints: np.ndarray
    order: np.ndarray
    clips: np.ndarray
    channels: np.ndarray
    keys: np.ndarray

    def arrays(self):
        return self.skins, self.joints, self.order, self.clips, self.channels, self.keys


def topological_order(nodes: Sequence[Node]) -> List[int]:
    """Parents before children (GltfSceneInstance::topological_order)."""
    depth = {}

    def d(i):
        if i not in depth:
            chain, j = [], i
            while j is not None and j not in depth:
                chain.append(j)
                j = nodes[j].parent
            base = -1 if j is None else depth[j]
            for k in reversed(chain):
                base += 1
                depth[k] = base
        return depth[i]

    return sorted(range(len(nodes)), key=lambda i: (d(i), i))


class AnimationData:
    """AnimationData::from_gltf_scene over a synthetic scene; `library` holds what r3_set_animations takes."""

    def __init__(self, nodes: Sequence[Node], skins: Sequence[Skin], animations: Sequence[Animation], order: Optional[List[int]] = None):
        order = topological_order(nodes) if order is None else order
        keys: List[np.ndarray] = []
        n_keys = 0

        def push(a):
            nonlocal n_keys
            a = np.ascontiguousarray(a, dtype=f32).reshape(-1)
            keys.append(a)
            n_keys += len(a)
            return n_keys - len(a)

        def track(t: Optional[Track]):
            r = np.zeros((), dtype=ANIM_CHANNEL_DTYPE["translation"])
            if t is None:
                r["times"] = ANIM_ABSENT
                return r
            r["times"] = push(t.times)
            r["count"] = len(t.times)
            r["values"] = push(t.values)
            r["value_count"] = len(t.values)
            return r

        skin_recs, joint_recs, order_out, clips, channels = [], [], [], [], []
        self.clip_of: Dict[Tuple[int, int], int] = {}
        for s, skin in enumerate(skins):
            node_to_joint = {n: k for k, n in enumerate(skin.joints)}
            first = len(joint_recs)
            skin_recs.append((first, len(skin.joints)))
            for k, n in enumerate(skin.joints):
                node = nodes[n]
                j = np.zeros((), dtype=ANIM_JOINT_DTYPE)
                j["bind_translation"], j["bind_rotation"], j["bind_scale"] = node.translation, node.rotation, node.scale
                j["parent"] = ANIM_NO_PARENT if node.parent is None else node_to_joint.get(node.parent, ANIM_PARENT_NOT_JOINT)
                j["inverse_bind"] = np.asarray(skin.inverse_bind[k], dtype=f32).reshape(16)
                joint_recs.append(j)
            order_out += [node_to_joint[n] for n in order if n in node_to_joint]
        for a, anim in enumerate(animations):
            for s, skin in enumerate(skins):
                self.clip_of[(a, s)] = len(clips)
                clips.append((s, len(channels), anim.duration))
                for n in skin.joints:
                    ch = np.zeros((), dtype=ANIM_CHANNEL_DTYPE)
                    nc = anim.channels.get(n)
                    ch["translation"], ch["rotation"], ch["scale"] = track(nc and nc.translation), track(nc and nc.rotation), track(nc and nc.scale)
                    ch["animated"] = nc is not None
                    channels.append(ch)
        self.library = Library(
            np.array(skin_recs, dtype=ANIM_SKIN_DTYPE), np.array(joint_recs, dtype=ANIM_JOINT_DTYPE),
            np.array(order_out, dtype=np.uint32), np.array(clips, dtype=ANIM_CLIP_DTYPE),
            np.array(channels, dtype=ANIM_CHANNEL_DTYPE), np.concatenate(keys) if keys else np.zeros(0, dtype=f32))
        self.n_skins = len(skins)

    def upload(self, backend):
        backend.set_animations(*self.library.arrays())

    def pose_jobs(self, frames: Sequence[Tuple[int, float, Dict[int, List[Tuple[int, int]]]]]):
        """pose_animation_frame(scene, animation, time) for each (animation, time, skeletons) of `frames` — one instance of a scene
        each; `skeletons` maps a skin to its skeletons' (joint_matrix_base_offset, joint_count) — as r3_set_pose_jobs records."""
        jobs, targets = [], []
        for animation, time, skeletons in frames:
            for s in range(self.n_skins):
                sk = skeletons.get(s, [])
                jobs.append((self.clip_of[(animation, s)], time, len(targets), len(sk)))
                targets += sk
        return np.array(jobs, dtype=POSE_JOB_DTYPE), np.array(targets, dtype=POSE_TARGET_DTYPE)


@dataclass
class ObjectLibrary:
    """The arrays of r3_anim_object_library."""
    nodes: np.ndarray
    clips: np.ndarray
    channels: np.ndarray
    keys: np.ndarray
    left_handed: bool

    def arrays(self):
        return self.nodes, self.clips, self.channels, self.keys, self.left_handed


class ObjectAnimationData:
    """The object-transform half of pose_animation_frame (lib.rs:192-212) over a synthetic scene: every animation becomes one clip with
    the channels of the nodes that carry objects (a channel of a node without an object sets nothing), every node its bind pose.
    `library` holds what r3_set_object_animations takes; `pose_jobs` turns pose_animation_frame calls into r3_set_object_pose_jobs
    records.  `left_handed` is renderer.handedness == Handedness::Left."""

    def __init__(self, nodes: Sequence[Node], animations: Sequence[Animation], left_handed: bool = False):
        keys: List[np.ndarray] = []
        n_keys = 0

        def track(t: Optional[Track]):
            nonlocal n_keys
            r = np.zeros((), dtype=ANIM_NODE_CHANNEL_DTYPE["translation"])
            if t is None:
                r["times"] = ANIM_ABSENT
                return r
            for name, a in (("times", t.times), ("values", t.values)):
                a = np.ascontiguousarray(a, dtype=f32).reshape(-1)
                r[name] = n_keys
                keys.append(a)
                n_keys += len(a)
            r["count"], r["value_count"] = len(t.times), len(t.values)
            return r

        node_recs = np.zeros(len(nodes), dtype=ANIM_NODE_DTYPE)
        for i, node in enumerate(nodes):
            node_recs[i]["bind_translation"], node_recs[i]["bind_rotation"], node_recs[i]["bind_scale"] = node.translation, node.rotation, node.scale
        clips, channels = [], []
        self.channel_of: Dict[Tuple[int, int], int] = {}   # (animation, node) -> channel within the clip
        for a, anim in enumerate(animations):
            first = len(channels)
            for n in sorted(anim.channels):
                if not nodes[n].objects:
                    continue
                nc = anim.channels[n]
                ch = np.zeros((), dtype=ANIM_NODE_CHANNEL_DTYPE)
                ch["translation"], ch["rotation"], ch["scale"] = track(nc.translation), track(nc.rotation), track(nc.scale)
                ch["node"] = n
                self.channel_of[(a, n)] = len(channels) - first
                channels.append(ch)
            clips.append((first, len(channels) - first, anim.duration))
        self.library = ObjectLibrary(node_recs, np.array(clips, dtype=ANIM_NODE_CLIP_DTYPE), np.array(channels, dtype=ANIM_NODE_CHANNEL_DTYPE),
                                     np.concatenate(keys) if keys else np.zeros(0, dtype=f32), left_handed)
        self.nodes = list(nodes)

    def upload(self, backend):
        backend.set_object_animations(*self.library.arrays())

    def pose_jobs(self, frames: Sequence[Tuple[int, float, int]]):
        """pose_animation_frame(scene, animation, time) for each (animation, time, slot_offset) of `frames` — one scene instance each,
        whose objects are the nodes' objects with their slots moved by slot_offset — as r3_set_object_pose_jobs records."""
        jobs, targets = [], []
        for animation, time, offset in frames:
            first = len(targets)
            for (a, n), ch in sorted(self.channel_of.items(), key=lambda kv: kv[1]):
                if a != animation:
                    continue
                targets += [(slot + offset, ch, center, radius) for slot, center, radius in self.nodes[n].objects]
            jobs.append((animation, time, first, len(targets) - first))
        out = np.zeros(len(targets), dtype=OBJECT_POSE_TARGET_DTYPE)
        for i, (slot, ch, center, radius) in enumerate(targets):
            out[i]["slot"], out[i]["channel"], out[i]["mesh_sphere_center"], out[i]["mesh_sphere_radius"] = slot, ch, center, radius
        return np.array(jobs, dtype=POSE_JOB_DTYPE), out
