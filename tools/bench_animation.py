"""Crowd animation benchmark: device posing (r3_pose_skeletons) and skinning from resident joint matrices (r3_skin_posed) against the
host path they replace (the oracle's pose on the CPU + r3_skin's per-frame upload and stream drain).  Prints one JSON line.

With --objects K > 0 each instance also carries K posed objects (one per animated node, translation / rotation / scale tracks of 60
keys), and the line gains "objects": the device time of r3_pose_objects (pose + the cull's dense copies) against the host path it
replaces — the oracle's object pose, then r3_update_objects and r3_update_object_sort_info of the posed slots, each ending in a drain.

Workload: --instances instances (default 4096) of a 65-joint humanoid-shaped skin of depth 10, two skeletons (primitives) per instance
of --vertices vertices each (default 1000), one clip with translation, rotation and scale channels of 60 keys on every joint.  The
instances share the two meshes' source attributes and each skeleton has its own skinned ranges, as SkeletonManager lays them out.

With --joint-writes the line gains "joint_writes": skeletons posed by the application (set_skeleton_joint_transforms) for 1 %, 10 % and
100 % of the skeletons per frame (--joint-write-fractions), each a write of 65 globals times the skin's shared inverse binds.  Per
fraction: the device time of joint_write_kernel (192 B per joint: 64 B matrix + 64 B inverse bind read, 64 B written) against the
3.35 TB/s data-sheet bandwidth, the host time of one call, and the frame rate and early flushes of --frames frame graphs that hold the
skinning node — r3_set_joint_matrices (host form) or r3_set_joint_matrices_device, then r3_skin_posed — against r3_skin of the whole
host joint array.

Usage: python tools/bench_animation.py [--instances N] [--vertices V] [--objects K] [--iters I] [--warmup W] [--joint-writes]"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

f32 = np.float32


def skinned_mesh(n_instances, n_vertices, seed=0):
    """Mesh words + one r3_skinning_input per skeleton: 2 meshes' source attributes, then per skeleton its updated position / normal."""
    from rend3_b200.layouts import ATTR_ABSENT, SKINNING_INPUT_DTYPE

    rng = np.random.default_rng(seed)
    parts, cursor = [], 0

    def push(a):
        nonlocal cursor
        raw = np.ascontiguousarray(a).view(np.uint32).reshape(-1)
        parts.append(raw)
        cursor += len(raw)
        return 4 * (cursor - len(raw))

    meshes = []
    for _ in range(2):
        nrm = rng.standard_normal((n_vertices, 3)).astype(f32)
        nrm /= np.linalg.norm(nrm, axis=1, keepdims=True).astype(f32)
        w = rng.random((n_vertices, 4)).astype(f32)
        meshes.append((push(rng.uniform(-1, 1, (n_vertices, 3)).astype(f32)), push(nrm), push(rng.integers(0, 65, (n_vertices, 4)).astype(np.uint16)),
                       push((w / w.sum(axis=1, keepdims=True)).astype(f32))))
    n_skel = 2 * n_instances
    recs = np.zeros(n_skel, dtype=SKINNING_INPUT_DTYPE)
    out_base = cursor
    for s in range(n_skel):
        p, n, j, w = meshes[s % 2]
        recs[s] = (p, n, ATTR_ABSENT, j, w, 4 * (out_base + 6 * n_vertices * s), 4 * (out_base + 6 * n_vertices * s + 3 * n_vertices), ATTR_ABSENT,
                   65 * s, n_vertices)
    parts.append(np.zeros(6 * n_vertices * n_skel, dtype=np.uint32))
    return np.concatenate(parts), recs


def pose_bytes(jobs, targets, library, n_keys):
    """Bytes pose_kernel requests per launch: job + targets, per joint its channel record (64 B), joint record (112 B), per track the
    binary search (ceil(log2 K) + 2 key times) and two key values, and 64 B per matrix stored."""
    joints = int(library.skins["joint_count"][0])
    search = (math.ceil(math.log2(n_keys)) + 2) * 4
    per_joint = 64 + 112 + 3 * search + 2 * (3 + 4 + 3) * 4
    reads = len(jobs) * (16 + joints * per_joint) + 8 * len(targets)
    writes = 64 * int(targets["joint_count"].sum())
    unique = library.channels.nbytes + library.joints.nbytes + library.keys.nbytes + jobs.nbytes + targets.nbytes
    return {"requested_read_bytes": reads, "written_bytes": writes, "distinct_read_bytes": unique}


def object_bench(args, b, device_ms):
    """r3_pose_objects over instances x objects posed objects against the host pose + r3_update_objects + r3_update_object_sort_info."""
    import animation_case
    import object_animation_case
    from oracle.objanim import load_objanim_oracle_backend
    from rend3_b200.animation import Animation, Node, NodeChannels, ObjectAnimationData

    rng = np.random.default_rng(1)
    k, duration = args.objects, 2.0
    nodes = [Node(None, rng.uniform(-3, 3, 3).astype(f32), animation_case._unit_quat(rng), (1.0, 1.0, 1.0),
                  [(i, rng.uniform(-1, 1, 3).astype(f32), f32(1.5))]) for i in range(k)]
    channels = {i: NodeChannels(animation_case._track(rng, 60, 3, duration), animation_case._track(rng, 60, 4, duration),
                                animation_case._track(rng, 60, 3, duration)) for i in range(k)}
    data = ObjectAnimationData(nodes, [Animation(channels, duration)], left_handed=True)
    jobs, targets = data.pose_jobs([(0, float(rng.uniform(0, duration)), i * k) for i in range(args.instances)])
    n = args.instances * k
    records = object_animation_case._records(n, rng)
    key, flags, loc = np.zeros(n, np.uint64), np.ones(n, np.uint8), rng.uniform(-9, 9, (n, 3)).astype(f32)
    b.set_objects(records)
    b.set_object_sort_info(key, flags, loc)
    data.upload(b)
    b.set_object_pose_jobs(jobs, targets)
    pose_ms = device_ms(b.pose_objects)
    got_r, got_l = b.readback_objects(0, n)

    orc = load_objanim_oracle_backend()
    orc.set_objects(records)
    orc.set_object_sort_info(key, flags, loc)
    data.upload(orc)
    orc.set_object_pose_jobs(jobs, targets)
    orc.pose_objects()
    t0 = time.perf_counter()
    for _ in range(5):
        orc.pose_objects()
    host_pose_ms = (time.perf_counter() - t0) * 1e3 / 5
    want_r, want_l = orc.readback_objects(0, n)
    orc.close()
    same = bool(np.array_equal(got_r.view(np.uint32).reshape(n, 32)[:, :30], want_r.view(np.uint32).reshape(n, 32)[:, :30])
                and np.array_equal(got_l.view(np.uint32), want_l.view(np.uint32)))

    slots = np.arange(n, dtype=np.uint32)
    def upload():
        b.update_objects(slots, want_r)
        b.update_object_sort_info(slots, key, flags, want_l)
    for _ in range(3):
        upload()
    t0 = time.perf_counter()
    reps = 20
    for _ in range(reps):
        upload()
    upload_ms = (time.perf_counter() - t0) * 1e3 / reps
    return {"instances": args.instances, "objects_per_instance": k, "objects_posed": n, "pose_objects_ms": round(pose_ms, 4),
            "host_alternative": {"oracle_object_pose_ms": round(host_pose_ms, 3),
                                 "update_objects_and_sort_info_ms": round(upload_ms, 3), "bytes_uploaded_per_frame": n * (128 + 4 + 4 + 8 + 1 + 12)},
            "device_pose_equals_oracle": same}


def joint_write_bench(args, b, recs, buf, device_ms):
    """r3_set_joint_matrices[_device] (set_skeleton_joint_transforms: globals times the skin's shared inverse binds) for a fraction of the
    skeletons per frame, against r3_skin of the whole host joint array.  Frames are recorded as frame graphs (r3_frame_begin / end) that
    hold the skinning node only: the write (or r3_skin) and r3_skin_posed."""
    import torch
    from rend3_b200.layouts import JOINT_WRITE_DTYPE

    rng = np.random.default_rng(3)
    n_skel, nj = len(recs), 65
    binds = rng.uniform(-1, 1, (nj, 16)).astype(f32)
    full = rng.uniform(-1, 1, (len(buf), 16)).astype(f32)   # what r3_skin uploads every frame
    reps = args.frames

    def frames(fn):
        """frames per second of `reps` frame graphs back to back, and early flushes per frame"""
        fn()
        b.sync()
        before = b.frame_graph_stats()["flushed"]
        t0 = time.perf_counter()
        for _ in range(reps):
            b.frame_begin()
            fn()
            b.frame_end()
        b.sync()
        dt = time.perf_counter() - t0
        return reps / dt, (b.frame_graph_stats()["flushed"] - before) / reps

    def host_ms(fn, n=50):
        fn()
        b.sync()
        t0 = time.perf_counter()
        for _ in range(n):
            fn()
        ms = (time.perf_counter() - t0) * 1e3 / n
        b.sync()
        return ms

    skin_fps, skin_flush = frames(lambda: b.skin(recs, full))
    out = {"skeletons": n_skel, "joints_per_skeleton": nj, "frames_per_measure": reps,
           "r3_skin_host_matrices": {"fps": round(skin_fps, 1), "early_flushes_per_frame": skin_flush, "bytes_uploaded_per_frame": full.nbytes},
           "fractions": {}}
    for frac in args.joint_write_fractions:
        n = max(1, round(frac * n_skel))
        chosen = np.sort(rng.choice(n_skel, n, replace=False))
        writes = np.zeros(n, dtype=JOINT_WRITE_DTYPE)
        writes["joint_matrix_base_offset"] = recs["joint_matrix_base_offset"][chosen]
        writes["joint_count"] = nj
        writes["first_matrix"] = nj * np.arange(n)
        mats = rng.uniform(-1, 1, (n * nj, 16)).astype(f32)
        dw, dm, db = (torch.from_numpy(a).cuda() for a in (writes.view(np.int32).reshape(-1, 4), mats, binds))
        torch.cuda.synchronize()
        host_call = lambda: b.set_joint_matrices(writes, mats, binds)
        dev_call = lambda: b.set_joint_matrices_device(dw, dm, db)
        b.set_skeletons(recs, buf)   # both forms start from the same buffer
        host_call()
        via_host = b.readback_joint_matrices(0, len(buf))
        b.set_skeletons(recs, buf)
        dev_call()
        same = bool(np.array_equal(b.readback_joint_matrices(0, len(buf)).view(np.uint32), via_host.view(np.uint32)))
        kernel_ms = device_ms(dev_call)
        joints = n * nj
        host_fps, host_flush = frames(lambda: (host_call(), b.skin_posed()))
        dev_fps, dev_flush = frames(lambda: (dev_call(), b.skin_posed()))
        out["fractions"][str(frac)] = {
            "skeletons_written": n, "joints_written": joints,
            "kernel_ms": round(kernel_ms, 5), "bytes_per_joint": 192,
            "kernel_bytes_per_s": 192 * joints / (kernel_ms * 1e-3),
            "share_of_3_35_tb_s": 192 * joints / (kernel_ms * 1e-3) / 3.35e12,
            "host_form": {"call_host_ms": round(host_ms(host_call), 4), "fps": round(host_fps, 1), "early_flushes_per_frame": host_flush,
                          "bytes_uploaded_per_frame": writes.nbytes + mats.nbytes + binds.nbytes},
            "device_form": {"call_host_ms": round(host_ms(dev_call, 200), 4), "fps": round(dev_fps, 1), "early_flushes_per_frame": dev_flush},
            "device_equals_host": same,
        }
        del dw, dm, db
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--instances", type=int, default=4096)
    ap.add_argument("--vertices", type=int, default=1000)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--objects", type=int, default=0, help="posed objects per instance (0: skeletons only)")
    ap.add_argument("--joint-writes", action="store_true", help="also time r3_set_joint_matrices[_device] against r3_skin (frame graphs)")
    ap.add_argument("--joint-write-fractions", type=lambda s: [float(x) for x in s.split(",")], default=[0.01, 0.1, 1.0])
    ap.add_argument("--frames", type=int, default=50, help="frame graphs per frame-rate measurement (--joint-writes)")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_animation needs a CUDA device")
    import animation_case
    import oracle
    from oracle.anim import load_anim_oracle_backend
    from rend3_b200.backend import load_cuda_backend

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    data, jobs, targets, buf = animation_case.crowd(args.instances)
    words, recs = skinned_mesh(args.instances, args.vertices)
    n_joints = int(targets["joint_count"].sum())

    b = load_cuda_backend(0)
    b.set_mesh_buffer(words)
    b.set_animations(*data.library.arrays())
    b.set_skeletons(recs, buf)
    b.set_pose_jobs(jobs, targets)
    stream = torch.cuda.ExternalStream(b.stream())

    def device_ms(fn):
        for _ in range(args.warmup):
            fn()
        b.sync()
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record(stream)
        for _ in range(args.iters):
            fn()
        stop.record(stream)
        stop.synchronize()
        return start.elapsed_time(stop) / args.iters

    # r3_set_pose_jobs is the per-frame host call of the new path (new times): host clock, the call ends in a stream synchronise
    for _ in range(3):
        b.set_pose_jobs(jobs, targets)
    t0 = time.perf_counter()
    for _ in range(50):
        b.set_pose_jobs(jobs, targets)
    set_jobs_ms = (time.perf_counter() - t0) * 1e3 / 50

    pose_ms = device_ms(b.pose_skeletons)
    skin_ms = device_ms(b.skin_posed)
    posed = b.readback_joint_matrices(0, len(buf))

    # frame-graph flushes per frame: posed path vs r3_skin with host matrices
    def flushes(fn):
        before = b.frame_graph_stats()["flushed"]
        b.frame_begin()
        fn()
        b.frame_end()
        b.sync()
        return b.frame_graph_stats()["flushed"] - before

    flush_posed = flushes(lambda: (b.pose_skeletons(), b.skin_posed()))
    flush_skin = flushes(lambda: b.skin(recs, posed))

    # r3_skin: per-frame upload of the joint matrices + launch + stream drain (host clock around a call that ends in a synchronise)
    for _ in range(3):
        b.skin(recs, posed)
    t0 = time.perf_counter()
    reps = 20
    for _ in range(reps):
        b.skin(recs, posed)
    skin_host_ms = (time.perf_counter() - t0) * 1e3 / reps

    # the host pose: the oracle (C, OpenMP over jobs) on this machine's cores
    threads = oracle.set_threads(os.cpu_count() or 1)
    orc = load_anim_oracle_backend()
    orc.set_animations(*data.library.arrays())
    orc.set_skeletons(recs[:0], buf)
    orc.set_pose_jobs(jobs, targets)
    orc.pose_skeletons()
    t0 = time.perf_counter()
    for _ in range(5):
        orc.pose_skeletons()
    host_pose_ms = (time.perf_counter() - t0) * 1e3 / 5
    same = bool(np.array_equal(orc.readback_joint_matrices(0, len(buf)).view(np.uint32), posed.view(np.uint32)))
    orc.close()
    objects = object_bench(args, b, device_ms) if args.objects > 0 else None
    joint_writes = joint_write_bench(args, b, recs, buf, device_ms) if args.joint_writes else None
    b.close()

    model = pose_bytes(jobs, targets, data.library, 60)
    joints_posed = len(jobs) * int(data.library.skins["joint_count"][0])
    print(json.dumps({
        "workload": {"instances": args.instances, "joints_per_skin": int(data.library.skins["joint_count"][0]), "skeletons": len(recs),
                     "vertices_per_skeleton": args.vertices, "keys_per_track": 60, "joint_matrices_written": n_joints},
        "gpu": smi[0] if smi else torch.cuda.get_device_name(0),
        "pose_skeletons_ms": round(pose_ms, 4), "skin_posed_ms": round(skin_ms, 4), "set_pose_jobs_host_ms": round(set_jobs_ms, 4),
        "set_pose_jobs_bytes": int(jobs.nbytes + targets.nbytes + 8 * len(jobs)),
        "joints_posed_per_s": joints_posed / (pose_ms * 1e-3),
        "pose_byte_model": model, "pose_requested_bytes_per_s": (model["requested_read_bytes"] + model["written_bytes"]) / (pose_ms * 1e-3),
        "early_flushes_per_frame": {"posed": flush_posed, "r3_skin": flush_skin},
        "host_alternative": {"oracle_pose_ms": round(host_pose_ms, 3), "oracle_threads": threads, "r3_skin_upload_and_sync_ms": round(skin_host_ms, 3),
                             "joint_bytes_uploaded_per_frame": 64 * len(buf)},
        "device_pose_equals_oracle": same,
        **({"objects": objects} if objects is not None else {}),
        **({"joint_writes": joint_writes} if joint_writes is not None else {}),
    }))


if __name__ == "__main__":
    main()
