"""Cost of meshes whose topology changes every frame, through the three ways new vertices and indices can reach the library.

Workloads (--workloads):
  iso     one isosurface-sized mesh: a 1024 x 1024 grid's capacity (1 048 576 vertices, 6 279 174 indices) with uv0, normals and
          tangents recomputed; each frame keeps the quads outside a disc that moves with the frame, vertices compacted;
  chunks  1000 terrain chunks of 32 x 32 vertices' capacity with uv0; each frame keeps a different random 30-100 % of each chunk's quads.
One object per mesh.  The remesh alone is timed (no rendering), each frame bracketed by r3_frame_begin / r3_frame_end:
  device   r3_remesh_meshes_device from CUDA tensors (enqueue only);
  host     r3_remesh_meshes from host arrays (copies, the kernels, one drain: a recorded frame flushes there);
  rebuild  what the reference does, restated: normals, tangents and mesh spheres in vectorised numpy (its time is reported apart), then
           r3_update_mesh_buffer of the written ranges, r3_update_objects and r3_update_object_sort_info; 2 frames.
Reported: kernel times by group from torch.profiler (the corner-list build apart from the four shared kernels and the validation),
the corner-list build against the byte model below, frames per second and early flushes per frame, and the card's name and power limit
read in the same run.  One JSON document to stdout (and --out).

Byte model of the corner-list build, per index of capacity: the key pass reads 4 B (stream) and writes 4 B (mesh buffer) + 8 B (key);
each radix pass reads the keys twice (histogram, scatter) and writes them once, 24 B; the list pass reads 8 B and writes 4 B; per vertex
of capacity 4 B of list start.  Passes: ceil(bits(vertex capacity) / 8), 3 for both workloads.

    python tools/remesh_cost.py [--workloads iso,chunks] [--frames 20]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import mesh_deform_case as dcase  # noqa: E402
import mesh_deform_reference as ref  # noqa: E402
from rend3_b200.backend import load_cuda_backend  # noqa: E402
from rend3_b200.layouts import ATTR_ABSENT, DEFORM_LEFT_HANDED, DEFORM_NORMALS, DEFORM_TANGENTS, OBJECT_DTYPE, REMESHABLE_MESH_DTYPE  # noqa: E402
from world_update_cost import card  # noqa: E402

f32 = np.float32
HBM_BYTES_PER_S = 3.35e12


class Workload:
    def __init__(self, name, nx, n_meshes, seed=0):
        self.name, self.nx, self.n = name, nx, n_meshes
        self.grid = dcase.grid(nx, nx, size=2.0)
        self.vcap, self.icap = len(self.grid.positions), len(self.grid.indices)
        self.rng = np.random.default_rng(seed)
        # layout: per mesh position, normal, tangent, uv0 ranges, then its indices
        words_per = self.vcap * 11 + self.icap
        self.records = np.zeros(n_meshes, REMESHABLE_MESH_DTYPE)
        self.objects = np.zeros(n_meshes, OBJECT_DTYPE)
        for i in range(n_meshes):
            b = 4 * i * words_per
            p, nrm, tan, uv, ix = b, b + 12 * self.vcap, b + 24 * self.vcap, b + 36 * self.vcap, b + 44 * self.vcap
            self.records[i] = (p, nrm, tan, uv, ATTR_ABSENT, ix // 4, self.icap, self.vcap, DEFORM_LEFT_HANDED | DEFORM_NORMALS | DEFORM_TANGENTS)
            o = self.objects[i]
            o["transform"] = np.eye(4, dtype=f32).reshape(-1)
            o["first_index"], o["index_count"], o["enabled"] = ix // 4, self.icap, 1
            o["attr_offset"] = (p, nrm, tan, uv, ATTR_ABSENT, ATTR_ABSENT)
        self.words = np.zeros(n_meshes * words_per, np.uint32)

    def frame(self, k):
        """(streams at capacity strides, per-mesh (positions, indices, uv)) of frame k"""
        quads = self.grid.indices.reshape(-1, 6)
        centre = self.grid.positions[quads[:, 0]][:, [0, 2]]
        out = dict(counts=np.zeros((self.n, 2), np.uint32), positions=np.zeros((self.n * self.vcap, 3), f32),
                   indices=np.zeros(self.n * self.icap, np.uint32), uv0=np.zeros((self.n * self.vcap, 2), f32))
        meshes = []
        for i in range(self.n):
            if self.n == 1:
                keep = ((centre[:, 0] - 0.5 * np.cos(0.3 * k)) ** 2 + (centre[:, 1] - 0.5 * np.sin(0.3 * k)) ** 2) > 0.1
            else:
                keep = self.rng.random(len(quads)) < self.rng.uniform(0.3, 1.0)
            kept = quads[keep].reshape(-1)
            used = np.zeros(self.vcap, bool)
            used[kept] = True
            remap = (np.cumsum(used) - 1).astype(np.uint32)
            pos, idx, uv = self.grid.positions[used], remap[kept], self.grid.uv[used]
            out["counts"][i] = (len(pos), len(idx))
            out["positions"][i * self.vcap:i * self.vcap + len(pos)] = pos
            out["uv0"][i * self.vcap:i * self.vcap + len(pos)] = uv
            out["indices"][i * self.icap:i * self.icap + len(idx)] = idx
            meshes.append((pos, idx, uv))
        return out, meshes


def setup(w):
    b = load_cuda_backend(0)
    b.set_objects(w.objects)
    b.set_object_sort_info(np.zeros(w.n, np.uint64), np.ones(w.n, np.uint8), np.zeros((w.n, 3), f32))
    b.set_object_mesh_spheres(np.zeros((w.n, 4), f32))
    b.set_mesh_buffer(w.words)
    b.set_remeshable_meshes(w.records, np.arange(w.n, dtype=np.uint32), np.arange(w.n, dtype=np.uint32))
    return b


def kernel_groups(b, dev_frames):
    import torch
    from torch.profiler import ProfilerActivity, profile

    for s in dev_frames[:2]:
        b.remesh_meshes_device(**s)
    b.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in dev_frames:
            b.remesh_meshes_device(**s)
        b.sync()
        torch.cuda.synchronize()
    groups = {"corner_lists": ("corner_", "scan_u32"), "validate": ("remesh_counts", "remesh_indices", "remesh_apply"), "copy": ("remesh_copy",),
              "shared_four": ("deform_",)}
    ms = {g: 0.0 for g in groups}
    for e in prof.key_averages():
        for g, names in groups.items():
            if any(n in e.key for n in names):
                ms[g] += e.device_time_total / 1000.0   # us -> ms
    return {g: v / len(dev_frames) for g, v in ms.items()}


def run(w, frames):
    import torch

    data = [w.frame(k) for k in range(frames)]
    b = setup(w)
    dev = [{k: torch.from_numpy(v).cuda() for k, v in s.items()} for s, _ in data]
    torch.cuda.synchronize()
    res = {"workload": w.name, "meshes": w.n, "vertex_capacity": w.n * w.vcap, "index_capacity": w.n * w.icap,
           "kernels_ms": kernel_groups(b, dev)}
    passes = (int(w.n * w.vcap).bit_length() + 7) // 8
    model = w.n * w.icap * (16 + 24 * passes + 12) + 4 * w.n * w.vcap
    res["corner_lists_bytes_model"] = model
    res["corner_lists_gbps"] = model / (res["kernels_ms"]["corner_lists"] * 1e-3) / 1e9
    res["corner_lists_share_of_hbm"] = res["corner_lists_gbps"] * 1e9 / HBM_BYTES_PER_S
    for form in ("device", "host"):
        s0 = b.frame_graph_stats()
        b.sync()
        t0 = time.perf_counter()
        for (h, _), d in zip(data, dev):
            b.frame_begin()
            if form == "device":
                b.remesh_meshes_device(**d)
            else:
                b.remesh_meshes(**h)
            b.frame_end()
        b.sync()
        dt = time.perf_counter() - t0
        s1 = b.frame_graph_stats()
        res[form] = {"fps": frames / dt, "early_flushes_per_frame": (s1["flushed"] - s0["flushed"]) / frames}
    b.close()
    # the reference's rebuild path: numpy build, then the blocking range, record and sort-info uploads
    b = setup(w)
    np_s, t_all = 0.0, time.perf_counter()
    slots = np.arange(w.n, dtype=np.uint32)
    n_rebuild = min(frames, 2)
    for _, meshes in data[:n_rebuild]:
        t = time.perf_counter()
        words, objs = [], w.objects.copy()
        for i, (pos, idx, uv) in enumerate(meshes):
            nrm = ref.normals(pos, idx, True)
            tan = ref.tangents(pos, nrm, uv, idx)
            sph = ref.mesh_sphere(pos)
            objs[i]["sphere_center"], objs[i]["sphere_radius"], objs[i]["index_count"] = sph[:3], sph[3], len(idx)
            words.append((i, [pos, nrm, tan, uv], idx))
        np_s += time.perf_counter() - t
        b.frame_begin()
        for i, attrs, idx in words:
            r = w.records[i]
            for off, a in zip((r["position_offset"], r["normal_offset"], r["tangent_offset"], r["uv0_offset"]), attrs):
                if len(a):
                    b.update_mesh_buffer(int(off), np.ascontiguousarray(a, f32).reshape(-1).view(np.uint32))
            if len(idx):
                b.update_mesh_buffer(4 * int(r["first_index"]), np.ascontiguousarray(idx, np.uint32))
        b.update_objects(slots, objs)
        b.update_object_sort_info(slots, np.zeros(w.n, np.uint64), np.ones(w.n, np.uint8), np.ascontiguousarray(objs["sphere_center"], f32))
        b.frame_end()
    b.sync()
    dt = time.perf_counter() - t_all
    res["rebuild"] = {"fps": n_rebuild / dt, "numpy_ms_per_frame": 1e3 * np_s / n_rebuild, "frames": n_rebuild}
    b.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="iso,chunks")
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--out")
    a = ap.parse_args()
    wl = {"iso": lambda: Workload("iso", 1024, 1), "chunks": lambda: Workload("chunks", 32, 1000)}
    doc = {"card": card(), "workloads": [run(wl[n](), a.frames) for n in a.workloads.split(",")]}
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        open(a.out, "w").write(s)


if __name__ == "__main__":
    main()
