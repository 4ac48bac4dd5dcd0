"""Cost of meshes that deform every frame, through the three ways new positions can reach the library.

Workloads (--workloads):
  ocean  one 1024 x 1024 grid with uv0: 1 048 576 vertices, 2 093 058 triangles, normals and tangents recomputed, one object;
  flags  4096 flags of 33 x 33 vertices with uv0 (2048 triangles each), one object each, on a 64 x 64 field.
Each frame moves every vertex (a travelling wave, computed before the timed window) and renders the world at 1280 x 720 with one
shadowed directional light, inside a frame graph.  Three contexts, alternated rep by rep, each submitting --frames frames and one r3_sync:
  device   r3_deform_meshes_device from CUDA tensors at the skinning node (enqueue only);
  host     r3_deform_meshes from host arrays at the skinning node (one copy, the kernels, one drain: the frame flushes there);
  rebuild  what the reference does, restated: the normals, tangents and mesh spheres in vectorised numpy, then r3_update_mesh_buffer of
           the position, normal and tangent ranges, r3_update_objects and r3_update_object_sort_info of the objects, before the frame.
           Its numpy time per frame is reported apart from the frame rate (numpy is not Rust); it runs 2 frames per rep.
Reported: the deform's kernels alone (CUDA events over --launches launches of r3_deform_meshes_device) against the byte model below,
frames per second (median of --reps), early flushes per frame (r3_frame_graph_stats), the host time of r3_set_deformable_meshes (which
builds the corner lists on the host), and the card's name and power limit, read in the same run.  One JSON document to stdout (and --out).

Byte model per deform (what the four kernels must move at least once): per vertex 12 B position in, 8 B uv0 (with tangents), 36 B of
position, normal and tangent out (24 without tangents), 12 B position re-read for the radius, 4 B corner-list start; per index 4 B index
and 4 B corner entry; per object 16 B mesh sphere + 64 B transform read, 16 + 16 + 4 + 16 + 12 B written.  A regular grid (6 corners per
vertex) comes to about 120 B per vertex.

    python tools/mesh_deform_cost.py [--workloads ocean,flags] [--reps 3] [--frames 8] [--launches 50]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import mesh_deform_case as case  # noqa: E402
import mesh_deform_reference as ref  # noqa: E402
from rend3_b200.backend import load_cuda_backend  # noqa: E402
from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings  # noqa: E402
from rend3_b200.scenes import bulk_object_records, cube_example_camera, eval_with_bulk_objects, trs_matrices  # noqa: E402
from rend3_b200.world import LEFT, DirectionalLight, Mesh, PbrMaterial, Renderer  # noqa: E402
from world_update_cost import card  # noqa: E402

f32 = np.float32
RES = (1280, 720)
HBM_BYTES_PER_S = 3.35e12


class Workload:
    """n_meshes equal grids laid out attribute after attribute in one mesh-buffer block, each described as its own mesh (its indices
    local to it), one object per mesh"""

    def __init__(self, name, nx, n_meshes, size, spacing, pull_back):
        g = case.grid(nx, nx, size=size)
        self.name, self.n_meshes, self.vc, self.ic = name, n_meshes, len(g.positions), len(g.indices)
        side = int(np.ceil(np.sqrt(n_meshes)))
        offs = np.stack(np.meshgrid(np.arange(side), np.arange(side)), -1).reshape(-1, 2)[:n_meshes].astype(f32) * f32(spacing)
        offs -= offs.mean(0)
        self.rest = (np.repeat(g.positions[None], n_meshes, 0)
                     + np.stack([offs[:, 0], np.zeros(n_meshes, f32), offs[:, 1]], -1)[:, None, :]).astype(f32).reshape(-1, 3)
        self.uv = np.tile(g.uv, (n_meshes, 1))
        self.local = np.tile(g.indices, n_meshes)
        self.global_idx = (self.local.reshape(n_meshes, -1) + (np.arange(n_meshes, dtype=np.uint32) * self.vc)[:, None]).reshape(-1)
        r = Renderer(LEFT, aspect_ratio=RES[0] / RES[1])
        r.add_material(PbrMaterial(albedo_value=(0.2, 0.4, 0.7, 1.0), roughness_factor=0.3))
        r.set_camera_data(cube_example_camera(pull_back))
        r.add_directional_light(DirectionalLight(color=(1, 1, 1), intensity=1.0, direction=(-1.0, -4.0, 2.0), distance=4 * pull_back,
                                                 resolution=2048))
        nrm = ref.normals(self.rest, self.global_idx, True)
        tan = ref.tangents(self.rest, nrm, self.uv, self.global_idx)
        big = r.add_mesh(Mesh([(0, self.rest), (3, self.uv), (1, nrm), (2, tan)], len(self.rest), self.local))
        m0 = r.meshes.pop(big)
        self.ranges, self.index_start = m0["ranges"], m0["index_start"]
        spheres = self.mesh_spheres(self.rest)
        for i in range(n_meshes):   # each grid as its own mesh, pointing into the block
            r.meshes.append(dict(ranges={k: v + i * self.vc * (8 if k == 3 else 12) for k, v in self.ranges.items()},
                                 index_start=self.index_start + i * self.ic * 4, index_count=self.ic, center=spheres[i, :3],
                                 radius=spheres[i, 3], vertex_count=self.vc, left_handed=True, normals_calculated=True,
                                 tangents_calculated=True))
        ids = np.arange(n_meshes)
        t = trs_matrices(np.zeros((n_meshes, 3), f32), np.tile(np.array([[0, 0, 0, 1]], f32), (n_meshes, 1)), np.ones((n_meshes, 1), f32))
        rec, loc = bulk_object_records(r, t, ids, np.zeros(n_meshes, np.uint32), capacity=n_meshes)
        self.ev = eval_with_bulk_objects(r, rec, loc, n_meshes, ids)
        self.meshes = case.deformable_records(r, list(range(n_meshes)))
        self.slots = np.arange(n_meshes, dtype=np.uint32)

    def mesh_spheres(self, pos):
        """per-mesh (centre, radius), vectorised over the equal meshes (numpy max / min: the rebuild path's cost, not R15's ties)"""
        p = pos.reshape(self.n_meshes, self.vc, 3)
        c = ((p.max(1) + p.min(1)) / f32(2)).astype(f32)
        d = (p - c[:, None, :]).astype(f32)
        r = np.sqrt(((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).astype(f32)).max(1)
        return np.concatenate([c, r[:, None]], 1).astype(f32)

    def frames(self, n):
        return [case.wave(self.rest, 0.3 * (k + 1)) for k in range(n)]

    def model_bytes(self):
        v, i, o = self.vc * self.n_meshes, self.ic * self.n_meshes, self.n_meshes
        return v * (12 + 8 + 36 + 12 + 4) + i * (4 + 4) + o * (16 + 64 + 16 + 16 + 4 + 16 + 12)


def rebuild(b, w, pos):
    """the reference's per-frame path, restated; returns its numpy seconds"""
    t0 = time.perf_counter()
    nrm = ref.normals(pos, w.global_idx, True)
    tan = ref.tangents(pos, nrm, w.uv, w.global_idx)
    sph = w.mesh_spheres(pos)
    rec = w.ev.object_buffer.copy()
    world = ref.apply_transform(rec["transform"], sph)
    rec["sphere_center"], rec["sphere_radius"] = world[:, :3], world[:, 3]
    numpy_s = time.perf_counter() - t0
    for slot, arr in ((0, pos), (1, nrm), (2, tan)):
        b.update_mesh_buffer(w.ranges[slot], arr)
    b.update_objects(w.slots, rec)
    flags = np.ones(w.n_meshes, np.uint8) | (w.ev.object_atomic[:w.n_meshes] << 1)
    b.update_object_sort_info(w.slots, w.ev.object_material_key[:w.n_meshes], flags, np.ascontiguousarray(world[:, :3]))
    return numpy_s


def measure(w, reps, n_frames, launches):
    import torch

    settings = BaseRenderGraphSettings(clear_color=(0.1, 0.1, 0.12, 1.0))
    frames = w.frames(n_frames)
    paths = {}
    for name in ("device", "host", "rebuild"):
        b = load_cuda_backend(0)
        g = BaseRenderGraph(b)
        g.add_to_graph(w.ev, RES, 1, settings, movable_objects=True)
        t0 = time.perf_counter()
        b.set_deformable_meshes(w.meshes, w.slots, np.arange(w.n_meshes, dtype=np.uint32))
        set_ms = (time.perf_counter() - t0) * 1e3
        paths[name] = dict(b=b, g=g, set_ms=set_ms, fps=[], flushes=[], numpy_ms=[])
    dev = paths["device"]["b"]
    stream = torch.cuda.ExternalStream(dev.stream())
    with torch.cuda.stream(stream):
        d_frames = [torch.from_numpy(f).to("cuda") for f in frames]
    torch.cuda.synchronize()
    # the kernels alone
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(5):
        dev.deform_meshes_device(d_frames[0])
    with torch.cuda.stream(stream):
        start.record(stream)
        for k in range(launches):
            dev.deform_meshes_device(d_frames[k % n_frames])
        stop.record(stream)
    stop.synchronize()
    kernel_ms = start.elapsed_time(stop) / launches
    for _ in range(reps):
        for name, p in paths.items():
            b, g = p["b"], p["g"]
            s0 = b.frame_graph_stats()
            numpy_s = 0.0
            b.sync()
            t0 = time.perf_counter()
            count = n_frames if name != "rebuild" else min(n_frames, 2)   # its numpy takes seconds per frame on the large worlds
            for k in range(count):
                if name == "device":
                    g.add_to_graph(w.ev, RES, 1, settings, upload=False, frame_graph=True, mesh_deforms=d_frames[k])
                elif name == "host":
                    g.add_to_graph(w.ev, RES, 1, settings, upload=False, frame_graph=True, mesh_deforms=frames[k])
                else:
                    numpy_s += rebuild(b, w, frames[k])
                    g.add_to_graph(w.ev, RES, 1, settings, upload=False, frame_graph=True)
            b.sync()
            dt = time.perf_counter() - t0
            s1 = b.frame_graph_stats()
            p["fps"].append(count / dt)
            p["flushes"].append((s1["flushed"] - s0["flushed"]) / count)
            p["numpy_ms"].append(numpy_s * 1e3 / count)
    # the three paths end on the same world: the device and host forms bit for bit
    last = {n: paths[n]["b"].readback_mesh_buffer(len(w.ev.mesh_buffer)) for n in ("device", "host")}
    out = dict(vertices=w.vc * w.n_meshes, triangles=w.ic * w.n_meshes // 3, meshes=w.n_meshes, frames_per_measure=n_frames,
               kernel_ms=round(kernel_ms, 5), model_bytes=w.model_bytes(), model_bytes_per_vertex=round(w.model_bytes() / (w.vc * w.n_meshes), 1),
               kernel_bytes_per_s=w.model_bytes() / (kernel_ms * 1e-3), share_of_3_35_tb_s=w.model_bytes() / (kernel_ms * 1e-3) / HBM_BYTES_PER_S,
               device_equals_host=bool(np.array_equal(last["device"], last["host"])))
    for name, p in paths.items():
        out[name] = dict(fps=round(statistics.median(p["fps"]), 1), early_flushes_per_frame=statistics.median(p["flushes"]),
                         set_deformable_meshes_ms=round(p["set_ms"], 2))
        if name == "rebuild":
            out[name]["numpy_ms_per_frame"] = round(statistics.median(p["numpy_ms"]), 2)
        p["b"].close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="ocean,flags")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    makers = {"ocean": lambda: Workload("ocean", 1024, 1, 200.0, 0.0, 30.0),
              "flags": lambda: Workload("flags", 33, 4096, 2.0, 3.0, 30.0)}
    result = dict(card())
    for name in a.workloads.split(","):
        result[name] = measure(makers[name](), a.reps, a.frames, a.launches)
        print(name, json.dumps(result[name]), file=sys.stderr, flush=True)
    doc = json.dumps(result)
    print(doc)
    if a.out:
        with open(a.out, "w") as f:
            f.write(doc + "\n")


if __name__ == "__main__":
    main()
