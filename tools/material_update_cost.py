"""Frame throughput of a world whose materials change every frame, through the three ways a material can reach the library.

World: --objects cubes with one material each (a per-object tint, as rend3 expresses it), 12 triangles per cube, one directional light
with a 2048^2 shadow map, 1920x1080, camera static.  Two kinds of world:
  opaque   no material discards per fragment: what the device form's conservative rule costs (it runs the alpha-testing raster kernels);
  cutout   a third of the materials are cutouts whose alpha comes from a texture (every path runs the alpha-testing kernels).
Every frame updates --fraction of the materials (1 %, 10 % and 100 %, drawn at random): a new albedo tint and emissive value.  Three
contexts, each submitting --frames frame graphs back to back and one r3_sync per rep, alternated rep by rep:
  set_materials  r3_set_materials of the whole table before r3_frame_begin (re-uploads 208 B per material and drains the stream);
  host_form      r3_update_materials of the changed materials inside the frame (one copy, one kernel, one drain: the frame flushes there);
  device         r3_update_materials_device from CUDA tensors written before the timed window (enqueue only: one graph launch).
Each frame's records are computed before the timed window, so only the library's material calls are timed; their host time per frame and
the early flushes per frame are reported with the frames per second (median of --reps).  The card's name and power limit are recorded
beside the numbers.  Writes one JSON document to stdout (and to --out when given).

    python tools/material_update_cost.py [--objects 1000,100000] [--reps 3] [--frames 8] [--fractions 0.01,0.1,1.0]
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
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from rend3_b200.backend import load_cuda_backend  # noqa: E402
from rend3_b200.layouts import MATERIAL_DTYPE  # noqa: E402
from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings  # noqa: E402
from rend3_b200.scenes import (bulk_object_records, cube_example_camera, eval_with_bulk_objects, random_unit_quaternions,  # noqa: E402
                               subdivided_cube_mesh, trs_matrices)
from rend3_b200.world import CUTOUT, LEFT, DirectionalLight, PbrMaterial, Renderer, Texture  # noqa: E402
from shadow_camera_cost import Timed  # noqa: E402
from world_update_cost import card  # noqa: E402

f32 = np.float32


def material_world(n_objects, cutout, resolution=(1920, 1080), seed=11):
    """(EvalOutput with one material per object, resolution).  The objects' sort keys come from their material's kind."""
    rng = np.random.default_rng(seed)
    r = Renderer(LEFT, aspect_ratio=resolution[0] / resolution[1])
    mesh = r.add_mesh(subdivided_cube_mesh(1, with_uv=True))
    tex = r.add_texture_2d(Texture(rng.integers(0, 256, (64, 64, 4), dtype=np.uint8), srgb=True))
    kinds = [r.add_material(PbrMaterial(albedo_value=(0.8, 0.8, 0.8, 1.0), roughness_factor=0.5)),
             r.add_material(PbrMaterial(albedo_texture=tex, roughness_factor=0.6, transparency=CUTOUT, alpha_cutout=0.5))]
    r.set_camera_data(cube_example_camera(8.0))
    r.add_directional_light(DirectionalLight(color=(1, 1, 1), intensity=0.6, direction=(-1.0, -4.0, 2.0), distance=100.0, resolution=2048))
    extent = 40.0 * (n_objects / 100_000) ** (1 / 3) if n_objects < 100_000 else 40.0
    t = trs_matrices(rng.uniform(-extent, extent, (n_objects, 3)).astype(f32), random_unit_quaternions(rng, n_objects),
                     rng.uniform(0.1, 0.3, (n_objects, 1)).astype(f32))
    kind = (rng.random(n_objects) < (1 / 3 if cutout else 0.0)).astype(np.uint32)
    rec, loc = bulk_object_records(r, t, np.full(n_objects, mesh), np.asarray(kinds, dtype=np.uint32)[kind], capacity=n_objects)
    ev = eval_with_bulk_objects(r, rec, loc, n_objects)
    ev.object_buffer["material_index"][:n_objects] = np.arange(n_objects, dtype=np.uint32)   # one material per object
    table = np.zeros(n_objects, dtype=MATERIAL_DTYPE)   # np.stack would promote the padded record dtype to a packed one
    for k, m in enumerate(kinds):
        table[kind == k] = r.materials[m].to_record()
    table["albedo"][:, :3] = rng.uniform(0.2, 1.0, (n_objects, 3)).astype(f32)
    ev.material_buffer = table
    return ev, resolution


def edits(table, fraction, n_frames, rng):
    """Per frame: (changed indices (ascending, uint32), their new records, the whole table after the frame)."""
    cur, out = table.copy(), []
    for _ in range(n_frames):
        changed = np.sort(rng.choice(len(cur), max(1, int(fraction * len(cur))), replace=False)).astype(np.uint32)
        s = changed.astype(np.int64)
        cur["albedo"][s, :3] = rng.uniform(0.2, 1.0, (len(s), 3)).astype(f32)
        cur["emissive"][s] = rng.uniform(0.0, 0.2, (len(s), 3)).astype(f32)
        out.append((changed, cur[s].copy(), cur.copy()))
    return out


def frame_throughput(a, ev, res, fraction):
    import torch

    settings = BaseRenderGraphSettings()
    steps = edits(ev.material_buffer, fraction, a.frames, np.random.default_rng(int(fraction * 1000)))
    dense = lambda idx: None if len(idx) == len(ev.material_buffer) else idx
    timed_calls = {"set_materials": {"set_materials"}, "host_form": {"update_materials"}, "device": {"update_materials_device"}}
    paths = {}
    for name, calls in timed_calls.items():
        b = load_cuda_backend(0)
        t = Timed(b, calls)
        g = BaseRenderGraph(t)
        g.upload_world(ev)
        if name == "device":
            with torch.cuda.stream(torch.cuda.ExternalStream(b.stream())):
                entries = [(None if dense(idx) is None else torch.from_numpy(idx.view(np.int32)).cuda(),
                            torch.from_numpy(np.ascontiguousarray(recs).view(np.uint8).reshape(-1, 208)).cuda()) for idx, recs, _ in steps]
            torch.cuda.synchronize()
        else:
            entries = [(dense(idx), recs, table) for idx, recs, table in steps]

        def frame(k, t=t, g=g, name=name, entries=entries):
            # the entries set absolute values: every rep makes the same edits, so the work per frame is the same
            if name == "set_materials":
                t.set_materials(entries[k][2])
                g.add_to_graph(ev, res, 1, settings, upload=False, frame_graph=True)
            else:
                g.add_to_graph(ev, res, 1, settings, upload=False, frame_graph=True, material_updates=entries[k][:2])
        for k in range(min(3, a.frames)):   # warm both graph parities
            frame(k)
        b.sync()
        paths[name] = dict(b=b, t=t, frame=frame, fps=[], call_ms=[], flushed=[])
    for _ in range(a.reps):
        for name, p in paths.items():
            b, t = p["b"], p["t"]
            t.seconds = 0.0
            f0 = b.frame_graph_stats()["flushed"]
            t0 = time.perf_counter()
            for k in range(a.frames):
                p["frame"](k)
            b.sync()
            dt = time.perf_counter() - t0
            p["fps"].append(a.frames / dt)
            p["call_ms"].append(1e3 * t.seconds / a.frames)
            p["flushed"].append((b.frame_graph_stats()["flushed"] - f0) / a.frames)
    out = {}
    for name, p in paths.items():
        out[name] = dict(fps_median=statistics.median(p["fps"]), fps=p["fps"], material_calls_host_ms_per_frame=statistics.median(p["call_ms"]),
                         early_flushes_per_frame=statistics.median(p["flushed"]))
        p["b"].close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--objects", default="1000,100000")
    ap.add_argument("--worlds", default="opaque,cutout")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--fractions", default="0.01,0.1,1.0")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    doc = dict(card(), config="n cubes (12 triangles) with one material each, one directional light (2048^2 shadow map), 1920x1080, camera "
               "static; opaque: no material discards per fragment; cutout: a third of the materials take alpha from a texture",
               frames_per_rep=a.frames, reps=a.reps, runs={})
    for n in [int(x) for x in a.objects.split(",")]:
        for world in a.worlds.split(","):
            ev, res = material_world(n, world == "cutout")
            for fr in [float(x) for x in a.fractions.split(",")]:
                doc["runs"][f"{n} {world} {fr:g}"] = frame_throughput(a, ev, res, fr)
                print(f"{n} {world} {fr:g}", json.dumps(doc["runs"][f"{n} {world} {fr:g}"]), file=sys.stderr, flush=True)
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(s)


if __name__ == "__main__":
    main()
