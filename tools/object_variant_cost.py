"""Frame throughput of a world whose objects switch levels of detail, through the three ways a slot's mesh change can reach the library.

World: --objects objects (default 100 000), each with a 4-level LOD chain of cubes (scenes.subdivided_cube_mesh(k) for k = 8, 4, 2, 1:
768, 192, 48 and 12 triangles) in one of three materials, one directional light with a 2048^2 shadow map, 1920x1080.  Every frame
switches --fraction of the objects (1 %, 10 % and 100 %) to another level, drawn at random.  Three contexts, each submitting --frames
frame graphs back to back and one r3_sync per rep, alternated rep by rep:
  update       r3_update_objects + r3_update_object_sort_info + r3_set_object_mesh_spheres of the changed slots (the re-add's records,
               sort entries and mesh spheres): the way in before the variant calls (each drains the stream);
  host_form    r3_switch_object_variants of the changed slots from host arrays (drains the stream once);
  device       r3_switch_object_variants_device from CUDA tensors written before the timed window (enqueue only: one graph launch).
Each frame's entries are computed before the timed window, so only the library's calls are timed; their host time per frame and the
early flushes per frame are reported with the frames per second (median of --reps), beside the card's name and power limit.  The slot
count and r3_debug_invocation_bound of the variant world are reported next to those of the equivalent presence pool (one prepared slot
per level, one of them enabled), computed from the same round_up(triangles, 256) terms.  Writes one JSON document to stdout (and --out).

    python tools/object_variant_cost.py [--objects 100000] [--reps 3] [--frames 8] [--fractions 0.01,0.1,1.0]
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
from object_variant_case import variant_record  # noqa: E402
from rend3_b200.backend import load_cuda_backend  # noqa: E402
from rend3_b200.layouts import OBJECT_VARIANT_DTYPE, VARIANT_GROUP_DTYPE  # noqa: E402
from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings  # noqa: E402
from rend3_b200.scenes import (bulk_object_records, cube_example_camera, eval_with_bulk_objects, random_unit_quaternions,  # noqa: E402
                               subdivided_cube_mesh, trs_matrices)
from rend3_b200.world import LEFT, DirectionalLight, PbrMaterial, Renderer  # noqa: E402
from shadow_camera_cost import Timed  # noqa: E402
from world_update_cost import card  # noqa: E402

f32 = np.float32
LEVELS = (8, 4, 2, 1)


def lod_world(n, resolution=(1920, 1080), seed=11):
    rng = np.random.default_rng(seed)
    r = Renderer(LEFT, aspect_ratio=resolution[0] / resolution[1])
    meshes = [r.add_mesh(subdivided_cube_mesh(k)) for k in LEVELS]
    mats = [r.add_material(PbrMaterial(albedo_value=(0.6, g, 1.0 - g, 1.0), roughness_factor=0.5)) for g in (0.25, 0.5, 0.75)]
    r.set_camera_data(cube_example_camera(8.0))
    r.add_directional_light(DirectionalLight(color=(1, 1, 1), intensity=0.6, direction=(-1.0, -4.0, 2.0), distance=100.0, resolution=2048))
    t = trs_matrices(rng.uniform(-40.0, 40.0, (n, 3)).astype(f32), random_unit_quaternions(rng, n), rng.uniform(0.05, 0.2, (n, 1)).astype(f32))
    mat = rng.integers(0, len(mats), n).astype(np.uint32)
    level = np.full(n, len(LEVELS) - 1, dtype=np.int64)
    rec, loc = bulk_object_records(r, t, np.asarray(meshes)[level], mat, capacity=n)
    ev = eval_with_bulk_objects(r, rec, loc, n, mesh_ids=np.asarray(meshes)[level])
    variants = np.array([variant_record(r, meshes[l], m) for m in range(len(mats)) for l in range(len(LEVELS))], dtype=OBJECT_VARIANT_DTYPE)
    groups = np.zeros(len(mats), dtype=VARIANT_GROUP_DTYPE)
    groups["first"], groups["count"] = len(LEVELS) * np.arange(len(mats)), len(LEVELS)
    return dict(r=r, meshes=meshes, ev=ev, t=t, mat=mat, level=level, variants=variants, groups=groups, res=resolution)


def switches(w, fraction, n_frames, rng):
    """Per frame: (changed slots (ascending, uint32), their new level (uint32), the levels after the frame)."""
    cur, out = w["level"].copy(), []
    for _ in range(n_frames):
        changed = np.sort(rng.choice(len(cur), max(1, int(fraction * len(cur))), replace=False))
        cur[changed] = (cur[changed] + rng.integers(1, len(LEVELS), len(changed))) % len(LEVELS)
        out.append((changed.astype(np.uint32), cur[changed].astype(np.uint32), cur.copy()))
    return out


def frame_throughput(a, w, fraction):
    import torch

    ev, res, settings = w["ev"], w["res"], BaseRenderGraphSettings()
    steps = switches(w, fraction, a.frames, np.random.default_rng(int(fraction * 1000)))
    timed_calls = {"update": {"update_objects", "update_object_sort_info", "set_object_mesh_spheres"},
                   "host_form": {"switch_object_variants"}, "device": {"switch_object_variants_device"}}
    key_of = np.array([m.key() for m in w["r"].materials], dtype=np.uint64)
    paths = {}
    for name, calls in timed_calls.items():
        b = load_cuda_backend(0)
        t = Timed(b, calls)
        g = BaseRenderGraph(t)
        g.upload_world(ev, movable_objects=True)
        b.set_object_variants(w["variants"], w["groups"], np.arange(len(w["mat"])), w["mat"])
        entries = []
        if name == "update":
            for changed, lvl, _ in steps:
                s = changed.astype(np.int64)
                mesh = np.asarray(w["meshes"])[lvl]
                rec, loc = bulk_object_records(w["r"], w["t"][s], mesh, w["mat"][s], capacity=len(s))
                ms = np.array([[*w["r"].meshes[k]["center"], w["r"].meshes[k]["radius"]] for k in mesh], dtype=f32)
                flags = np.full(len(s), 1 | 2, np.uint8)
                entries.append((changed, rec, key_of[w["mat"][s]], flags, loc, ms))
        elif name == "host_form":
            entries = [(changed, lvl) for changed, lvl, _ in steps]
        else:
            with torch.cuda.stream(torch.cuda.ExternalStream(b.stream())):
                entries = [(torch.from_numpy(changed.view(np.int32)).cuda(), torch.from_numpy(lvl.view(np.int32)).cuda()) for changed, lvl, _ in steps]
            torch.cuda.synchronize()

        def frame(k, t=t, g=g, name=name, entries=entries):
            # the entries set absolute levels: every rep makes the same switches, so the work per frame is the same
            if name == "update":
                s, rec, key, flags, loc, ms = entries[k]
                t.update_objects(s, rec)
                t.update_object_sort_info(s, key, flags, loc)
                t.set_object_mesh_spheres(ms, s)
                g.add_to_graph(ev, res, 1, settings, upload=False, frame_graph=True)
            elif name == "host_form":
                g.add_to_graph(ev, res, 1, settings, upload=False, frame_graph=True, object_variants=(entries[k][0], entries[k][1]))
            else:
                g.add_to_graph(ev, res, 1, settings, upload=False, frame_graph=True, object_variants=(entries[k][0], entries[k][1]))
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
        out[name] = dict(fps_median=statistics.median(p["fps"]), fps=p["fps"], variant_calls_host_ms_per_frame=statistics.median(p["call_ms"]),
                         early_flushes_per_frame=statistics.median(p["flushed"]))
        if name == "device":
            out["variant_world_invocation_bound"] = p["b"].debug_invocation_bound()[0]
        p["b"].close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--objects", type=int, default=100_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--fractions", default="0.01,0.1,1.0")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    w = lod_world(a.objects)
    tris = np.array([12 * k * k for k in LEVELS], dtype=np.int64)
    term = (tris + 255) // 256 * 256
    doc = dict(card(), config=f"{a.objects} objects with a 4-level LOD chain ({', '.join(str(int(x)) for x in tris)} triangles), one directional "
               f"light (2048^2 shadow map), {w['res'][0]}x{w['res'][1]}, camera static", frames_per_rep=a.frames, reps=a.reps,
               slots=dict(variant_world=a.objects, presence_pool=a.objects * len(LEVELS)),
               invocation_bound=dict(variant_world=int(a.objects * term.max()), presence_pool=int(a.objects * term.sum())), fractions={})
    for fr in [float(x) for x in a.fractions.split(",")]:
        doc["fractions"][f"{fr:g}"] = frame_throughput(a, w, fr)
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(s)


if __name__ == "__main__":
    main()
