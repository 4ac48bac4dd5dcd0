"""Frame throughput of a pool world whose objects come and go, through the three ways a slot's presence can reach the library.

Pool world: --slots prepared slots (default 250 000) of 12-triangle cubes, the first --present of them (default 75 000) present, one
directional light with a 2048^2 shadow map, 1920x1080.  The culling buffers are sized for every slot, live or not (256 invocations per
slot), so three contexts of 1 M slots do not fit in 80 GB; the default leaves room for them.  Every frame switches --fraction of the pool (1 %, 10 % and 100 %): that many
slots, drawn at random, change state.  Three contexts, each submitting --frames frame graphs back to back and one r3_sync per rep,
alternated rep by rep so that clock and thermal drift fall on all of them:
  update       r3_update_objects + r3_update_object_sort_info of the changed slots, records and flags as the pool's state gives them
               (object_presence_case.pool_state): the way in before r3_set_objects_enabled (both drain the stream);
  host_form    r3_set_objects_enabled of the changed slots from host arrays (drains the stream once);
  device       r3_set_objects_enabled_device from CUDA tensors written before the timed window (enqueue only: one graph launch).
Each frame's entries are computed before the timed window, so only the library's presence calls are timed; their host time per frame and
the early flushes per frame are reported with the frames per second (median of --reps).  The card's name and power limit are recorded
beside the numbers.  Writes one JSON document to stdout (and to --out when given).

    python tools/object_presence_cost.py [--reps 3] [--frames 8] [--fractions 0.01,0.1,1.0]
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
from object_presence_case import pool_state  # noqa: E402
from rend3_b200.backend import load_cuda_backend  # noqa: E402
from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings  # noqa: E402
from rend3_b200.scenes import (bulk_object_records, cube_example_camera, eval_with_bulk_objects, random_unit_quaternions,  # noqa: E402
                               subdivided_cube_mesh, trs_matrices)
from rend3_b200.world import LEFT, DirectionalLight, PbrMaterial, Renderer  # noqa: E402
from shadow_camera_cost import Timed  # noqa: E402
from world_update_cost import card  # noqa: E402

f32 = np.float32


def pool_world(n_slots, n_present, resolution=(1920, 1080), seed=11):
    rng = np.random.default_rng(seed)
    r = Renderer(LEFT, aspect_ratio=resolution[0] / resolution[1])
    mesh = r.add_mesh(subdivided_cube_mesh(1))
    mats = [r.add_material(PbrMaterial(albedo_value=(0.6, g, 1.0 - g, 1.0), roughness_factor=0.5)) for g in (0.25, 0.5, 0.75)]
    r.set_camera_data(cube_example_camera(8.0))
    r.add_directional_light(DirectionalLight(color=(1, 1, 1), intensity=0.6, direction=(-1.0, -4.0, 2.0), distance=100.0, resolution=2048))
    t = trs_matrices(rng.uniform(-40.0, 40.0, (n_slots, 3)).astype(f32), random_unit_quaternions(rng, n_slots),
                     rng.uniform(0.05, 0.2, (n_slots, 1)).astype(f32))
    rec, loc = bulk_object_records(r, t, np.full(n_slots, mesh), rng.integers(0, len(mats), n_slots).astype(np.uint32), capacity=n_slots)
    ev = eval_with_bulk_objects(r, rec, loc, n_slots)
    present = np.zeros(n_slots, dtype=bool)
    present[:n_present] = True
    return ev, present, resolution


def switches(present, fraction, n_frames, rng):
    """Per frame: (changed slots (ascending, uint32), their new presence (uint8), the pool's presence after the frame)."""
    cur, out = present.copy(), []
    for _ in range(n_frames):
        changed = np.sort(rng.choice(len(cur), max(1, int(fraction * len(cur))), replace=False)).astype(np.uint32)
        cur[changed] = ~cur[changed]
        out.append((changed, cur[changed].astype(np.uint8), cur.copy()))
    return out


def frame_throughput(a, ev, present, res, fraction):
    import torch

    settings = BaseRenderGraphSettings()
    steps = switches(present, fraction, a.frames, np.random.default_rng(int(fraction * 1000)))
    start = pool_state(ev, present)
    timed_calls = {"update": {"update_objects", "update_object_sort_info"}, "host_form": {"set_objects_enabled"},
                   "device": {"set_objects_enabled_device"}}
    paths = {}
    for name, calls in timed_calls.items():
        b = load_cuda_backend(0)
        t = Timed(b, calls)
        g = BaseRenderGraph(t)
        g.upload_world(ev)
        b.set_objects(start[0])
        b.set_object_sort_info(ev.object_material_key, start[1], ev.object_location)
        entries = []
        if name == "update":
            for changed, _, cur in steps:
                rec, flags = pool_state(ev, cur)
                s = changed.astype(np.int64)
                entries.append((changed, rec[s], ev.object_material_key[s], flags[s], ev.object_location[s]))
        elif name == "host_form":
            entries = [(changed, on) for changed, on, _ in steps]
        else:
            with torch.cuda.stream(torch.cuda.ExternalStream(b.stream())):
                entries = [(torch.from_numpy(changed.view(np.int32)).cuda(), torch.from_numpy(on).cuda()) for changed, on, _ in steps]
            torch.cuda.synchronize()

        def frame(k, t=t, g=g, name=name, entries=entries):
            # the entries set absolute states: every rep makes the same switches, so the work per frame is the same
            if name == "update":
                s, rec, key, flags, loc = entries[k]
                t.update_objects(s, rec)
                t.update_object_sort_info(s, key, flags, loc)
                g.add_to_graph(ev, res, 1, settings, upload=False, frame_graph=True)
            elif name == "host_form":
                g.add_to_graph(ev, res, 1, settings, upload=False, frame_graph=True, object_presence=(entries[k][0], entries[k][1]))
            else:
                g.add_to_graph(ev, res, 1, settings, upload=False, frame_graph=True, object_presence=entries[k])
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
        out[name] = dict(fps_median=statistics.median(p["fps"]), fps=p["fps"], presence_calls_host_ms_per_frame=statistics.median(p["call_ms"]),
                         early_flushes_per_frame=statistics.median(p["flushed"]))
        p["b"].close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=250_000)
    ap.add_argument("--present", type=int, default=75_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--fractions", default="0.01,0.1,1.0")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ev, present, res = pool_world(a.slots, a.present)
    doc = dict(card(), config=f"pool of {a.slots} slots (12-triangle cubes), {a.present} present at the start, one directional light "
               f"(2048^2 shadow map), {res[0]}x{res[1]}, camera static", frames_per_rep=a.frames, reps=a.reps, fractions={})
    for fr in [float(x) for x in a.fractions.split(",")]:
        doc["fractions"][f"{fr:g}"] = frame_throughput(a, ev, present, res, fr)
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(s)


if __name__ == "__main__":
    main()
