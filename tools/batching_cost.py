"""Frame cost of batch_objects on the device against the host path, for a world with a few high-poly meshes.

A 200k-cube field (config-1 shape, one directional light: a viewport and a shadow camera) in which a few objects use a 76,800-triangle
cube, so that a batch can reach the dispatch limit.  Each number is the host time of one whole frame submitted as a frame graph, ending
in r3_sync, median of --reps after --warmup; the device context and a context created with R3_HOST_BATCHING=1 are alternated frame by
frame, so that clock and thermal drift fall on both.  Records the early flushes of the frame graph per frame, the batching path, and the
card name and its power limit beside the numbers.  Writes one JSON document to stdout (and to --out when given).

    python tools/batching_cost.py [--reps 21] [--objects 200000] [--big 4]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rend3_b200.backend import CAMERA_VIEWPORT, load_cuda_backend  # noqa: E402
from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings  # noqa: E402
from rend3_b200.scenes import cube_field_scene  # noqa: E402
from world_update_cost import card  # noqa: E402

BIG_TRIANGLES = 12 * 80 * 80


def world(n, big, resolution):
    """cube_field_scene with subdivisions (1, 2, 80), then every 76,800-triangle object but `big` of them switched to a 12-triangle cube
    (same unit bounds, so the bounding spheres stay valid)."""
    ev = cube_field_scene(n_objects=n, seed=1, resolution=resolution, subdivisions=(1, 2, 80))
    rec = ev.object_buffer
    is_big = rec["index_count"] == 3 * BIG_TRIANGLES
    small = np.flatnonzero(rec["index_count"] == 36)[0]
    keep = np.flatnonzero(is_big)[:big]
    swap = is_big.copy()
    swap[keep] = False
    for f in ("first_index", "index_count", "attr_offset"):
        rec[f][swap] = rec[f][small]
    return ev, len(keep)


def context(ev, resolution, host):
    if host:
        os.environ["R3_HOST_BATCHING"] = "1"
    else:
        os.environ.pop("R3_HOST_BATCHING", None)
    b = load_cuda_backend(0)
    g = BaseRenderGraph(b)
    g.add_to_graph(ev, resolution, 1, BaseRenderGraphSettings(), frame_graph=True)   # uploads (read R3_HOST_BATCHING) and allocates
    b.sync()
    os.environ.pop("R3_HOST_BATCHING", None)
    return b, g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--objects", type=int, default=200_000)
    ap.add_argument("--big", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = (1920, 1080)
    ev, n_big = world(args.objects, args.big, res)
    ctx = {name: context(ev, res, name == "host") for name in ("device", "host")}
    times = {k: [] for k in ctx}
    flushes = {k: [] for k in ctx}
    for r in range(args.warmup + args.reps):
        for k, (b, g) in ctx.items():
            before = b.frame_graph_stats()["flushed"]
            t0 = time.perf_counter()
            g.add_to_graph(ev, res, 1, BaseRenderGraphSettings(), upload=False, frame_graph=True)
            b.sync()
            t = (time.perf_counter() - t0) * 1e3
            if r >= args.warmup:
                times[k].append(t)
                flushes[k].append(b.frame_graph_stats()["flushed"] - before)
    result = {"card": card(), "objects": args.objects, "objects_with_76800_triangles": n_big, "resolution": list(res), "cameras": 1 + len(ev.shadows),
              "reps": args.reps, "warmup": args.warmup, "clock": "host perf_counter around one frame-graph frame, ending in r3_sync"}
    for k, (b, _) in ctx.items():
        result[k] = {"frame_ms_median": round(statistics.median(times[k]), 3), "frame_ms_min": round(min(times[k]), 3),
                     "flushed_frames": sum(1 for f in flushes[k] if f), "timed_frames": len(flushes[k]),
                     "batching": b.batching_info(CAMERA_VIEWPORT), "frame_graph_stats": b.frame_graph_stats()}
        b.close()
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
