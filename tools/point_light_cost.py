"""Frame throughput of config 5 with every point light moving every frame, through the three ways the lights can reach the shading.

Config 5 (4400 meshes / ~500k triangles, 64 point lights + 4 directional lights with 2048^2 shadow maps, 3840x2160), camera static, each of
the 64 lights on its own circle.  Three contexts, each submitting --frames frame graphs back to back and one r3_sync per rep, alternated rep
by rep so that clock and thermal drift fall on all of them:
  device            r3_set_point_light_sources once; every frame r3_update_point_light_sources_device from CUDA tensors + r3_evaluate_point_lights
                    (enqueue only: the frame stays one graph launch);
  host_form         the same with r3_update_point_light_sources from host arrays (it drains the stream, so the frame flushes early);
  set_point_lights  world.py's evaluated buffer uploaded with r3_set_point_lights before r3_frame_begin (drains the stream between frames).
The moved lights of every frame are computed before the timed window (on the device for the device path), so only the library's light
calls are timed; their host time per frame and the early flushes per frame are reported with the frames per second (median of --reps).

With --parent DIR (a built checkout of the parent commit), `bench.py --gpus 1` runs --bench-reps times in DIR and in this tree,
alternating, and the config-5 resolve kernel's stage time and frame time of each run are reported: whether reading the point-light count
from the device costs the shading anything.  The card's name and power limit are recorded beside the numbers.  Writes one JSON document to
stdout (and to --out when given).

    python tools/point_light_cost.py [--reps 5] [--frames 32] [--parent DIR --bench-reps 3 --bench-steps 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from rend3_b200.backend import load_cuda_backend  # noqa: E402
from rend3_b200.configs import config5  # noqa: E402
from rend3_b200.layouts import POINT_LIGHT_DTYPE  # noqa: E402
from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings  # noqa: E402
from shadow_camera_cost import Timed  # noqa: E402
from world_update_cost import card  # noqa: E402

f32 = np.float32


def moved_lights(ev, n_frames):
    """Per frame: (handles, POINT_LIGHT_SOURCE_DTYPE records, live bytes) of every handle, and world.py's evaluated buffer of them."""
    src, live = ev.point_sources
    out = []
    for k in range(n_frames):
        s = src.copy()
        phase = np.arange(len(s), dtype=f32) * f32(0.37) + f32(0.2 * k)
        s["position"][:, 0] += f32(2.0) * np.cos(phase)
        s["position"][:, 2] += f32(2.0) * np.sin(phase)
        pl = np.zeros(int(live.sum()), dtype=POINT_LIGHT_DTYPE)
        lv = s[live != 0]
        pl["position"][:, :3], pl["position"][:, 3] = lv["position"], f32(1.0)
        pl["color"] = lv["color"] * lv["intensity"][:, None]
        pl["radius"] = lv["radius"]
        buf = np.array([len(pl), 0, 0, 0], dtype=np.uint32).tobytes() + pl.tobytes()
        out.append((np.arange(len(s), dtype=np.uint32), s, live.copy(), buf))
    return out


def frame_throughput(a):
    import torch

    ev, res = config5()
    steps = moved_lights(ev, a.frames)
    settings = BaseRenderGraphSettings()
    timed_calls = {"device": {"update_point_light_sources_device", "evaluate_point_lights"},
                   "host_form": {"update_point_light_sources", "evaluate_point_lights"}, "set_point_lights": {"set_point_lights"}}
    paths = {}
    for name, calls in timed_calls.items():
        b = load_cuda_backend(0)
        t = Timed(b, calls)
        g = BaseRenderGraph(t)
        device_sources = name != "set_point_lights"
        g.add_to_graph(ev, res, 1, settings, frame_graph=True, device_shadow_cameras=True, device_point_lights=device_sources)   # uploads
        updates = []
        if name == "device":
            with torch.cuda.stream(torch.cuda.ExternalStream(b.stream())):
                for h, s, lv, _ in steps:
                    updates.append((torch.from_numpy(h.view(np.int32)).cuda(), torch.from_numpy(s.view(f32).reshape(-1, 8)).cuda(),
                                    torch.from_numpy(lv).cuda()))
            torch.cuda.synchronize()
        elif name == "host_form":
            updates = [(h, s, lv) for h, s, lv, _ in steps]

        def frame(k, t=t, g=g, name=name, updates=updates):
            if name == "set_point_lights":
                t.set_point_lights(steps[k][3])
                g.add_to_graph(ev, res, 1, settings, upload=False, frame_graph=True, device_shadow_cameras=True)
            else:
                g.add_to_graph(ev, res, 1, settings, upload=False, frame_graph=True, device_shadow_cameras=True, device_point_lights=True,
                               point_light_updates=updates[k])
        for k in range(3):                        # warm both graph parities
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
        out[name] = dict(fps_median=statistics.median(p["fps"]), fps=p["fps"], light_calls_host_ms_per_frame=statistics.median(p["call_ms"]),
                         early_flushes_per_frame=statistics.median(p["flushed"]))
        p["b"].close()
    return out


def find(doc, key):
    if isinstance(doc, dict):
        if key in doc:
            return doc[key]
        for v in doc.values():
            r = find(v, key)
            if r is not None:
                return r
    return None


def bench_runs(a):
    """bench.py in the parent checkout and in this tree, alternated run by run: config 5's resolve stage time and frame time."""
    rows = {"parent": [], "this": []}
    for _ in range(a.bench_reps):
        for name, cwd in (("parent", a.parent), ("this", ROOT)):
            r = subprocess.run([sys.executable, "bench.py", "--gpus", "1", "--steps", str(a.bench_steps), "--warmup", "2", "--no-dynamic"],
                               cwd=cwd, capture_output=True, text=True)
            line = [l for l in r.stdout.splitlines() if l.startswith("{")]
            if r.returncode != 0 or not line:
                rows[name].append({"error": (r.stderr or r.stdout)[-400:]})
                continue
            doc = json.loads(line[-1])
            fwd = find(doc, "forward") or {}
            rows[name].append({"resolve_ms": find(fwd, "resolve_kernel").get("kernel_ms_per_frame") if find(fwd, "resolve_kernel") else None,
                               "frame_ms": fwd.get("frame_ms")})
    summary = {}
    for name, rs in rows.items():
        ok = [r for r in rs if r.get("resolve_ms") is not None]
        summary[name] = dict(runs=rs, resolve_ms_median=statistics.median([r["resolve_ms"] for r in ok]) if ok else None,
                             frame_ms_median=statistics.median([r["frame_ms"] for r in ok]) if ok else None)
    return summary


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--parent", default=None, help="a built checkout of the parent commit: compare bench.py's config-5 resolve time")
    ap.add_argument("--bench-reps", type=int, default=3)
    ap.add_argument("--bench-steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    doc = dict(card(), config="config5 3840x2160, 4400 meshes, 64 point lights moving every frame, 4 directional lights (device shadow cameras), "
               "camera static", frames_per_rep=a.frames, reps=a.reps)
    doc["paths"] = frame_throughput(a)
    if a.parent:
        doc["bench_config5_resolve"] = bench_runs(a)
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(s)


if __name__ == "__main__":
    main()
