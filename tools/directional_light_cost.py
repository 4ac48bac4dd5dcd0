"""Frame throughput of config 3 with every directional light turning and changing colour and intensity every frame, through the three
ways such a change can reach the device, and the time of directional_light_change_kernel alone.

Config 3 (200k objects, 4 directional lights with 2048^2 shadow maps, 4 point lights, 3840x2160), camera static.  Every frame all four
lights move along a sun arc and change colour and intensity.  Three contexts, each submitting --frames frame graphs back to back and one
r3_sync per rep, alternated rep by rep so that clock and thermal drift fall on all of them:
  set          r3_set_directional_light_sources with the changed list, inside the frame (it drains the stream: the frame flushes early);
  host_form    r3_update_directional_light_sources from host records (enqueue only: the frame stays one graph launch);
  device_form  r3_update_directional_light_sources_device from a CUDA tensor (enqueue only).
The changes of every frame are computed before the timed window (uploaded to the device for the device form), so only the library's
light calls are timed: their host time per frame (the change call plus r3_evaluate_shadow_cameras) and the early flushes per frame are
reported with the frames per second (median of --reps).  The kernel alone is timed with CUDA events around --kernel-launches back-to-back
launches of each form, queued behind a sleep kernel so that the events see the device's rate rather than the host's.  The card's name
and power limit are read in the same run.  Writes one JSON document to stdout (and to --out).

    python tools/directional_light_cost.py [--reps 5] [--frames 32] [--kernel-launches 512]
    python tools/directional_light_cost.py --dry-run      (no device: the world and the changes at a tiny size, checked against world.py)
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
from rend3_b200.configs import config3  # noqa: E402
from rend3_b200.layouts import DIRECTIONAL_LIGHT_CHANGE_DTYPE  # noqa: E402
from rend3_b200.world import LEFT  # noqa: E402

TURN = 1 | 2 | 4   # colour, intensity, direction; distance stays


def sun_changes(n_lights, n_frames):
    """Per frame, one change per light of colour, intensity and direction: a direction on a sun arc (never along +-Y), a warm-to-white colour and an intensity
    that follow the sun's height."""
    out = []
    for k in range(n_frames):
        c = np.zeros(n_lights, dtype=DIRECTIONAL_LIGHT_CHANGE_DTYPE)
        theta = 0.35 + 0.04 * k + 0.5 * np.arange(n_lights)
        h = np.sin(theta)
        c["index"] = np.arange(n_lights)
        c["mask"] = TURN
        c["direction"] = np.stack([np.cos(theta), -(0.2 + np.abs(h)), 0.3 * (np.arange(n_lights) - 1.5)], axis=1)
        c["color"] = np.stack([np.ones(n_lights), 0.6 + 0.4 * np.abs(h), 0.4 + 0.6 * np.abs(h)], axis=1)
        c["intensity"] = 0.15 + 0.1 * np.abs(h)
        out.append(c)
    return out


def applied(sources, changes):
    """The sources after the changes (update_from_changes field by field, in array order)."""
    s = sources.copy()
    for e in changes:
        i, m = int(e["index"]), int(e["mask"])
        if m & 1:
            s[i]["color"] = e["color"]
        if m & 2:
            s[i]["intensity"] = e["intensity"]
        if m & 4:
            s[i]["direction"] = e["direction"]
        if m & 8:
            s[i]["distance"] = e["distance"]
    return s


def dry_run(a):
    """No device: config 3 at a tiny size, the changes, and the per-frame sources of the set path checked against world.py's
    update_directional_light of the same lights."""
    from rend3_b200.world import DirectionalLight, DirectionalLightChange, Renderer

    ev, res = config3((64, 36), n_objects=2000)
    src = ev.directional_sources
    changes = sun_changes(len(src), a.frames)
    assert len(src) == 4 and all(c.shape == (4,) and c.dtype.itemsize == 48 for c in changes)
    r = Renderer(LEFT)
    handles = [r.add_directional_light(DirectionalLight(tuple(s["color"]), float(s["intensity"]), tuple(s["direction"]), float(s["distance"]),
                                                        int(s["resolution"]))) for s in src]
    for c in changes:
        want = applied(src, c)
        for e in c:
            h = next(h for h in handles if r.directional_shadow_index(h) == int(e["index"]))
            r.update_directional_light(h, DirectionalLightChange(color=tuple(e["color"]), intensity=float(e["intensity"]),
                                                                 direction=tuple(e["direction"])))
        got = r.evaluate().directional_sources
        assert got.tobytes() == want.tobytes(), "the set path's sources differ from world.py's updated lights"
    return dict(dry_run=True, resolution=res, lights=len(src), frames=len(changes), change_bytes_per_frame=int(changes[0].nbytes))


def frame_throughput(a):
    import torch

    from rend3_b200.backend import load_cuda_backend
    from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings
    from shadow_camera_cost import Timed

    ev, res = config3()
    changes = sun_changes(len(ev.directional_sources), a.frames)
    sources = [applied(ev.directional_sources, c) for c in changes]
    aw, ah = ev.shadow_target_size
    left = ev.camera.handedness == LEFT
    settings = BaseRenderGraphSettings()
    timed_calls = {"set": {"set_directional_light_sources", "evaluate_shadow_cameras"},
                   "host_form": {"update_directional_light_sources", "evaluate_shadow_cameras"},
                   "device_form": {"update_directional_light_sources_device", "evaluate_shadow_cameras"}}
    paths = {}
    for name, calls in timed_calls.items():
        b = load_cuda_backend(0)
        t = Timed(b, calls)
        g = BaseRenderGraph(t)
        g.add_to_graph(ev, res, 1, settings, frame_graph=True, device_shadow_cameras=True)   # uploads the world
        per_frame = changes
        if name == "device_form":
            with torch.cuda.stream(torch.cuda.ExternalStream(b.stream())):
                per_frame = [torch.from_numpy(c.view(np.uint8).reshape(-1, 48)).cuda() for c in changes]
            torch.cuda.synchronize()

        class SetInFrame:
            """the set path: the changed list re-set where the update would be enqueued, inside the frame bracket"""
            def __init__(self, t, k):
                self.t, self.k = t, k

            def __getattr__(self, n):
                return getattr(self.t, n)

            def evaluate_shadow_cameras(self, loc):
                self.t.set_directional_light_sources(sources[self.k], aw, ah, left)
                self.t.evaluate_shadow_cameras(loc)

        def frame(k, t=t, g=g, name=name, per_frame=per_frame, SetInFrame=SetInFrame):
            if name == "set":
                g.backend = SetInFrame(t, k)
                g.add_to_graph(ev, res, 1, settings, upload=False, frame_graph=True, device_shadow_cameras=True)
                g.backend = t
            else:
                g.add_to_graph(ev, res, 1, settings, upload=False, frame_graph=True, device_shadow_cameras=True,
                               directional_changes=per_frame[k])
        for k in range(3):                        # warm both graph parities
            frame(k)
        b.sync()
        paths[name] = dict(b=b, t=t, frame=frame, fps=[], call_ms=[], flushed=[], keep=per_frame)
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


def kernel_time(a):
    """directional_light_change_kernel alone on config 3's four lights: CUDA events around --kernel-launches back-to-back launches of each
    form, enqueued while the stream is held by a sleep kernel so that the events time the device, not the Python submission rate."""
    import torch

    from rend3_b200.backend import load_cuda_backend

    ev, _ = config3((64, 36), n_objects=2000)   # the same four lights; the kernel never reads the objects
    b = load_cuda_backend(0)
    b.set_directional_light_sources(ev.directional_sources, *ev.shadow_target_size, True)
    host = sun_changes(len(ev.directional_sources), 1)[0]
    stream = torch.cuda.ExternalStream(b.stream())
    with torch.cuda.stream(stream):
        dev = torch.from_numpy(host.view(np.uint8).reshape(-1, 48)).cuda()
    torch.cuda.synchronize()
    out = {}
    for name, call in (("host_form", lambda: b.update_directional_light_sources(host)),
                       ("device_form", lambda: b.update_directional_light_sources_device(dev))):
        for _ in range(50):
            call()
        b.sync()
        us, host_us = [], []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(stream):
                torch.cuda._sleep(100_000_000)   # ~50 ms at 1.98 GHz: longer than enqueueing the launches below
            e0.record(stream)
            t0 = time.perf_counter()
            for _ in range(a.kernel_launches):
                call()
            host_us.append(1e6 * (time.perf_counter() - t0) / a.kernel_launches)
            e1.record(stream)
            e1.synchronize()
            us.append(1e3 * e0.elapsed_time(e1) / a.kernel_launches)
        out[name] = dict(device_us_per_launch_median=statistics.median(us), device_us_per_launch=us,
                         host_us_per_call_median=statistics.median(host_us), launches=a.kernel_launches)
    b.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--kernel-launches", type=int, default=512)
    ap.add_argument("--dry-run", action="store_true", help="no device: build the world and the changes at a tiny size and check them")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.dry_run:
        doc = dry_run(a)
    else:
        from world_update_cost import card

        doc = dict(card(), config="config3 3840x2160, 200k objects, 4 directional lights (2048^2, device shadow cameras) turning and "
                   "changing colour and intensity every frame, 4 point lights, camera static", frames_per_rep=a.frames, reps=a.reps)
        doc["paths"] = frame_throughput(a)
        doc["kernel"] = kernel_time(a)
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(s)


if __name__ == "__main__":
    main()
