"""Frame throughput of a walkthrough with the shadow cameras evaluated on the host against the device.

Config 3 (200k objects, 4 directional lights with 2048^2 shadow maps, 4 point lights, 3840x2160) with the camera moving every frame and the
world static.  Two contexts, alternated rep by rep so that clock and thermal drift fall on both:
  host    the caller evaluates the shadow cameras and uploads the light buffer with r3_set_directional_lights every frame (it drains the
          stream, so the next frame cannot be recorded before the previous one has finished);
  device  r3_set_directional_light_sources once; every frame r3_evaluate_shadow_cameras + r3_shadow_uniform_upload (enqueue only).
Each rep submits --frames frame graphs back to back and ends with one r3_sync; the number is frames per second over that window, median
of --reps.  The host-side cameras are computed before the timed window, so only the library's per-frame light calls are timed; their host
time per frame is reported too.  The card's name and power limit are recorded beside the numbers.  Writes one JSON document to stdout
(and to --out when given).

    python tools/shadow_camera_cost.py [--reps 7] [--frames 32]
"""
import argparse
import dataclasses
import json
import os
import statistics
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from rend3_b200 import glam  # noqa: E402
from rend3_b200.backend import load_cuda_backend  # noqa: E402
from rend3_b200.configs import config3  # noqa: E402
from rend3_b200.layouts import DIRECTIONAL_LIGHT_DTYPE  # noqa: E402
from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings  # noqa: E402
from rend3_b200.world import Camera, CameraState, DirectionalLight, ShadowDesc, shadow_camera  # noqa: E402
from world_update_cost import card  # noqa: E402

f32 = np.float32


def frames(ev, n):
    """n EvalOutputs of a camera sliding 3 cm per frame (across shadow texels: 100 / 2048 = 4.9 cm), with host-evaluated cameras."""
    base = ev.camera
    out = []
    for k in range(n):
        view = glam.mul(base.view, glam.from_translation((-0.03 * k, 0.0, -0.02 * k)))
        cam = CameraState(Camera(base.data.projection, view), base.handedness, base.aspect_ratio)
        shadows, dl = [], np.frombuffer(ev.directional_buffer[16:], dtype=DIRECTIONAL_LIGHT_DTYPE).copy()
        for i, s in enumerate(ev.directional_sources):
            light = DirectionalLight(tuple(s["color"]), float(s["intensity"]), tuple(s["direction"]), float(s["distance"]), int(s["resolution"]))
            sc = shadow_camera(light, cam)
            shadows.append(ShadowDesc(tuple(int(v) for v in s["offset"]), int(s["size"]), i, sc))
            dl[i]["view_proj"] = sc.view_proj.reshape(16)
        buf = np.array([len(dl), 0, 0, 0], dtype=np.uint32).tobytes() + dl.tobytes()
        out.append(dataclasses.replace(ev, camera=cam, shadows=shadows, directional_buffer=buf))
    return out


class Timed:
    """Forwards to a backend and sums the host time of the named entry points."""

    def __init__(self, b, names):
        self.b, self.names, self.seconds = b, names, 0.0

    def __getattr__(self, name):
        attr = getattr(self.b, name)
        if name not in self.names:
            return attr

        def timed(*a, **k):
            t0 = time.perf_counter()
            r = attr(*a, **k)
            self.seconds += time.perf_counter() - t0
            return r
        return timed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ev, res = config3()
    evs = frames(ev, a.frames)
    settings = BaseRenderGraphSettings()
    paths = {}
    for name, device in (("host", False), ("device", True)):
        b = load_cuda_backend(0)
        t = Timed(b, {"set_directional_lights"} if not device else {"evaluate_shadow_cameras", "shadow_uniform_upload"})
        g = BaseRenderGraph(t)
        g.add_to_graph(evs[0], res, 1, settings, frame_graph=True, device_shadow_cameras=device)   # uploads and allocates
        for e in evs[:3]:                                                                        # warm both graph parities
            if not device:
                t.set_directional_lights(e.directional_buffer, *e.shadow_target_size)
            g.add_to_graph(e, res, 1, settings, upload=False, frame_graph=True, device_shadow_cameras=device)
        b.sync()
        paths[name] = dict(b=b, t=t, g=g, device=device, fps=[], call_ms=[], flushed=[])
    for _ in range(a.reps):
        for name, p in paths.items():
            b, t, g = p["b"], p["t"], p["g"]
            t.seconds = 0.0
            f0 = b.frame_graph_stats()["flushed"]
            t0 = time.perf_counter()
            for e in evs:
                if not p["device"]:
                    t.set_directional_lights(e.directional_buffer, *e.shadow_target_size)
                g.add_to_graph(e, res, 1, settings, upload=False, frame_graph=True, device_shadow_cameras=p["device"])
            b.sync()
            dt = time.perf_counter() - t0
            p["fps"].append(len(evs) / dt)
            p["call_ms"].append(1e3 * t.seconds / len(evs))
            p["flushed"].append((b.frame_graph_stats()["flushed"] - f0) / len(evs))
    doc = dict(card(), config="config3 3840x2160, 200k objects, 4 directional + 4 point lights, camera moving every frame",
               frames_per_rep=a.frames, reps=a.reps)
    for name, p in paths.items():
        doc[name] = dict(fps_median=statistics.median(p["fps"]), fps=p["fps"], light_calls_host_ms_per_frame=statistics.median(p["call_ms"]),
                         early_flushes_per_frame=statistics.median(p["flushed"]))
        p["b"].close()
    doc["device_over_host_fps"] = doc["device"]["fps_median"] / doc["host"]["fps_median"]
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(s)


if __name__ == "__main__":
    main()
