"""What a texture that changes every frame costs through each way its texels can reach the device.

Three workloads, each rendering a textured full-screen quad (or, for the sky, the skybox alone) at 640x360 in frame graphs:
  video   one 3840x2160 RGBA8 level per frame.  set: r3_set_textures of the whole table; update: r3_update_textures of the level's bytes;
          host_form: r3_write_texture_regions; device_form: r3_write_texture_regions_device from a CUDA tensor.
  pages   1024 random 128x128 BC7 pages (16 KB each) into sixteen 4096^2 BC7 textures.  device_form against one cudaMemcpy2DAsync per
          page into a device buffer of the same layout (the library does not hand out its blob, so the per-page copies go to a stand-in
          of the same size and pitches: the same copies the application would make with a bare pointer).
  sky     six 512^2 RGBA32F faces per frame.  set: r3_set_skybox; device_form: r3_write_texture_regions_device.
Every write call runs through the graph's before_resolve hook, which is inside the recorded frame and before the pass that samples the
texture; the set / update / host forms drain the stream there (an early flush).  Reported per method: frames per second over --frames frames (median of --reps), host ms per write call,
early flushes per frame, and the plan + copy kernels' time (CUDA events around --kernel-reps back-to-back device-form calls) against the
least time HBM allows, 2 x bytes / 3.35 TB/s (H100 SXM data sheet).  The card's name and power limit are read in the same run.  Writes
one JSON document to stdout (and to --out).

    python tools/texture_write_cost.py [--reps 3] [--frames 16] [--kernel-reps 20]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rend3_b200 import glam  # noqa: E402
from rend3_b200.layouts import SKYBOX_FACE, TEXTURE_REGION_DTYPE  # noqa: E402
from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings  # noqa: E402
from rend3_b200.world import LEFT, Camera, MeshBuilder, Object, PbrMaterial, Renderer, Texture  # noqa: E402

HBM = 3.35e12
RES = (640, 360)


def quad_world(textures):
    r = Renderer(LEFT, aspect_ratio=RES[0] / RES[1])
    pos = [(-1, -1, 0.5), (-1, 1, 0.5), (1, 1, 0.5), (1, -1, 0.5)]
    mesh = MeshBuilder.new(pos, LEFT).with_indices([0, 1, 2, 0, 2, 3]).with_vertex_texture_coordinates_0([((x + 1) / 2, (1 - y) / 2) for x, y, _ in pos]).build()
    handles = [r.add_texture_2d(t) for t in textures]
    mat = r.add_material(PbrMaterial(albedo_texture=handles[0], unlit=True))
    r.add_object(Object(r.add_mesh(mesh), mat, glam.identity()))
    r.set_camera_data(Camera(("raw", glam.identity()), glam.identity()))
    return r


def region_array(rows):
    a = np.zeros(len(rows), dtype=TEXTURE_REGION_DTYPE)
    for k, row in enumerate(rows):
        a[k] = row
    return a


def cudart():
    for name in ("libcudart.so", "libcudart.so.12", "/usr/local/cuda/lib64/libcudart.so"):
        try:
            return ctypes.CDLL(name)
        except OSError:
            pass
    raise RuntimeError("libcudart not found")


def frames(b, ev, graph, n, write):
    """n frame graphs with write(k) inside each; (frames per second, host ms per write call, early flushes per frame)."""
    calls = []

    def timed(k):
        t = time.perf_counter()
        out = write(k)
        calls.append(time.perf_counter() - t)
        return out
    s0 = b.frame_graph_stats()
    b.sync()
    t0 = time.perf_counter()
    for k in range(n):
        graph.add_to_graph(ev, RES, 1, BaseRenderGraphSettings(), upload=False, frame_graph=True, before_resolve=lambda k=k: timed(k))
    b.sync()
    wall = time.perf_counter() - t0
    s1 = b.frame_graph_stats()
    return n / wall, 1e3 * statistics.median(calls), (s1["flushed"] - s0["flushed"]) / n


def kernel_ms(b, call, reps):
    import torch

    stream = torch.cuda.ExternalStream(b.stream())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    call()
    b.sync()
    with torch.cuda.stream(stream):
        e0.record(stream)
        for _ in range(reps):
            call()
        e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def run_methods(b, ev, methods, args):
    graph = BaseRenderGraph(b)
    graph.add_to_graph(ev, RES, 1, BaseRenderGraphSettings())
    for name, fn in methods.items():                                         # warm up every shape
        frames(b, ev, graph, 2, fn)
    res = {name: [] for name in methods}
    for _ in range(args.reps):                                               # alternated, rep by rep
        for name, fn in methods.items():
            res[name].append(frames(b, ev, graph, args.frames, fn))
    return {name: {"frames_per_s": statistics.median(r[0] for r in v), "host_ms_per_call": statistics.median(r[1] for r in v),
                   "flushes_per_frame": statistics.median(r[2] for r in v)} for name, v in res.items()}


def video(args, load):
    import torch

    rng = np.random.default_rng(1)
    w, h = 3840, 2160
    r = quad_world([Texture(rng.integers(0, 256, (h, w, 4), dtype=np.uint8), mips="none")])
    ev = r.evaluate()
    b = load()
    frames_host = [rng.integers(0, 256, w * h * 4, dtype=np.uint8) for _ in range(2)]
    frames_dev = [torch.from_numpy(f).cuda() for f in frames_host]
    regions = region_array([(0, 0, 0, 0, 0, w, h, 4 * w, 0)])
    d_regions = torch.from_numpy(regions.view(np.uint8).reshape(1, 40).copy()).cuda()
    off = int(ev.texture_descs[0]["byte_offset"])
    torch.cuda.synchronize()

    methods = {"set": lambda k: b.set_textures(ev.texture_descs, ev.texture_texels),
               "update": lambda k: b.update_textures(0, ev.texture_descs[:0], off, frames_host[k % 2]),
               "host_form": lambda k: b.write_texture_regions(regions, frames_host[k % 2]),
               "device_form": lambda k: b.write_texture_regions_device(d_regions, frames_dev[k % 2])}
    out = run_methods(b, ev, methods, args)
    ms = kernel_ms(b, lambda: b.write_texture_regions_device(d_regions, frames_dev[0]), args.kernel_reps)
    out["kernels"] = {"ms": ms, "bytes": w * h * 4, "hbm_floor_ms": 2 * w * h * 4 / HBM * 1e3}
    b.close()
    return out


def pages(args, load):
    import torch

    rng = np.random.default_rng(2)
    n_tex, size, page, n_pages = 16, 4096, 128, 1024
    blocks = size // 4
    from rend3_b200.layouts import TEXFMT_BC7_RGBA_UNORM, TEXTURE_DESC_DTYPE
    descs = np.zeros(n_tex, TEXTURE_DESC_DTYPE)
    level = blocks * blocks * 16
    for i in range(n_tex):
        descs[i] = (size, size, 1, TEXFMT_BC7_RGBA_UNORM, i * level)
    b = load()
    b.set_textures(descs, np.zeros(n_tex * level, np.uint8))
    slots = rng.choice(n_tex * (size // page) ** 2, n_pages, replace=False)
    page_bytes = (page // 4) ** 2 * 16
    rows = []
    for k, s in enumerate(slots):
        t, p = divmod(int(s), (size // page) ** 2)
        py, px = divmod(p, size // page)
        rows.append((k * page_bytes, t, 0, px * page, py * page, page, page, (page // 4) * 16, 0))
    regions = region_array(rows)
    d_regions = torch.from_numpy(regions.view(np.uint8).reshape(-1, 40).copy()).cuda()
    d_src = torch.from_numpy(rng.integers(0, 256, n_pages * page_bytes, dtype=np.uint8)).cuda()
    stand_in = torch.empty(n_tex * level, dtype=torch.uint8, device="cuda")
    rt = cudart()
    rt.cudaMemcpy2DAsync.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_size_t,
                                     ctypes.c_int, ctypes.c_void_p]
    stream = b.stream()
    pitch = blocks * 16

    def memcpy2d():
        for row in regions:
            dst = stand_in.data_ptr() + int(row["texture"]) * level + (int(row["y"]) // 4) * pitch + (int(row["x"]) // 4) * 16
            rc = rt.cudaMemcpy2DAsync(dst, pitch, d_src.data_ptr() + int(row["src_offset"]), int(row["src_pitch"]), int(row["src_pitch"]),
                                      page // 4, 3, stream)
            assert rc == 0, rc
    torch.cuda.synchronize()
    out = {}
    for name, call in (("device_form", lambda: b.write_texture_regions_device(d_regions, d_src)), ("memcpy2d_per_page", memcpy2d)):
        host = []
        for _ in range(3):
            t = time.perf_counter()
            call()
            host.append(time.perf_counter() - t)
        b.sync()
        t0 = time.perf_counter()
        for _ in range(args.frames):
            call()
        b.sync()
        out[name] = {"calls_per_s": args.frames / (time.perf_counter() - t0), "host_ms_per_call": 1e3 * statistics.median(host),
                     "gpu_ms": kernel_ms(b, call, args.kernel_reps)}
    out["bytes"] = n_pages * page_bytes
    out["hbm_floor_ms"] = 2 * n_pages * page_bytes / HBM * 1e3
    b.close()
    return out


def sky(args, load):
    import torch

    rng = np.random.default_rng(3)
    n = 512
    r = Renderer(LEFT, aspect_ratio=RES[0] / RES[1])
    r.set_camera_data(Camera(("perspective", 90.0, 0.1), glam.identity()))
    faces = [rng.standard_normal((n, n, 4)).astype(np.float32) for _ in range(6)]
    r.set_skybox(faces, srgb=False, mips="none")
    ev = r.evaluate()
    b = load()
    face_bytes = n * n * 16
    regions = region_array([(f * face_bytes, SKYBOX_FACE(f), 0, 0, 0, n, n, n * 16, 0) for f in range(6)])
    d_regions = torch.from_numpy(regions.view(np.uint8).reshape(-1, 40).copy()).cuda()
    d_faces = [torch.from_numpy(rng.standard_normal(6 * n * n * 4).astype(np.float32)).cuda() for _ in range(2)]
    torch.cuda.synchronize()

    out = run_methods(b, ev, {"set": lambda k: b.set_skybox(ev.skybox_desc, ev.skybox_texels),
                              "device_form": lambda k: b.write_texture_regions_device(d_regions, d_faces[k % 2])}, args)
    out["kernels"] = {"ms": kernel_ms(b, lambda: b.write_texture_regions_device(d_regions, d_faces[0]), args.kernel_reps),
                      "bytes": 6 * face_bytes, "hbm_floor_ms": 2 * 6 * face_bytes / HBM * 1e3}
    b.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--kernel-reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from rend3_b200.backend import load_cuda_backend

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    load = lambda: load_cuda_backend(0)   # noqa: E731
    doc = {"card": card, "resolution": RES, "video": video(args, load), "pages": pages(args, load), "sky": sky(args, load)}
    text = json.dumps(doc, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
