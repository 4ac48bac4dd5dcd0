"""Per-step cost of moving objects: r3_update_objects + r3_update_object_sort_info against r3_set_object_transforms (host form) and
r3_set_object_transforms_device (device form).

On the 10 M-object cull + bake world of bench.py (same seeded generator) and on a 200 k-slot world, for 1 % / 10 % / 100 % of the slots
moved per step, the three paths alternate in the same run; each is followed by the cull + bake step.  Times are CUDA events on the
library's stream (step: from before the update to after the cull + bake; kernel: around the device-form call alone), medians of --steps
after --warmup, repeated --runs times.  Bytes per second use the algorithmic 256 B per moved object (64 matrix + 16 mesh sphere read;
80 record + 80 dense copies + 12 location written; 4 slot read in the sparse form).  Host time is perf_counter around the calls alone.
Prints the card's name and power limit read in the same run and one JSON line.  Fails without a GPU.

    python tools/object_transform_cost.py [--steps 21] [--runs 3] [--sizes 200000,10000000] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rend3_b200.backend import CAMERA_VIEWPORT, CB_BAKE, CB_CULL, load_cuda_backend  # noqa: E402
from rend3_b200.routines import per_camera_header  # noqa: E402
from rend3_b200.scenes import cloud_camera, object_cloud_records  # noqa: E402

BYTES_PER_OBJECT = 256
f32 = np.float32


def card(torch):
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                               timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        power = f"unknown ({type(e).__name__})"
    return {"gpu": name, "power_limit": power}


def host_records(rec, ms, slots, mats):
    """The bytes today's path uploads: the records with the moved transform and sphere, and the locations (float32, the rule's order)."""
    m = mats.reshape(-1, 4, 4)
    s = ms[slots]
    part = rec[slots].copy()
    ls = [(m[:, a, 0] * m[:, a, 0] + m[:, a, 1] * m[:, a, 1]) + m[:, a, 2] * m[:, a, 2] for a in range(3)]
    part["transform"] = mats
    for r in range(3):
        part["sphere_center"][:, r] = ((m[:, 0, r] * s[:, 0] + m[:, 1, r] * s[:, 1]) + m[:, 2, r] * s[:, 2]) + m[:, 3, r]
    part["sphere_radius"] = np.sqrt(np.fmax(ls[0], np.fmax(ls[1], ls[2]))) * s[:, 3]
    return part, np.ascontiguousarray(m[:, 3, :3])


def world_section(torch, n, steps, warmup, runs):
    rec = object_cloud_records(n, seed=4)
    rng = np.random.default_rng(5)
    key = rng.integers(0, 3, n).astype(np.uint64)
    flags = (1 | 2 * (key != 2) | 4 * (key == 2)).astype(np.uint8)
    ms = np.zeros((n, 4), f32)
    ms[:, 3] = np.sqrt(f32(3.0))                                    # unit cube mesh
    header = per_camera_header(cloud_camera(), CAMERA_VIEWPORT, (1920, 1080), 1, n)
    b = load_cuda_backend(0)
    b.set_objects(rec)
    b.set_object_sort_info(key, flags, np.ascontiguousarray(rec["sphere_center"]))
    b.set_object_mesh_spheres(ms)
    stream = torch.cuda.ExternalStream(b.stream())
    rows = []
    for frac in (0.01, 0.10, 1.0):
        k = int(n * frac)
        slots = None if k == n else np.sort(rng.choice(n, k, replace=False)).astype(np.uint32)
        idx = np.arange(n) if slots is None else slots
        mats = np.ascontiguousarray(rec["transform"][idx])
        mats[:, 12:15] += f32(0.25)
        part, loc = host_records(rec, ms, idx, mats)
        pk, pf = key[idx], flags[idx]
        upd_slots = idx.astype(np.uint32)
        pinned = torch.from_numpy(mats).pin_memory()
        pinned_np = pinned.numpy()
        with torch.cuda.stream(stream):
            d_base = pinned.to("cuda")
            d_mats = torch.empty_like(d_base)
            d_slots = None if slots is None else torch.from_numpy(slots.view(np.int32)).to("cuda")
        b.sync()

        def cull():
            b.object_uniform_upload(CAMERA_VIEWPORT, header, CB_BAKE | CB_CULL)

        def update_path():
            b.update_objects(upd_slots, part)
            b.update_object_sort_info(upd_slots, pk, pf, loc)

        def host_form():
            b.set_object_transforms(pinned_np, slots)

        def device_form():
            with torch.cuda.stream(stream):
                torch.add(d_base, 0.0, out=d_mats)                   # the producer: a torch op on the context's stream
            b.set_object_transforms_device(d_mats, d_slots)

        variants = {"update_objects+sort_info": update_path, "set_object_transforms": host_form, "set_object_transforms_device": device_form}
        result = {name: {"step_ms": [], "host_ms": []} for name in variants}
        kernel_ms = []
        for _ in range(runs):
            t = {name: ([], []) for name in variants}
            kt = []
            for i in range(warmup + steps):
                for name, fn in variants.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    b.sync()
                    e0.record(stream)
                    h0 = time.perf_counter()
                    fn()
                    h1 = time.perf_counter()
                    cull()
                    e1.record(stream)
                    b.sync()
                    if i >= warmup:
                        t[name][0].append(e0.elapsed_time(e1))
                        t[name][1].append((h1 - h0) * 1e3)
                # the kernel alone: the device form between two events, its producer outside them
                k0, k1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                k0.record(stream)
                b.set_object_transforms_device(d_mats, d_slots)
                k1.record(stream)
                b.sync()
                if i >= warmup:
                    kt.append(k0.elapsed_time(k1))
            for name in variants:
                result[name]["step_ms"].append(round(statistics.median(t[name][0]), 4))
                result[name]["host_ms"].append(round(statistics.median(t[name][1]), 4))
            kernel_ms.append(round(statistics.median(kt), 4))
        best = min(kernel_ms)
        rows.append({"slots": n, "moved": k, "fraction": frac, "form": "dense" if slots is None else "sparse", "paths": result,
                     "kernel_ms": kernel_ms, "kernel_model_bytes": k * BYTES_PER_OBJECT,
                     "kernel_gb_per_s_best_run": round(k * BYTES_PER_OBJECT / (best * 1e-3) / 1e9, 1) if best > 0 else None})
    # a graphed frame that moves objects with the device form: early flushes after the first frame
    before = b.frame_graph_stats()
    for _ in range(4):
        b.frame_begin()
        b.set_object_transforms_device(d_mats, d_slots)
        b.object_uniform_upload(CAMERA_VIEWPORT, header, CB_BAKE | CB_CULL)
        b.frame_end()
    b.sync()
    after = b.frame_graph_stats()
    b.close()
    return rows, {"frames": after["frames"] - before["frames"], "graphed": after["graphed"] - before["graphed"],
                  "early_flushes": after["flushed"] - before["flushed"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--sizes", default="200000,10000000")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        sys.exit("object_transform_cost.py needs a CUDA device: there is nothing to measure without one")
    out = {"card": card(torch), "steps": args.steps, "warmup": args.warmup, "runs": args.runs,
           "clock": "CUDA events on the library's stream; host_ms is perf_counter around the update calls", "bytes_per_object_model": BYTES_PER_OBJECT,
           "worlds": []}
    for n in (int(s) for s in args.sizes.split(",")):
        rows, graph = world_section(torch, n, args.steps, args.warmup, args.runs)
        out["worlds"].append({"slots": n, "rows": rows, "graphed_device_form_frames": graph})
    text = json.dumps(out)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
