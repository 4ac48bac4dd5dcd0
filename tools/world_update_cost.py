"""Per-frame upload cost of the incremental world updates against the full uploads they replace.

Each number is the host time of one upload call, ending in a stream sync (the calls block until the caller's bytes are consumed),
median of --reps after --warmup, the two variants alternated so that clock and thermal drift fall on both.  Records the card
name and its power limit beside the numbers.  Writes one JSON document to stdout (and to --out when given).

    python tools/world_update_cost.py [--reps 21] [--sizes 200000,1000000,10000000]
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
from rend3_b200.backend import load_cuda_backend  # noqa: E402
from rend3_b200.layouts import TEXTURE_DESC_DTYPE  # noqa: E402
from rend3_b200.scenes import object_cloud_records  # noqa: E402


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                               timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        power = f"unknown ({type(e).__name__})"
    return {"gpu": name, "power_limit": power}


def timed(b, fn):
    t0 = time.perf_counter()
    fn()
    b.sync()
    return (time.perf_counter() - t0) * 1e3


def alternate(b, variants, reps, warmup, setup=None):
    """variants: {name: fn}; returns {name: median ms}."""
    times = {k: [] for k in variants}
    for r in range(warmup + reps):
        for k, fn in variants.items():
            if setup:
                setup(k)
            t = timed(b, fn)
            if r >= warmup:
                times[k].append(t)
    return {k: round(statistics.median(v), 3) for k, v in times.items()}


def sort_info(n, seed):
    rng = np.random.default_rng(seed)
    key = rng.integers(0, 3, n).astype(np.uint64)
    flags = (1 | 2 * (key != 2) | 4 * (key == 2)).astype(np.uint8)
    return key, flags


def objects_section(b, sizes, reps, warmup):
    out = []
    for n in sizes:
        rec = object_cloud_records(n, seed=4)
        key, flags = sort_info(n, 5)
        loc = np.ascontiguousarray(rec["sphere_center"])
        b.set_objects(rec)
        b.set_object_sort_info(key, flags, loc)
        rng = np.random.default_rng(6)
        for frac in (0.01, 0.10):
            slots = np.sort(rng.choice(n, int(n * frac), replace=False)).astype(np.uint32)
            part, pk, pf, pl = rec[slots], key[slots], flags[slots], loc[slots]

            def full():
                b.set_objects(rec)
                b.set_object_sort_info(key, flags, loc)

            def incremental():
                b.update_objects(slots, part)
                b.update_object_sort_info(slots, pk, pf, pl)
            ms = alternate(b, {"full": full, "incremental": incremental}, reps, warmup)
            out.append({"slots": n, "changed_fraction": frac, "full_ms": ms["full"], "incremental_ms": ms["incremental"],
                        "full_h2d_bytes": n * (128 + 21), "incremental_h2d_bytes": len(slots) * (128 + 4 + 20)})
    return out


def growth_section(sizes, reps, warmup):
    """Grow the object buffer by 1 %: r3_resize_objects (device copy) vs r3_set_objects of the grown array.  A fresh context per
    repetition, so that every resize really reallocates (r3_set_objects sizes the buffer exactly)."""
    out = []
    for n in sizes:
        rec = object_cloud_records(n, seed=4)
        m = n + n // 100
        grown = np.zeros(m, dtype=rec.dtype)
        grown[:n] = rec
        times = {"resize": [], "set_objects": []}
        for r in range(warmup + reps):
            for k in times:
                b = load_cuda_backend(0)
                b.set_objects(rec)
                b.sync()
                t = timed(b, (lambda: b.resize_objects(m)) if k == "resize" else (lambda: b.set_objects(grown)))
                b.close()
                if r >= warmup:
                    times[k].append(t)
        out.append({"slots": n, "grown_to": m, "resize_ms": round(statistics.median(times["resize"]), 3),
                    "set_objects_ms": round(statistics.median(times["set_objects"]), 3)})
    return out


def mesh_section(b, reps, warmup):
    base = np.random.default_rng(7).integers(0, 2 ** 32, (1 << 30) // 4, dtype=np.uint32)
    out = []
    for mb in (1, 64):
        extra = np.random.default_rng(8).integers(0, 2 ** 32, (mb << 20) // 4, dtype=np.uint32)
        whole = np.concatenate([base, extra])
        b.set_mesh_buffer(base)
        grow_ms = timed(b, lambda: b.update_mesh_buffer(base.nbytes, extra))   # the first append past the capacity: grows the buffer
        ms = alternate(b, {"full": lambda: b.set_mesh_buffer(whole), "append": lambda: b.update_mesh_buffer(base.nbytes, extra)}, reps, warmup)
        out.append({"mesh_bytes": base.nbytes, "appended_bytes": extra.nbytes, "full_ms": ms["full"], "append_ms": ms["append"],
                    "append_with_growth_ms": round(grow_ms, 3)})
        del whole
    return out


def texture_section(b, reps, warmup):
    size, count = 1024, 256                                   # 256 RGBA8 textures of 4 MB: a 1 GB table
    descs = np.zeros(count + 1, dtype=TEXTURE_DESC_DTYPE)
    descs["width"], descs["height"], descs["mip_count"], descs["format"] = size, size, 1, 0
    descs["byte_offset"] = np.arange(count + 1, dtype=np.uint64) * size * size * 4
    texels = np.random.default_rng(9).integers(0, 256, (count + 1) * size * size * 4, dtype=np.uint8)
    head = texels[:count * size * size * 4]
    tail = texels[count * size * size * 4:]
    b.set_textures(descs[:count], head)
    grow_ms = timed(b, lambda: b.update_textures(count, descs[count:], int(descs[count]["byte_offset"]), tail))
    ms = alternate(b, {"full": lambda: b.set_textures(descs, texels),
                       "append": lambda: b.update_textures(count, descs[count:], int(descs[count]["byte_offset"]), tail)}, reps, warmup)
    return {"table_bytes": head.nbytes, "appended_bytes": tail.nbytes, "full_ms": ms["full"], "append_ms": ms["append"],
            "append_with_growth_ms": round(grow_ms, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sizes", default="200000,1000000,10000000")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    sizes = [int(s) for s in args.sizes.split(",")]
    b = load_cuda_backend(0)
    result = {"card": card(), "reps": args.reps, "warmup": args.warmup, "clock": "host perf_counter around the call, ending in r3_sync",
              "objects": objects_section(b, sizes, args.reps, args.warmup)}
    b.close()
    result["object_growth"] = growth_section([s for s in sizes if s >= 1_000_000], max(5, args.reps // 2), 1)
    b = load_cuda_backend(0)
    result["mesh"] = mesh_section(b, args.reps, args.warmup)
    b.close()
    b = load_cuda_backend(0)
    result["textures"] = texture_section(b, args.reps, args.warmup)
    b.close()
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
