"""What taking the sphere centre from the transform's translation does to the 10 M-object cull + bake, against a built parent checkout.

A slot whose bounding-sphere centre has exactly the bit patterns of its translation column carries a centre bit; the fused cull + bake
then reads its 4-byte radius instead of the 16-byte sphere (52 B + 3 bits per object instead of 64 B + 2 bits).  Three measurements,
the card's name and power limit recorded beside them:
  (a) `bench.py --gpus 1 --steps S --warmup W` run --runs times in --parent and in this tree, alternating run by run: the headline
      ms_per_step and value, roofline.kernel_ms, forward.frame_ms, forward.config3.frame_ms and the dynamic / e2e rows;
  (b) the cull + bake step alone (r3_object_uniform_upload with CB_BAKE | CB_CULL, CUDA events on the library's stream, --world-steps
      steps after a warm-up) on bench.py's 10 M-object world, in both trees, alternating, with 100 %, 50 % (random slots) and 0 % of
      the slots centred — the others' centre moved one ulp in x off the translation — and a hash of each world's visible list, which
      must agree between the trees;
  (c) the share of slots with the bit in the config 3 (a 20 k-object sample), config 4 and config 5 worlds.

    python tools/cull_bake_cost.py --parent DIR [--runs 5] [--steps 50] [--warmup 5] [--world-runs 3] [--world-steps 50] [--out FILE]
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.abspath(__file__)
N_OBJECTS = 10_000_000
SHARES = (1.0, 0.5, 0.0)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    name, _, limit = q.splitlines()[0].partition(",") if q else ("unknown", "", "unknown")
    return {"gpu": name.strip(), "power_limit": limit.strip()}


def centred(rec):
    """Per slot: the sphere centre has the bit patterns of the translation (transform elements 12-14)."""
    return np.all(rec["transform"][:, 12:15].view(np.uint32) == rec["sphere_center"].view(np.uint32), axis=1)


def off_centre(rec, share, seed=5):
    """`rec` with (1 - share) of its slots (random ones) moved off the centre bit: centre x one ulp towards +inf."""
    out = rec.copy()
    n = len(out)
    keep = np.zeros(n, dtype=bool)
    if share >= 1.0:
        keep[:] = True
    elif share > 0.0:
        keep[np.random.default_rng(seed).choice(n, int(n * share), replace=False)] = True
    c = out["sphere_center"]
    c[~keep, 0] = np.nextafter(c[~keep, 0], np.float32(np.inf))
    return out


def world_worker(tree, steps, warmup):
    """(b) inside one tree: imports the library of `tree` and times the cull + bake on the three worlds."""
    sys.path.insert(0, tree)
    import torch

    from rend3_b200.backend import CAMERA_VIEWPORT, CB_BAKE, CB_CULL, load_cuda_backend
    from rend3_b200.routines import per_camera_header
    from rend3_b200.scenes import cloud_camera, object_cloud_records

    base = object_cloud_records(N_OBJECTS, seed=4)     # bench.py's world (rank 0)
    header = per_camera_header(cloud_camera(), CAMERA_VIEWPORT, (1920, 1080), 1, N_OBJECTS)
    b = load_cuda_backend(0)
    stream = torch.cuda.ExternalStream(b.stream())
    out = {}
    for share in SHARES:
        rec = off_centre(base, share)
        b.set_objects(rec)
        for _ in range(warmup):
            b.object_uniform_upload(CAMERA_VIEWPORT, header, CB_BAKE | CB_CULL)
        b.sync()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(steps):
            b.object_uniform_upload(CAMERA_VIEWPORT, header, CB_BAKE | CB_CULL)
        e1.record(stream)
        e1.synchronize()
        vis = b.readback_visible(CAMERA_VIEWPORT)
        out[f"{int(share * 100)}%"] = {"ms_per_step": e0.elapsed_time(e1) / steps, "centred_share": float(centred(rec).mean()),
                                       "visible": int(len(vis)), "visible_sha16": hashlib.sha256(np.ascontiguousarray(vis).tobytes()).hexdigest()[:16]}
    b.close()
    print(json.dumps(out), flush=True)


def find(doc, *path):
    for k in path:
        if not isinstance(doc, dict) or k not in doc:
            return None
        doc = doc[k]
    return doc


def bench_row(doc):
    return {"ms_per_step": doc["ms_per_step"], "value": doc["value"], "kernel_ms": find(doc, "roofline", "kernel_ms"),
            "forward_frame_ms": find(doc, "forward", "frame_ms"), "config3_frame_ms": find(doc, "forward", "config3", "frame_ms"),
            "dynamic_ms_per_step": {str(r["updated_fraction"]): r["ms_per_step"] for r in (doc.get("dynamic") or [])},
            "e2e_value": find(doc, "e2e", "value")}


def run_json(cmd, cwd):
    t0 = time.perf_counter()
    r = subprocess.run(cmd, cwd=cwd, capture_output=True, text=True)
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode != 0 or not line:
        return {"error": (r.stderr or r.stdout)[-600:]}, time.perf_counter() - t0
    return json.loads(line[-1]), time.perf_counter() - t0


def spread(rows, key):
    v = [r[key] for r in rows if r.get(key) is not None]
    return {"median": statistics.median(v), "min": min(v), "max": max(v)} if v else None


def bench_runs(a):
    """(a) bench.py in the parent checkout and in this tree, alternated run by run."""
    trees = (("parent", a.parent), ("this", ROOT))
    rows = {name: [] for name, _ in trees}
    for _ in range(a.runs):
        for name, tree in trees:
            doc, secs = run_json([sys.executable, "bench.py", "--gpus", "1", "--steps", str(a.steps), "--warmup", str(a.warmup)], tree)
            rows[name].append(dict(bench_row(doc), seconds=round(secs, 1)) if "error" not in doc else doc)
    out = {"runs": rows}
    for name, rs in rows.items():
        ok = [r for r in rs if "error" not in r]
        out[name] = {k: spread(ok, k) for k in ("ms_per_step", "value", "kernel_ms", "forward_frame_ms", "config3_frame_ms", "e2e_value")}
        out[name]["dynamic_ms_per_step"] = {f: spread([{"v": r["dynamic_ms_per_step"].get(f)} for r in ok], "v") for f in ("0.01", "0.1", "1.0")}
    p, t = out["parent"]["ms_per_step"], out["this"]["ms_per_step"]
    if p and t:
        out["headline"] = {"median_ratio": t["median"] / p["median"], "every_run_faster": t["max"] < p["min"]}
    return out


def world_runs(a):
    """(b) the three centre worlds in both trees, alternated run by run."""
    trees = (("parent", a.parent), ("this", ROOT))
    rows = {name: [] for name, _ in trees}
    for _ in range(a.world_runs):
        for name, tree in trees:
            doc, _ = run_json([sys.executable, HERE, "--world-worker", tree, "--world-steps", str(a.world_steps)], ROOT)
            rows[name].append(doc)
    out = {"runs": rows}
    for share in SHARES:
        key = f"{int(share * 100)}%"
        per = {}
        for name, rs in rows.items():
            ok = [r[key] for r in rs if key in r]
            per[name] = {"ms_per_step": spread(ok, "ms_per_step"), "visible_sha16": sorted({r["visible_sha16"] for r in ok})}
        if per["parent"]["ms_per_step"] and per["this"]["ms_per_step"]:
            per["median_ratio"] = per["this"]["ms_per_step"]["median"] / per["parent"]["ms_per_step"]["median"]
        per["same_visible_list"] = per["parent"]["visible_sha16"] == per["this"]["visible_sha16"] and len(per["this"]["visible_sha16"]) == 1
        out[key] = per
    return out


def shares():
    """(c) share of (enabled) slots whose sphere centre is bit for bit the translation."""
    sys.path.insert(0, ROOT)
    from rend3_b200 import configs
    from rend3_b200.scenes import object_cloud_records

    rec4 = object_cloud_records(N_OBJECTS, seed=4)
    out = {"config4 (bench.py world, all slots)": float(centred(rec4).mean())}
    for name, (ev, _) in (("config3 (20 k-object sample, enabled slots)", configs.config3(n_objects=20_000)),
                          ("config5 (enabled slots)", configs.config5())):
        rec = ev.object_buffer
        en = rec["enabled"] != 0
        out[name] = float(centred(rec[en]).mean())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", help="a built checkout of the parent commit")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--world-runs", type=int, default=3)
    ap.add_argument("--world-steps", type=int, default=50)
    ap.add_argument("--skip-bench", action="store_true", help="only (b) and (c)")
    ap.add_argument("--world-worker", metavar="TREE", help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.world_worker:
        return world_worker(a.world_worker, a.world_steps, 5)
    if not a.parent:
        ap.error("--parent DIR is required")
    a.parent = os.path.abspath(a.parent)
    doc = {"card": card(), "objects": N_OBJECTS, "centre_share": shares()}
    if not a.skip_bench:
        doc["bench"] = bench_runs(a)
    doc["centre_worlds"] = world_runs(a)
    doc["card_after"] = card()
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(s)


if __name__ == "__main__":
    main()
