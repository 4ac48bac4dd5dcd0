"""batch_objects on the device closes batches at the dispatch limit (max_dispatch_count x 256 invocations, batching.rs:194-209) like the
host path and the oracle: bit-identical batch and region tables at limits from 0 to 65535, through every sort tier, the frame-wide
sort, back-to-front objects, NaN distances and moving split points; whole frames of worlds with 76,800-triangle meshes against the
oracle; and such a world stays on the device, so a frame graph is not flushed."""
import numpy as np
import pytest

from rend3_b200.backend import CAMERA_VIEWPORT, CB_CULL, R3Error, load_cuda_backend
from rend3_b200.configs import config1
from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings, per_camera_header
from rend3_b200.scenes import cloud_camera, cube_field_scene, object_cloud_records

from batch_split_cases import CASES, assert_same_tables, expected_tables, load
from oracle import load_oracle_backend
from harness import compare_frame_state

pytestmark = pytest.mark.gpu
LIMITS = [0, 1, 2, 3, 255, 256, 65535]


def _device(monkeypatch):
    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    return load_cuda_backend(0)


def _upload_host(monkeypatch, fn):
    """The host path is chosen when the sort info is uploaded (R3_HOST_BATCHING is read there)."""
    monkeypatch.setenv("R3_HOST_BATCHING", "1")
    try:
        fn()
    finally:
        monkeypatch.delenv("R3_HOST_BATCHING")


def _check_device_info(b, what, camera=CAMERA_VIEWPORT):
    info = b.batching_info(camera)
    assert info["path"].startswith("device") and info["overflow"] == 0, f"{what}: {info}"
    return info


@pytest.mark.parametrize("frame_sort", ["0", "1"])
def test_hand_made_cases_at_every_limit(monkeypatch, frame_sort):
    """Each tiny world at its own limit equals the hand-made tables; at every limit of LIMITS the device equals the host path and the oracle."""
    monkeypatch.setenv("R3_FRAME_SORT", frame_sort)
    dev, orc = _device(monkeypatch), load_oracle_backend()
    host = load_cuda_backend(0)
    for name, c in sorted(CASES.items()):
        for md in [c["max_dispatch"]] + LIMITS:
            cc = dict(c, max_dispatch=md)
            load(dev, cc)
            load(orc, cc)
            _upload_host(monkeypatch, lambda: load(host, cc))
            what = f"{name} at max_dispatch_count {md}"
            _check_device_info(dev, what)
            assert host.batching_info(CAMERA_VIEWPORT)["path"] == "host"
            bd, rd = dev.readback_batches(CAMERA_VIEWPORT)
            bo, ro = orc.readback_batches(CAMERA_VIEWPORT)
            bh, rh = host.readback_batches(CAMERA_VIEWPORT)
            assert_same_tables(bd, rd, bo, ro, what + " (device vs oracle)")
            assert_same_tables(bh, rh, bo, ro, what + " (host vs oracle)")
            if md == c["max_dispatch"]:
                want_b, want_r = expected_tables(c)
                # the contexts carry the previous case's invocations over (the oracle's, equal to the device's, are checked above)
                want_b["object_culling_information"]["previous_global_invocation"] = bo["object_culling_information"]["previous_global_invocation"]
                assert_same_tables(bd, rd, want_b, want_r, what + " (device vs hand-made)")
    dev.close(), host.close()


def random_world(n, seed, big_fraction=0.002, nan_fraction=0.01):
    """n visible objects: 0-300 triangles, a few 20k-80k triangle ones, material keys 0-2, random atomic / back-to-front flags and
    some NaN locations."""
    rng = np.random.default_rng(seed)
    rec = object_cloud_records(n, seed=seed, extent=100.0, disabled_fraction=0.0)
    rec["sphere_radius"][:] = 1.0e6
    tris = rng.integers(0, 301, n)
    big = rng.random(n) < big_fraction
    tris[big] = rng.integers(20_000, 80_001, int(big.sum()))
    rec["index_count"] = (tris * 3).astype(np.uint32)
    key = rng.integers(0, 3, n).astype(np.uint64)
    flags = (1 | 2 * rng.integers(0, 2, n) | 4 * rng.integers(0, 2, n)).astype(np.uint8)
    loc = rec["sphere_center"].copy()
    loc[rng.random(n) < nan_fraction] = np.nan
    return rec, key, flags, loc


def _run_frames(backends, world, locations, md, host_backend, monkeypatch, what):
    """Upload the world, then per frame batch the viewport and a shadow camera (it sorts by the viewport's distance too,
    batching.rs:156-157) on every backend and compare both cameras' tables."""
    rec, key, flags, loc = world
    n = len(rec)
    cameras = (CAMERA_VIEWPORT, 0)
    headers = {cam: per_camera_header(cloud_camera(), cam, (1920, 1080) if cam == CAMERA_VIEWPORT else (1024, 1024), 1, n) for cam in cameras}

    def upload(b):
        b.set_objects(rec)
        b.set_object_sort_info(key, flags, loc)
        for cam in cameras:
            b.object_uniform_upload(cam, headers[cam], CB_CULL)
    for b in backends:
        upload(b)
    _upload_host(monkeypatch, lambda: upload(host_backend))
    dev, orc = backends
    for f, vp in enumerate(locations):
        for b in (dev, orc, host_backend):
            for cam in cameras:
                b.batch_objects(cam, np.asarray(vp, dtype=np.float32), md)
        for cam in cameras:
            w = f"{what}, frame {f}, camera {cam:#x}"
            info = _check_device_info(dev, w, cam)
            bd, rd = dev.readback_batches(cam)
            bo, ro = orc.readback_batches(cam)
            bh, rh = host_backend.readback_batches(cam)
            assert_same_tables(bd, rd, bo, ro, w + " (device vs oracle)")
            assert_same_tables(bh, rh, bo, ro, w + " (host vs oracle)")
            assert info["batches"] == len(bo) and info["regions"] == len(ro)
    return orc.visible_count(CAMERA_VIEWPORT), len(bo)


@pytest.mark.parametrize("frame_sort", ["0", "1"])
@pytest.mark.parametrize("n,limits", [(5000, LIMITS), (100_000, [3, 256, 65535]), (600_000, [256, 65535])])
def test_random_worlds_in_every_sort_tier(monkeypatch, frame_sort, n, limits):
    """<= 8192 (one-CTA sort), <= 524288 (cooperative sort) and > 524288 (multi-launch sort) visible objects; three frames each with the
    viewport moving, so the sort order and the split points move and the previous-invocation maps are carried over."""
    monkeypatch.setenv("R3_FRAME_SORT", frame_sort)
    world = random_world(n, seed=n % 97 + 3)
    locations = [(0.0, 0.0, 0.0), (40.0, -10.0, 5.0), (-60.0, 25.0, 80.0)]
    for md in limits:
        dev, orc = _device(monkeypatch), load_oracle_backend()
        host = load_cuda_backend(0)
        nv, _ = _run_frames((dev, orc), world, locations, md, host, monkeypatch, f"n={n} max_dispatch_count={md} frame sort {frame_sort}")
        assert nv == n
        dev.close(), host.close()


def test_world_that_reaches_the_batch_bound(monkeypatch):
    """Every object alone in its batch behind the leading empty one: nv + 1 batches, the bound the tables are sized with."""
    n = 3000
    rec = object_cloud_records(n, seed=8, extent=50.0, disabled_fraction=0.0)
    rec["sphere_radius"][:] = 1.0e6
    rec["index_count"] = 3 * 256
    world = (rec, np.zeros(n, dtype=np.uint64), np.full(n, 3, dtype=np.uint8), rec["sphere_center"].copy())
    for md in (0, 1):
        dev, orc = _device(monkeypatch), load_oracle_backend()
        host = load_cuda_backend(0)
        _, nb = _run_frames((dev, orc), world, [(0.0, 0.0, 0.0)], md, host, monkeypatch, f"bound, max_dispatch_count={md}")
        assert nb == n + 1
        dev.close(), host.close()


def test_launches_without_a_big_mesh_are_unchanged(monkeypatch):
    """A world no batch of which can reach the limit records the sort and the three build launches, as before the partition existed; one
    that can adds the partition's launches, a number fixed by the capacity alone."""
    monkeypatch.setenv("R3_FRAME_SORT", "0")
    n = 2000
    rec, key, flags, loc = random_world(n, seed=5, big_fraction=0.0)
    header = per_camera_header(cloud_camera(), CAMERA_VIEWPORT, (1920, 1080), 1, n)
    b = _device(monkeypatch)
    b.set_objects(rec)
    b.set_object_sort_info(key, flags, loc)
    b.object_uniform_upload(CAMERA_VIEWPORT, header, CB_CULL)
    b.batch_objects(CAMERA_VIEWPORT, np.zeros(3, dtype=np.float32))   # the first call also sums the padded triangle counts once
    counts = {}
    for md in (65535, 1, 1, 65535):
        l0 = b.launch_count()
        b.batch_objects(CAMERA_VIEWPORT, np.zeros(3, dtype=np.float32), md)
        counts.setdefault(md, set()).add(b.launch_count() - l0)
        _check_device_info(b, f"max_dispatch_count {md}")
    assert counts[65535] == {1 + 3}, counts                  # one-CTA sort + build, scan, finalize
    bound = min(n + 1, (n + 255) // 256 + 2 * (int(((rec["index_count"] // 3 + 255) // 256 * 256).sum()) // 256) + 3)
    steps = (bound - 1).bit_length()                        # ceil(log2(bound))
    assert counts[1] == {1 + 3 + 5 + steps}, counts          # + tile scan, tile offsets, next, K doubling steps, count, scatter
    b.close()


def test_config1_frame_launches_are_unchanged(monkeypatch):
    """BASELINE config 1 (10k cubes of 12 and 48 triangles, one shadowed directional light) at the default limit takes no partition:
    a steady-state frame issues 40 kernel launches, as it did before batches could split on the device."""
    monkeypatch.delenv("R3_FRAME_SORT", raising=False)
    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    ev, res = config1()
    b = load_cuda_backend(0, parity_target=False)         # as bench.py runs it: no f32 parity copy of the shading result
    g = BaseRenderGraph(b)
    g.add_to_graph(ev, res, 1, BaseRenderGraphSettings())
    per_frame = []
    for _ in range(2):
        l0 = b.launch_count()
        g.add_to_graph(ev, res, 1, BaseRenderGraphSettings(), upload=False)
        per_frame.append(b.launch_count() - l0)
    _check_device_info(b, "config 1")
    assert per_frame == [40, 40], per_frame
    b.close()


def test_worlds_past_2_31_invocations_keep_their_paths(monkeypatch):
    """A padded total of 2^31 or more invocations: with a mesh that lets a batch reach the dispatch limit the world batches on the host,
    as it always did; without one the device path refuses it, as before."""
    n = 28_000                                               # 28,000 x 76,800 = 2.15 G invocations
    rec = object_cloud_records(n, seed=9, extent=50.0, disabled_fraction=0.0)
    rec["sphere_radius"][:] = 1.0e6
    rec["index_count"] = 3 * 76_800
    header = per_camera_header(cloud_camera(), CAMERA_VIEWPORT, (1920, 1080), 1, n)
    b = _device(monkeypatch)
    b.set_objects(rec)
    b.set_object_sort_info(np.zeros(n, dtype=np.uint64), np.full(n, 3, dtype=np.uint8), rec["sphere_center"].copy())
    b.object_uniform_upload(CAMERA_VIEWPORT, header, CB_CULL)
    b.batch_objects(CAMERA_VIEWPORT, np.zeros(3, dtype=np.float32))               # 256 x 76,800 >= 65535 x 256
    assert b.batching_info(CAMERA_VIEWPORT)["path"] == "host"
    assert b.batch_counts(CAMERA_VIEWPORT)[0] == (n + 217) // 218                 # 218 such meshes per batch
    with pytest.raises(R3Error, match="2\\^31"):
        b.batch_objects(CAMERA_VIEWPORT, np.zeros(3, dtype=np.float32), 100_000)  # 256 x 76,800 < 100000 x 256: no batch reaches it
    b.close()


# ------------------------------------------------------------------ whole frames
RES = (192, 112)


def big_mesh_field(mixed):
    return cube_field_scene(n_objects=90, seed=21, resolution=RES, n_dir_lights=1, shadow_resolution=256, shadow_distance=60.0, pull_back=6.0,
                            extent=10.0, subdivisions=(1, 2, 80), material_count=6 if mixed else 1, mixed_transparency=mixed)


@pytest.mark.parametrize("samples,mixed,limit", [(1, False, 65535), (4, False, 65535), (1, True, 65535), (4, True, 300), (1, False, 1000)])
def test_frames_with_big_meshes_match_oracle(monkeypatch, samples, mixed, limit):
    """A cube field with 76,800-triangle cubes: batched on the device at the default limit (it went to the host before) and at small limits
    set through the routines, frames equal to the oracle's, viewport and shadow camera."""
    ev = big_mesh_field(mixed)
    cuda, orc = _device(monkeypatch), load_oracle_backend()
    for b in (cuda, orc):
        BaseRenderGraph(b, max_compute_workgroups_per_dimension=limit).add_to_graph(ev, RES, samples, BaseRenderGraphSettings(clear_color=(0.1, 0.1, 0.2, 1.0)))
    _check_device_info(cuda, f"samples {samples}")
    compare_frame_state(cuda, orc, ev, [CAMERA_VIEWPORT, 0], what=f"big meshes, {samples} samples, mixed={mixed}, limit {limit}", f16_samples=samples > 1)
    bo, _ = orc.readback_batches(CAMERA_VIEWPORT)
    if limit < 65535:
        assert len(bo) > 2, "the small limit must split the batches"
    cuda.close()


@pytest.mark.parametrize("host", [False, True])
def test_big_mesh_world_keeps_the_frame_graph(monkeypatch, host):
    """Five frame-graph frames of the opaque big-mesh field: the device path flushes at most once (the first frame allocates); the host
    path flushes every frame.  The frames equal the oracle's either way."""
    monkeypatch.setenv("R3_FRAME_GRAPH", "1")
    if host:
        monkeypatch.setenv("R3_HOST_BATCHING", "1")
    else:
        monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    ev = big_mesh_field(False)
    b, orc = load_cuda_backend(0), load_oracle_backend()
    graphs = {id(x): BaseRenderGraph(x) for x in (b, orc)}
    for frame in range(5):
        for x in (b, orc):
            graphs[id(x)].add_to_graph(ev, RES, 1, BaseRenderGraphSettings(), upload=(frame == 0))
        if frame in (0, 4):
            compare_frame_state(b, orc, ev, [CAMERA_VIEWPORT, 0], what=f"graph frame {frame}, host={host}")
    assert b.batching_info(CAMERA_VIEWPORT)["path"].startswith("host" if host else "device")
    st = b.frame_graph_stats()
    assert st["frames"] == 5, st
    if host:
        assert st["flushed"] == 5, st
    else:
        assert st["flushed"] <= 1 and st["graphed"] >= 4, st
    b.close()
