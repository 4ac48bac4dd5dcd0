"""Objects that come and go — r3_set_objects_enabled, r3_set_objects_enabled_device — against the same presence states fed through
r3_update_objects + r3_update_object_sort_info (bit for bit) and the CPU oracle given the states as full uploads (within the parity
tolerance), plus the blend routine's bookkeeping, the frame graph, the dense form's bit words and the calls' validation."""
import ctypes

import numpy as np
import pytest

from harness import (assert_same_frame, assert_same_ldr, check_declared_and_exported, cull_and_batch, expect_error, hdr_close,
                     settings, to_device, unbound_backend)
from object_presence_case import pool_state, pool_world, state_eval, switch_script, update_path
from rend3_b200.backend import CAMERA_VIEWPORT, load_cuda_backend

E_INVALID, E_STATE = -1, -5
RES = (256, 160)


# ------------------------------------------------------------------ without a GPU
def test_library_exports_both_entry_points_with_the_headers_signatures():
    check_declared_and_exported(("int r3_set_objects_enabled(r3_ctx*, const uint32_t* slots_or_null, const uint8_t* enabled, uint32_t n);",
                                 "int r3_set_objects_enabled_device(r3_ctx*, const uint32_t* d_slots_or_null, const uint8_t* d_enabled, uint32_t n);"),
                                (None, None, None, 0))


@pytest.mark.parametrize("enabled,slots", [
    (np.ones((4, 2), np.uint8), None),                          # 2-d flags
    (np.ones(4, np.float32), None),                             # float flags
    (np.ones(4, np.int32), None),                               # 4-byte flags
    (np.ones(4, np.uint8), np.arange(3)),                       # lengths differ
    (np.ones(3, np.uint8), np.array([0.0, 1.0, 2.0])),          # float slots
    (np.ones(3, np.uint8), np.array([[0, 1, 2]])),              # 2-d slots
    (np.ones(2, np.uint8), np.array([-1, 3])),                  # negative slot
    (np.ones(1, np.uint8), np.array([1 << 32], np.int64)),      # beyond uint32
], ids=["2d-flags", "float-flags", "int32-flags", "length", "float-slots", "2d-slots", "negative", "wide"])
def test_host_wrapper_rejects_bad_shapes_and_dtypes_before_calling(enabled, slots):
    with pytest.raises(AssertionError, match="enabled|slots"):
        unbound_backend().set_objects_enabled(enabled, slots)


def test_device_wrapper_rejects_host_and_mistyped_tensors_before_calling():
    torch = pytest.importorskip("torch")
    b = unbound_backend()
    for enabled, slots in ((torch.ones(4, dtype=torch.uint8), None),                  # a host tensor
                           (np.ones(4, np.uint8), None)):                             # a numpy array
        with pytest.raises(AssertionError):
            b.set_objects_enabled_device(enabled, slots)
    with pytest.raises(AssertionError):
        b.set_objects_enabled_device(None, None)                                     # no length


def test_pool_state_equals_world_add_and_remove():
    """The expected-state builder against world.Renderer: a slot removed through remove_object draws nothing from the next evaluate on
    (enabled 0) and is no longer live one evaluate later; a present slot keeps its record bytes, key and location.  pool_state says
    'disabled and not live' at once — the documented departure, which changes no image."""
    from rend3_b200.scenes import subdivided_cube_mesh
    from rend3_b200.world import BLEND, LEFT, Object, PbrMaterial, Renderer

    r = Renderer(LEFT)
    mesh = r.add_mesh(subdivided_cube_mesh(1))
    mats = [r.add_material(PbrMaterial()), r.add_material(PbrMaterial(albedo_value=(1, 1, 1, 0.5), transparency=BLEND))]
    rng = np.random.default_rng(3)
    for i in range(40):
        t = np.eye(4, dtype=np.float32)
        t[3, :3] = rng.uniform(-5, 5, 3)
        r.add_object(Object(mesh, mats[i % 2], t))
    pool = r.evaluate()
    present = np.zeros(len(pool.object_buffer), dtype=bool)
    present[:40] = True
    gone = np.array([0, 5, 31, 32, 39])
    present[gone] = False
    for h in gone:
        r.remove_object(int(h))
    first, second = r.evaluate(), r.evaluate()
    rec, flags = pool_state(pool, present)
    assert np.array_equal(rec["enabled"] != 0, first.object_buffer["enabled"] != 0), "enabled words"
    assert np.array_equal(flags & 1, second.object_live), "live bits once the handles are reclaimed"
    assert np.array_equal(first.object_live[gone], np.ones(len(gone), np.uint8)), "world.py keeps a removed object live for one frame"
    keep = np.flatnonzero(present)
    for f in rec.dtype.names:
        assert rec[f][keep].tobytes() == first.object_buffer[f][keep].tobytes(), f
    assert np.array_equal(pool.object_material_key[keep], second.object_material_key[keep])
    assert pool.object_location[keep].tobytes() == second.object_location[keep].tobytes()
    assert np.array_equal(flags >> 1, pool_state(pool, np.ones_like(present))[1] >> 1), "flags bits 1-2 never change"


# ------------------------------------------------------------------ GPU
def device_entries(b, present, slots):
    """(slots as int32, enabled as uint8) CUDA tensors on the context's stream; slots None stays None (dense)."""
    flags = np.ascontiguousarray(present[slots] if slots is not None else present).astype(np.uint8)
    d_slots = None if slots is None else to_device(b, np.asarray(slots, dtype=np.uint32).view(np.int32))
    return d_slots, to_device(b, flags)


def same_fields(a, b):
    """Records equal field by field (the record ends in padding, which numpy's structured copies do not carry)."""
    return len(a) == len(b) and all(a[f].tobytes() == b[f].tobytes() for f in a.dtype.names)


@pytest.mark.gpu
@pytest.mark.parametrize("samples,host", [(1, False), (4, False), (1, True)], ids=["x1", "x4", "x1-host-batching"])
def test_gpu_switches_equal_the_update_path_and_the_oracle(monkeypatch, samples, host):
    """Nine frames of a pool with opaque, cutout and blend slots, a shadowed light and point lights: random subsets, all off, all on, the
    word edges, one visible slot off / on / off in successive frames.  The device form (sparse lists) and the host form (dense) equal a
    context fed the same states through r3_update_objects + r3_update_object_sort_info in every artefact, bit for bit; with device
    batching the oracle, given each state as a full upload, agrees within the parity tolerance."""
    from oracle import load_oracle_backend
    from rend3_b200.routines import BaseRenderGraph

    if host:
        monkeypatch.setenv("R3_HOST_BATCHING", "1")
    else:
        monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    w = pool_world(n_objects=2000)
    ev, n = w.ev, len(w.ev.object_buffer)
    ctx = {"update": load_cuda_backend(0, parity_target=True), "host": load_cuda_backend(0, parity_target=True), "device": load_cuda_backend(0, parity_target=True)}
    graphs = {k: BaseRenderGraph(x) for k, x in ctx.items()}
    orc = None if host else load_oracle_backend()
    go = None if host else BaseRenderGraph(orc)
    for k, g in graphs.items():
        g.add_to_graph(ev, RES, samples, settings())
    vis = ctx["device"].readback_visible(CAMERA_VIEWPORT)
    watch = int(vis[len(vis) // 2])
    keep = []
    for frame, (present, changed) in enumerate(switch_script(n, np.random.default_rng(samples), watch)):
        update_path(ctx["update"], ev, present, changed)
        graphs["update"].add_to_graph(ev, RES, samples, settings(), upload=False)
        graphs["host"].add_to_graph(ev, RES, samples, settings(), upload=False, object_presence=(None, present))
        entries = device_entries(ctx["device"], present, changed[::-1].copy())   # descending: order does not matter
        keep.append(entries)
        graphs["device"].add_to_graph(ev, RES, samples, settings(), upload=False, object_presence=entries)
        for name in ("host", "device"):
            assert_same_frame(ctx[name], ctx["update"], ev, f"frame {frame}, {name} form")
            assert_same_ldr(ctx[name], ctx["update"], f"frame {frame}, {name} form")
        rec, _ = ctx["device"].readback_objects(0, n, locations=False)
        want, _ = pool_state(ev, present)
        assert same_fields(rec, ctx["update"].readback_objects(0, n, locations=False)[0]), f"frame {frame}: records"
        assert np.array_equal(rec["enabled"], want["enabled"]), f"frame {frame}: enabled words"
        if orc is not None:
            go.add_to_graph(state_eval(ev, present), RES, samples, settings())
            for cam in [CAMERA_VIEWPORT] + list(range(len(ev.shadows))):
                assert np.array_equal(ctx["device"].readback_visible(cam), orc.readback_visible(cam)), f"frame {frame} camera {cam}: oracle"
            assert np.array_equal(ctx["device"].readback_depth().view(np.uint32), orc.readback_depth().view(np.uint32)), f"frame {frame}: oracle depth"
            hdr_close(ctx["device"].readback_hdr_f32(), orc.readback_hdr_f32(), f"frame {frame}: oracle hdr", samples != 1)
        if frame == 2:
            assert ctx["device"].visible_count(CAMERA_VIEWPORT) == 0, "all off"
    for x in ctx.values():
        x.close()
    if orc is not None:
        orc.close()


@pytest.mark.gpu
def test_gpu_despawned_object_leaves_the_predicted_pass_and_a_spawned_one_joins_the_residual_pass(monkeypatch):
    """Frame N-1 draws slot X; frame N despawns it with the device form while the predicted pass replays frame N-1's list, which holds X:
    X is not drawn (vs_main's disabled-object test).  Frame N+1 spawns it again: the predicted list (frame N's) lacks X and the residual
    pass draws it.  Depth is compared with the frames before, images with the update path, bit for bit."""
    from rend3_b200.routines import BaseRenderGraph

    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    w = pool_world(n_objects=600, blend=False)
    ev, n = w.ev, len(w.ev.object_buffer)
    dev, upd = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True)
    gd, gu = BaseRenderGraph(dev), BaseRenderGraph(upd)
    for g in (gd, gu):
        g.add_to_graph(ev, RES, 1, settings())
        g.add_to_graph(ev, RES, 1, settings(), upload=False)   # frame N-1: a predicted list exists
    depth_drawn = dev.readback_depth().copy()
    vis = dev.readback_visible(CAMERA_VIEWPORT)
    present = np.ones(n, dtype=bool)
    # the slot nearest the camera among the visible ones: it covers pixels no other object does
    x = int(vis[np.argmin(np.linalg.norm(ev.object_location[vis] - ev.camera.location(), axis=1))])
    keep = []
    for frame, on in (("N", False), ("N+1", True)):
        present[x] = on
        keep.append(device_entries(dev, present, np.array([x])))
        gd.add_to_graph(ev, RES, 1, settings(), upload=False, object_presence=keep[-1])
        update_path(upd, ev, present, [x])
        gu.add_to_graph(ev, RES, 1, settings(), upload=False)
        assert_same_frame(dev, upd, ev, f"frame {frame}")
        if not on:
            assert x not in dev.readback_visible(CAMERA_VIEWPORT)
            assert dev.readback_depth().tobytes() != depth_drawn.tobytes(), "the despawned slot is still drawn"
        else:
            assert x in dev.readback_visible(CAMERA_VIEWPORT)
            assert dev.readback_depth().tobytes() == depth_drawn.tobytes(), "the spawned slot is not drawn"
    dev.close(), upd.close()


@pytest.mark.gpu
def test_gpu_switching_frames_stay_one_graph(monkeypatch):
    """Six recorded frames of a pool without key-2 slots: the device form switches different slots each frame, spawned slots are placed
    with r3_set_object_transforms_device in the same frame and another slot is posed by r3_pose_objects.  graphed == 6, flushed == 0,
    and every artefact equals the same frames run eagerly, bit for bit."""
    import object_animation_case as anim_cases
    from rend3_b200.animation import Animation, Node, NodeChannels, ObjectAnimationData
    from rend3_b200.routines import BaseRenderGraph
    from rend3_b200.scenes import cube_field_scene

    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    res = (256, 144)
    ev = cube_field_scene(n_objects=300, seed=7, resolution=res, n_dir_lights=2, shadow_resolution=256)
    assert not (ev.object_material_key == 2).any()
    n = len(ev.object_buffer)
    ms = ev.object_mesh_sphere
    rng = np.random.default_rng(5)
    live = np.flatnonzero(ev.object_live)
    posed = rng.choice(live, 4, replace=False)
    pool = np.setdiff1d(live, posed)
    nodes, channels = [], {}
    for i, s in enumerate(posed):
        t = ev.object_buffer["transform"][s].reshape(4, 4)[3, :3]
        nodes.append(Node(None, t, anim_cases._unit_quat(rng), (0.7, 0.7, 0.7), [(int(s), ms[s, :3].copy(), np.float32(ms[s, 3]))]))
        channels[i] = NodeChannels(anim_cases.key_track([0.0, 2.0], [t, t + rng.uniform(-1, 1, 3).astype(np.float32)]))
    data = ObjectAnimationData(nodes, [Animation(channels, 2.0)], left_handed=True)
    graph_b, eager_b = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True)
    graphs = {id(x): BaseRenderGraph(x) for x in (graph_b, eager_b)}
    for x in (graph_b, eager_b):
        graphs[id(x)].upload_world(ev, device_shadow_cameras=True, movable_objects=True)
        data.upload(x)
        x.set_object_pose_jobs(*data.pose_jobs([(0, 0.0, 0)]))
        graphs[id(x)].add_to_graph(ev, res, 1, settings(), upload=False, posed_objects=True, device_shadow_cameras=True, frame_graph=False)
    present = np.ones(n, dtype=bool)
    keep = []
    for frame in range(6):
        off = rng.choice(pool[present[pool]], 20, replace=False)
        on = rng.choice(pool[~present[pool]], min(10, int((~present[pool]).sum())), replace=False) if frame else np.zeros(0, np.int64)
        present[off], present[on] = False, True
        slots = np.concatenate([off, on]).astype(np.uint32)
        mats = np.tile(np.eye(4, dtype=np.float32).reshape(16), (len(on), 1))
        mats[:, 12:15] = rng.uniform(-8, 8, (len(on), 3))                  # spawned slots are placed in the same frame
        t = 0.3 * frame
        before = graph_b.frame_graph_stats()
        for x in (graph_b, eager_b):
            x.set_object_pose_jobs(*data.pose_jobs([(0, t, 0)]))
            d_slots, d_enabled = device_entries(x, present, slots)
            moved = (to_device(x, on.astype(np.uint32).view(np.int32)), to_device(x, mats)) if len(on) else None
            keep.append((d_slots, d_enabled, moved))
            graphs[id(x)].add_to_graph(ev, res, 1, settings(), upload=False, posed_objects=True, device_shadow_cameras=True,
                                       frame_graph=x is graph_b, object_presence=(d_slots, d_enabled), object_transforms=moved)
        after = graph_b.frame_graph_stats()
        assert after["flushed"] == before["flushed"], f"frame {frame} flushed early"
        assert_same_frame(graph_b, eager_b, ev, f"frame {frame}: graph vs eager")
        assert_same_ldr(graph_b, eager_b, f"frame {frame}")
        vis = graph_b.readback_visible(CAMERA_VIEWPORT)
        assert not np.isin(vis, np.flatnonzero(~present)).any(), f"frame {frame}: an absent slot is visible"
    stats = graph_b.frame_graph_stats()
    assert stats["graphed"] == 6 and stats["flushed"] == 0, stats
    graph_b.close(), eager_b.close()


@pytest.mark.gpu
def test_gpu_blend_routine_bookkeeping(monkeypatch):
    """Host form: despawning the only live key-2 object turns the blend routine off (a recorded frame stops flushing) and spawning it turns
    it on.  Device form: with key-2 slots, none present, the image equals the one the exact rule gives, bit for bit, though the routine
    runs (the recorded frame flushes).  After r3_set_object_sort_info the exact rule is back."""
    from rend3_b200.routines import BaseRenderGraph

    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    w = pool_world(n_objects=800, blend=True)
    ev, n = w.ev, len(w.ev.object_buffer)
    blend = np.flatnonzero(ev.object_material_key == 2)
    assert len(blend) >= 2
    present = np.ones(n, dtype=bool)
    present[blend[1:]] = False                                           # one key-2 object present
    exact, dev = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True)
    ge, gd = BaseRenderGraph(exact), BaseRenderGraph(dev)

    def frame(g, b, **kw):
        before = b.frame_graph_stats()["flushed"]
        g.add_to_graph(ev, RES, 1, settings(), upload=False, frame_graph=True, **kw)
        return b.frame_graph_stats()["flushed"] - before
    for g, b in ((ge, exact), (gd, dev)):
        g.upload_world(ev)
        b.set_objects_enabled(present)
        assert frame(g, b) > 0, "a present key-2 object: the blend routine runs and the frame flushes"
    present[blend[0]] = False
    exact.set_objects_enabled(np.zeros(1, np.uint8), np.array([blend[0]]))
    keep = device_entries(dev, present, np.array([blend[0]]))
    assert frame(ge, exact) == 0, "no key-2 object is live: the blend routine is off"
    assert frame(gd, dev, object_presence=keep) > 0, "after the device form any key-2 slot runs the routine"
    assert_same_frame(dev, exact, ev, "device form, no key-2 object present")
    assert_same_ldr(dev, exact, "device form, no key-2 object present")
    assert frame(ge, exact) == 0 and frame(gd, dev) > 0, "the conservative rule holds until r3_set_object_sort_info"
    assert_same_frame(dev, exact, ev, "device form, second frame")
    _, flags = pool_state(ev, present)
    dev.set_object_sort_info(ev.object_material_key, flags, ev.object_location)
    assert frame(gd, dev) == 0, "the exact rule is back"
    present[blend[0]] = True
    exact.set_objects_enabled(np.ones(1, np.uint8), np.array([blend[0]]))
    assert frame(ge, exact) > 0, "spawning a key-2 object turns the routine on"
    exact.close(), dev.close()


def cloud(n, seed=3):
    from rend3_b200.scenes import object_cloud_records

    rec = object_cloud_records(n, seed=seed, extent=60.0)
    rec["enabled"] = 1
    rng = np.random.default_rng(seed)
    key = rng.integers(0, 3, n).astype(np.uint64)
    flags = (1 | 2 * rng.integers(0, 2, n) | 4 * (key == 2)).astype(np.uint8)
    return rec, key, flags, rec["sphere_center"].copy()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1000, 1024, 33])
def test_gpu_dense_form_equals_sparse_form(monkeypatch, n):
    """The dense form (whole bit words, ragged last word and a partial range by atomics) equals the sparse form over the same slots, and
    both equal the update path: records, visible list, MV / MVP, batches and regions."""
    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    rec, key, flags, loc = cloud(n)
    rng = np.random.default_rng(n)
    ctx = {"dense": load_cuda_backend(0, parity_target=False), "sparse": load_cuda_backend(0, parity_target=False), "update": load_cuda_backend(0, parity_target=False)}
    for x in ctx.values():
        x.set_objects(rec)
        x.set_object_sort_info(key, flags, loc)
    present = np.ones(n, dtype=bool)
    keep = []
    for step, k in enumerate((n, n, n - 7, min(45, n), 1)):                     # whole range twice, then prefixes that end inside a word
        new = present.copy()
        new[:k] = rng.random(k) < 0.5
        changed = np.flatnonzero(new != present)
        present = new
        d = device_entries(ctx["dense"], present[:k], None)
        keep.append(d)
        ctx["dense"].set_objects_enabled_device(d[1])
        perm = rng.permutation(k).astype(np.uint32)
        s = device_entries(ctx["sparse"], present, perm)
        keep.append(s)
        ctx["sparse"].set_objects_enabled_device(s[1], s[0])
        ev_like = type("E", (), {})()
        ev_like.object_buffer, ev_like.object_material_key, ev_like.object_location = rec, key, loc
        ev_like.object_live, ev_like.object_atomic, ev_like.object_back_to_front = flags & 1, (flags >> 1) & 1, (flags >> 2) & 1
        update_path(ctx["update"], ev_like, present, changed)
        out = {name: cull_and_batch(x, n) for name, x in ctx.items()}
        recs = {name: x.readback_objects(0, n, locations=False)[0] for name, x in ctx.items()}
        assert out["dense"] == out["sparse"] == out["update"], f"step {step}: cull / batch differ"
        assert same_fields(recs["dense"], recs["update"]) and same_fields(recs["sparse"], recs["update"]), f"step {step}: records differ"
    for x in ctx.values():
        x.close()


@pytest.mark.gpu
def test_gpu_without_sort_info_the_enabled_bits_decide(monkeypatch):
    """No r3_set_object_sort_info: both forms switch the enabled bits alone, which decide the visible list as after r3_update_objects."""
    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    n = 1000
    rec, _, _, _ = cloud(n, seed=9)
    ctx = {"host": load_cuda_backend(0, parity_target=False), "device": load_cuda_backend(0, parity_target=False), "update": load_cuda_backend(0, parity_target=False)}
    for x in ctx.values():
        x.set_objects(rec)
    rng = np.random.default_rng(1)
    present = rng.random(n) < 0.6
    slots = np.flatnonzero(~present).astype(np.uint32)
    ctx["host"].set_objects_enabled(present)
    keep = device_entries(ctx["device"], present, slots)
    ctx["device"].set_objects_enabled_device(keep[1], keep[0])
    want = rec.copy()
    want["enabled"] = present
    ctx["update"].update_objects(slots, want[slots])
    out = {name: cull_and_batch(x, n, batch=False) for name, x in ctx.items()}
    assert out["host"] == out["update"] and out["device"] == out["update"]
    vis = np.frombuffer(out["device"][0], dtype=np.uint32)
    assert len(vis) > 0 and present[vis].all()
    for x in ctx.values():
        x.close()


@pytest.mark.gpu
def test_gpu_validation_and_dropped_slots(monkeypatch):
    """The host form rejects an out-of-range slot, a slot named twice, a null pointer and too many dense flags with R3_E_INVALID and
    leaves the context unchanged (records, next frame); both forms return R3_E_STATE before r3_set_objects and with borrowed records;
    the device form drops out-of-range slots and writes the rest."""
    import torch

    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    n = 500
    rec, key, flags, loc = cloud(n, seed=4)
    b = load_cuda_backend(0, parity_target=False)
    one = np.ones(1, np.uint8)
    b.set_objects_enabled(np.zeros(0, np.uint8))                                    # n == 0: R3_OK before any state exists
    expect_error(E_STATE, b.set_objects_enabled, one, np.array([0]))
    d_one = to_device(b, one)
    expect_error(E_STATE, b.set_objects_enabled_device, d_one, None)
    ref = load_cuda_backend(0, parity_target=False)                                                               # the same frames without the rejected calls
    for x in (b, ref):
        x.set_objects(rec)
        x.set_object_sort_info(key, flags, loc)
        cull_and_batch(x, n)
    before_rec = b.readback_objects(0, n, locations=False)[0]
    expect_error(E_INVALID, b.set_objects_enabled, np.zeros(2, np.uint8), np.array([3, n]))         # slot 3 is not written either
    expect_error(E_INVALID, b.set_objects_enabled, np.zeros(3, np.uint8), np.array([4, 9, 4]))      # one slot named twice
    expect_error(E_INVALID, b.set_objects_enabled, np.zeros(n + 1, np.uint8))                       # dense: more flags than slots
    s = np.array([1, 2], np.uint32)
    rc = b.lib.r3_set_objects_enabled(b.ctx, s.ctypes.data_as(ctypes.c_void_p), None, ctypes.c_uint32(2))
    assert rc == E_INVALID, "null flags"
    assert same_fields(b.readback_objects(0, n, locations=False)[0], before_rec), "a rejected call wrote something"
    assert cull_and_batch(b, n) == cull_and_batch(ref, n), "a rejected call changed the next frame"
    ref.close()
    # the device form drops out-of-range slots
    slots = np.array([5, n, 77, 0xFFFFFFFF, n + 31, 499], dtype=np.uint32)
    d_slots = to_device(b, slots.view(np.int32))
    d_off = to_device(b, np.zeros(len(slots), np.uint8))
    b.set_objects_enabled_device(d_off, d_slots)
    got = b.readback_objects(0, n, locations=False)[0]
    assert np.array_equal(np.flatnonzero(got["enabled"] == 0), [5, 77, 499])
    cull_and_batch(b, n)
    assert not np.isin(b.readback_visible(CAMERA_VIEWPORT), [5, 77, 499]).any()
    # borrowed records
    dev = torch.from_numpy(rec.view(np.uint8).copy()).cuda()
    torch.cuda.synchronize()
    b.set_objects_device(dev.data_ptr(), n)
    expect_error(E_STATE, b.set_objects_enabled, one, np.array([0]))
    expect_error(E_STATE, b.set_objects_enabled_device, d_one, None)
    b.sync()
    assert dev.cpu().numpy().tobytes() == rec.view(np.uint8).tobytes()
    b.close()
    del d_slots, d_off, d_one
