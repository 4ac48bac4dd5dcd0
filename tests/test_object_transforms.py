"""Objects moved in bulk — r3_set_object_mesh_spheres, r3_set_object_transforms, r3_set_object_transforms_device — against the numpy
float32 restatement of rule R12's object half (tests/object_transform_case.py), the CPU oracle and, on the GPU, a context fed the same
bytes through r3_update_objects + r3_update_object_sort_info."""
import numpy as np
import pytest

import object_transform_case as cases
from harness import assert_same_frame, check_declared_and_exported, cull_and_batch_defined, expect_error, on_stream, to_device
from object_anim_reference import set_object_transform
from object_transform_case import apply, move_objects, moved_records, same_bits, same_records
from rend3_b200.backend import CAMERA_VIEWPORT, load_cuda_backend

from oracle.objtransforms import load_objtransforms_oracle_backend

f32 = np.float32
E_INVALID, E_STATE = -1, -5


def setup_world(b, rec, key, flags, loc, ms):
    b.set_objects(rec)
    b.set_object_sort_info(key, flags, loc)
    b.set_object_mesh_spheres(ms)


# ------------------------------------------------------------------ without a GPU
def test_restatement_equals_the_scalar_rule_and_the_oracle_bit_for_bit():
    """Seeded matrices and the rule's edges (row 3 of (+0, +0, -0, 1) and arbitrary, negative and zero scale, an inf axis giving a NaN
    location, NaN entries that f32::max ignores, zero-radius and zero mesh spheres): array restatement == scalar restatement == oracle,
    dense and sparse."""
    em, es, names = cases.edge_matrices()
    mats = np.concatenate([em, cases.seeded_matrices(500)])
    rec, key, flags, loc, ms = cases.world(len(mats) + 40)
    ms[:len(em)] = es
    sph, l = move_objects(mats, ms[:len(mats)])
    with np.errstate(all="ignore"):
        for i in range(len(em) + 20):
            _, c, r, p = set_object_transform(mats[i].reshape(4, 4), ms[i, :3], ms[i, 3])
            assert same_bits(sph[i], np.append(c, r)) and same_bits(l[i], p), names[i] if i < len(names) else i
    k = names.index("inf in an axis: NaN location")
    assert np.isnan(l[k]).any() and not np.isnan(mats[k, 12:15]).any()
    k = names.index("NaN in one axis: f32::max ignores it")
    assert sph[k, 3] == f32(3.0) * ms[k, 3]
    orc = load_objtransforms_oracle_backend()
    setup_world(orc, rec, key, flags, loc, ms)
    orc.set_object_transforms(mats)
    want_r, want_l = moved_records(rec, loc, ms, mats)
    got_r, got_l = orc.readback_objects(0, len(rec))
    assert same_records(got_r, want_r) and same_bits(got_l, want_l)
    # sparse, in descending order, over the slots the dense call left alone and some it wrote
    slots = np.arange(len(rec) - 1, len(rec) - 101, -1).astype(np.uint32)
    orc.set_object_transforms(mats[:100], slots)
    want_r, want_l = moved_records(want_r, want_l, ms, mats[:100], slots)
    got_r, got_l = orc.readback_objects(0, len(rec))
    assert same_records(got_r, want_r) and same_bits(got_l, want_l)
    orc.close()


def test_restatement_equals_world_set_object_transform():
    """world.Renderer.set_object_transform + evaluate() writes the same records and locations, and evaluate() reports the mesh spheres."""
    from rend3_b200.world import LEFT, Object, PbrMaterial, Renderer
    from rend3_b200.scenes import subdivided_cube_mesh

    r = Renderer(LEFT)
    meshes = [r.add_mesh(subdivided_cube_mesh(k)) for k in (1, 2)]
    mat = r.add_material(PbrMaterial())
    start = cases.seeded_matrices(40, seed=1)
    for i in range(40):
        r.add_object(Object(meshes[i % 2], mat, start[i].reshape(4, 4)))
    ev = r.evaluate()
    ms = ev.object_mesh_sphere
    assert ms.shape == (len(ev.object_buffer), 4) and np.all(ms[:40, 3] > 0) and not ms[40:].any()
    moved = cases.seeded_matrices(40, seed=2)
    slots = np.arange(0, 40, 3)
    for s in slots:
        r.set_object_transform(int(s), moved[s].reshape(4, 4))
    ev2 = r.evaluate()
    want_r, want_l = moved_records(ev.object_buffer, ev.object_location, ms, moved[slots], slots)
    assert same_records(ev2.object_buffer, want_r) and same_bits(ev2.object_location, want_l)


def check_rejections(b):
    """Call-order and argument errors of a context; every rejected call leaves records, locations and spheres as they were."""
    rec, key, flags, loc, ms = cases.world(200)
    mats = cases.seeded_matrices(200)
    b.set_object_transforms(np.zeros((0, 16), f32))                                   # n == 0: R3_OK before any state exists
    expect_error(E_STATE, b.set_object_transforms, mats[:1])                          # before r3_set_objects
    b.set_objects(rec)
    b.set_object_sort_info(key, flags, loc)
    expect_error(E_STATE, b.set_object_transforms, mats[:1])                          # before the mesh spheres
    b.set_object_mesh_spheres(ms[:150])
    expect_error(E_STATE, b.set_object_transforms, mats[:1])                          # spheres do not cover every slot
    expect_error(E_INVALID, b.set_object_mesh_spheres, ms[:2], np.array([3, 150], np.uint32))   # beyond the sphere count
    expect_error(E_INVALID, b.set_object_mesh_spheres, ms[:2], np.array([3, 3], np.uint32))
    b.set_object_mesh_spheres(ms)
    b.set_object_mesh_spheres(ms[10:12] * f32(2), np.array([7, 5], np.uint32))        # sparse spheres
    ms = ms.copy()
    ms[7], ms[5] = ms[10] * f32(2), ms[11] * f32(2)
    expect_error(E_INVALID, b.set_object_transforms, mats[:2], np.array([3, 200], np.uint32))   # slot 3 is not written either
    expect_error(E_INVALID, b.set_object_transforms, mats[:3], np.array([4, 9, 4], np.uint32))  # one slot named twice
    expect_error(E_INVALID, b.set_object_transforms, np.zeros((201, 16), f32))                  # dense: more matrices than slots
    got_r, got_l = b.readback_objects(0, 200)
    assert same_records(got_r, rec) and same_bits(got_l, loc), "a rejected call wrote something"
    b.set_object_transforms(mats[:12], np.arange(12, dtype=np.uint32))
    want_r, want_l = moved_records(rec, loc, ms, mats[:12])
    got_r, got_l = b.readback_objects(0, 200)
    assert same_records(got_r, want_r) and same_bits(got_l, want_l), "the sparse spheres are used"
    # r3_set_objects keeps the spheres; a larger world than they cover is R3_E_STATE until they are set again
    larger = np.zeros(208, dtype=rec.dtype)
    larger[:200] = rec
    b.set_objects(larger)
    expect_error(E_STATE, b.set_object_transforms, mats[:1])
    b.set_objects(rec)
    b.set_object_transforms(mats[:1])


def test_oracle_rejections_and_state_rules():
    orc = load_objtransforms_oracle_backend()
    check_rejections(orc)
    orc.close()


def test_library_exports_the_three_entry_points_with_the_headers_signatures():
    check_declared_and_exported(("int r3_set_object_mesh_spheres(r3_ctx*, const uint32_t* slots_or_null, const float* center_radius , uint32_t n);",
                                 "int r3_set_object_transforms(r3_ctx*, const uint32_t* slots_or_null, const float* mat4s , uint32_t n);",
                                 "int r3_set_object_transforms_device(r3_ctx*, const uint32_t* d_slots_or_null, const float* d_mat4s, uint32_t n);"),
                                (None, None, None, 0))


# ------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("form", ["host", "device"])
def test_gpu_records_equal_the_oracle(form):
    """Records and locations after dense and sparse moves of 1 .. 300 000 objects == the oracle's; sparse lists that put 32 updates in one
    bit word, lists in descending order, shuffled lists; untouched slots and every cold field keep their bytes."""
    n = 300_000
    rec, key, flags, loc, ms = cases.world(n)
    em, es, _ = cases.edge_matrices()
    mats = cases.seeded_matrices(n)
    mats[:len(em)] = em
    ms[:len(em)] = es
    rng = np.random.default_rng(17)
    b, orc = load_cuda_backend(0, parity_target=False), load_objtransforms_oracle_backend()
    for x in (b, orc):
        setup_world(x, rec, key, flags, loc, ms)
    steps = [(k, None) for k in (1, 31, 32, 33, 1000, n)]
    steps += [(32, np.arange(64, 96)), (32, np.arange(127, 95, -1)), (5000, np.sort(rng.choice(n, 5000, replace=False))[::-1]),
              (100_000, rng.permutation(n)[:100_000]), (1, np.array([n - 1]))]
    keep = []
    for i, (k, slots) in enumerate(steps):
        m = np.roll(mats, 7 * i, axis=0)[:k]
        s = None if slots is None else np.ascontiguousarray(slots, dtype=np.uint32)
        keep.append(apply(b, form, m, s))
        orc.set_object_transforms(m, s)
        got_r, got_l = b.readback_objects(0, n)
        want_r, want_l = orc.readback_objects(0, n)
        assert same_records(got_r, want_r) and same_bits(got_l, want_l), f"step {i}: {k} objects, slots {'dense' if s is None else 'sparse'}"
        if i == 0:
            assert same_records(got_r[1:], rec[1:]) and got_l[1:].tobytes() == loc[1:].tobytes(), "untouched slots changed"
    for f in rec.dtype.names:
        if f not in ("transform", "sphere_center", "sphere_radius"):
            assert got_r[f].tobytes() == rec[f].tobytes(), f"cold field {f} changed"
    b.close(), orc.close()


@pytest.mark.gpu
def test_gpu_cull_bake_after_moves_equals_oracle_and_the_update_path(monkeypatch):
    """Visible list and every MV / MVP word after a move == the oracle's == a context fed the same bytes through r3_update_objects +
    r3_update_object_sort_info, for both forms; a slot goes affine -> non-affine -> affine, and a disabled slot moves and stays disabled."""
    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    n = 4000
    rec, key, flags, loc, ms = cases.world(n, seed=11)
    disabled = int(np.flatnonzero(rec["enabled"] == 0)[0])
    rng = np.random.default_rng(23)
    ctx = {"host": load_cuda_backend(0, parity_target=False), "device": load_cuda_backend(0, parity_target=False),
           "update": load_cuda_backend(0, parity_target=False), "oracle": load_objtransforms_oracle_backend()}
    for x in ctx.values():
        setup_world(x, rec, key, flags, loc, ms)
    cur_r, cur_l = rec, loc
    keep = []
    for step in range(3):
        slots = np.unique(np.concatenate([rng.choice(n, 400, replace=False), [disabled, 64, 65]])).astype(np.uint32)
        mats = cases.seeded_matrices(len(slots), seed=30 + step, extent=40.0)
        if step == 1:                                                 # row 3 leaves (+0, +0, +0, 1) for slots 64 (-0) and 65 (arbitrary)
            mats[np.searchsorted(slots, 64), 11] = f32(-0.0)
            mats[np.searchsorted(slots, 65), 3::4] = (0.01, 0.02, -0.01, 1.1)
        cur_r, cur_l = moved_records(cur_r, cur_l, ms, mats, slots)
        out = {}
        for name, x in ctx.items():
            if name == "update":
                x.update_objects(slots, cur_r[slots])
                x.update_object_sort_info(slots, key[slots], flags[slots], cur_l[slots])
            else:
                keep.append(apply(x, "device" if name == "device" else "host", mats, slots))
            out[name] = cull_and_batch_defined(x, n)
        for name in ("host", "device"):
            assert out[name][:2] == out["oracle"][:2], f"step {step}, {name} form: visible list / MV / MVP differ from the oracle"
            assert out[name] == out["update"], f"step {step}, {name} form: differs from the update path"
        vis = np.frombuffer(out["device"][0], dtype=np.uint32)
        assert len(vis) > 0
    got_r, _ = ctx["device"].readback_objects(0, n)
    assert got_r["enabled"][disabled] == 0 and not np.array_equal(got_r["transform"][disabled], rec["transform"][disabled])
    mv = ctx["device"].readback_object_matrices(CAMERA_VIEWPORT, disabled, 1)
    assert mv.tobytes() == ctx["update"].readback_object_matrices(CAMERA_VIEWPORT, disabled, 1).tobytes(), "a disabled slot is not baked on either path"
    for x in ctx.values():
        x.close()


@pytest.mark.gpu
@pytest.mark.parametrize("host", [False, True], ids=["device_batching", "host_batching"])
def test_gpu_batching_sorts_by_moved_locations(monkeypatch, host):
    """Batch and region tables == the oracle's on both batching paths while two back-to-front blend objects swap places by being moved
    with the device form; the host path takes the moved locations from the device in the drain it makes for the visible list."""
    if host:
        monkeypatch.setenv("R3_HOST_BATCHING", "1")
    else:
        monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    n = 4000
    rec, key, flags, loc, ms = cases.world(n, seed=12)
    pair = np.array([100, 2000], dtype=np.uint32)
    rec["enabled"][pair] = 1
    key[pair], flags[pair] = 2, 1 | 4
    b, orc = load_cuda_backend(0, parity_target=False), load_objtransforms_oracle_backend()
    for x in (b, orc):
        setup_world(x, rec, key, flags, loc, ms)
    vp = (0.0, 0.0, -30.0)
    orders, keep = [], []
    for z in ((0.0, 10.0), (20.0, 5.0)):
        mats = np.tile(np.eye(4, dtype=f32).reshape(16), (2, 1))
        mats[:, 14] = z
        keep.append(apply(b, "device", mats, pair))
        orc.set_object_transforms(mats, pair)
        got, want = cull_and_batch_defined(b, n, vp), cull_and_batch_defined(orc, n, vp)
        assert got == want, f"z={z}: batches differ from the oracle"
        assert b.batching_info(CAMERA_VIEWPORT)["path"] == ("host" if host else "device")
        bt, _ = b.readback_batches(CAMERA_VIEWPORT)
        ids = [int(i) for bb in bt for i in bb["object_culling_information"]["object_id"][:int(bb["total_objects"])]]
        orders.append([s for s in ids if s in (100, 2000)])
    assert len(orders[0]) == 2 and orders[0] == orders[1][::-1], f"the blend pair must swap places: {orders}"
    b.close(), orc.close()


@pytest.mark.gpu
def test_gpu_rejections_dropped_slots_and_growth():
    """The host form's rejections and the R3_E_STATE rules as on the oracle; a borrowed object buffer refuses both forms; the device form
    drops out-of-range slots and changes nothing else; after r3_resize_objects a new slot (zero mesh sphere until set) can be moved."""
    import torch

    b = load_cuda_backend(0, parity_target=False)
    check_rejections(b)
    b.close()
    n = 1000
    rec, key, flags, loc, ms = cases.world(n)
    mats = cases.seeded_matrices(64)
    b = load_cuda_backend(0, parity_target=False)
    setup_world(b, rec, key, flags, loc, ms)
    slots = np.array([5, n, 77, 0xFFFFFFFF, n + 31, 999], dtype=np.uint32)
    keep = apply(b, "device", mats[:6], slots)
    want_r, want_l = moved_records(rec, loc, ms, mats[:6], slots.astype(np.int64))
    got_r, got_l = b.readback_objects(0, n)
    assert same_records(got_r, want_r) and same_bits(got_l, want_l)
    assert np.array_equal(np.flatnonzero((got_r["transform"] != rec["transform"]).any(axis=1)), [5, 77, 999])
    # growth: the spheres grow with zeros, a sparse sphere write and a move of the new slots equal the rule
    b.resize_objects(n + 40)
    new = np.arange(n, n + 40, dtype=np.uint32)
    b.set_object_mesh_spheres(ms[:20], new[:20])
    keep = apply(b, "device", mats[:40], new)
    grown_r, grown_l = np.zeros(n + 40, rec.dtype), np.zeros((n + 40, 3), f32)
    grown_r[:n], grown_l[:n] = want_r, want_l
    grown_ms = np.zeros((n + 40, 4), f32)
    grown_ms[:n], grown_ms[n:n + 20] = ms, ms[:20]
    want_r, want_l = moved_records(grown_r, grown_l, grown_ms, mats[:40], new)
    got_r, got_l = b.readback_objects(0, n + 40)
    assert same_records(got_r, want_r) and same_bits(got_l, want_l)
    # borrowed records
    dev = torch.from_numpy(rec.view(np.uint8).copy()).cuda()
    torch.cuda.synchronize()
    b.set_objects_device(dev.data_ptr(), n)
    expect_error(E_STATE, b.set_object_transforms, mats[:1])
    expect_error(E_STATE, b.set_object_transforms_device, keep[0], None, 1)
    expect_error(E_INVALID, b.set_object_transforms_device, keep[0].data_ptr() + 4, None, 1)   # misaligned matrices
    b.sync()
    assert dev.cpu().numpy().tobytes() == rec.view(np.uint8).tobytes()
    b.close()
    del keep


@pytest.mark.gpu
def test_gpu_moved_frames_stay_one_graph():
    """Seven frames of a left-handed cube field through add_to_graph with the frame graph on: 60 objects moved every frame by the device
    form from a tensor written on the context's stream, together with posed_objects on other slots and device_shadow_cameras.  No early
    flush; graph == eager == a context given the same bytes by r3_update_objects + r3_update_object_sort_info, bit for bit in every
    artefact (HDR included); records, locations, the viewport's visible list, MV / MVP and depth == the oracle's (which gets the host's
    light bytes, so the shadowed shading is held to the CUDA contexts only)."""
    import torch

    import object_animation_case as anim_cases
    from rend3_b200.animation import Animation, Node, NodeChannels, ObjectAnimationData
    from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings
    from rend3_b200.scenes import cube_field_scene

    res = (256, 144)
    ev = cube_field_scene(n_objects=300, seed=7, resolution=res, n_dir_lights=2, shadow_resolution=256)
    n = len(ev.object_buffer)
    ms = ev.object_mesh_sphere
    rng = np.random.default_rng(5)
    live = np.flatnonzero(ev.object_live)
    chosen = rng.choice(live, 100, replace=False)
    moved, posed = np.sort(chosen[:60]).astype(np.uint32), chosen[60:]
    nodes, channels = [], {}
    for i, s in enumerate(posed):
        t = ev.object_buffer["transform"][s].reshape(4, 4)[3, :3]
        nodes.append(Node(None, t, anim_cases._unit_quat(rng), (0.7, 0.7, 0.7), [(int(s), ms[s, :3].copy(), f32(ms[s, 3]))]))
        channels[i] = NodeChannels(anim_cases.key_track([0.0, 2.0], [t, t + rng.uniform(-1, 1, 3).astype(f32)]))
    data = ObjectAnimationData(nodes, [Animation(channels, 2.0)], left_handed=True)
    settings = BaseRenderGraphSettings(clear_color=(0.1, 0.05, 0.1, 1.0))
    graph_b, eager_b, update_b = (load_cuda_backend(0, parity_target=True) for _ in range(3))
    orc = load_objtransforms_oracle_backend()
    graphs = {id(x): BaseRenderGraph(x) for x in (graph_b, eager_b, update_b, orc)}
    for x in (graph_b, eager_b, update_b, orc):
        dsc = x is not orc
        graphs[id(x)].upload_world(ev, device_shadow_cameras=dsc, movable_objects=True)
        data.upload(x)
        x.set_object_pose_jobs(*data.pose_jobs([(0, 0.0, 0)]))
        graphs[id(x)].add_to_graph(ev, res, 1, settings, upload=False, posed_objects=True, device_shadow_cameras=dsc, frame_graph=False)
    base = ev.object_buffer["transform"][moved].copy()
    d_base = {id(x): to_device(x, base) for x in (graph_b, eager_b)}
    d_mats = {id(x): on_stream(x, lambda: torch.empty((len(moved), 16), dtype=torch.float32, device="cuda")) for x in (graph_b, eager_b)}
    d_slots = {id(x): to_device(x, moved.view(np.int32)) for x in (graph_b, eager_b)}
    cur_r, cur_l = ev.object_buffer, ev.object_location
    for frame, t in enumerate([0.0, 0.3, 0.7, 1.1, 1.6, 2.0, 2.5]):
        offset = np.zeros(16, f32)
        offset[12:15] = (0.4 * t, -0.3 * t, 0.2 * t)
        scale = f32(1.0 + 0.1 * t)
        mats = (base * scale + offset).astype(f32)                   # one f32 multiply and one f32 add per entry, as torch does below
        cur_r, cur_l = moved_records(cur_r, cur_l, ms, mats, moved)
        flushed = graph_b.frame_graph_stats()["flushed"]
        for x in (graph_b, eager_b, update_b, orc):
            x.set_object_pose_jobs(*data.pose_jobs([(0, t, 0)]))
            kw = dict(upload=False, posed_objects=True, device_shadow_cameras=x is not orc, frame_graph=x is graph_b)
            if x in (graph_b, eager_b):
                def produce(x=x):
                    torch.mul(d_base[id(x)], float(scale), out=d_mats[id(x)])
                    d_mats[id(x)].add_(torch.from_numpy(offset).to("cuda"))
                on_stream(x, produce)
                graphs[id(x)].add_to_graph(ev, res, 1, settings, object_transforms=(d_slots[id(x)], d_mats[id(x)]), **kw)
            elif x is update_b:
                x.update_objects(moved, cur_r[moved])
                x.update_object_sort_info(moved, ev.object_material_key[moved], (ev.object_live[moved] & 1) | ((ev.object_atomic[moved] & 1) << 1)
                                          | ((ev.object_back_to_front[moved] & 1) << 2), cur_l[moved])
                graphs[id(x)].add_to_graph(ev, res, 1, settings, **kw)
            else:
                graphs[id(x)].add_to_graph(ev, res, 1, settings, object_transforms=(moved, mats), **kw)
        assert graph_b.frame_graph_stats()["flushed"] == flushed, f"frame {frame} flushed early"
        assert_same_frame(graph_b, eager_b, ev, f"frame {frame}: graph vs eager")
        assert_same_frame(graph_b, update_b, ev, f"frame {frame}: device form vs the update path")
        (rg, lg), (ro, lo) = graph_b.readback_objects(0, n), orc.readback_objects(0, n)
        assert same_records(rg, ro) and same_bits(lg, lo), f"frame {frame}: records differ from the oracle"
        assert same_records(rg[moved], cur_r[moved]) and same_bits(lg[moved], cur_l[moved]), f"frame {frame}: records differ from the restatement"
        assert np.array_equal(graph_b.readback_visible(CAMERA_VIEWPORT), orc.readback_visible(CAMERA_VIEWPORT))
        assert graph_b.readback_object_matrices(CAMERA_VIEWPORT, 0, n).tobytes() == orc.readback_object_matrices(CAMERA_VIEWPORT, 0, n).tobytes()
        assert np.array_equal(graph_b.readback_depth().view(np.uint32), orc.readback_depth().view(np.uint32)), f"frame {frame}: depth differs"
    stats = graph_b.frame_graph_stats()
    assert stats["graphed"] == 7 and stats["flushed"] == 0, stats
    for x in (graph_b, eager_b, update_b, orc):
        x.close()
