"""Incremental world updates — r3_update_object_sort_info, r3_resize_objects, r3_update_mesh_buffer, r3_update_textures — against
full uploads.  A context fed the whole world every frame (A) is the reference for one fed only the changes (B): every artefact of every
frame must be bit-identical, and B agrees with the oracle as the parity tests require."""
import itertools

import numpy as np
import pytest

import cull_scenes as scenes
from harness import assert_same_frame, compare_frame_state, cull_and_batch, expect_error
from world_update_scene import ChangingWorld, merge, upload_delta
from rend3_b200.backend import CAMERA_VIEWPORT, CB_BAKE, CB_CULL, load_cuda_backend
from rend3_b200.layouts import PCU_MULTISAMPLED, TEXTURE_DESC_DTYPE
from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings, per_camera_header
from rend3_b200.scenes import cloud_camera, object_cloud_records

from oracle import load_oracle_backend

pytestmark = pytest.mark.gpu
RES = (256, 160)
SETTINGS = BaseRenderGraphSettings(clear_color=(0.1, 0.05, 0.1, 1.0), ambient_color=(0.02, 0.02, 0.02, 1.0))
E_INVALID, E_STATE = -1, -5


def script(w: ChangingWorld, blend: bool = True):
    """Frames 1-11 of changes; yields (frame, delta)."""
    yield 1, w.move(0.01)
    yield 2, w.move(0.10)
    killed = w.live_slots(0.03)
    yield 3, w.kill(killed)
    yield 4, w.revive(killed)
    opaque = np.flatnonzero((w.mat_ids == 0) & w.enabled)[:80]
    yield 5, w.set_material(opaque, 1)                      # material key 0 -> 1
    yield 6, w.set_material(opaque, 2 if blend else 3)      # 1 -> 2 (blend), or back to an opaque key
    yield 7, w.wide_key(int(opaque[0]), 64)                 # one key >= 64: the host batching for this frame
    yield 8, merge(w.set_material(opaque[:1], 2 if blend else 3), w.grow(extra=64, used=40))
    yield 9, w.replace_texture(0)
    d = w.move(0.01)
    slots, key, flags, loc = d.sort                         # stale entries for five slots, listed before their final ones
    d.sort = (np.concatenate([slots[:5], slots]), np.concatenate([key[:5] + 1, key]), np.concatenate([flags[:5] ^ 1, flags]),
              np.concatenate([loc[:5] + 99.0, loc]))
    yield 10, d
    yield 11, w.move(0.10)


def contexts():
    return load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True)


@pytest.mark.parametrize("frame_sort,host", [("0", False), ("1", False), ("0", True)])
def test_incremental_updates_equal_full_uploads(monkeypatch, frame_sort, host):
    """Twelve frames of a changing textured cube field: moves of 1 % and 10 % of the objects, objects killed and revived, material keys
    0 -> 1 -> 2 and one key >= 64 for a frame, objects added by a growth of the object buffer plus updates, a mesh appended past the
    buffer's capacity and used by the new objects, a texture appended and another replaced.  B equals A bit for bit every frame, its
    batching path goes device -> host -> device, and on three frames B equals the oracle.  (Some later frames differ from the oracle with
    full uploads as well: the previous-invocation entries of the batch tables when the batching path changes or the object count grows,
    and the readable length of the residual index list after objects are revived.  A and B agree there, so those frames are held to A.)"""
    monkeypatch.setenv("R3_FRAME_SORT", frame_sort)
    if host:
        monkeypatch.setenv("R3_HOST_BATCHING", "1")
    else:
        monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    w = ChangingWorld(n_objects=3000)
    a, b = contexts()
    orc = load_oracle_backend() if frame_sort == "0" and not host else None
    ga, gb = BaseRenderGraph(a), BaseRenderGraph(b)
    go = BaseRenderGraph(orc) if orc else None
    device = "device, frame-wide sort" if frame_sort == "1" else "device"
    paths = []
    for frame, d in itertools.chain([(0, None)], script(w)):   # lazily: each change is made right before its frame
        ga.add_to_graph(w.ev, RES, 1, SETTINGS)
        if d is not None:
            upload_delta(b, w.ev, d)
        gb.add_to_graph(w.ev, RES, 1, SETTINGS, upload=(frame == 0))
        assert_same_frame(a, b, w.ev, f"frame {frame}")
        paths.append(b.batching_info(CAMERA_VIEWPORT)["path"])
        if go is not None:
            go.add_to_graph(w.ev, RES, 1, SETTINGS)
            if frame in (0, 1, 6):   # the first frame; a move; blend objects
                compare_frame_state(b, orc, w.ev, [CAMERA_VIEWPORT, 0, 1], what=f"oracle, frame {frame}", f16_samples=True)
    assert paths == (["host"] * 12 if host else [device] * 7 + ["host"] + [device] * 4), paths
    assert len(w.ev.object_buffer) == 3064 and b.visible_count(CAMERA_VIEWPORT) > 0
    a.close(), b.close()


# ------------------------------------------------------------------ edge cases of the sort info and the object buffer
def cloud_world(n, seed=3):
    rec = object_cloud_records(n, seed=seed, extent=60.0)
    rng = np.random.default_rng(seed)
    key = rng.integers(0, 3, n).astype(np.uint64)
    flags = (1 | 2 * rng.integers(0, 2, n) | 4 * (key == 2)).astype(np.uint8)
    return rec, key, flags, rec["sphere_center"].copy()


def assert_same_objects(a, b, n, what):
    ra, rb = (cull_and_batch(x, n) + [x.batching_info(CAMERA_VIEWPORT)["path"]] for x in (a, b))
    for k, name in enumerate(("visible list", "MV/MVP", "batches", "regions", "batching path")):
        assert ra[k] == rb[k], f"{what}: {name} differs"
    return np.frombuffer(ra[0], np.uint32)


def test_duplicate_slots_and_shared_live_words(monkeypatch):
    """A slot listed twice takes its later entry; slots of one live-bit word — the last, partial one included — change in one call."""
    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    n = 1000                                                         # 1000 = 31 * 32 + 8: the last live word is partial
    rec, key, flags, loc = cloud_world(n)
    a, b = contexts()
    for x in (a, b):
        x.set_objects(rec)
        x.set_object_sort_info(key, flags, loc)
    slots = np.array([5, 9, 5, 0, 1, 31, 32, 33, 63, 992, 995, 999, 5], dtype=np.uint32)
    k2 = (key[slots] + 1) % 3
    f2 = (flags[slots] ^ 1).astype(np.uint8)                        # live bits flip, within shared words
    l2 = loc[slots] + np.float32(3.0)
    k2[2], f2[2], l2[2] = 0, 7, (1.0, 1.0, 1.0)                      # slot 5's middle entry, overridden by the last
    k2[-1], f2[-1], l2[-1] = 2, 5, (-4.0, 2.0, 8.0)
    b.update_object_sort_info(slots, k2, f2, l2)
    key2, flags2, loc2 = key.copy(), flags.copy(), loc.copy()
    for i, s in enumerate(slots):                                    # in order: the last entry of a slot wins
        key2[s], flags2[s], loc2[s] = k2[i], f2[i], l2[i]
    a.set_object_sort_info(key2, flags2, loc2)
    assert_same_objects(a, b, n, "duplicates")
    a.close(), b.close()


def test_resize_1000_1001_70001(monkeypatch):
    """The object buffer grows 1000 -> 1001 -> 70001 in place (zero records, sort info grown with zeros), new slots filled by updates;
    each step equals r3_set_objects + r3_set_object_sort_info of the same contents, through the device and the host batching."""
    for host in (False, True):
        if host:
            monkeypatch.setenv("R3_HOST_BATCHING", "1")
        else:
            monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
        rec, key, flags, loc = cloud_world(70001, seed=8)
        a, b = contexts()
        cur = 1000
        b.set_objects(rec[:cur])
        b.set_object_sort_info(key[:cur], flags[:cur], loc[:cur])
        for new in (1001, 70001):
            b.resize_objects(new)
            full_rec, full_key, full_flags, full_loc = np.zeros(new, rec.dtype), np.zeros(new, np.uint64), np.zeros(new, np.uint8), np.zeros((new, 3), np.float32)
            full_rec[:cur], full_key[:cur], full_flags[:cur], full_loc[:cur] = rec[:cur], key[:cur], flags[:cur], loc[:cur]
            a.set_objects(full_rec)
            a.set_object_sort_info(full_key, full_flags, full_loc)
            assert_same_objects(a, b, new, f"resize to {new} (host={host})")
            fill = np.arange(cur, new, 2, dtype=np.uint32)             # every other new slot gets an object; the rest stay zero records
            b.update_objects(fill, rec[fill])
            b.update_object_sort_info(fill, key[fill], flags[fill], loc[fill])
            full_rec[fill], full_key[fill], full_flags[fill], full_loc[fill] = rec[fill], key[fill], flags[fill], loc[fill]
            a.set_objects(full_rec)
            a.set_object_sort_info(full_key, full_flags, full_loc)
            vis = assert_same_objects(a, b, new, f"filled to {new} (host={host})")
            if new - cur > 1000:
                assert np.any(vis >= cur), "some of the new objects are visible"
            cur = new
        a.close(), b.close()


def test_rejections_leave_the_context_unchanged(monkeypatch):
    """Every rejected call (bad slot, shrink, borrowed records, connected exchange / peer plumbing, misaligned mesh or texel ranges, a gap
    in the texture table, bad descriptors) returns its error, and the next frame still equals the full-upload context's."""
    import torch

    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    w = ChangingWorld(n_objects=600, seed=21)
    a, b = contexts()
    ga, gb = BaseRenderGraph(a), BaseRenderGraph(b)
    ev, n = w.ev, len(w.ev.object_buffer)

    def frame(what):
        ga.add_to_graph(ev, RES, 1, SETTINGS)
        gb.add_to_graph(ev, RES, 1, SETTINGS, upload=(what == "first"))
        assert_same_frame(a, b, ev, what)

    frame("first")
    mesh_before = b.readback_mesh_buffer(len(ev.mesh_buffer))
    s = np.array([3, n], dtype=np.uint32)                            # the second slot is out of range: nothing is written, not even slot 3
    expect_error(E_INVALID, b.update_object_sort_info, s, np.array([2, 0], np.uint64), np.array([0, 0], np.uint8), np.zeros((2, 3), np.float32))
    expect_error(E_INVALID, b.resize_objects, n - 1)
    ex = b.exchange_create(CAMERA_VIEWPORT, 1, 0, n)
    b.exchange_connect(CAMERA_VIEWPORT, ex)
    expect_error(E_STATE, b.resize_objects, n + 10)
    b.exchange_destroy(CAMERA_VIEWPORT)
    handles = b.peer_create(1, 0)
    b.peer_connect(handles)
    expect_error(E_STATE, b.resize_objects, n + 10)
    b.peer_destroy()
    expect_error(E_INVALID, b.update_mesh_buffer, 2, np.zeros(4, np.uint32))
    expect_error(E_INVALID, b.update_mesh_buffer, 0, np.zeros(6, np.uint8))
    t = len(ev.texture_descs)
    good = ev.texture_descs[:1].copy()
    expect_error(E_INVALID, b.update_textures, t + 1, good, 0, np.zeros(0, np.uint8))            # would leave a gap
    expect_error(E_INVALID, b.update_textures, t, good, 8, np.zeros(32, np.uint8))               # texels not 16-aligned
    bad = good.copy()
    bad["byte_offset"] = len(ev.texture_texels)                                                 # mip chain past the blob
    expect_error(E_INVALID, b.update_textures, t, bad, len(ev.texture_texels), np.zeros(16, np.uint8))
    bad = good.copy()
    bad["format"] = 255
    expect_error(E_INVALID, b.update_textures, 0, bad, 0, np.zeros(0, np.uint8))
    assert np.array_equal(b.readback_mesh_buffer(len(ev.mesh_buffer)), mesh_before)
    frame("after the rejections")
    # borrowed records: the growth is refused while the caller owns the buffer
    dev = torch.from_numpy(ev.object_buffer.view(np.uint8).copy()).cuda()
    b.set_objects_device(dev.data_ptr(), n)
    expect_error(E_STATE, b.resize_objects, n + 10)
    b.set_objects(ev.object_buffer)
    del dev
    frame("after borrowed records")
    # a count of 0 is a no-op
    b.update_object_sort_info(np.zeros(0, np.uint32), np.zeros(0, np.uint64), np.zeros(0, np.uint8), np.zeros((0, 3), np.float32))
    b.update_mesh_buffer(0, np.zeros(0, np.uint32))
    b.update_textures(0, np.zeros(0, TEXTURE_DESC_DTYPE), 0, np.zeros(0, np.uint8))
    b.resize_objects(n)
    d = w.move(0.05)
    upload_delta(b, ev, d)
    frame("after a move")
    a.close(), b.close()


# ------------------------------------------------------------------ mesh growth
def test_skinned_ranges_survive_mesh_growth():
    """r3_skin's output is part of the megabuffer: a growth keeps it, the gap before the appended range reads 0."""
    import skinning_case

    words, inputs, joints, _ = skinning_case.build(seed=2, vertex_counts=(257, 5000, 1), joints_per_skeleton=(3, 16, 1))
    a, b = load_cuda_backend(0), load_cuda_backend(0)
    for x in (a, b):
        x.set_mesh_buffer(words)
        x.skin(inputs, joints)
    skinned = a.readback_mesh_buffer(len(words))
    assert not np.array_equal(skinned, words)
    extra = np.random.default_rng(3).integers(0, 2 ** 32, 3 * len(words), dtype=np.uint32)   # past the capacity: the buffer grows
    b.update_mesh_buffer(4 * (len(words) + 16), extra)
    got = b.readback_mesh_buffer(len(words) + 16 + len(extra))
    assert np.array_equal(got[:len(words)], skinned), "the skinned ranges must survive the growth"
    assert not got[len(words):len(words) + 16].any(), "the gap reads 0"
    assert np.array_equal(got[len(words) + 16:], extra)
    a.close(), b.close()


def test_mesh_end_scene_built_through_growth():
    """cull_scenes' index runs at the end of the mesh, uploaded range by range: once into a buffer that grows, once into a larger stale
    one whose words past the end must still read 0.  The triangle cull matches the restated cull.wgsl."""
    s, end, stale = scenes.mesh_end_scene()
    for with_stale in (False, True):
        b = load_cuda_backend(0)
        if with_stale:
            b.set_mesh_buffer(stale)
            b.set_mesh_buffer(s.mesh[:100])
        else:
            b.update_mesh_buffer(0, s.mesh[:100])
        b.update_mesh_buffer(400, s.mesh[100:end - 40])
        b.update_mesh_buffer(4 * (end - 40), s.mesh[end - 40:])
        assert np.array_equal(b.readback_mesh_buffer(end), s.mesh)
        b.set_objects(s.objects)
        hdr = scenes.ortho_header(256, 256, PCU_MULTISAMPLED, len(s.objects))
        got = scenes.run_cull(b, s, hdr)
        want = scenes.reference_for(got, s, hdr, None)
        scenes.assert_matches(got, want, s, f"mesh end through growth, stale={with_stale}")
        assert want["pass32"][:2].all()
        b.close()


# ------------------------------------------------------------------ frame graphs
def test_updates_between_frame_graphs(monkeypatch):
    """Updates between r3_frame_begin / r3_frame_end brackets: after the first frame every frame of B is one graph launch with no early
    flush — also after the mesh and the texture blob grew — and every frame equals A's."""
    monkeypatch.setenv("R3_FRAME_GRAPH", "1")
    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    w = ChangingWorld(n_objects=1500, seed=5, blend=False)
    a, b = contexts()
    ga, gb = BaseRenderGraph(a), BaseRenderGraph(b)
    flushes = []
    steps = [(0, None), (1, lambda: w.move(0.01)), (2, lambda: w.move(0.1)), (3, lambda: w.kill(w.live_slots(0.02))),
             (4, lambda: w.set_material(np.flatnonzero(w.mat_ids == 0)[:50], 1)), (5, lambda: w.replace_texture(1))]
    for frame, change in steps:
        d = change() if change else None
        ga.add_to_graph(w.ev, RES, 1, SETTINGS)
        if d is not None:
            upload_delta(b, w.ev, d)
        before = b.frame_graph_stats()["flushed"]
        gb.add_to_graph(w.ev, RES, 1, SETTINGS, upload=(frame == 0))
        flushes.append(b.frame_graph_stats()["flushed"] - before)
        assert_same_frame(a, b, w.ev, f"graph frame {frame}")
    # a mesh appended past the capacity and a texture appended (both grow on the host side of the bracket), used by existing slots
    g = w.grow(extra=0, used=0)
    d = merge(g, w.set_material(np.flatnonzero(w.enabled)[:30], len(w.r.materials) - 1))
    ga.add_to_graph(w.ev, RES, 1, SETTINGS)
    upload_delta(b, w.ev, d)
    before = b.frame_graph_stats()["flushed"]
    gb.add_to_graph(w.ev, RES, 1, SETTINGS, upload=False)
    flushes.append(b.frame_graph_stats()["flushed"] - before)
    assert_same_frame(a, b, w.ev, "graph frame after the growth")
    st = b.frame_graph_stats()
    assert st["frames"] == len(flushes) and st["graphed"] == len(flushes) - 1, st   # the first frame allocates: one early flush
    assert flushes[1:] == [0] * (len(flushes) - 1), f"early flushes per frame: {flushes}"
    a.close(), b.close()


# ------------------------------------------------------------------ scale
def test_ten_million_slots_one_percent_moved(monkeypatch):
    """10 M slots from the config-4 generator, 1 % of them moved per frame for three frames: the visible list, a seeded sample of MV/MVP
    and the viewport's device batch tables equal the full-upload context's."""
    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    n = 10_000_000
    rec = object_cloud_records(n, seed=4)
    rec["index_count"] = 0   # cull-only, as config 4: 10 M slots of 256 padded invocations each would exceed the device batching's 2^31 bound
    rng = np.random.default_rng(40)
    key = rng.integers(0, 3, n).astype(np.uint64)
    flags = (1 | 2 * (key != 2) | 4 * (key == 2)).astype(np.uint8)
    loc = rec["sphere_center"].copy()
    header = per_camera_header(cloud_camera(), CAMERA_VIEWPORT, (1920, 1080), 1, n)
    a, b = load_cuda_backend(0), load_cuda_backend(0)
    for x in (a, b):
        x.set_objects(rec)
        x.set_object_sort_info(key, flags, loc)
    sample = np.sort(rng.choice(n, 4096, replace=False))
    for frame in range(3):
        slots = np.sort(rng.choice(n, n // 100, replace=False)).astype(np.uint32)
        t = rec["transform"][slots].reshape(-1, 16)
        shift = rng.uniform(-20.0, 20.0, (len(slots), 3)).astype(np.float32)
        t[:, 12:15] += shift
        rec["transform"][slots] = t
        rec["sphere_center"][slots] += shift
        loc[slots] = rec["sphere_center"][slots]
        a.set_objects(rec)
        a.set_object_sort_info(key, flags, loc)
        b.update_objects(slots, rec[slots])
        b.update_object_sort_info(slots, key[slots], flags[slots], loc[slots])
        for x in (a, b):
            x.object_uniform_upload(CAMERA_VIEWPORT, header, CB_BAKE | CB_CULL)
            x.batch_objects(CAMERA_VIEWPORT, np.zeros(3, dtype=np.float32))
        assert np.array_equal(a.readback_visible(CAMERA_VIEWPORT), b.readback_visible(CAMERA_VIEWPORT)), f"frame {frame}: visible list"
        for i in sample:
            assert a.readback_object_matrices(CAMERA_VIEWPORT, int(i), 1).tobytes() == b.readback_object_matrices(CAMERA_VIEWPORT, int(i), 1).tobytes(), \
                f"frame {frame}: MV/MVP of slot {i}"
        assert b.batching_info(CAMERA_VIEWPORT)["path"].startswith("device")
        ba, ra = a.readback_batches(CAMERA_VIEWPORT)
        bb, rb = b.readback_batches(CAMERA_VIEWPORT)
        assert ba.tobytes() == bb.tobytes() and ra.tobytes() == rb.tobytes(), f"frame {frame}: batch tables"
    a.close(), b.close()
