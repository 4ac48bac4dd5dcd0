"""Objects that switch between prepared mesh and material variants — r3_set_object_variants, r3_switch_object_variants,
r3_switch_object_variants_device — against the re-added world fed through r3_update_objects + r3_update_object_sort_info +
r3_set_object_mesh_spheres (bit for bit) and the CPU oracle given the re-added world (within the parity tolerance), plus the frame graph,
the invocation bound, the blend routine's bookkeeping, the dense form, validation and the ordering with the other per-object calls."""
import ctypes
import os
import re

import numpy as np
import pytest

from harness import ROOT, assert_same_frame, check_declared_and_exported, cull_and_batch, expect_error, settings, to_device, unbound_backend
from object_variant_case import PARTNER_OPAQUE, VariantWorld, expected_bound, update_path
from rend3_b200.backend import CAMERA_VIEWPORT, load_cuda_backend
from rend3_b200.layouts import OBJECT_VARIANT_DTYPE, VARIANT_GROUP_DTYPE, VARIANT_NONE

E_INVALID, E_STATE = -1, -5
RES = (256, 160)
DECLS = (
    "int r3_set_object_variants(r3_ctx*, const r3_object_variant* variants, uint32_t n_variants, const r3_variant_group* groups, uint32_t n_groups, const uint32_t* slots, const uint32_t* slot_groups, uint32_t n_listed);",
    "int r3_switch_object_variants(r3_ctx*, const uint32_t* slots_or_null, const uint32_t* choices, uint32_t n);",
    "int r3_switch_object_variants_device(r3_ctx*, const uint32_t* d_slots_or_null, const uint32_t* d_choices, uint32_t n);",
    "int r3_readback_object_variants(r3_ctx*, uint32_t* out, uint32_t first, uint32_t n);",
)


# ------------------------------------------------------------------ without a GPU
def test_library_exports_the_four_entry_points_with_the_headers_signatures():
    check_declared_and_exported(DECLS, lambda decl: [None] * decl.count(",") + [0])


def test_variant_record_layout_equals_the_c_header():
    text = open(os.path.join(ROOT, "include", "r3_layouts.h")).read()
    body = re.search(r"typedef struct r3_object_variant \{(.*?)\} r3_object_variant;", text, re.S).group(1)
    offsets = {m.group(1): int(m.group(2)) for m in re.finditer(r"(\w+)(?:\[\d+\])?;\s*/\*\s*@(\d+)", body)}
    assert offsets == {name: OBJECT_VARIANT_DTYPE.fields[name][1] for name in OBJECT_VARIANT_DTYPE.names}
    assert re.search(r"sizeof\(r3_object_variant\) == 64", text) and OBJECT_VARIANT_DTYPE.itemsize == 64
    assert re.search(r"sizeof\(r3_variant_group\) == 8", text) and VARIANT_GROUP_DTYPE.itemsize == 8
    for name in OBJECT_VARIANT_DTYPE.names:
        if name != "first_index":
            assert f"offsetof(r3_object_variant, {name}) == {offsets[name]}" in text, name


@pytest.mark.parametrize("choices,slots", [
    (np.zeros((4, 2), np.uint32), None),                        # 2-d choices
    (np.zeros(4, np.float32), None),                            # float choices
    (np.zeros(4, np.uint32), np.arange(3)),                     # lengths differ
    (np.zeros(2, np.uint32), np.array([-1, 3])),                # negative slot
    (np.array([1 << 32]), None),                                # beyond uint32
], ids=["2d", "float", "length", "negative", "wide"])
def test_host_wrappers_reject_bad_shapes_and_dtypes_before_calling(choices, slots):
    with pytest.raises(AssertionError, match="choices|slots"):
        unbound_backend().switch_object_variants(choices, slots)


def test_set_and_device_wrappers_reject_bad_arguments_before_calling():
    torch = pytest.importorskip("torch")
    b = unbound_backend()
    v, g = np.zeros(2, OBJECT_VARIANT_DTYPE), np.zeros(1, VARIANT_GROUP_DTYPE)
    for args in ((np.zeros(2, np.uint32), g), (v, np.zeros(1, np.uint32)), (v, g, np.arange(3), np.zeros(2)), (v, g, np.arange(2), None)):
        with pytest.raises(AssertionError):
            b.set_object_variants(*args)
    for choices in (torch.zeros(4, dtype=torch.int32), np.zeros(4, np.uint32), None):   # a host tensor, a numpy array, no length
        with pytest.raises(AssertionError):
            b.switch_object_variants_device(choices)


def test_expected_state_equals_world_readd_object():
    """VariantWorld.choose (the vectorised re-add the GPU tests hold the calls to) against world.Renderer: the same objects added one by
    one, then readd_object with each switched slot's mesh and material, then evaluate — records, mesh spheres, keys, flags, locations."""
    from world_update_scene import sort_flags

    from rend3_b200.world import Object

    w = VariantWorld(n_objects=60, seed=3)
    r, n = w.r, w.n
    t = w._transforms(np.arange(n))
    handles = [r.add_object(Object(int(w.mesh_ids[i]), int(w.mat_ids[i]), t[i])) for i in range(n)]
    rng = np.random.default_rng(1)
    for step in range(4):
        choices = rng.integers(0, 4, n).astype(np.uint32)
        d = w.choose(choices)
        for s in d.objects:
            v = w.variants[w.variant_of(int(s), int(choices[s]))]
            mesh = w.lod_mesh[int(choices[s]) & 1]
            assert v["first_index"] == r.meshes[mesh]["index_start"] // 4
            r.readd_object(handles[s], mesh, int(v["material_index"]))
        ev = r.evaluate()
        for f in ev.object_buffer.dtype.names:
            assert ev.object_buffer[f][:n].tobytes() == w.ev.object_buffer[f][:n].tobytes(), f"step {step}: {f}"
        assert ev.object_mesh_sphere[:n].tobytes() == w.mesh_spheres.tobytes(), f"step {step}: mesh spheres"
        assert np.array_equal(ev.object_material_key[:n], w.ev.object_material_key[:n])
        assert np.array_equal(sort_flags(ev)[:n], sort_flags(w.ev)[:n])
        assert ev.object_location[:n].tobytes() == w.ev.object_location[:n].tobytes(), f"step {step}: locations"
        # the variant table says the same as the re-add: key and flags bits 1-2 of the chosen variant
        v = w.variants[w.variant_of(np.arange(n), w.choice)]
        assert np.array_equal(v["material_key"], ev.object_material_key[:n])
        assert np.array_equal(v["sort_flags"], sort_flags(ev)[:n] & 6)
        assert np.array_equal(v["index_count"], ev.object_buffer["index_count"][:n])


# ------------------------------------------------------------------ GPU
def u32_tensor(b, a):
    return to_device(b, np.asarray(a, dtype=np.uint32).view(np.int32))


def same_fields(a, b):
    return len(a) == len(b) and all(a[f].tobytes() == b[f].tobytes() for f in a.dtype.names)


def prepare(graph, b, w, samples=1):
    """The first frame, then the mesh spheres and the variant set (every slot listed)."""
    graph.add_to_graph(w.ev, RES, samples, settings())
    b.set_object_mesh_spheres(w.mesh_spheres)
    b.set_object_variants(w.variants, w.groups, np.arange(w.n), w.slot_groups)


@pytest.mark.gpu
@pytest.mark.parametrize("samples,host", [(1, False), (4, False), (1, True)], ids=["x1", "x4", "x1-host-batching"])
def test_gpu_switches_equal_the_update_path_and_the_oracle(monkeypatch, samples, host):
    """Nine frames of a world with opaque, cutout and blend variants, two shadowed lights and point lights; every frame picks LODs by
    distance with a moving threshold and swaps materials of a random subset.  The host form (dense) and the device form (sparse, the
    changed slots in descending order) equal the update path in every artefact bit for bit, records and locations included; with
    device batching the oracle, given the re-added world, gives the same visible lists and depth."""
    from oracle import load_oracle_backend
    from rend3_b200.routines import BaseRenderGraph

    if host:
        monkeypatch.setenv("R3_HOST_BATCHING", "1")
    else:
        monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    w = VariantWorld(n_objects=2000)
    n = w.n
    ctx = {"update": load_cuda_backend(0, parity_target=True), "host": load_cuda_backend(0, parity_target=True), "device": load_cuda_backend(0, parity_target=True)}
    graphs = {k: BaseRenderGraph(x) for k, x in ctx.items()}
    for k, x in ctx.items():
        prepare(graphs[k], x, w, samples)
    orc = None if host else load_oracle_backend()
    go = None if host else BaseRenderGraph(orc)
    if go is not None:
        go.add_to_graph(w.ev, RES, samples, settings())   # the frame before: every predicted pass replays the same previous frame
    rng = np.random.default_rng(samples)
    swap = np.zeros(n, dtype=bool)
    keep = []
    cam = w.ev.camera.location()
    for frame, threshold in enumerate((12.0, 16.0, 8.0, 30.0, 0.0, 14.0, 14.0, 20.0, 10.0)):
        flip = rng.choice(n, n // 8, replace=False)
        swap[flip] = ~swap[flip]
        choices = w.lod_choices(cam, threshold, swap)
        changed = np.flatnonzero(choices != w.choice)
        d = w.choose(choices)
        update_path(ctx["update"], w, d)
        graphs["update"].add_to_graph(w.ev, RES, samples, settings(), upload=False)
        graphs["host"].add_to_graph(w.ev, RES, samples, settings(), upload=False, object_variants=(None, choices))
        entries = (u32_tensor(ctx["device"], changed[::-1]), u32_tensor(ctx["device"], choices[changed[::-1]]))
        keep.append(entries)
        graphs["device"].add_to_graph(w.ev, RES, samples, settings(), upload=False, object_variants=entries)
        want_rec, want_loc = ctx["update"].readback_objects(0, n)
        for name in ("host", "device"):
            assert_same_frame(ctx[name], ctx["update"], w.ev, f"frame {frame}, {name} form")
            assert ctx[name].readback_ldr().tobytes() == ctx["update"].readback_ldr().tobytes(), f"frame {frame}, {name}: LDR"
            rec, loc = ctx[name].readback_objects(0, n)
            assert same_fields(rec, want_rec), f"frame {frame}, {name}: records"
            assert loc.tobytes() == want_loc.tobytes(), f"frame {frame}, {name}: sort locations"
            assert same_fields(rec, w.ev.object_buffer[:n]), f"frame {frame}, {name}: records against the re-added world"
        got = ctx["device"].readback_object_variants(0, n)
        assert np.array_equal(got[changed], w.variant_of(changed, choices[changed])), f"frame {frame}: current variants"
        if orc is not None:
            go.add_to_graph(w.ev, RES, samples, settings())
            for c in [CAMERA_VIEWPORT] + list(range(len(w.ev.shadows))):
                assert np.array_equal(ctx["device"].readback_visible(c), orc.readback_visible(c)), f"frame {frame} camera {c}: oracle"
            assert np.array_equal(ctx["device"].readback_depth().view(np.uint32), orc.readback_depth().view(np.uint32)), f"frame {frame}: oracle depth"
    for x in ctx.values():
        x.close()
    if orc is not None:
        orc.close()


@pytest.mark.gpu
def test_gpu_device_picked_lods_stay_one_graph(monkeypatch):
    """Six recorded frames of a world without key-2 variants: a torch producer on the context's stream picks every object's LOD from
    its distance to a moving point and swaps some materials; the device form applies the choices inside the frame.  Every frame is one
    graph with no early flush, the frames equal the same frames run eagerly bit for bit, and the read-back variants are the producer's."""
    import torch

    from rend3_b200.routines import BaseRenderGraph

    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    w = VariantWorld(n_objects=1500, blend=False, partner=PARTNER_OPAQUE)
    assert not (w.variants["material_key"] == 2).any()
    n = w.n
    graph_b, eager_b = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True)
    graphs = {id(x): BaseRenderGraph(x) for x in (graph_b, eager_b)}
    for x in (graph_b, eager_b):
        prepare(graphs[id(x)], x, w)
        graphs[id(x)].add_to_graph(w.ev, RES, 1, settings(), upload=False, frame_graph=x is graph_b)   # graphs instantiated
    before = graph_b.frame_graph_stats()
    pos = {id(x): to_device(x, w.translation) for x in (graph_b, eager_b)}
    keep = []
    for frame in range(6):
        point = np.array([np.cos(frame), 0.5, np.sin(frame)], dtype=np.float32) * 10.0
        for x in (graph_b, eager_b):
            with torch.cuda.stream(torch.cuda.ExternalStream(x.stream())):
                p = pos[id(x)]
                d = torch.linalg.vector_norm(p - torch.from_numpy(point).to("cuda"), dim=1)
                swap = (torch.arange(n, device="cuda") % 7 == frame).to(torch.int32)
                choices = ((d > 12.0).to(torch.int32) + 2 * swap).contiguous()
            keep.append(choices)
            graphs[id(x)].add_to_graph(w.ev, RES, 1, settings(), upload=False, frame_graph=x is graph_b, object_variants=(None, choices))
        after = graph_b.frame_graph_stats()
        assert after["flushed"] == before["flushed"], f"frame {frame} flushed early"
        assert_same_frame(graph_b, eager_b, w.ev, f"frame {frame}: graph vs eager")
        want = w.variant_of(np.arange(n), keep[-1].cpu().numpy().astype(np.uint32))
        assert np.array_equal(graph_b.readback_object_variants(0, n), want), f"frame {frame}: current variants"
    stats = graph_b.frame_graph_stats()
    assert stats["graphed"] - before["graphed"] == 6 and stats["flushed"] == before["flushed"], stats
    graph_b.close(), eager_b.close()


@pytest.mark.gpu
def test_gpu_invocation_bound_takes_the_groups_largest_level(monkeypatch):
    """After the set call the bound is the sum of round_up(max(index_count, group max) / 3, 256); switching every slot to its smallest
    and then to its largest level leaves it unchanged without a flush; removing the set restores the old bound."""
    from rend3_b200.routines import BaseRenderGraph

    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    w = VariantWorld(n_objects=1200, blend=False, partner=PARTNER_OPAQUE)
    b = load_cuda_backend(0, parity_target=False)
    g = BaseRenderGraph(b)
    g.add_to_graph(w.ev, RES, 1, settings())
    b.set_object_mesh_spheres(w.mesh_spheres)
    counts = w.ev.object_buffer["index_count"]
    old = b.debug_invocation_bound()
    assert old == expected_bound(counts, np.zeros_like(counts))
    listed = np.arange(0, w.n, 3)
    b.set_object_variants(w.variants, w.groups, listed, w.slot_groups[listed])
    floors = np.zeros(w.n, np.int64)
    floors[listed] = [w.variants["index_count"][4 * gr:4 * gr + 4].max() for gr in w.slot_groups[listed]]
    bound = b.debug_invocation_bound()
    assert bound == expected_bound(counts, floors)
    flushed = b.frame_graph_stats()["flushed"]
    for lod in (1, 0, 1):
        keep = (u32_tensor(b, listed), u32_tensor(b, np.full(len(listed), lod)))
        g.add_to_graph(w.ev, RES, 1, settings(), upload=False, frame_graph=True, object_variants=keep)
        assert b.debug_invocation_bound() == bound
    assert b.frame_graph_stats()["flushed"] == flushed, "a switch flushed a recorded frame"
    b.set_object_variants(np.zeros(0, OBJECT_VARIANT_DTYPE), np.zeros(0, VARIANT_GROUP_DTYPE))
    rec = b.readback_objects(0, w.n, locations=False)[0]
    assert b.debug_invocation_bound() == expected_bound(rec["index_count"], np.zeros_like(counts))
    b.close()


@pytest.mark.gpu
def test_gpu_blend_routine_bookkeeping(monkeypatch):
    """Host form: swapping the only blended object to an opaque variant stops the blend routine (forward_stats[3] == 0, a recorded frame
    no longer flushes).  Device form: the routine keeps running while some variant has key 2.  The images are equal either way."""
    from rend3_b200.routines import BaseRenderGraph

    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    w = VariantWorld(n_objects=600, blend=False, partner={0: 2, 1: 0, 2: 0, 3: 1})   # group 0 swaps to blend
    opaque0 = np.flatnonzero(w.slot_groups == 0)
    vis = None
    hb, db = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True)
    gh, gd = BaseRenderGraph(hb), BaseRenderGraph(db)
    for g, b in ((gh, hb), (gd, db)):
        prepare(g, b, w)
        vis = b.readback_visible(CAMERA_VIEWPORT)
    cand = np.intersect1d(vis, opaque0)
    x = int(cand[np.argmin(np.linalg.norm(w.translation[cand] - w.ev.camera.location(), axis=1))])   # nearest: its fragments are seen
    lod = int(w.choice[x]) & 1

    def frame(g, b, **kw):
        before = b.frame_graph_stats()["flushed"]
        g.add_to_graph(w.ev, RES, 1, settings(), upload=False, frame_graph=True, **kw)
        return b.frame_graph_stats()["flushed"] - before
    hb.switch_object_variants(np.array([lod + 2]), np.array([x]))          # the only blended object
    db.switch_object_variants(np.array([lod + 2]), np.array([x]))
    assert frame(gh, hb) > 0 and frame(gd, db) > 0 and hb.forward_stats()[3] > 0
    hb.switch_object_variants(np.array([lod]), np.array([x]))
    keep = (u32_tensor(db, [x]), u32_tensor(db, [lod]))
    assert frame(gh, hb) == 0 and hb.forward_stats()[3] == 0, "no blended object: the routine is off"
    assert frame(gd, db, object_variants=keep) > 0, "after the device form any key-2 variant runs the routine"
    assert db.readback_hdr_f16().tobytes() == hb.readback_hdr_f16().tobytes() and db.readback_ldr().tobytes() == hb.readback_ldr().tobytes()
    hb.close(), db.close()


def cloud_world(n):
    from rend3_b200.scenes import object_cloud_records

    rec = object_cloud_records(n, seed=5, extent=60.0)
    rec["enabled"] = 1
    key = np.zeros(n, np.uint64)
    flags = np.full(n, 1 | 2, np.uint8)
    variants = np.zeros(6, OBJECT_VARIANT_DTYPE)
    variants["first_index"], variants["index_count"] = rec["first_index"][0], [36, 12, 24, 36, 6, 3]
    variants["attr_offset"] = rec["attr_offset"][0]
    variants["material_key"] = [0, 1, 3, 0, 1, 5]
    variants["sort_flags"] = [2, 0, 4, 6, 2, 0]
    variants["mesh_sphere"] = np.random.default_rng(1).uniform(-0.5, 1.5, (6, 4)).astype(np.float32)
    groups = np.zeros(2, VARIANT_GROUP_DTYPE)
    groups["first"], groups["count"] = [0, 3], [3, 3]
    return rec, key, flags, rec["sphere_center"].copy(), variants, groups


def cloud_context(n, mesh_words):
    rec, key, flags, loc, variants, groups = cloud_world(n)
    b = load_cuda_backend(0, parity_target=False)
    b.set_objects(rec)
    b.set_object_sort_info(key, flags, loc)
    b.set_mesh_buffer(mesh_words)
    b.set_object_mesh_spheres(np.tile(np.array([0.1, 0.2, 0.3, 1.0], np.float32), (n, 1)))
    return b, rec, variants, groups


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1000, 1024, 33])
def test_gpu_dense_form_equals_sparse_form(monkeypatch, n):
    """The dense form (whole centre-bit words, a ragged last word by atomics, unlisted slots and choices past the group kept as they
    were) equals the sparse form over the same entries: records, locations, visible list, MV / MVP, batches and current variants."""
    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    words = np.arange(4096, dtype=np.uint32) % 3
    ctx = {k: cloud_context(n, words) for k in ("dense", "sparse")}
    rng = np.random.default_rng(n)
    listed = np.flatnonzero(rng.random(n) < 0.9)
    sg = rng.integers(0, 2, len(listed)).astype(np.uint32)
    for b, rec, variants, groups in ctx.values():
        b.set_object_variants(variants, groups, listed, sg)
    keep = []
    for step, k in enumerate((n, n - 7, min(45, n), 1)):
        choices = rng.integers(0, 4, k).astype(np.uint32)                # 3 is past every group: dropped
        b = ctx["dense"][0]
        d = u32_tensor(b, choices)
        keep.append(d)
        b.switch_object_variants_device(d)
        perm = rng.permutation(k).astype(np.uint32)
        b = ctx["sparse"][0]
        s = (u32_tensor(b, perm), u32_tensor(b, choices[perm]))
        keep.append(s)
        b.switch_object_variants_device(s[1], s[0])
        out = {name: cull_and_batch(c[0], n) for name, c in ctx.items()}
        assert out["dense"] == out["sparse"], f"step {step}: cull / batch differ"
        (rd, ld), (rs, ls) = ctx["dense"][0].readback_objects(0, n), ctx["sparse"][0].readback_objects(0, n)
        assert same_fields(rd, rs) and ld.tobytes() == ls.tobytes(), f"step {step}: records differ"
        assert np.array_equal(ctx["dense"][0].readback_object_variants(0, n), ctx["sparse"][0].readback_object_variants(0, n))
    cur = ctx["dense"][0].readback_object_variants(0, n)
    assert (cur[np.setdiff1d(np.arange(n), listed)] == VARIANT_NONE).all(), "an unlisted slot was switched"
    for c in ctx.values():
        c[0].close()


@pytest.mark.gpu
def test_gpu_validation_leaves_the_context_unchanged(monkeypatch):
    """Every R3_E_INVALID / R3_E_STATE case of the set and host switch calls leaves records, locations, current variants and the next
    frame as they were; the device form drops unlisted slots and out-of-range choices and applies the rest."""
    import torch

    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    n = 500
    words = np.arange(4096, dtype=np.uint32) % 3
    b = load_cuda_backend(0, parity_target=False)
    rec, key, flags, loc, variants, groups = cloud_world(n)
    one = np.zeros(1, np.uint32)
    expect_error(E_STATE, b.set_object_variants, variants, groups, np.array([0]), one)          # before r3_set_objects
    expect_error(E_STATE, b.switch_object_variants, one, np.array([0]))
    b.close()
    b, rec, variants, groups = cloud_context(n, words)
    ref, _, _, _ = cloud_context(n, words)
    listed = np.arange(0, n, 2)
    sg = (listed % 4 == 0).astype(np.uint32)
    expect_error(E_STATE, b.switch_object_variants, one, np.array([0]))                          # before a set
    for x in (b, ref):
        x.set_object_variants(variants, groups, listed, sg)
        x.switch_object_variants(np.ones(len(listed), np.uint32), listed)

    def snapshot(x):
        r, l = x.readback_objects(0, n)
        return r, l.tobytes(), x.readback_object_variants(0, n).tobytes(), x.debug_invocation_bound()
    base = snapshot(b)

    def bad(**change):
        v = variants.copy()
        for f, val in change.items():
            v[f][1] = val
        return v
    attr = variants["attr_offset"][1].copy()
    attr[2] = 6
    no_pos = variants["attr_offset"][1].copy()
    no_pos[0] = 0xFFFFFFFF
    g_empty, g_past = groups.copy(), groups.copy()
    g_empty["count"][1] = 0
    g_past["count"][1] = 4
    invalid_sets = [
        (bad(first_index=len(words) - 2), groups, listed, sg),          # index range past the mesh buffer
        (bad(index_count=10), groups, listed, sg),                      # not triangles
        (bad(attr_offset=attr), groups, listed, sg),                    # offset not a multiple of 4
        (bad(attr_offset=no_pos), groups, listed, sg),                  # no position
        (bad(sort_flags=1), groups, listed, sg),                        # the live bit
        (bad(sort_flags=8), groups, listed, sg),                        # an unknown bit
        (variants, g_empty, listed, sg),                                # an empty group
        (variants, g_past, listed, sg),                                 # a group past the variants
        (variants, groups, np.array([3, n]), np.zeros(2, np.uint32)),   # a slot past the slot count
        (variants, groups, np.array([3, 9, 3]), np.zeros(3, np.uint32)),   # a slot named twice
        (variants, groups, np.array([3]), np.array([2], np.uint32)),    # a group index past n_groups
    ]
    for i, args in enumerate(invalid_sets):
        expect_error(E_INVALID, b.set_object_variants, *args)
    rc = b.lib.r3_set_object_variants(b.ctx, None, ctypes.c_uint32(2), None, ctypes.c_uint32(0), None, None, ctypes.c_uint32(0))
    assert rc == E_INVALID, "null variants"
    expect_error(E_INVALID, b.switch_object_variants, np.zeros(2, np.uint32), np.array([0, 1]))      # slot 1 is unlisted
    expect_error(E_INVALID, b.switch_object_variants, np.zeros(2, np.uint32), np.array([0, 0]))      # named twice
    expect_error(E_INVALID, b.switch_object_variants, np.array([0, 3], np.uint32), np.array([0, 2])) # choice past the group
    expect_error(E_INVALID, b.switch_object_variants, np.zeros(n, np.uint32))                        # dense: slot 1 is unlisted
    expect_error(E_INVALID, b.switch_object_variants, one, np.array([n]))                            # past the slot count
    now = snapshot(b)
    assert same_fields(now[0], base[0]) and now[1:] == base[1:], "a rejected call wrote something"
    assert cull_and_batch(b, n) == cull_and_batch(ref, n), "a rejected call changed the next frame"
    # a mesh buffer shorter than the set's indices
    b.set_mesh_buffer(words[:8])
    expect_error(E_STATE, b.switch_object_variants, one, np.array([0]))
    expect_error(E_STATE, b.switch_object_variants_device, u32_tensor(b, one), u32_tensor(b, [0]))
    b.set_mesh_buffer(words)
    # the device form drops unlisted slots and choices past the group
    slots = np.array([0, 1, 2, n, 0xFFFFFFFF, 4, 6], np.uint32)
    choices = np.array([2, 0, 5, 0, 0, 0, 2], np.uint32)
    keep = (u32_tensor(b, slots), u32_tensor(b, choices))
    b.switch_object_variants_device(keep[1], keep[0])
    ref.switch_object_variants(np.array([2, 0, 2], np.uint32), np.array([0, 4, 6]))
    r1, l1 = b.readback_objects(0, n)
    r2, l2 = ref.readback_objects(0, n)
    assert same_fields(r1, r2) and l1.tobytes() == l2.tobytes()
    assert b.readback_object_variants(0, n).tobytes() == ref.readback_object_variants(0, n).tobytes()
    assert cull_and_batch(b, n) == cull_and_batch(ref, n)
    # borrowed records
    dev = torch.from_numpy(rec.view(np.uint8).copy()).cuda()
    torch.cuda.synchronize()
    b.set_objects_device(dev.data_ptr(), n)
    expect_error(E_STATE, b.switch_object_variants, one, np.array([0]))
    expect_error(E_STATE, b.set_object_variants, variants, groups, listed, sg)
    b.sync()
    b.close(), ref.close()


@pytest.mark.gpu
def test_gpu_overlap_with_dynamic_mesh_sets_and_ordering_with_moves(monkeypatch):
    """A slot in both a deformable (or remeshable) set and the variant set is rejected in both call orders.  In one frame, a switch then
    r3_set_object_transforms_device gives the move's location with the new mesh sphere; a move then a switch gives the add's location."""
    from rend3_b200.layouts import DEFORMABLE_MESH_DTYPE, REMESHABLE_MESH_DTYPE

    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    n = 64
    words = np.arange(4096, dtype=np.uint32) % 3
    b, rec, variants, groups = cloud_context(n, words)
    dm = np.zeros(1, DEFORMABLE_MESH_DTYPE)
    dm["position_offset"], dm["normal_offset"], dm["tangent_offset"], dm["uv0_offset"] = rec["attr_offset"][0][0], 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF
    dm["first_index"], dm["index_count"], dm["vertex_count"] = rec["first_index"][0], rec["index_count"][0], 3
    rm = np.zeros(1, REMESHABLE_MESH_DTYPE)
    rm["position_offset"], rm["normal_offset"] = rec["attr_offset"][0][0], rec["attr_offset"][0][1]
    rm["tangent_offset"], rm["uv0_offset"], rm["color0_offset"] = 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF
    rm["first_index"], rm["index_capacity"], rm["vertex_capacity"] = rec["first_index"][0], rec["index_count"][0], 3
    for setter, mesh in ((b.set_deformable_meshes, dm), (b.set_remeshable_meshes, rm)):
        b.set_mesh_buffer(np.zeros(4096, np.uint32))                 # indices 0: below vertex_count
        setter(mesh, np.array([5]), np.array([0]))
        expect_error(E_INVALID, b.set_object_variants, variants, groups, np.array([4, 5]), np.array([0, 1], np.uint32))
        setter(mesh[:0])
        b.set_object_variants(variants, groups, np.array([4, 5]), np.array([0, 1], np.uint32))
        expect_error(E_INVALID, setter, mesh, np.array([5]), np.array([0]))
        setter(mesh, np.array([6]), np.array([0]))                   # disjoint slots are fine
        setter(mesh[:0])
        b.set_object_variants(np.zeros(0, OBJECT_VARIANT_DTYPE), np.zeros(0, VARIANT_GROUP_DTYPE))
    b.set_mesh_buffer(words)
    b.set_object_variants(variants, groups, np.arange(n), np.zeros(n, np.uint32))
    mats = np.tile(np.eye(4, dtype=np.float32).reshape(16), (2, 1))
    mats[:, 12:15] = [[3.0, -2.0, 5.0], [-4.0, 1.0, 2.0]]
    ms = variants["mesh_sphere"][2]
    keep = []
    for order in ("switch-move", "move-switch"):
        s = 10 if order == "switch-move" else 11
        m = (u32_tensor(b, [s]), to_device(b, mats[:1] if s == 10 else mats[1:]))
        c = (u32_tensor(b, [s]), u32_tensor(b, [2]))
        keep += [m, c]
        b.frame_begin()
        if order == "switch-move":
            b.switch_object_variants_device(c[1], c[0])
            b.set_object_transforms_device(m[1], m[0])
        else:
            b.set_object_transforms_device(m[1], m[0])
            b.switch_object_variants_device(c[1], c[0])
        b.frame_end()
        r, loc = b.readback_objects(s, 1)
        t = (mats[0] if s == 10 else mats[1]).reshape(4, 4)
        centre = (t[0, :3] * ms[0] + t[1, :3] * ms[1] + t[2, :3] * ms[2] + t[3, :3]).astype(np.float32)
        assert r["sphere_center"][0].tobytes() == centre.tobytes(), f"{order}: world sphere of the new mesh sphere"
        assert r["index_count"][0] == variants["index_count"][2]
        want_loc = t[3, :3] if order == "switch-move" else centre      # the move's translation / the add's sphere centre
        assert loc[0].tobytes() == want_loc.astype(np.float32).tobytes(), f"{order}: location"
    b.close()
