"""Materials that change — r3_update_materials, r3_update_materials_device, r3_readback_materials — against r3_set_materials of
world.py's full table (bit for bit) and the CPU oracle given the full tables (within the parity tolerance), plus the conservative
alpha-testing rule after the device form, the frame graph, the transparency-change recipe, growth and the calls' validation."""
import ctypes
import os

import numpy as np
import pytest

from harness import (ROOT, assert_same_frame, assert_same_ldr, check_declared_and_exported, expect_error, hdr_close, on_stream, settings,
                     to_device, unbound_backend)
from material_update_case import CUTOUT_VALUE, EMISSIVE, OPAQUE_VALUE, MaterialWorld, frames, updates
from rend3_b200.backend import CAMERA_VIEWPORT, load_cuda_backend
from rend3_b200.layouts import MATERIAL_DTYPE
E_INVALID, E_STATE = -1, -5
RES = (256, 160)


# ------------------------------------------------------------------ without a GPU
def test_library_exports_the_three_entry_points_with_the_headers_signatures():
    check_declared_and_exported(("int r3_update_materials(r3_ctx*, const uint32_t* indices_or_null, const r3_material* records, uint32_t n);",
                                 "int r3_update_materials_device(r3_ctx*, const uint32_t* d_indices_or_null, const r3_material* d_records, uint32_t n);",
                                 "int r3_readback_materials(r3_ctx*, r3_material* out, uint32_t first, uint32_t n);"),
                                (None, None, None, 0))


def test_material_record_layout():
    """GpuMaterialData: 208 bytes, the offsets r3_layouts.h asserts, a whole number of float4s (the scatter's lanes)."""
    layout = open(os.path.join(ROOT, "include", "r3_layouts.h")).read()
    assert 'R3_STATIC_ASSERT(sizeof(r3_material) == 208, "GpuMaterialData");' in layout
    assert MATERIAL_DTYPE.itemsize == 208 and MATERIAL_DTYPE.itemsize % 16 == 0
    offsets = {name: MATERIAL_DTYPE.fields[name][1] for name in MATERIAL_DTYPE.names}
    assert offsets["textures"] == 0 and offsets["uv_transform0"] == 48 and offsets["uv_transform1"] == 96
    assert offsets["albedo"] == 144 and offsets["emissive"] == 160 and offsets["roughness"] == 172
    assert offsets["alpha_cutout"] == 200 and offsets["flags"] == 204


@pytest.mark.parametrize("records,indices", [
    (np.zeros(4, np.uint8), None),                                     # bytes, not records
    (np.zeros((2, 2), MATERIAL_DTYPE), None),                          # 2-d records
    (np.zeros(3, MATERIAL_DTYPE), np.arange(2)),                       # lengths differ
    (np.zeros(3, MATERIAL_DTYPE), np.array([0.0, 1.0, 2.0])),          # float indices
    (np.zeros(2, MATERIAL_DTYPE), np.array([[0, 1]])),                 # 2-d indices
    (np.zeros(2, MATERIAL_DTYPE), np.array([-1, 3])),                  # negative index
    (np.zeros(1, MATERIAL_DTYPE), np.array([1 << 32], np.int64)),      # beyond uint32
], ids=["bytes", "2d-records", "length", "float-indices", "2d-indices", "negative", "wide"])
def test_host_wrapper_rejects_bad_shapes_and_dtypes_before_calling(records, indices):
    with pytest.raises(AssertionError, match="records|indices"):
        unbound_backend().update_materials(records, indices)


def test_device_wrapper_rejects_host_and_mistyped_tensors_before_calling():
    torch = pytest.importorskip("torch")
    b = unbound_backend()
    for records, indices in ((torch.zeros(2, 208, dtype=torch.uint8), None),          # a host tensor
                             (np.zeros(2, MATERIAL_DTYPE), None)):                     # a numpy array
        with pytest.raises(AssertionError):
            b.update_materials_device(records, indices)
    with pytest.raises(AssertionError):
        b.update_materials_device(None, None)                                         # no length


def test_world_update_material_marks_exactly_the_stale_indices():
    """Renderer.update_material: evaluate() names each updated index once, sorted, and nothing the next time; the table equals the
    records of the current materials; the per-slot keys change only when a material's transparency changes, and only for its
    objects."""
    from dataclasses import replace

    from rend3_b200.world import BLEND, CUTOUT

    w = MaterialWorld(n_objects=60)
    r = w.r
    ev0 = r.evaluate()
    assert len(r.evaluate().material_stale) == 0
    w.edit(EMISSIVE, emissive=(1.0, 0.0, 0.0))
    w.edit(OPAQUE_VALUE, roughness_factor=0.0)
    w.edit(EMISSIVE, emissive=(0.0, 1.0, 0.0))
    ev1 = r.evaluate()
    assert ev1.material_stale.dtype == np.uint32 and list(ev1.material_stale) == [OPAQUE_VALUE, EMISSIVE]
    assert ev1.material_buffer[EMISSIVE]["emissive"].tolist() == [0.0, 1.0, 0.0]
    for i, m in enumerate(r.materials):
        assert ev1.material_buffer[i].tobytes() == m.to_record().tobytes()
    assert np.array_equal(ev1.object_material_key, ev0.object_material_key), "no transparency change, no key change"
    assert len(r.evaluate().material_stale) == 0
    r.update_material(OPAQUE_VALUE, replace(r.materials[OPAQUE_VALUE], transparency=BLEND))
    r.update_material(CUTOUT_VALUE, replace(r.materials[CUTOUT_VALUE], alpha_cutout=0.2, transparency=CUTOUT))
    ev2 = r.evaluate()
    assert list(ev2.material_stale) == [OPAQUE_VALUE, CUTOUT_VALUE]
    uses = np.array([e is not None and int(e["rec"]["material_index"]) == OPAQUE_VALUE for e in r.objects[:len(ev2.object_buffer)]]
                    + [False] * (len(ev2.object_buffer) - len(r.objects)))
    assert uses.any()
    changed = np.flatnonzero(ev2.object_material_key != ev0.object_material_key)
    assert np.array_equal(changed, np.flatnonzero(uses)) and (ev2.object_material_key[changed] == BLEND).all()
    assert (ev2.object_back_to_front[changed] == 1).all() and (ev2.object_atomic[changed] == 0).all()


# ------------------------------------------------------------------ GPU
def device_updates(b, indices, records):
    """(indices as int32 or None, records as uint8 (n, 208)) CUDA tensors on the context's stream."""
    rec = to_device(b, np.ascontiguousarray(records).view(np.uint8).reshape(-1, 208))
    return (None if indices is None else to_device(b, np.asarray(indices, dtype=np.uint32).view(np.int32))), rec


def same_table(a, b):
    """Material tables equal field by field (the record's padding is not carried by numpy's structured copies)."""
    return len(a) == len(b) and all(a[f].tobytes() == b[f].tobytes() for f in a.dtype.names)


@pytest.mark.gpu
@pytest.mark.parametrize("samples,host", [(1, False), (4, False), (1, True)], ids=["x1", "x4", "x1-host-batching"])
def test_gpu_updates_equal_the_full_upload_and_the_oracle(monkeypatch, samples, host):
    """Seven frames of material edits (albedo, emissive, roughness 0, metallic, uv_transform0, texture slots one of them past the table,
    ALBEDO_ACTIVE off and on, alpha_cutout; the last frame edits every material, the dense form).  The device form in graph frames and
    the host form equal r3_set_materials of world.py's full table in every artefact, bit for bit; r3_readback_materials returns that
    table; with device batching the oracle, given the full table, agrees within the parity tolerance plus one rgba16f step (the
    blend routine's layers are stored in rgba16f)."""
    from oracle import load_oracle_backend
    from rend3_b200.routines import BaseRenderGraph

    if host:
        monkeypatch.setenv("R3_HOST_BATCHING", "1")
    else:
        monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    w = MaterialWorld()
    ev = w.r.evaluate()
    ctx = {"full": load_cuda_backend(0, parity_target=True), "host": load_cuda_backend(0, parity_target=True), "device": load_cuda_backend(0, parity_target=True)}
    graphs = {k: BaseRenderGraph(x) for k, x in ctx.items()}
    orc = None if host else load_oracle_backend()
    go = None if host else BaseRenderGraph(orc)
    for g in graphs.values():
        g.add_to_graph(ev, RES, samples, settings())
    keep = []
    for frame, (label, ev) in enumerate(frames(w)):
        what = f"frame {frame} ({label})"
        indices, records = updates(ev)
        assert len(records) > 0
        ctx["full"].set_materials(ev.material_buffer)
        graphs["full"].add_to_graph(ev, RES, samples, settings(), upload=False)
        graphs["host"].add_to_graph(ev, RES, samples, settings(), upload=False, material_updates=(indices, records))
        d = device_updates(ctx["device"], None if indices is None else indices[::-1].copy(),   # descending: order does not matter
                           records if indices is None else records[::-1].copy())
        keep.append(d)
        graphs["device"].add_to_graph(ev, RES, samples, settings(), upload=False, frame_graph=True, material_updates=d)
        for name in ("host", "device"):
            assert_same_frame(ctx[name], ctx["full"], ev, f"{what}, {name} form")
            assert_same_ldr(ctx[name], ctx["full"], f"{what}, {name} form")
            assert same_table(ctx[name].readback_materials(0, len(ev.material_buffer)), ev.material_buffer), f"{what}, {name} form: table"
        if orc is not None:
            go.add_to_graph(ev, RES, samples, settings())
            for cam in [CAMERA_VIEWPORT] + list(range(len(ev.shadows))):
                assert np.array_equal(ctx["device"].readback_visible(cam), orc.readback_visible(cam)), f"{what} camera {cam}: oracle"
            assert np.array_equal(ctx["device"].readback_depth().view(np.uint32), orc.readback_depth().view(np.uint32)), f"{what}: oracle depth"
            # the blend routine stores every layer in rgba16f (at 1x too), so a 1e-7 difference in a layer's shaded colour can land on
            # the other side of a half-precision rounding: the bound is TOL plus one rgba16f step, as for 4x samples
            hdr_close(ctx["device"].readback_hdr_f32(), orc.readback_hdr_f32(), f"{what}: oracle hdr", True)
    for x in ctx.values():
        x.close()
    if orc is not None:
        orc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("count", [1000, 33])
def test_gpu_dense_form_equals_sparse_form(count):
    """Arbitrary record bytes: the device form dense and sparse (permuted), the host form dense and sparse, and r3_set_materials of the
    expected table read back the same bytes; the table is the expected one after every step."""
    rng = np.random.default_rng(count)
    mat = lambda u8: np.ascontiguousarray(u8).view(MATERIAL_DTYPE).reshape(-1)       # raw rows as records, padding included
    table = rng.integers(0, 256, (count, 208), dtype=np.uint8)
    ctx = {k: load_cuda_backend(0, parity_target=False) for k in ("device-dense", "device-sparse", "host-dense", "host-sparse", "full")}
    for x in ctx.values():
        x.set_materials(mat(table))
    keep = []
    for step, k in enumerate((count, count // 2, 1)):
        new = rng.integers(0, 256, (k, 208), dtype=np.uint8)
        table = table.copy()
        table[:k] = new
        perm = rng.permutation(k)
        d = device_updates(ctx["device-dense"], None, mat(new))
        keep.append(d)
        ctx["device-dense"].update_materials_device(d[1], d[0])
        s = device_updates(ctx["device-sparse"], perm, mat(new[perm]))
        keep.append(s)
        ctx["device-sparse"].update_materials_device(s[1], s[0])
        ctx["host-dense"].update_materials(mat(new))
        ctx["host-sparse"].update_materials(mat(new[perm]), perm)
        ctx["full"].set_materials(mat(table))
        for name, x in ctx.items():
            got = x.readback_materials(0, count).view(np.uint8).reshape(count, 208)
            assert np.array_equal(got, table), f"step {step}: {name}"
    for x in ctx.values():
        x.close()


@pytest.mark.gpu
@pytest.mark.parametrize("samples", [1, 4])
def test_gpu_conservative_alpha_testing_is_safe(monkeypatch, samples):
    """A world where no material discards per fragment: device-form frames (which run the alpha-testing raster kernels) equal host-form
    frames bit for bit.  Then a device update that turns the cutout material into a per-fragment cutout (alpha from a texture) discards
    in the shadow and forward passes exactly where the full-upload path does — and the frame differs from the one before."""
    from rend3_b200.routines import BaseRenderGraph

    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    w = MaterialWorld(discard=False)
    ev = w.r.evaluate()
    host, dev = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True)
    gh, gd = BaseRenderGraph(host), BaseRenderGraph(dev)
    gh.add_to_graph(ev, RES, samples, settings())
    gd.add_to_graph(ev, RES, samples, settings())
    keep = []
    for frame, (label, ev) in enumerate(frames(w)):
        indices, records = updates(ev)
        gh.add_to_graph(ev, RES, samples, settings(), upload=False, material_updates=(indices, records))
        keep.append(device_updates(dev, indices, records))
        gd.add_to_graph(ev, RES, samples, settings(), upload=False, frame_graph=True, material_updates=keep[-1])
        assert_same_frame(dev, host, ev, f"frame {frame} ({label})")
        assert_same_ldr(dev, host, f"frame {frame} ({label})")
    sw, sh = ev.shadow_target_size
    before = (dev.readback_depth().tobytes(), dev.readback_shadow_atlas(sw, sh).tobytes())
    w.edit(CUTOUT_VALUE, albedo_texture=w.textures[1], albedo_value=None, alpha_cutout=0.5)
    ev = w.r.evaluate()
    assert list(ev.material_stale) == [CUTOUT_VALUE]
    host.set_materials(ev.material_buffer)                                            # the full-upload path, exact rule
    keep.append(device_updates(dev, *updates(ev)))
    gh.add_to_graph(ev, RES, samples, settings(), upload=False)
    gd.add_to_graph(ev, RES, samples, settings(), upload=False, frame_graph=True, material_updates=keep[-1])
    assert_same_frame(dev, host, ev, "per-fragment cutout")
    assert_same_ldr(dev, host, "per-fragment cutout")
    assert dev.readback_depth().tobytes() != before[0], "the per-fragment cutout changed nothing in the forward pass"
    assert dev.readback_shadow_atlas(sw, sh).tobytes() != before[1], "the per-fragment cutout changed nothing in the shadow pass"
    host.close(), dev.close()


@pytest.mark.gpu
def test_gpu_graph_frames_stay_one_launch(monkeypatch):
    """Recorded frames update materials from a torch tensor that a kernel on the context's stream rewrites every frame (an emissive
    pulse and an albedo fade).  No frame flushes early; the graphs are instantiated again at most once per frame parity, when the
    raster variant first changes; every frame equals a context fed the same records through r3_set_materials, bit for bit."""
    import torch

    from rend3_b200.routines import BaseRenderGraph

    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    w = MaterialWorld(discard=False, blend=False)
    ev = w.r.evaluate()
    graph_b, full = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True)
    gg, gf = BaseRenderGraph(graph_b), BaseRenderGraph(full)
    gg.add_to_graph(ev, RES, 1, settings())
    gf.add_to_graph(ev, RES, 1, settings())
    for _ in range(2):                                                                # both frame parities recorded once
        gg.add_to_graph(ev, RES, 1, settings(), upload=False, frame_graph=True)
        gf.add_to_graph(ev, RES, 1, settings(), upload=False)
    first = graph_b.frame_graph_stats()
    assert first["flushed"] == 0, first
    pulse = np.array([EMISSIVE, CUTOUT_VALUE, OPAQUE_VALUE], dtype=np.uint32)
    table = ev.material_buffer.copy()
    d_idx = to_device(graph_b, pulse.view(np.int32))
    d_rec = to_device(graph_b, table[pulse.astype(np.int64)].view(np.uint8).reshape(-1, 208)).view(torch.float32)   # (3, 52)
    for frame in range(6):
        t = 0.2 * (frame + 1)

        def rewrite():                                                                # the producer, on the context's stream
            d_rec[0, 40:43] = torch.tensor([t, 2.0 * t, 0.5], device="cuda")          # emissive @160
            d_rec[1, 39] = 0.9 - 0.1 * frame                                          # albedo alpha @156: a fade through the cutout
            d_rec[2, 43] = 0.1 * frame                                                # roughness @172
        on_stream(graph_b, rewrite)
        gg.add_to_graph(ev, RES, 1, settings(), upload=False, frame_graph=True, material_updates=(d_idx, d_rec))
        table[EMISSIVE]["emissive"] = (np.float32(t), np.float32(2.0) * np.float32(t), 0.5)
        table[CUTOUT_VALUE]["albedo"][3] = np.float32(0.9 - 0.1 * frame)
        table[OPAQUE_VALUE]["roughness"] = np.float32(0.1 * frame)
        full.set_materials(table)
        gf.add_to_graph(ev, RES, 1, settings(), upload=False)
        assert_same_frame(graph_b, full, ev, f"frame {frame}")
        assert_same_ldr(graph_b, full, f"frame {frame}")
    stats = graph_b.frame_graph_stats()
    print("frame graph stats", first, stats)
    assert stats["graphed"] == first["graphed"] + 6 and stats["flushed"] == 0, stats
    assert stats["instantiations"] - first["instantiations"] <= 2, (first, stats)
    graph_b.close(), full.close()


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host-form", "device-form"])
def test_gpu_transparency_change_by_the_documented_recipe(monkeypatch, device):
    """An opaque material becomes a blend material: r3_update_materials (or its device form) plus r3_update_object_sort_info of the
    slots that use it moves those objects into the blend routine; every artefact equals r3_set_materials + r3_set_object_sort_info."""
    from dataclasses import replace

    from rend3_b200.routines import BaseRenderGraph
    from rend3_b200.world import BLEND
    from world_update_scene import sort_flags

    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    w = MaterialWorld(blend=False)
    ev0 = w.r.evaluate()
    recipe, full = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True)
    gr, gf = BaseRenderGraph(recipe), BaseRenderGraph(full)
    gr.add_to_graph(ev0, RES, 1, settings())
    gf.add_to_graph(ev0, RES, 1, settings())
    _, regions = recipe.readback_batches(CAMERA_VIEWPORT)
    assert not (regions["material_key"] == 2).any()
    w.r.update_material(OPAQUE_VALUE, replace(w.r.materials[OPAQUE_VALUE], albedo_value=(0.9, 0.4, 0.1, 0.5), transparency=BLEND))
    ev = w.r.evaluate()
    slots = np.flatnonzero(ev.object_material_key != ev0.object_material_key).astype(np.uint32)
    assert len(slots) > 0
    indices, records = updates(ev)
    keep = None
    if device:
        keep = device_updates(recipe, indices, records)
        recipe.update_materials_device(keep[1], keep[0])
    else:
        recipe.update_materials(records, indices)
    s = slots.astype(np.int64)
    recipe.update_object_sort_info(slots, ev.object_material_key[s], sort_flags(ev)[s], ev.object_location[s])
    full.set_materials(ev.material_buffer)
    full.set_object_sort_info(ev.object_material_key, sort_flags(ev), ev.object_location)
    gr.add_to_graph(ev, RES, 1, settings(), upload=False)
    gf.add_to_graph(ev, RES, 1, settings(), upload=False)
    assert_same_frame(recipe, full, ev, "transparency change")
    assert_same_ldr(recipe, full, "transparency change")
    _, regions = recipe.readback_batches(CAMERA_VIEWPORT)
    assert (regions["material_key"] == 2).any(), "the objects did not move into the blend routine"
    recipe.close(), full.close()
    del keep


@pytest.mark.gpu
def test_gpu_validation_growth_and_dropped_indices(monkeypatch):
    """Host form: a repeated index, a null pointer, index 0xFFFFFFFF and the dense form past the count each return R3_E_INVALID and leave
    the table as it was.  Growth by the host form (zeros in between, contents kept), then r3_update_objects pointing objects at the new
    material, renders like a full upload.  Device form: R3_E_STATE on an empty table, R3_E_INVALID for the dense form past the count and
    a misaligned record pointer, and out-of-range indices are dropped."""
    from rend3_b200.routines import BaseRenderGraph
    from rend3_b200.world import PbrMaterial

    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    w = MaterialWorld(n_objects=300)
    ev = w.r.evaluate()
    n = len(ev.material_buffer)
    b = load_cuda_backend(0, parity_target=True)
    one = ev.material_buffer[:1].copy()
    keep = [device_updates(b, None, one)]
    expect_error(E_STATE, b.update_materials_device, keep[0][1], None)                # empty table
    b.update_materials(one[:0])                                                      # n == 0: R3_OK on an empty table
    ref = load_cuda_backend(0, parity_target=True)
    g, gref = BaseRenderGraph(b), BaseRenderGraph(ref)
    g.add_to_graph(ev, RES, 1, settings())
    gref.add_to_graph(ev, RES, 1, settings())
    table = b.readback_materials(0, n)
    assert same_table(table, ev.material_buffer)
    recs = ev.material_buffer[:2].copy()
    recs["emissive"] = 5.0
    expect_error(E_INVALID, b.update_materials, recs, np.array([1, 1]))                # one index named twice
    expect_error(E_INVALID, b.update_materials, recs, np.array([3, 0xFFFFFFFF]))       # index 0xFFFFFFFF (3 is not written either)
    expect_error(E_INVALID, b.update_materials, np.zeros(n + 1, MATERIAL_DTYPE))       # dense past the count
    idx = np.array([1, 2], np.uint32)
    assert b.lib.r3_update_materials(b.ctx, idx.ctypes.data_as(ctypes.c_void_p), None, ctypes.c_uint32(2)) == E_INVALID, "null records"
    assert same_table(b.readback_materials(0, n), table), "a rejected call wrote something"
    expect_error(E_INVALID, b.readback_materials, 0, n + 1)
    # growth: material n + 2, zeros at n and n + 1; objects moved onto it render like a full upload of the grown table
    grow = w.r.add_material(PbrMaterial(albedo_value=(1.0, 0.1, 0.6, 1.0), emissive=(0.3, 0.0, 0.3), roughness_factor=0.2))
    assert grow == n
    new = np.zeros(1, MATERIAL_DTYPE)
    new[0] = w.r.materials[grow].to_record()
    b.update_materials(new, np.array([n + 2]))
    grown = np.zeros(n + 3, MATERIAL_DTYPE)
    grown[:n], grown[n + 2] = ev.material_buffer, new[0]
    assert same_table(b.readback_materials(0, n + 3), grown)
    slots = np.flatnonzero(ev.object_live)[::7].astype(np.uint32)
    obj = ev.object_buffer[slots.astype(np.int64)].copy()
    obj["material_index"] = n + 2
    for x in (b, ref):
        x.update_objects(slots, obj)
    ref.set_materials(grown)
    g.add_to_graph(ev, RES, 1, settings(), upload=False)
    gref.add_to_graph(ev, RES, 1, settings(), upload=False)
    assert_same_frame(b, ref, ev, "grown table")
    assert_same_ldr(b, ref, "grown table")
    # device form: dense past the count, misaligned records, dropped indices
    d = device_updates(b, None, np.zeros(n + 4, MATERIAL_DTYPE))
    keep.append(d)
    expect_error(E_INVALID, b.update_materials_device, d[1], None)
    expect_error(E_INVALID, b.update_materials_device, d[1].data_ptr() + 4, None, 1)
    drop = np.array([1, n + 3, 4, 0xFFFFFFFF, n + 40], np.uint32)
    recs = np.zeros(len(drop), MATERIAL_DTYPE)
    recs["roughness"] = np.arange(len(drop), dtype=np.float32) + 0.5
    d = device_updates(b, drop, recs)
    keep.append(d)
    b.update_materials_device(d[1], d[0])
    got = b.readback_materials(0, n + 3)
    want = grown.copy()
    want[1], want[4] = recs[0], recs[2]
    assert same_table(got, want), "out-of-range indices were not dropped"
    b.close(), ref.close()
