"""Meshes that deform every frame — r3_set_deformable_meshes, r3_deform_meshes, r3_deform_meshes_device — against rule R15's numpy
restatement (tests/mesh_deform_reference.py) of rebuilding each mesh from the new positions and re-adding its objects: the mesh buffer,
the mesh spheres, the records with their sort locations, and whole frames against a context (and the oracle) fed the rebuilt world."""
import ctypes
import os

import numpy as np
import pytest

import mesh_deform_case as case
import mesh_deform_reference as ref
from harness import ROOT, assert_same_frame, check_declared_and_exported, expect_error, on_stream, to_device, unbound_backend
from mesh_deform_case import bits, canon, canon_records
from rend3_b200 import world
from rend3_b200.backend import load_cuda_backend
from rend3_b200.layouts import ATTR_ABSENT, DEFORM_NORMALS, DEFORM_TANGENTS, DEFORMABLE_MESH_DTYPE, OBJECT_DTYPE

f32 = np.float32
E_INVALID, E_STATE = -1, -5
RES = (256, 160)


# ------------------------------------------------------------------ without a GPU
def test_library_exports_the_entry_points_with_the_headers_signatures():
    decls = {
        "int r3_set_deformable_meshes(r3_ctx*, const r3_deformable_mesh* meshes, uint32_t n_meshes, const uint32_t* object_slots, "
        "const uint32_t* object_meshes, uint32_t n_objects);": (None, None, 0, None, None, 0),
        "int r3_deform_meshes(r3_ctx*, const float* positions, uint64_t n_floats);": (None, None, ctypes.c_uint64(0)),
        "int r3_deform_meshes_device(r3_ctx*, const float* d_positions, uint64_t n_floats);": (None, None, ctypes.c_uint64(0)),
        "int r3_readback_deformable_mesh_spheres(r3_ctx*, float* out , uint32_t first, uint32_t n);": (None, None, 0, 0),
    }
    check_declared_and_exported(decls, decls.get)


def test_deformable_mesh_layout_matches_c_header():
    import subprocess
    import tempfile

    src = "\n".join(["#include <stdio.h>", "#include <stddef.h>", f'#include "{ROOT}/include/r3_layouts.h"', "int main(void){",
                     'printf("size %zu\\n", sizeof(r3_deformable_mesh));',
                     'printf("flags_lh %u\\nflags_n %u\\nflags_t %u\\n", R3_DEFORM_LEFT_HANDED, R3_DEFORM_NORMALS, R3_DEFORM_TANGENTS);']
                    + [f'printf("{f} %zu\\n", offsetof(r3_deformable_mesh, {f}));' for f in DEFORMABLE_MESH_DTYPE.names] + ["return 0;}"])
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(c, "w").write(src)
        subprocess.run(["/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc", c, "-o", exe], check=True)
        out = dict(l.split() for l in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(out["size"]) == DEFORMABLE_MESH_DTYPE.itemsize == 32
    for f in DEFORMABLE_MESH_DTYPE.names:
        assert int(out[f]) == DEFORMABLE_MESH_DTYPE.fields[f][1], f
    from rend3_b200.layouts import DEFORM_LEFT_HANDED
    assert (int(out["flags_lh"]), int(out["flags_n"]), int(out["flags_t"])) == (DEFORM_LEFT_HANDED, DEFORM_NORMALS, DEFORM_TANGENTS)


FINITE_SPECS = [case.grid(11, 7), case.double_sided(case.grid(5, 4)), case.fan(512), case.grid(6, 9, uv=False)]


@pytest.mark.parametrize("spec", FINITE_SPECS, ids=["grid", "double-sided", "fan", "no-uv"])
@pytest.mark.parametrize("left", [True, False], ids=["left", "right"])
def test_restatement_equals_world_normals_and_tangents_on_finite_meshes(spec, left):
    """np.add.at in triangle order gives world.py's per-triangle loop bit for bit, wherever the sums stay finite"""
    pos = case.wave(spec.positions, 0.7)
    n_ref = world.calculate_normals(pos, spec.indices, left)
    n = ref.normals(pos, spec.indices, left)
    assert np.array_equal(bits(n), bits(n_ref))
    if spec.uv is not None:
        assert np.array_equal(bits(ref.tangents(pos, n, spec.uv, spec.indices)), bits(world.calculate_tangents(pos, n_ref, spec.uv, spec.indices)))


def test_restatement_equals_world_normals_with_repeated_corners():
    rng = np.random.default_rng(1)
    pos = (rng.standard_normal((1500, 3)) * 1e3).astype(f32)
    idx = rng.integers(0, 1500, size=(6000, 3)).astype(np.uint32)
    idx[:50, 1] = idx[:50, 0]
    assert np.array_equal(bits(ref.normals(pos, idx.reshape(-1), True)), bits(world.calculate_normals(pos, idx.reshape(-1), True)))


def test_parallel_bbox_equals_the_sequential_sse_fold_with_nan_and_signed_zero_everywhere():
    """R15's reduction against a literal _mm_max_ps / _mm_min_ps fold: one NaN, +0.0 and -0.0 ties and both at every position"""
    rng = np.random.default_rng(2)
    for n in (1, 2, 3, 7, 33):
        base = rng.choice(np.array([0.0, -0.0, 1.0, -1.0, 2.0], f32), (n, 3)).astype(f32)
        variants = [base]
        for at in range(n):
            for v in (np.nan, 0.0, -0.0, np.inf, -np.inf):
                p = base.copy()
                p[at] = f32(v)
                variants.append(p)
                q = p.copy()
                q[(at + 1) % n, 1] = np.nan
                variants.append(q)
        for p in variants:
            mx, mn = ref.bbox_r15(p)
            sx, sn = ref.bbox_sequential(p)
            assert np.array_equal(bits(mx), bits(sx)) and np.array_equal(bits(mn), bits(sn)), p


def test_mesh_sphere_agrees_with_bounding_sphere_from_mesh_where_that_is_exact():
    """world.bounding_sphere_from_mesh takes numpy's max / min: the same without NaN or ±0 ties; with a -0.0 / +0.0 tie numpy keeps the
    first and SSE the later, so the centre's sign of zero can differ there (world.py is left as it is)"""
    rng = np.random.default_rng(4)
    for n in (1, 5, 100, 4097):
        p = rng.standard_normal((n, 3)).astype(f32)
        c, r = world.bounding_sphere_from_mesh(p)
        s = ref.mesh_sphere(p)
        assert np.array_equal(bits(s[:3]), bits(c)) and bits(s[3:])[0] == bits([r])[0]
    # a ±0 tie: the fold takes the later vertex's zero, whichever order (numpy's choice there is its own)
    tie = np.array([[0.0, 1.0, 0.0], [-0.0, -1.0, -0.0]], f32)
    assert bits(ref.bbox_r15(tie)[0])[0] == bits([-0.0])[0] and bits(ref.bbox_r15(tie[::-1])[0])[0] == bits([0.0])[0]
    # a NaN before the last vertex: numpy's box is NaN, the fold starts over after it
    nan_first = np.array([[np.nan, 0, 0], [1, 0, 0], [2, 0, 0]], f32)
    assert np.isnan(world.bounding_sphere_from_mesh(nan_first)[0][0]) and ref.mesh_sphere(nan_first)[0] == f32(1.5)
    assert np.array_equal(bits(ref.mesh_sphere(np.zeros((0, 3), f32))), np.zeros(4, np.uint32))


def test_wrappers_reject_bad_arrays_before_calling():
    b = unbound_backend()
    with pytest.raises(AssertionError, match="meshes"):
        b.set_deformable_meshes(np.zeros(4, np.uint32))
    with pytest.raises(AssertionError, match="one mesh per slot"):
        b.set_deformable_meshes(np.zeros(1, DEFORMABLE_MESH_DTYPE), [0, 1], [0])
    for p in (np.zeros((4, 3), np.float64), np.zeros(12, f32), np.zeros((4, 4), f32)):
        with pytest.raises(AssertionError, match="positions"):
            b.deform_meshes(p)
    with pytest.raises(AssertionError, match="positions"):
        b.deform_meshes_device(np.zeros((4, 3), f32))
    with pytest.raises(AssertionError, match="n_floats"):
        b.deform_meshes_device(1 << 20)


# ------------------------------------------------------------------ on the GPU
def check_state(b, w, new_pos, what):
    """the mesh buffer, per-mesh spheres, records and sort locations against the restatement; returns the expected arrays"""
    ev = w.ev
    pos = np.concatenate(new_pos) if new_pos else np.zeros((0, 3), f32)
    words, objs, loc, ms, spheres = ref.deform_expected(ev.mesh_buffer, ev.object_buffer, ev.object_location, ev.object_mesh_sphere,
                                                        w.meshes, pos, w.slots, w.object_meshes)
    got = b.readback_mesh_buffer(len(ev.mesh_buffer))
    bad = np.flatnonzero(got != words)
    assert len(bad) == 0, f"{what}: {len(bad)} mesh words differ, first at {bad[:8]}"
    assert np.array_equal(canon(b.readback_deformable_mesh_spheres(0, len(w.meshes))), canon(spheres)), f"{what}: mesh spheres"
    recs, l = b.readback_objects(0, len(ev.object_buffer))
    ra, rb = np.frombuffer(canon_records(recs), np.uint8).reshape(len(recs), -1), np.frombuffer(canon_records(objs), np.uint8).reshape(len(objs), -1)
    differ = np.flatnonzero((ra != rb).any(1))
    assert len(differ) == 0, f"{what}: records of slots {differ[:8]} differ"
    assert np.array_equal(canon(l), canon(loc)), f"{what}: sort locations"
    return words, objs, loc, ms


def positions_for(w, t, specials=False):
    return [case.wave(p, t, seed=i, specials=specials and i % 2 == 0) for i, p in enumerate(w.rest)]


@pytest.mark.gpu
@pytest.mark.parametrize("handedness", [world.LEFT, world.RIGHT])
@pytest.mark.parametrize("form", ["host", "device"])
def test_gpu_edge_cases_equal_the_restatement(handedness, form):
    """every edge mesh in one set (left- and right-handed grids with uv0, a double-sided mesh, a 4096-triangle fan, repeated corners and
    unreferenced vertices, r = inf, authored normals, no uv0, an empty mesh) deformed twice, the second time with NaN, inf and ±0
    positions, bit for bit against R15"""
    w = case.build_world(case.edge_specs(), handedness=handedness)
    b = load_cuda_backend(0)
    case.upload(b, w.ev)
    b.set_deformable_meshes(w.meshes, w.slots, w.object_meshes)
    for k, specials in enumerate((False, True)):
        new_pos = positions_for(w, 0.5 + k, specials)
        pos = np.concatenate(new_pos)
        if form == "host":
            b.deform_meshes(pos)
        else:
            d = to_device(b, pos)
            b.deform_meshes_device(d)
            b.sync()
        check_state(b, w, new_pos, f"{handedness} {form} deform {k}")
        # the next deform starts from the rebuilt world: fold this one into the expectation's inputs
        words, objs, loc, ms = ref.deform_expected(w.ev.mesh_buffer, w.ev.object_buffer, w.ev.object_location, w.ev.object_mesh_sphere,
                                                   w.meshes, pos, w.slots, w.object_meshes)[:4]
        w.ev.mesh_buffer, w.ev.object_buffer, w.ev.object_location, w.ev.object_mesh_sphere = words, objs, loc, ms
    b.close()


@pytest.mark.gpu
def test_gpu_one_million_vertex_grid():
    """the ocean of tools/mesh_deform_cost.py: 1024 x 1024 vertices with uv0, 2 093 058 triangles, normals and tangents recomputed"""
    w = case.build_world([case.grid(1024, 1024, size=200.0)], objects_per_mesh=1, undeformed_objects=0, vectorised=True)
    b = load_cuda_backend(0)
    case.upload(b, w.ev)
    b.set_deformable_meshes(w.meshes, w.slots, w.object_meshes)
    new_pos = positions_for(w, 1.3)
    b.deform_meshes(np.concatenate(new_pos))
    check_state(b, w, new_pos, "1M grid")
    b.close()


@pytest.mark.gpu
def test_gpu_identity_deform_leaves_the_uploaded_world():
    """cube meshes built by MeshBuilder without normals, with and without uv0, deformed to their own positions: the mesh buffer and the
    records and locations stay bit-identical to the upload"""
    from rend3_b200.scenes import subdivided_cube_mesh

    specs = []
    for k, uv in ((1, False), (2, True), (3, False), (4, True)):
        m = subdivided_cube_mesh(k, with_uv=uv)
        specs.append(case.MeshSpec(m.attributes[0][1], m.indices, next((a for s, a in m.attributes if s == 3), None)))
    w = case.build_world(specs, objects_per_mesh=5)
    b = load_cuda_backend(0)
    case.upload(b, w.ev)
    b.set_deformable_meshes(w.meshes, w.slots, w.object_meshes)
    b.deform_meshes(np.concatenate(w.rest))
    assert np.array_equal(b.readback_mesh_buffer(len(w.ev.mesh_buffer)), w.ev.mesh_buffer)
    recs, loc = b.readback_objects(0, len(w.ev.object_buffer))
    assert recs.tobytes() == w.ev.object_buffer.tobytes()
    assert np.array_equal(bits(loc), bits(w.ev.object_location))
    b.close()


@pytest.mark.gpu
def test_gpu_deform_then_move_takes_the_moves_location_with_the_new_mesh_sphere():
    w = case.build_world([case.grid(9, 9), case.fan(64)], objects_per_mesh=3)
    b = load_cuda_backend(0)
    case.upload(b, w.ev)
    b.set_deformable_meshes(w.meshes, w.slots, w.object_meshes)
    new_pos = positions_for(w, 2.0)
    b.deform_meshes(np.concatenate(new_pos))
    words, objs, loc, ms = check_state(b, w, new_pos, "deform")
    mats = case.trs_matrices(np.array([[1, 2, 3], [-4, 0.5, 2]], f32), case.random_unit_quaternions(np.random.default_rng(9), 2),
                             np.array([[2.0], [0.5]], f32))
    moved = w.slots[[0, 4]]
    b.set_object_transforms(mats.reshape(-1, 16), moved)
    recs, l = b.readback_objects(0, len(objs))
    sph = ref.apply_transform(mats.reshape(-1, 16), ms[moved.astype(np.int64)])
    for i, s in enumerate(moved):
        assert recs[s]["transform"].tobytes() == mats[i].reshape(16).tobytes()
        assert np.array_equal(bits(np.r_[recs[s]["sphere_center"], recs[s]["sphere_radius"]]), bits(sph[i]))
        assert np.array_equal(bits(l[s]), bits(world.glam.transform_point3(mats[i], np.zeros(3, f32))))   # the move's location
    b.close()


def cloth_world(t=None):
    """a waving cloth (a 48 x 32 grid with uv0), a flag on a pole and a few of its copies, under the cube example's camera"""
    specs = [case.grid(48, 32, size=6.0), case.grid(16, 12, size=2.0)]
    if t is None:
        return case.build_world(specs, objects_per_mesh=2, extent=3.0), specs
    rest = [s.positions for s in specs]
    return case.rebuilt_world(specs, [case.wave(p, t) for p in rest], objects_per_mesh=2, extent=3.0), specs


@pytest.mark.gpu
def test_gpu_cloth_frames_in_one_graph_equal_the_rebuilt_world_and_the_oracle(monkeypatch):
    """Recorded frames deform the cloth from a device tensor rewritten on the context's stream: no early flush; every frame equals, bit
    for bit in every artefact, a context uploaded with the world rebuilt from the same positions, and the oracle's frame of that world in
    visible lists and depth (HDR within the parity tolerance); the host form gives the device form's bits"""
    import torch

    import oracle
    from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings

    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    settings = BaseRenderGraphSettings(clear_color=(0.1, 0.05, 0.1, 1.0))
    w, specs = cloth_world()
    dev, host = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True)
    gd, gh = BaseRenderGraph(dev), BaseRenderGraph(host)
    for b, g in ((dev, gd), (host, gh)):
        g.add_to_graph(w.ev, RES, 1, settings, movable_objects=True)
        b.set_deformable_meshes(w.meshes, w.slots, w.object_meshes)
    full = load_cuda_backend(0, parity_target=True)                  # fed the rebuilt world every frame, as the reference would be
    gf = BaseRenderGraph(full)
    gf.add_to_graph(w.ev, RES, 1, settings)
    rest = np.concatenate(w.rest)
    d_pos = to_device(dev, rest)
    for _ in range(2):
        gd.add_to_graph(w.ev, RES, 1, settings, upload=False, frame_graph=True, mesh_deforms=d_pos)
        gh.add_to_graph(w.ev, RES, 1, settings, upload=False, mesh_deforms=rest)
        gf.add_to_graph(w.ev, RES, 1, settings, upload=False)
    first = dev.frame_graph_stats()
    assert first["flushed"] == 0, first
    for frame in range(3):
        t = 0.4 * (frame + 1)
        new = [case.wave(p, t) for p in w.rest]
        on_stream(dev, lambda: d_pos.copy_(torch.from_numpy(np.concatenate(new)).to("cuda")))
        gd.add_to_graph(w.ev, RES, 1, settings, upload=False, frame_graph=True, mesh_deforms=d_pos)
        gh.add_to_graph(w.ev, RES, 1, settings, upload=False, mesh_deforms=np.concatenate(new))
        assert_same_frame(dev, host, w.ev, f"frame {frame}: device form against host form")
        assert dev.readback_hdr_f32().tobytes() == host.readback_hdr_f32().tobytes()
        rebuilt, _ = cloth_world(t)
        gf.add_to_graph(rebuilt.ev, RES, 1, settings)
        assert_same_frame(dev, full, rebuilt.ev, f"frame {frame}: deformed against rebuilt")
        assert dev.readback_hdr_f32().tobytes() == full.readback_hdr_f32().tobytes()
        orc = oracle.load_oracle_backend()
        BaseRenderGraph(orc).add_to_graph(rebuilt.ev, RES, 1, settings)
        assert np.array_equal(dev.readback_visible(0xFFFFFFFF), orc.readback_visible(0xFFFFFFFF)), f"frame {frame}: visible list"
        assert dev.readback_depth().tobytes() == orc.readback_depth().tobytes(), f"frame {frame}: depth"
        hd, ho = dev.readback_hdr_f32(), orc.readback_hdr_f32()
        err = np.abs(hd - ho) / np.maximum(1.0, np.abs(ho))
        assert err.max() <= 1e-4, f"frame {frame}: HDR differs from the oracle by {err.max()}"
    stats = dev.frame_graph_stats()
    print("frame graph stats", first, stats)
    assert stats["graphed"] == first["graphed"] + 3 and stats["flushed"] == 0, stats
    dev.close(), host.close(), full.close()


@pytest.mark.gpu
def test_gpu_validation_leaves_the_context_unchanged():
    import torch

    w = case.build_world([case.grid(6, 5), case.fan(16), case.grid(4, 4, uv=False)], objects_per_mesh=2)
    b = load_cuda_backend(0)
    case.upload(b, w.ev)
    n_v = sum(int(m["vertex_count"]) for m in w.meshes)
    pos = np.concatenate(positions_for(w, 0.3))
    expect_error(E_STATE, b.deform_meshes, pos)                                       # no set yet
    expect_error(E_STATE, b.readback_deformable_mesh_spheres, 0, 1)
    words0 = b.readback_mesh_buffer(len(w.ev.mesh_buffer))
    recs0 = b.readback_objects(0, len(w.ev.object_buffer))[0]

    def bad(mutate=None, slots=None, meshes_of=None):
        m = w.meshes.copy()
        if mutate:
            mutate(m)
        expect_error(E_INVALID, b.set_deformable_meshes, m, w.slots if slots is None else slots,
                     w.object_meshes if meshes_of is None else meshes_of)
    bad(lambda m: m["flags"].__setitem__(0, m["flags"][0] | 0x100))                           # unknown flag
    bad(lambda m: m["position_offset"].__setitem__(0, ATTR_ABSENT))                            # no positions
    bad(lambda m: m["position_offset"].__setitem__(0, m["position_offset"][0] + 2))            # not a multiple of 4
    bad(lambda m: m["normal_offset"].__setitem__(1, ATTR_ABSENT))                              # normals recomputed without a range
    bad(lambda m: m["uv0_offset"].__setitem__(0, ATTR_ABSENT))                                 # tangents without uv0
    bad(lambda m: m["flags"].__setitem__(2, m["flags"][2] | DEFORM_TANGENTS))                  # tangents without tangent / uv0 ranges
    bad(lambda m: m["index_count"].__setitem__(0, m["index_count"][0] - 1))                    # not a multiple of 3
    bad(lambda m: m["vertex_count"].__setitem__(1, 5))                                         # an index >= vertex_count
    bad(lambda m: m["first_index"].__setitem__(2, len(w.ev.mesh_buffer) - 3))                  # indices outside the buffer
    bad(lambda m: m["vertex_count"].__setitem__(2, len(w.ev.mesh_buffer)))                     # positions outside the buffer
    bad(lambda m: m["tangent_offset"].__setitem__(0, m["normal_offset"][0]))                   # two written ranges overlap
    bad(lambda m: m["position_offset"].__setitem__(1, m["first_index"][1] * 4))                # a write over indices
    bad(lambda m: m["position_offset"].__setitem__(0, m["uv0_offset"][0]))                     # a write over uv0
    bad(slots=w.slots[[0, 0, 1, 2, 3, 4]])                                                     # a slot named twice
    bad(slots=np.r_[w.slots[:-1], len(w.ev.object_buffer)].astype(np.uint32))                  # a slot past the slot count
    bad(meshes_of=np.r_[w.object_meshes[:-1], 3].astype(np.uint32))                            # an object mesh past the set
    bad(meshes_of=w.object_meshes[::-1].copy())                                                # records that draw other meshes
    assert np.array_equal(b.readback_mesh_buffer(len(w.ev.mesh_buffer)), words0)
    assert b.readback_objects(0, len(w.ev.object_buffer))[0].tobytes() == recs0.tobytes()
    expect_error(E_STATE, b.deform_meshes, pos)                                       # still no set

    b.set_deformable_meshes(w.meshes, w.slots, w.object_meshes)
    expect_error(E_INVALID, b.deform_meshes, pos[:-1])                                # wrong n_floats
    d = to_device(b, pos)
    expect_error(E_INVALID, b.deform_meshes_device, d.data_ptr() + 2, 3 * n_v)         # misaligned
    expect_error(E_INVALID, b.deform_meshes_device, d.data_ptr(), 3 * n_v + 3)         # wrong n_floats
    expect_error(E_INVALID, b.readback_deformable_mesh_spheres, 2, 2)                 # past the set
    b.set_object_mesh_spheres(w.ev.object_mesh_sphere[:int(w.slots.max())])            # spheres no longer cover a listed slot
    expect_error(E_STATE, b.deform_meshes, pos)
    expect_error(E_STATE, b.deform_meshes_device, d)
    b.set_object_mesh_spheres(w.ev.object_mesh_sphere)
    b.update_mesh_buffer(int(w.meshes["position_offset"][0]), w.ev.mesh_buffer[int(w.meshes["position_offset"][0]) // 4:][:6])   # not indices
    b.deform_meshes(pos)
    check_state(b, w, positions_for(w, 0.3), "after the rejected calls")
    fi = int(w.meshes["first_index"][1])
    b.update_mesh_buffer(4 * fi, w.ev.mesh_buffer[fi:fi + 3])                          # into an index range: the set is stale
    expect_error(E_STATE, b.deform_meshes, pos)
    b.set_deformable_meshes(w.meshes, w.slots, w.object_meshes)
    b.deform_meshes(pos)
    b.set_mesh_buffer(w.ev.mesh_buffer)                                               # a new buffer: the set is gone
    expect_error(E_STATE, b.deform_meshes_device, d)
    b.set_deformable_meshes(w.meshes, w.slots, w.object_meshes)
    dev_recs = torch.from_numpy(w.ev.object_buffer.view(np.uint8).copy()).cuda()
    b.set_objects_device(dev_recs.data_ptr(), len(w.ev.object_buffer))               # a borrowed object buffer
    expect_error(E_STATE, b.deform_meshes, pos)
    torch.cuda.synchronize()
    b.close()
