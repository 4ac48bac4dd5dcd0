"""Meshes whose topology changes every frame — r3_set_remeshable_meshes, r3_remesh_meshes, r3_remesh_meshes_device — against rule
R15's restatement (tests/mesh_deform_reference.py, through tests/remesh_case.py) of rebuilding each mesh from its new vertices and
indices and re-adding its objects: the mesh buffer, the mesh spheres, the records with their index counts and sort locations, the
invocation bound, and whole frames against a context fed the rebuilt world."""
import ctypes
import os

import numpy as np
import pytest

import remesh_case as case
from harness import ROOT, assert_same_frame, check_declared_and_exported, expect_error, on_stream, to_device, unbound_backend
from mesh_deform_case import bits, canon, canon_records
from rend3_b200 import world
from rend3_b200.backend import R3Error, load_cuda_backend
from rend3_b200.layouts import (ATTR_ABSENT, DEFORM_TANGENTS, REMESH_APPLIED, REMESH_INDEX_OUT_OF_RANGE, REMESH_NOT_TRIANGLES,
                                REMESH_OVER_CAPACITY, REMESHABLE_MESH_DTYPE)

f32 = np.float32
E_INVALID, E_STATE = -1, -5
RES = (256, 160)


# ------------------------------------------------------------------ without a GPU
def test_library_exports_the_entry_points_with_the_headers_signatures():
    u64 = ctypes.c_uint64(0)
    decls = {
        "int r3_set_remeshable_meshes(r3_ctx*, const r3_remeshable_mesh* meshes, uint32_t n_meshes, const uint32_t* object_slots, "
        "const uint32_t* object_meshes, uint32_t n_objects);": (None, None, 0, None, None, 0),
        "int r3_remesh_meshes(r3_ctx*, const uint32_t* counts, const float* positions, const uint32_t* indices, const float* normals, "
        "const float* tangents, const float* uv0, const uint32_t* color0, uint64_t n_vertices, uint64_t n_indices);":
            (None,) * 8 + (u64, u64),
        "int r3_remesh_meshes_device(r3_ctx*, const uint32_t* d_counts, const float* d_positions, const uint32_t* d_indices, "
        "const float* d_normals, const float* d_tangents, const float* d_uv0, const uint32_t* d_color0, uint64_t n_vertices, "
        "uint64_t n_indices);": (None,) * 8 + (u64, u64),
        "int r3_readback_remesh_status(r3_ctx*, uint32_t* status, uint32_t* counts_or_null , uint32_t first, uint32_t n);": (None, None, None, 0, 0),
        "int r3_debug_invocation_bound(r3_ctx*, uint64_t out[2]);": (None, None),
    }
    check_declared_and_exported(decls, decls.get)


def test_remeshable_mesh_layout_matches_c_header():
    import subprocess
    import tempfile

    src = "\n".join(["#include <stdio.h>", "#include <stddef.h>", f'#include "{ROOT}/include/r3_layouts.h"', "int main(void){",
                     'printf("size %zu\\n", sizeof(r3_remeshable_mesh));',
                     'printf("st %u %u %u %u\\n", R3_REMESH_APPLIED, R3_REMESH_OVER_CAPACITY, R3_REMESH_NOT_TRIANGLES, R3_REMESH_INDEX_OUT_OF_RANGE);']
                    + [f'printf("{f} %zu\\n", offsetof(r3_remeshable_mesh, {f}));' for f in REMESHABLE_MESH_DTYPE.names] + ["return 0;}"])
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(c, "w").write(src)
        subprocess.run(["/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc", c, "-o", exe], check=True)
        lines = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines()
    out = {l.split()[0]: l.split()[1:] for l in lines}
    assert int(out["size"][0]) == REMESHABLE_MESH_DTYPE.itemsize == 48
    for f in REMESHABLE_MESH_DTYPE.names:
        assert int(out[f][0]) == REMESHABLE_MESH_DTYPE.fields[f][1], f
    assert [int(x) for x in out["st"]] == [REMESH_APPLIED, REMESH_OVER_CAPACITY, REMESH_NOT_TRIANGLES, REMESH_INDEX_OUT_OF_RANGE]


def test_wrappers_reject_bad_arrays_before_calling():
    b = unbound_backend()
    with pytest.raises(AssertionError, match="meshes"):
        b.set_remeshable_meshes(np.zeros(4, np.uint32))
    with pytest.raises(AssertionError, match="one mesh per slot"):
        b.set_remeshable_meshes(np.zeros(1, REMESHABLE_MESH_DTYPE), [0, 1], [0])
    good = dict(counts=np.zeros((1, 2), np.uint32), positions=np.zeros((4, 3), f32), indices=np.zeros(6, np.uint32))
    for name, bad in (("counts", np.zeros((1, 3), np.uint32)), ("positions", np.zeros((4, 3), np.float64)), ("positions", np.zeros(12, f32)),
                      ("indices", np.zeros((2, 3), np.uint32)), ("indices", np.zeros(6, np.float32)), ("uv0", np.zeros((4, 3), f32)),
                      ("normals", np.zeros((5, 3), f32)), ("color0", np.zeros((4, 4), np.uint8))):
        with pytest.raises(AssertionError, match=name):
            b.remesh_meshes(**{**good, name: bad})
    with pytest.raises(AssertionError, match="indices"):
        b.remesh_meshes(good["counts"], good["positions"], None)
    with pytest.raises(AssertionError, match="counts"):
        b.remesh_meshes_device(**good)   # host arrays to the device form


@pytest.mark.parametrize("left", [True, False], ids=["left", "right"])
def test_restatement_equals_world_rebuild_on_finite_meshes(left):
    """the restatement's prefixes of every range, index_count and world spheres equal world.py's MeshBuilder::build + add_mesh + add of
    the new vertices and indices (a fresh world holding only the rebuilt meshes)"""
    hand = world.LEFT if left else world.RIGHT
    ks = case.kinds()
    w = case.build_world(ks, handedness=hand)
    ev = w.ev
    for step in (1, 3):
        frames = [case.frame_for(k, step) for k in ks]
        words, objs, loc, ms, spheres = case.expected(ev.mesh_buffer, ev.object_buffer, ev.object_location, ev.object_mesh_sphere, w, frames)
        for i, (k, f) in enumerate(zip(ks, frames)):
            if len(f.positions) == 0:
                continue
            kk = case.Kind(k.name, f, k.uv, k.color, k.own_normals, k.own_tangents)
            r = world.Renderer(hand, aspect_ratio=1.0)
            mid = case.add_capacity_mesh(r, kk, hand)
            m, rm = r.meshes[mid], w.records[i]
            for slot, off in ((0, "position_offset"), (1, "normal_offset"), (2, "tangent_offset"), (3, "uv0_offset"), (5, "color0_offset")):
                if slot not in m["ranges"]:
                    assert rm[off] == ATTR_ABSENT
                    continue
                a, n = int(m["ranges"][slot]) // 4, int(rm[off]) // 4
                size = {0: 3, 1: 3, 2: 3, 3: 2, 5: 1}[slot] * len(f.positions)
                assert np.array_equal(words[n:n + size], r.mesh_words[a:a + size]), f"{k.name} step {step}: attribute {slot}"
            fi = int(rm["first_index"])
            assert np.array_equal(words[fi:fi + len(f.indices)], f.indices)
            assert np.array_equal(bits(spheres[i][:3]), bits(m["center"])) and bits(spheres[i][3:])[0] == bits([m["radius"]])[0], k.name
            for s in w.slots[w.object_meshes == i]:
                assert objs[s]["index_count"] == len(f.indices)


# ------------------------------------------------------------------ on the GPU
def byte_copy(records):
    """a copy that keeps the bytes between the fields, which numpy's copy of a structured array need not"""
    return np.frombuffer(bytearray(np.ascontiguousarray(records).tobytes()), dtype=records.dtype)


class State:
    """the expected mesh buffer, records, locations and per-slot mesh spheres, folded forward remesh after remesh"""

    def __init__(self, w):
        ev = w.ev
        self.w, self.words, self.objs = w, np.array(ev.mesh_buffer), byte_copy(ev.object_buffer)
        self.loc, self.ms = np.array(ev.object_location, f32), np.array(ev.object_mesh_sphere, f32)
        self.spheres = np.zeros((len(w.records), 4), f32)
        self.counts = np.zeros((len(w.records), 2), np.uint32)

    def apply(self, frames, applied=None):
        self.words, self.objs, self.loc, self.ms, sph = case.expected(self.words, self.objs, self.loc, self.ms, self.w, frames, applied)
        idx = [i for i in range(len(frames)) if applied is None or applied[i]]
        self.spheres[idx] = sph
        for i in idx:
            self.counts[i] = (len(frames[i].positions), len(frames[i].indices))

    def check(self, b, what):
        got = b.readback_mesh_buffer(len(self.words))
        bad = np.flatnonzero(got != self.words)
        assert len(bad) == 0, f"{what}: {len(bad)} mesh words differ, first at {bad[:8]}"
        assert np.array_equal(canon(b.readback_deformable_mesh_spheres(0, len(self.spheres))), canon(self.spheres)), f"{what}: mesh spheres"
        recs, l = b.readback_objects(0, len(self.objs))
        ra = np.frombuffer(canon_records(recs), np.uint8).reshape(len(recs), -1)
        rb = np.frombuffer(canon_records(self.objs), np.uint8).reshape(len(recs), -1)
        differ = np.flatnonzero((ra != rb).any(1))
        assert len(differ) == 0, f"{what}: records of slots {differ[:8]} differ"
        assert np.array_equal(canon(l), canon(self.loc)), f"{what}: sort locations"
        assert np.array_equal(b.readback_remesh_status(0, len(self.counts))[1], self.counts), f"{what}: counts in force"


def remesh(b, form, s):
    if form == "host":
        b.remesh_meshes(**s)
        return

    b.remesh_meshes_device(**{k: to_device(b, v) for k, v in s.items()})
    b.sync()


@pytest.mark.gpu
@pytest.mark.parametrize("handedness", [world.LEFT, world.RIGHT])
@pytest.mark.parametrize("form", ["host", "device"])
def test_gpu_edge_cases_equal_the_restatement(handedness, form):
    """every kind in one set (grids kept by a mask, colour0 without uv0, the 4096-triangle fan, repeated corners with unreferenced
    vertices, supplied normals, supplied normals and tangents): counts at capacity, shrink, counts of 0, grow, and NaN / inf / ±0
    positions, bit for bit"""
    ks = case.kinds()
    w = case.build_world(ks, handedness=handedness)
    b = load_cuda_backend(0)
    case.upload(b, w.ev)
    b.set_remeshable_meshes(w.records, w.slots, w.object_meshes)
    st = State(w)
    for step, nan in ((0, False), (1, False), (2, False), (3, False), (0, True), (4, True)):
        frames = [case.frame_for(k, step, seed=i, nan=nan) for i, k in enumerate(ks)]
        remesh(b, form, case.streams(w, frames))
        st.apply(frames)
        st.check(b, f"{handedness} {form} step {step} nan {nan}")
        assert (b.readback_remesh_status(0, len(ks))[0] == REMESH_APPLIED).all()
    b.close()


@pytest.mark.gpu
def test_gpu_validation_leaves_failing_meshes_and_their_objects_as_they_were():
    """the device form: each reason leaves its mesh and objects bit-identical to the previous frame, reports its status and applies the
    others; the host form rejects the whole call and writes nothing"""
    ks = case.kinds()
    w = case.build_world(ks)
    b = load_cuda_backend(0)
    case.upload(b, w.ev)
    b.set_remeshable_meshes(w.records, w.slots, w.object_meshes)
    st = State(w)
    frames = [case.frame_for(k, 1, seed=i) for i, k in enumerate(ks)]
    remesh(b, "device", case.streams(w, frames))
    st.apply(frames)
    st.check(b, "first frame")
    nxt = [case.frame_for(k, 3, seed=i) for i, k in enumerate(ks)]
    s = case.streams(w, nxt)
    ib = np.r_[0, np.cumsum(w.records["index_capacity"].astype(np.int64))]
    s["counts"][0, 0] = w.records["vertex_capacity"][0] + 1                              # more vertices than capacity
    s["counts"][1, 1] = w.records["index_capacity"][1] + 3                               # more indices than capacity
    s["counts"][2, 1] -= 1                                                               # not triangles
    s["indices"][ib[3] + s["counts"][3, 1] - 1] = s["counts"][3, 0]                      # an index == vertex_count
    reasons = [REMESH_OVER_CAPACITY, REMESH_OVER_CAPACITY, REMESH_NOT_TRIANGLES, REMESH_INDEX_OUT_OF_RANGE, REMESH_APPLIED, REMESH_APPLIED]
    before = b.readback_mesh_buffer(len(st.words))
    expect_error(E_INVALID, b.remesh_meshes, **s)                                        # host form: all or nothing
    assert np.array_equal(b.readback_mesh_buffer(len(st.words)), before)
    st.check(b, "after the rejected host call")
    remesh(b, "device", s)
    applied = [r == REMESH_APPLIED for r in reasons]
    st.apply(nxt, applied)
    st.check(b, "after the device call with failing meshes")
    assert list(b.readback_remesh_status(0, len(ks))[0]) == reasons
    remesh(b, "device", case.streams(w, nxt))                                            # the failing meshes come back
    st.apply(nxt)
    st.check(b, "after a valid call")
    b.close()


@pytest.mark.gpu
def test_gpu_set_rejects_bad_input_and_the_state_rules_hold():
    import torch

    ks = case.kinds()[:3]
    w = case.build_world(ks, objects_per_mesh=2)
    b = load_cuda_backend(0)
    case.upload(b, w.ev)
    frames = [case.frame_for(k, 1) for k in ks]
    s = case.streams(w, frames)
    expect_error(E_STATE, b.remesh_meshes, **s)                                          # no set yet
    expect_error(E_STATE, b.readback_remesh_status, 0, 1)
    words0 = b.readback_mesh_buffer(len(w.ev.mesh_buffer))
    recs0 = b.readback_objects(0, len(w.ev.object_buffer))[0]
    bound0 = b.debug_invocation_bound()

    none = np.zeros(0, np.uint32)

    def bad(msg, mutate=None, slots=None, meshes_of=None, objects=True):
        """rejected with `msg`; the record checks run without listed objects, so that only the check named can reject them"""
        m = w.records.copy()
        if mutate:
            mutate(m)
        with pytest.raises(R3Error) as e:
            b.set_remeshable_meshes(m, (w.slots if slots is None else slots) if objects else none,
                                    (w.object_meshes if meshes_of is None else meshes_of) if objects else none)
        assert e.value.code == E_INVALID and msg in str(e.value), str(e.value)
    n_words = len(w.ev.mesh_buffer)
    bad("unknown flag bits", lambda m: m["flags"].__setitem__(0, m["flags"][0] | 0x100), objects=False)
    bad("without positions", lambda m: m["position_offset"].__setitem__(0, ATTR_ABSENT), objects=False)
    bad("not a multiple of 4", lambda m: m["color0_offset"].__setitem__(1, m["color0_offset"][1] + 2), objects=False)
    bad("normals recomputed without a normal range", lambda m: m["normal_offset"].__setitem__(1, ATTR_ABSENT), objects=False)
    bad("tangents recomputed without", lambda m: m["flags"].__setitem__(1, m["flags"][1] | DEFORM_TANGENTS), objects=False)
    bad("outside the mesh buffer", lambda m: m["vertex_capacity"].__setitem__(2, n_words), objects=False)
    bad("outside the mesh buffer", lambda m: m["index_capacity"].__setitem__(2, n_words), objects=False)
    bad("overlaps another range", lambda m: m["uv0_offset"].__setitem__(2, m["uv0_offset"][0]), objects=False)   # shared uv0: both write it
    bad("overlaps another range", lambda m: m["position_offset"].__setitem__(1, m["first_index"][1] * 4), objects=False)   # over indices
    bad("does not draw its mesh", lambda m: m["index_capacity"].__setitem__(0, m["index_capacity"][0] - 3))   # a record draws more
    bad("does not draw its mesh", lambda m: m["color0_offset"].__setitem__(1, ATTR_ABSENT))                    # a record's colour differs
    bad("named twice", slots=w.slots[[0, 0, 1, 2, 3, 4]])
    bad("slot beyond the object buffer", slots=np.r_[w.slots[:-1], len(w.ev.object_buffer)].astype(np.uint32))
    bad("object mesh out of range", meshes_of=np.r_[w.object_meshes[:-1], 3].astype(np.uint32))
    bad("does not draw its mesh", meshes_of=w.object_meshes[::-1].copy())                                     # records of other meshes
    assert np.array_equal(b.readback_mesh_buffer(len(w.ev.mesh_buffer)), words0)
    assert b.readback_objects(0, len(w.ev.object_buffer))[0].tobytes() == recs0.tobytes()
    assert b.debug_invocation_bound() == bound0
    expect_error(E_STATE, b.remesh_meshes, **s)                                           # still no set

    b.set_remeshable_meshes(w.records, w.slots, w.object_meshes)
    expect_error(E_STATE, b.deform_meshes, np.zeros((3, 3), f32))                         # the deform calls belong to the other set
    short = {k: (v if k in ("counts", "indices") else v[:-1]) for k, v in s.items()}
    expect_error(E_INVALID, b.remesh_meshes, **short)                                    # not the capacity
    expect_error(E_INVALID, b.remesh_meshes, **{k: v for k, v in s.items() if k != "uv0"})   # a stream some mesh reads
    st = State(w)
    b.update_mesh_buffer(4 * int(w.records["first_index"][0]), w.ev.mesh_buffer[int(w.records["first_index"][0]):][:6])
    b.remesh_meshes(**s)                                                                  # a write into the set's ranges changes nothing
    st.words[int(w.records["first_index"][0]):][:6] = w.ev.mesh_buffer[int(w.records["first_index"][0]):][:6]
    st.apply(frames)
    st.check(b, "after a mesh-buffer write")
    b.set_object_mesh_spheres(w.ev.object_mesh_sphere[:int(w.slots.max())])              # spheres no longer cover a listed slot
    expect_error(E_STATE, b.remesh_meshes, **s)
    b.set_object_mesh_spheres(w.ev.object_mesh_sphere)
    b.set_mesh_buffer(w.ev.mesh_buffer)                                                   # a new buffer: the set is gone
    expect_error(E_STATE, b.remesh_meshes, **s)
    b.set_remeshable_meshes(w.records, w.slots, w.object_meshes)
    from mesh_deform_case import deformable_records

    b.set_objects(w.ev.object_buffer)                                                     # the records of the uploaded world again
    b.set_deformable_meshes(deformable_records(w.renderer, [0, 1, 2]), w.slots, w.object_meshes)   # replaces the remesh set
    expect_error(E_STATE, b.remesh_meshes, **s)
    expect_error(E_STATE, b.readback_remesh_status, 0, 1)
    assert b.debug_invocation_bound() == bound0                                            # no floors
    b.set_remeshable_meshes(w.records, w.slots, w.object_meshes)
    dev_recs = torch.from_numpy(w.ev.object_buffer.view(np.uint8).copy()).cuda()
    b.set_objects_device(dev_recs.data_ptr(), len(w.ev.object_buffer))                   # a borrowed object buffer
    expect_error(E_STATE, b.remesh_meshes, **s)
    torch.cuda.synchronize()
    b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("how", ["update_objects", "set_objects"])
def test_gpu_deform_keeps_a_rewritten_index_count_within_the_bound(how):
    """A deformable set has no invocation floors, so a deform must leave index_count as the host last wrote it: after a listed slot's
    record is given fewer indices (r3_update_objects, or a reload with r3_set_objects that keeps the set), the recomputed bound counts
    the new value, and a deform must not write the set's larger one back under it"""
    import mesh_deform_case as dcase

    w = dcase.build_world([dcase.grid(9, 9), dcase.fan(64)], objects_per_mesh=2)
    b = load_cuda_backend(0)
    dcase.upload(b, w.ev)
    b.set_deformable_meshes(w.meshes, w.slots, w.object_meshes)
    recs = byte_copy(w.ev.object_buffer)
    s = int(w.slots[0])
    recs[s]["index_count"] = 3
    if how == "update_objects":
        b.update_objects(np.array([s], np.uint32), recs[s:s + 1])
    else:
        b.set_objects(recs)
    bound = b.debug_invocation_bound()
    assert bound == padded_bound(recs["index_count"])
    b.deform_meshes(np.concatenate([dcase.wave(p, 0.7) for p in w.rest]))
    got = b.readback_objects(0, len(recs))[0]
    assert np.array_equal(got["index_count"], recs["index_count"])
    assert b.debug_invocation_bound() == bound and padded_bound(got["index_count"])[0] <= bound[0]
    b.close()


def padded_bound(index_counts):
    t = (np.asarray(index_counts, np.int64) // 3 + 255) // 256 * 256
    return int(t.sum()), int(t.max()) if len(t) else 0


@pytest.mark.gpu
@pytest.mark.parametrize("host_batching", [False, True], ids=["device-batching", "host-batching"])
def test_gpu_invocation_bound_keeps_the_capacities_and_frames_equal_the_rebuilt_world(monkeypatch, host_batching):
    """after shrinking every mesh and an invalidating r3_update_objects of an unrelated slot, the bound the culling buffers are sized with
    still counts every listed slot's capacity; only then a frame grows every mesh back to capacity, and every artefact of it equals a
    context uploaded with the rebuilt world"""
    from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings

    if host_batching:
        monkeypatch.setenv("R3_HOST_BATCHING", "1")
    else:
        monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    settings = BaseRenderGraphSettings(clear_color=(0.1, 0.05, 0.1, 1.0))
    ks = case.kinds()
    w = case.build_world(ks, objects_per_mesh=3, extent=3.0)
    b, full = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True)
    g, gf = BaseRenderGraph(b), BaseRenderGraph(full)
    g.add_to_graph(w.ev, RES, 1, settings, movable_objects=True)
    gf.add_to_graph(w.ev, RES, 1, settings)
    b.set_remeshable_meshes(w.records, w.slots, w.object_meshes)
    st = State(w)
    small = [case.frame_for(k, 1, seed=i) for i, k in enumerate(ks)]
    g.add_to_graph(w.ev, RES, 1, settings, upload=False, remeshes=case.streams(w, small))
    st.apply(small)
    gf.add_to_graph(rebuilt_ev(w.ev, st), RES, 1, settings)   # the same frame history: the culling predicts from the previous frame
    unrelated = int(np.setdiff1d(np.arange(len(w.ev.object_buffer)), w.slots)[0])
    b.update_objects(np.array([unrelated], np.uint32), st.objs[unrelated:unrelated + 1])   # invalidates the cached bound
    caps = st.objs["index_count"].astype(np.int64)
    caps[w.slots] = w.records["index_capacity"][w.object_meshes]
    assert b.debug_invocation_bound() == padded_bound(caps)
    assert padded_bound(caps)[0] > padded_bound(st.objs["index_count"])[0]
    for step in (0, 3):
        frames = [case.frame_for(k, step, seed=i) for i, k in enumerate(ks)]
        g.add_to_graph(w.ev, RES, 1, settings, upload=False, remeshes=case.streams(w, frames))
        st.apply(frames)
        st.check(b, f"step {step}")
        rebuilt = rebuilt_ev(w.ev, st)
        gf.add_to_graph(rebuilt, RES, 1, settings)
        assert_same_frame_within_bound(b, full, rebuilt, f"step {step}: remeshed against rebuilt")
    b.close(), full.close()


class _RangesOnly:
    """an index list whose length assert_same_frame does not compare: only the draw calls' ranges of it are read"""

    def __init__(self, x):
        self.x = x

    def __len__(self):
        return 0

    def __getitem__(self, k):
        return self.x[k]


def assert_same_frame_within_bound(a, b, ev, what):
    """harness.assert_same_frame, with the index lists compared over the draw calls' ranges only and the culling results
    over their common length: the remeshed context sizes those buffers by the capacities (the invocation floors), the rebuilt one by
    the counts"""

    ra, rb = a.readback_indices, b.readback_indices
    ca, cb = a.readback_culling_results, b.readback_culling_results

    def common(x, y):
        n = min(len(x), len(y))
        return x[:n], y[:n]
    a.readback_indices = lambda cam, part: _RangesOnly(ra(cam, part))
    b.readback_indices = lambda cam, part: _RangesOnly(rb(cam, part))
    a.readback_culling_results = lambda cam, part: common(ca(cam, part), cb(cam, part))[0]
    b.readback_culling_results = lambda cam, part: common(ca(cam, part), cb(cam, part))[1]
    try:
        assert_same_frame(a, b, ev, what)
    finally:
        del a.readback_indices, b.readback_indices, a.readback_culling_results, b.readback_culling_results


def rebuilt_ev(ev, st):
    """the world the reference's rebuild leaves: the same evaluation with the rebuilt meshes' words, records, locations and spheres"""
    import copy

    out = copy.copy(ev)
    out.mesh_buffer, out.object_buffer, out.object_location, out.object_mesh_sphere = st.words.copy(), byte_copy(st.objs), st.loc.copy(), st.ms.copy()
    return out


@pytest.mark.gpu
def test_gpu_isosurface_frames_in_one_graph_equal_the_rebuilt_world(monkeypatch):
    """A torch-on-CUDA producer keeps the quads of a grid under a moving mask and compacts their vertices with cumsum, every frame, on
    the context's stream; recorded frames remesh from those tensors with no early flush, and every frame equals a context fed the
    rebuilt world in every artefact"""
    import torch

    from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings

    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    settings = BaseRenderGraphSettings(clear_color=(0.1, 0.05, 0.1, 1.0))
    nx, ny = 24, 16
    ks = [case.Kind("grid", case.masked_grid(nx, ny, np.ones((ny - 1, nx - 1), bool), size=4.0), True, False, False, False)]
    w = case.build_world(ks, objects_per_mesh=2, extent=2.0)
    dev, full = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True)
    gd, gf = BaseRenderGraph(dev), BaseRenderGraph(full)
    gd.add_to_graph(w.ev, RES, 1, settings, movable_objects=True)
    dev.set_remeshable_meshes(w.records, w.slots, w.object_meshes)
    gf.add_to_graph(w.ev, RES, 1, settings)
    grid = case.dcase.grid(nx, ny, size=4.0)
    surface = case.dcase.wave(grid.positions, 0.5)   # not flat: no depth ties between the overlapping objects
    cap_v, cap_i = int(w.records["vertex_capacity"][0]), int(w.records["index_capacity"][0])
    with torch.cuda.stream(torch.cuda.ExternalStream(dev.stream())):
        quads = torch.from_numpy(grid.indices.reshape(-1, 6).astype(np.int64)).cuda()
        qc = torch.from_numpy(grid.positions.reshape(-1, 3)[grid.indices.reshape(-1, 6)[:, 0]][:, [0, 2]].copy()).cuda()
        base = torch.from_numpy(surface).cuda()
        uv_all = torch.from_numpy(grid.uv).cuda()
        out = dict(counts=torch.zeros((1, 2), dtype=torch.int32, device="cuda"), positions=torch.zeros((cap_v, 3), device="cuda"),
                   indices=torch.zeros(cap_i, dtype=torch.int32, device="cuda"), uv0=torch.zeros((cap_v, 2), device="cuda"))

    def produce(t):
        """the mask: quads whose corner lies outside a circle moving with t; vertices used by a kept quad, compacted by cumsum"""
        keep = ((qc[:, 0] - 0.8 * np.cos(t)) ** 2 + (qc[:, 1] - 0.8 * np.sin(t)) ** 2) > 0.6
        kept = quads[keep].reshape(-1)
        used = torch.zeros(len(base), dtype=torch.bool, device="cuda")
        used[kept] = True
        remap = torch.cumsum(used.to(torch.int64), 0) - 1
        nv, ni = int(used.sum().item()), len(kept)
        out["positions"][:nv] = base[used]
        out["uv0"][:nv] = uv_all[used]
        out["indices"][:ni] = remap[kept].to(torch.int32)
        out["counts"][0, 0], out["counts"][0, 1] = nv, ni
        return keep.cpu().numpy()

    st = State(w)

    def step(t):
        """one recorded frame from the producer's tensors, and the rebuilt world's frame on `full` (the same frame history)"""
        keep = on_stream(dev, lambda: produce(t))
        gd.add_to_graph(w.ev, RES, 1, settings, upload=False, frame_graph=True, remeshes=out)
        f = case.masked_grid(nx, ny, keep.reshape(ny - 1, nx - 1), size=4.0)   # its indices and uv0; positions: the producer's surface
        f.positions = surface[np.isin(np.arange(len(grid.positions)), grid.indices.reshape(-1, 6)[keep].reshape(-1))]
        st.apply([f])
        rebuilt = rebuilt_ev(w.ev, st)
        gf.add_to_graph(rebuilt, RES, 1, settings)
        return rebuilt

    for t in (0.0, 0.0):   # two warm frames record the graph's topology
        step(t)
    first = dev.frame_graph_stats()
    assert first["flushed"] == 0, first
    for frame in range(3):
        rebuilt = step(0.9 * (frame + 1))
        st.check(dev, f"frame {frame}")
        assert_same_frame_within_bound(dev, full, rebuilt, f"frame {frame}: remeshed against rebuilt")
    stats = dev.frame_graph_stats()
    print("frame graph stats", first, stats)
    assert stats["graphed"] == first["graphed"] + 3 and stats["flushed"] == 0, stats
    dev.close(), full.close()
