"""Animated nodes' objects posed on the device (r3_set_object_animations, r3_set_object_pose_jobs, r3_pose_objects, r3_readback_objects)
against the float32 restatement of the object-transform half of rend3-anim's pose_animation_frame (tests/object_anim_reference.py,
rule R12), its float64 twin, the existing world path (world.Renderer.set_object_transform) and the oracle (oracle/r3_oracle_objanim.c);
then cull + bake, batching and whole frames after the pose."""
import os

import numpy as np
import pytest

import animation_case
import object_animation_case as cases
from anim_reference import same_bits
from harness import cull_and_batch_defined
from object_animation_case import run, sort_info
from object_anim_reference import node_matrix, pose_objects, posed_records, set_object_transform
from rend3_b200 import glam
from rend3_b200.animation import NodeChannels
from rend3_b200.backend import CAMERA_VIEWPORT, R3Error, load_cuda_backend
from rend3_b200.layouts import ANIM_NODE_CHANNEL_DTYPE, ANIM_NODE_CLIP_DTYPE, ANIM_NODE_DTYPE, OBJECT_POSE_TARGET_DTYPE

from oracle.objanim import load_objanim_oracle_backend

f32 = np.float32
E_INVALID, E_STATE = -1, -5
CASES = {"right": lambda: cases.case(seed=1), "left": lambda: cases.case(seed=2, left_handed=True),
         "many_jobs_left": lambda: cases.case(seed=3, left_handed=True, instances=300)}


def words(r):
    """The 30 defined words of each record (the last two are padding, which numpy's structured copies do not carry)."""
    return np.ascontiguousarray(r).view(np.uint32).reshape(len(r), 32)[:, :30]


def same_records(a, b):
    """Records equal word for word, a NaN matched by any NaN (the bits of a NaN are not part of rule R12)."""
    fa, fb = words(a), words(b)
    return same_bits(fa[:, :20].view(f32), fb[:, :20].view(f32)) and np.array_equal(fa[:, 20:], fb[:, 20:])


# ------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", list(CASES))
def test_oracle_equals_float32_restatement_bit_for_bit(name):
    data, jobs, targets, records, loc = CASES[name]()
    want_r, want_l = posed_records(data.library, jobs, targets, records, loc)
    orc = load_objanim_oracle_backend()
    got_r, got_l = run(orc, data, jobs, targets, records, loc)
    orc.close()
    assert same_records(got_r, want_r) and same_bits(got_l, want_l)
    posed = np.zeros(len(records), bool)
    posed[targets["slot"]] = True
    assert np.array_equal(words(got_r[~posed]), words(records[~posed])) and np.array_equal(got_l[~posed], loc[~posed]), "slots no target names are kept"
    assert np.isfinite(got_r["transform"][posed]).any()
    assert np.isnan(got_r["transform"][posed]).any() == bool(np.isnan(jobs["time"]).any()), "the NaN time must reach the records"
    assert np.array_equal(got_r["enabled"], records["enabled"]) and np.array_equal(got_r["attr_offset"], records["attr_offset"])


@pytest.mark.parametrize("left", [False, True])
def test_restatement_equals_world_set_object_transform(left):
    """On finite times the restatement's record and location equal world.Renderer.set_object_transform(h, matrix) + evaluate()."""
    from rend3_b200.scenes import subdivided_cube_mesh
    from rend3_b200.world import LEFT, RIGHT, Object, PbrMaterial, Renderer

    data, jobs, targets, _, _ = cases.case(seed=4, left_handed=left)
    jobs = jobs[np.isfinite(jobs["time"])]
    r = Renderer(LEFT if left else RIGHT)
    mesh = r.add_mesh(subdivided_cube_mesh(1))
    mat = r.add_material(PbrMaterial())
    center, radius = r.meshes[mesh]["center"], r.meshes[mesh]["radius"]
    n = int(targets["slot"].max()) + 1
    handles = [r.add_object(Object(mesh, mat, glam.identity())) for _ in range(n)]
    assert handles == list(range(n))
    tg = targets.copy()
    tg["mesh_sphere_center"], tg["mesh_sphere_radius"] = center, radius
    ev0 = r.evaluate()
    checked = 0
    for job in jobs:
        for k in range(int(job["target_count"])):
            t = tg[int(job["first_target"]) + k]
            m = node_matrix(data.library, job["clip"], t["channel"], job["time"])
            if not np.isfinite(m).all():
                continue
            r.set_object_transform(int(t["slot"]), m)
            ev = r.evaluate()
            one = np.array([job])
            one["first_target"], one["target_count"] = int(job["first_target"]) + k, 1
            want_r, want_l = posed_records(data.library, one, tg, ev0.object_buffer, ev0.object_location)
            s = int(t["slot"])
            assert np.array_equal(words(ev.object_buffer[s:s + 1]), words(want_r[s:s + 1])), f"slot {s}"
            assert ev.object_location[s].tobytes() == want_l[s].tobytes(), f"slot {s}: location"
            checked += 1
    assert checked > 50


def test_float32_restatement_is_close_to_float64():
    data, jobs, targets, records, loc = cases.case(seed=5)
    jobs = jobs[np.isfinite(jobs["time"])]
    a, b = pose_objects(data.library, jobs, targets, records, loc), pose_objects(data.library, jobs, targets, records, loc, np.float64)
    for x, y in zip(a, b):
        ok = np.isfinite(y)
        assert np.max(np.abs(x[ok] - y[ok]) / np.maximum(1.0, np.abs(y[ok]))) <= 1e-5


def _pose_one(data, t=0.5, center=(0.0, 0.0, 0.0), radius=1.0):
    """Poses slot 0 on the oracle, checks it against the restatement; returns (record, location)."""
    jobs, targets = data.pose_jobs([(0, t, 0)])
    records, loc = cases._records(2, np.random.default_rng(0)), np.full((2, 3), 7.0, f32)
    orc = load_objanim_oracle_backend()
    got_r, got_l = run(orc, data, jobs, targets, records, loc)
    orc.close()
    want_r, want_l = posed_records(data.library, jobs, targets, records, loc)
    assert same_records(got_r, want_r) and same_bits(got_l, want_l)
    return got_r[0], got_l[0]


def test_quirk_absent_tracks_take_the_bind_pose_not_identity():
    q = np.array([0.0, 0.6, 0.0, 0.8], f32)
    rec, _ = _pose_one(cases.single_node(NodeChannels(), (1.0, 2.0, 3.0), q, (2.0, 3.0, 4.0)))
    assert np.array_equal(rec["transform"], glam.from_scale_rotation_translation((2.0, 3.0, 4.0), q, (1.0, 2.0, 3.0)).reshape(16))
    only_t = NodeChannels(cases.key_track([0.0, 1.0], [[5.0, 5.0, 5.0], [5.0, 5.0, 5.0]]))
    rec, _ = _pose_one(cases.single_node(only_t, (1.0, 2.0, 3.0), q, (2.0, 3.0, 4.0)))
    assert np.array_equal(rec["transform"], glam.from_scale_rotation_translation((2.0, 3.0, 4.0), q, (5.0, 5.0, 5.0)).reshape(16)), \
        "rotation and scale fall back to the bind pose per property"


def test_quirk_left_handed_row_3_is_not_affine():
    rec, _ = _pose_one(cases.single_node(left_handed=True))
    row3 = rec["transform"].reshape(4, 4)[:, 3]
    assert row3.view(np.uint32).tolist() == [0, 0, 0x80000000, 0x3F800000], "(+0, +0, -0, 1): the affine bit test must fail"
    assert rec["transform"][10] == -1.0
    rec, _ = _pose_one(cases.single_node(left_handed=False))
    assert rec["transform"].reshape(4, 4)[:, 3].view(np.uint32).tolist() == [0, 0, 0, 0x3F800000]


def test_quirk_location_is_the_translation_not_the_sphere_centre():
    rec, loc = _pose_one(cases.single_node(translation=(1.0, 2.0, 3.0), center=(0.5, -1.0, 2.0)))
    assert np.array_equal(loc, [1.0, 2.0, 3.0])
    assert np.array_equal(rec["sphere_center"], [1.5, 1.0, 5.0]), "add_object would have stored this centre as the location"
    rec, loc = _pose_one(cases.single_node(scale=(np.inf, 1.0, 1.0)))   # a bind scale (a lerp of an infinite key would give NaN)
    assert np.isnan(loc).all() and np.isinf(rec["transform"][0]), "inf * 0 in transform_point3a: a NaN location"


def test_quirk_f32_max_ignores_a_nan_length_squared():
    m = glam.from_scale_rotation_translation((2.0, 3.0, 1.0), (0.0, 0.0, 0.0, 1.0), (0.0, 0.0, 0.0))
    m[0, 0] = np.nan
    _, _, r, _ = set_object_transform(m, (0, 0, 0), 1.0)
    assert r == 3.0, "f32::max(NaN, x) is x; Python's max would give NaN here"
    nan_scale = NodeChannels(None, None, cases.key_track([0.0], [[np.nan, 3.0, 2.0]]))
    rec, _ = _pose_one(cases.single_node(nan_scale))
    assert np.isnan(rec["transform"][0]) and rec["sphere_radius"] == 3.0


def _invalid_libraries(lib):
    nodes, clips, channels, keys, left = lib.arrays()
    out = []

    def variant(what, **kw):
        a = dict(nodes=nodes.copy(), clips=clips.copy(), channels=channels.copy(), keys=keys.copy())
        for k, fn in kw.items():
            fn(a[k])
        out.append((what, (a["nodes"], a["clips"], a["channels"], a["keys"], left)))

    tr = int(np.flatnonzero(channels["translation"]["times"] != 0xFFFFFFFF)[0])
    t0 = int(channels[tr]["translation"]["times"])
    variant("NaN duration", clips=lambda a: a["duration"].__setitem__(0, np.nan))
    variant("negative duration", clips=lambda a: a["duration"].__setitem__(0, -1.0))
    variant("clip channels out of range", clips=lambda a: a["first_channel"].__setitem__(0, len(channels)))
    variant("channel node out of range", channels=lambda a: a["node"].__setitem__(0, len(nodes)))
    variant("empty key channel", channels=lambda a: a["translation"]["count"].__setitem__(tr, 0))
    variant("fewer values than times", channels=lambda a: a["translation"]["value_count"].__setitem__(tr, a["translation"]["count"][tr] - 1))
    variant("key range outside the blob", channels=lambda a: a["translation"]["times"].__setitem__(tr, len(keys)))
    variant("NaN key time", keys=lambda a: a.__setitem__(t0, np.nan))
    variant("negative key time", keys=lambda a: a.__setitem__(t0, -1.0))
    return out


def _invalid_jobs(jobs, targets, n_slots):
    out = []
    j = jobs.copy(); j["clip"][0] = 99; out.append(("clip out of range", j, targets))
    j = jobs.copy(); j["first_target"][-1] = len(targets); out.append(("targets out of range", j, targets))
    t = targets.copy(); t["channel"][0] = 10_000; out.append(("target channel beyond the clip", jobs, t))
    t = targets.copy(); t["slot"][0] = n_slots; out.append(("slot beyond the object buffer", jobs, t))
    t = targets.copy(); t["slot"][1] = t["slot"][0]; out.append(("one slot named twice", jobs, t))
    j = jobs.copy(); j["first_target"][1], j["target_count"][1] = j["first_target"][0], j["target_count"][0]
    out.append(("two jobs over the same targets", j, targets))
    return out


def check_rejections(b):
    """Every invalid call is rejected; afterwards the records are those r3_set_objects gave, and the first pose runs the last accepted
    jobs against the last accepted library."""
    data, jobs, targets, records, loc = cases.case(seed=6)
    want_r, want_l = posed_records(data.library, jobs, targets, records, loc)
    b.set_objects(records)
    b.set_object_sort_info(*sort_info(len(records)), loc)
    data.upload(b)
    b.set_object_pose_jobs(jobs, targets)
    for what, arrays in _invalid_libraries(data.library):
        with pytest.raises(R3Error) as e:
            b.set_object_animations(*arrays)
        assert e.value.code == E_INVALID, what
    for what, jb, tg in _invalid_jobs(jobs, targets, len(records)):
        with pytest.raises(R3Error) as e:
            b.set_object_pose_jobs(jb, tg)
        assert e.value.code == E_INVALID, what
    with pytest.raises(R3Error) as e:
        b.readback_objects(len(records) - 1, 2)
    assert e.value.code == E_INVALID
    r, l = b.readback_objects(0, len(records))
    assert np.array_equal(words(r), words(records)) and np.array_equal(l, loc), "rejected calls must not touch the records"
    b.pose_objects()
    r, l = b.readback_objects(0, len(records))
    assert same_records(r, want_r) and same_bits(l, want_l), "the accepted library and jobs must survive the rejected calls"


def check_state_errors(b):
    data, jobs, targets, records, loc = cases.case(seed=7)
    for call in (b.pose_objects, lambda: b.set_object_pose_jobs(jobs, targets)):
        with pytest.raises(R3Error) as e:
            call()
        assert e.value.code == E_STATE
    data.upload(b)
    with pytest.raises(R3Error) as e:
        b.pose_objects()
    assert e.value.code == E_STATE, "no jobs yet"
    b.set_object_pose_jobs(jobs[:0], targets[:0])
    with pytest.raises(R3Error) as e:
        b.pose_objects()
    assert e.value.code == E_STATE, "pose_objects before set_objects"
    b.set_objects(records)
    b.set_object_pose_jobs(jobs, targets)
    b.pose_objects()
    data.upload(b)
    with pytest.raises(R3Error) as e:
        b.pose_objects()
    assert e.value.code == E_STATE, "a new library drops the jobs"


def test_oracle_rejects_every_invalid_input_and_keeps_its_state():
    for check in (check_rejections, check_state_errors):
        b = load_objanim_oracle_backend()
        check(b)
        b.close()


def test_object_animation_layouts_match_c_header():
    import subprocess
    import tempfile

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    probes = {"r3_anim_node": ANIM_NODE_DTYPE, "r3_anim_node_channel": ANIM_NODE_CHANNEL_DTYPE, "r3_anim_node_clip": ANIM_NODE_CLIP_DTYPE,
              "r3_object_pose_target": OBJECT_POSE_TARGET_DTYPE}
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{root}/include/rend3_b200.h"', "int main(void){"]
    for name, dt in probes.items():
        lines.append(f'printf("{name} %zu\\n", sizeof({name}));')
        lines += [f'printf("{name}.{f} %zu\\n", offsetof({name}, {f}));' for f in dt.names]
    lines.append('printf("lib.left_handed %zu\\n", offsetof(r3_anim_object_library, left_handed));')
    lines.append("return 0;}")
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(src, "w").write("\n".join(lines))
        subprocess.run(["/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc", src, "-o", exe], check=True)
        out = dict(l.split() for l in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines())
    for name, dt in probes.items():
        assert int(out[name]) == dt.itemsize, name
        for f in dt.names:
            assert int(out[f"{name}.{f}"]) == dt.fields[f][1], f"{name}.{f}"
    from rend3_b200.backend import _AnimObjectLibrary

    assert int(out["lib.left_handed"]) == _AnimObjectLibrary.left_handed.offset


# ------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_gpu_pose_equals_oracle_bit_for_bit(name):
    data, jobs, targets, records, loc = CASES[name]()
    orc = load_objanim_oracle_backend()
    want_r, want_l = run(orc, data, jobs, targets, records, loc)
    orc.close()
    b = load_cuda_backend(0)
    got_r, got_l = run(b, data, jobs, targets, records, loc)
    b.close()
    assert same_records(got_r, want_r) and same_bits(got_l, want_l)
    posed = np.zeros(len(records), bool)
    posed[targets["slot"]] = True
    assert np.array_equal(words(got_r[~posed]), words(records[~posed])), "slots no target names are unchanged"


@pytest.mark.gpu
def test_gpu_crowd_equals_oracle():
    data, jobs, targets, records, loc = cases.case(seed=8, instances=4096)
    assert len(jobs) == 4096 and len(targets) > 4 * 4096
    orc = load_objanim_oracle_backend()
    want = run(orc, data, jobs, targets, records, loc)
    orc.close()
    b = load_cuda_backend(0)
    got = run(b, data, jobs, targets, records, loc)
    b.close()
    assert same_records(got[0], want[0]) and same_bits(got[1], want[1])


@pytest.mark.gpu
def test_gpu_rejects_every_invalid_input_and_keeps_its_state():
    for check in (check_rejections, check_state_errors):
        b = load_cuda_backend(0)
        check(b)
        b.close()
    # a borrowed object buffer: every object-animation call but the readback is refused, and nothing changes
    import torch

    data, jobs, targets, records, loc = cases.case(seed=9)
    b = load_cuda_backend(0)
    b.set_objects(records)
    data.upload(b)
    b.set_object_pose_jobs(jobs, targets)
    dev = torch.from_numpy(records.view(np.uint8).copy()).cuda()
    torch.cuda.synchronize()
    b.set_objects_device(dev.data_ptr(), len(records))
    for call in (b.pose_objects, lambda: b.set_object_pose_jobs(jobs, targets), lambda: data.upload(b)):
        with pytest.raises(R3Error) as e:
            call()
        assert e.value.code == E_STATE
    b.sync()
    assert dev.cpu().numpy().tobytes() == records.view(np.uint8).tobytes()
    b.close()


# cull + bake and batching after the pose: a cloud of objects, some of them posed, seen by the cloud camera
def cloud_scene(left, seed=11, n=4000, blend_pair=False):
    from rend3_b200.animation import Animation, Node, ObjectAnimationData
    from rend3_b200.scenes import object_cloud_records

    rec = object_cloud_records(n, seed=seed, extent=60.0)
    rng = np.random.default_rng(seed)
    key = rng.integers(0, 3, n).astype(np.uint64)
    flags = (1 | 2 * rng.integers(0, 2, n) | 4 * (key == 2)).astype(np.uint8)
    nodes, channels = [], {}
    posed = rng.choice(n, 300, replace=False)
    for i, s in enumerate(posed):
        t = rec["transform"][s].reshape(4, 4)[3, :3]
        c = rec["sphere_center"][s] - t
        nodes.append(Node(None, t, cases._unit_quat(rng), rng.uniform(0.5, 1.5, 3).astype(f32), [(int(s), c.astype(f32), f32(rec["sphere_radius"][s]))]))
        if i % 4 != 3:
            channels[i] = NodeChannels(cases.key_track([0.0, 1.0], [t, t + rng.uniform(-8, 8, 3).astype(f32)]),
                                       cases.key_track([0.0, 1.0], [cases._unit_quat(rng), cases._unit_quat(rng)]) if i % 2 else None,
                                       cases.key_track([0.0, 0.5, 1.0], rng.uniform(0.3, 2.0, (3, 3))) if i % 3 else None)
    if blend_pair:   # two blend objects sorted back to front, which swap places along the view axis between t = 0 and t = 1
        for i, (z0, z1) in enumerate(((0.0, 20.0), (10.0, 5.0))):
            s = int(posed[i])
            key[s], flags[s] = 2, 1 | 4
            channels[i] = NodeChannels(cases.key_track([0.0, 1.0], [[0.0, 0.0, z0], [0.0, 0.0, z1]]))
    data = ObjectAnimationData(nodes, [Animation(channels, 1.0)], left)
    return rec, key, flags, rec["sphere_center"].copy(), data


@pytest.mark.gpu
@pytest.mark.parametrize("left", [False, True], ids=["right", "left"])
def test_gpu_cull_bake_after_pose_equals_oracle_and_host_posed_upload(monkeypatch, left):
    """Visible list and every MV / MVP word after the pose == the oracle's == the same world posed on the host and uploaded through
    r3_update_objects + r3_update_object_sort_info.  Left-handed poses have row 3 (+0, +0, -0, 1): rows_w is read."""
    monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    rec, key, flags, loc, data = cloud_scene(left)
    n = len(rec)
    out = {}
    for t in (0.0, 0.37, 1.0):
        jobs, targets = data.pose_jobs([(0, t, 0)])
        want_r, want_l = posed_records(data.library, jobs, targets, rec, loc)
        slots = np.sort(targets["slot"])
        for name, b in (("cuda", load_cuda_backend(0)), ("oracle", load_objanim_oracle_backend()), ("host", load_cuda_backend(0))):
            b.set_objects(rec)
            b.set_object_sort_info(key, flags, loc)
            if name == "host":
                b.update_objects(slots, want_r[slots])
                b.update_object_sort_info(slots, key[slots], flags[slots], want_l[slots])
            else:
                data.upload(b)
                b.set_object_pose_jobs(jobs, targets)
                b.pose_objects()
            out[name] = cull_and_batch_defined(b, n)
            b.close()
        assert out["cuda"][:2] == out["oracle"][:2], f"t={t}: visible list / MV / MVP differ from the oracle"
        assert out["cuda"] == out["host"], f"t={t}: differs from the host-posed upload"
        assert len(out["cuda"][0]) > 0
    if left:
        assert (want_r["transform"][slots][:, 11].view(np.uint32) == 0x80000000).sum() > 100


@pytest.mark.gpu
@pytest.mark.parametrize("host", [False, True], ids=["device_batching", "host_batching"])
def test_gpu_batching_sorts_by_posed_locations(monkeypatch, host):
    """Batch records == the oracle's on both batching paths, over two poses in which two back-to-front blend objects swap order; the
    host path sorts by the posed locations it takes from the device with the visible list."""
    if host:
        monkeypatch.setenv("R3_HOST_BATCHING", "1")
    else:
        monkeypatch.delenv("R3_HOST_BATCHING", raising=False)
    rec, key, flags, loc, data = cloud_scene(True, blend_pair=True)
    n = len(rec)
    b, orc = load_cuda_backend(0), load_objanim_oracle_backend()
    for x in (b, orc):
        x.set_objects(rec)
        x.set_object_sort_info(key, flags, loc)
        data.upload(x)
    orders = []
    vp = (0.0, 0.0, -30.0)
    pair_slots = {int(data.nodes[0].objects[0][0]), int(data.nodes[1].objects[0][0])}
    for t in (0.0, 1.0):
        for x in (b, orc):
            x.set_object_pose_jobs(*data.pose_jobs([(0, t, 0)]))
            x.pose_objects()
        got, want = cull_and_batch_defined(b, n, vp), cull_and_batch_defined(orc, n, vp)
        assert got == want, f"t={t}: batches differ from the oracle"
        assert b.batching_info(CAMERA_VIEWPORT)["path"] == ("host" if host else "device")
        bt, _ = b.readback_batches(CAMERA_VIEWPORT)
        ids = [int(i) for bb in bt for i in bb["object_culling_information"]["object_id"][:int(bb["total_objects"])]]
        orders.append([s for s in ids if s in pair_slots])
    assert len(orders[0]) == 2 and orders[0] == orders[1][::-1], f"the blend pair must swap places: {orders}"
    b.close(), orc.close()


@pytest.mark.gpu
def test_gpu_posed_frames_stay_one_graph():
    """Six frames through add_to_graph(posed_objects=True, posed_skinning=True) with the frame graph on and the time changing per frame:
    no early flush, graph == eager bit for bit, the oracle's shading within 1e-4.  Between frames 2 and 3 the graphed context gets an
    r3_update_objects of the posed slots with their stale add-time records, and still renders the posed frame."""
    from rend3_b200.animation import Animation, Node, ObjectAnimationData
    from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings

    ev, rec, skel = animation_case._posed_cube_world()
    rng = np.random.default_rng(3)
    slots = rng.choice(len(ev.object_buffer), 40, replace=False)
    nodes, channels = [], {}
    for i, s in enumerate(slots):
        t = ev.object_buffer["transform"][s].reshape(4, 4)[3, :3]
        nodes.append(Node(None, t, cases._unit_quat(rng), (0.7, 0.7, 0.7), [(int(s), np.zeros(3, f32), f32(1.8))]))
        channels[i] = NodeChannels(cases.key_track([0.0, 2.0], [t, t + rng.uniform(-1, 1, 3).astype(f32)]),
                                   cases.key_track([0.0, 1.0, 2.0], [cases._unit_quat(rng) for _ in range(3)]) if i % 2 else None)
    data = ObjectAnimationData(nodes, [Animation(channels, 2.0)], left_handed=True)
    settings = BaseRenderGraphSettings(clear_color=(0.1, 0.05, 0.1, 1.0))
    graph_b, eager_b, orc = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True), load_objanim_oracle_backend()
    runs = [(graph_b, True), (eager_b, False), (orc, False)]
    graphs = {id(b): BaseRenderGraph(b) for b, _ in runs}
    for b, _ in runs:
        graphs[id(b)].upload_world(ev)
        b.set_animations(*skel.library.arrays())
        b.set_skeletons(rec, np.zeros((4, 16), f32))
        b.set_pose_jobs(*skel.pose_jobs([(0, 0.0, {0: [(0, 4)]})]))
        data.upload(b)
        b.set_object_pose_jobs(*data.pose_jobs([(0, 0.0, 0)]))
        graphs[id(b)].add_to_graph(ev, (256, 144), 1, settings, upload=False, posed_skinning=True, posed_objects=True, frame_graph=False)
    for frame, t in enumerate([0.0, 0.3, 0.7, 1.1, 1.6, 2.5]):
        out = []
        flushed = graph_b.frame_graph_stats()["flushed"]
        for b, fg in runs:
            b.set_pose_jobs(*skel.pose_jobs([(0, t, {0: [(0, 4)]})]))
            b.set_object_pose_jobs(*data.pose_jobs([(0, t, 0)]))
            if frame == 3 and b is graph_b:   # stale add-time records over the posed slots: the next pose overwrites them
                b.update_objects(slots.astype(np.uint32), ev.object_buffer[slots])
            graphs[id(b)].add_to_graph(ev, (256, 144), 1, settings, upload=False, posed_skinning=True, posed_objects=True, frame_graph=fg)
            out.append((b.readback_hdr_f32().copy(), b.readback_objects(0, len(ev.object_buffer))))
        assert graph_b.frame_graph_stats()["flushed"] == flushed, f"frame {frame} flushed early"
        (hg, (rg, lg)), (he, (re_, le)), (ho, (ro, lo)) = out
        assert np.array_equal(hg.view(np.uint32), he.view(np.uint32)) and np.array_equal(words(rg), words(re_)) and np.array_equal(lg, le), \
            f"frame {frame}: graph != eager"
        assert same_records(rg, ro) and same_bits(lg, lo), f"frame {frame}: posed records differ from the oracle"
        assert not np.array_equal(rg[slots]["transform"], ev.object_buffer[slots]["transform"])
        err = np.abs(hg - ho) / np.maximum(1.0, np.abs(ho))
        assert err.max() <= 1e-4, f"frame {frame}: shading differs from the oracle by {err.max()}"
    stats = graph_b.frame_graph_stats()
    assert stats["graphed"] == 6 and stats["flushed"] == 0, stats
    for b, _ in runs:
        b.close()
