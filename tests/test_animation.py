"""Skeletal animation posed on the device (r3_set_animations, r3_set_skeletons, r3_set_pose_jobs, r3_pose_skeletons, r3_skin_posed,
r3_readback_joint_matrices) against the float32 restatement of rend3-anim's pose_animation_frame (tests/anim_reference.py, rule R12),
its float64 twin, and the oracle (oracle/r3_oracle_anim.c)."""
import numpy as np
import pytest

import animation_case as cases
from anim_reference import pose as pose_f32, pose_f64, same_bits
from rend3_b200 import glam
from rend3_b200.animation import Animation, AnimationData, Node, NodeChannels, Skin, Track
from rend3_b200.backend import R3Error
from rend3_b200.layouts import (ANIM_CHANNEL_DTYPE, ANIM_CLIP_DTYPE, ANIM_JOINT_DTYPE, ANIM_SKIN_DTYPE, POSE_JOB_DTYPE, POSE_TARGET_DTYPE,
                                SKINNING_INPUT_DTYPE)

from oracle.anim import load_anim_oracle_backend

f32 = np.float32
E_INVALID, E_STATE = -1, -5
NO_SKELETONS = np.zeros(0, dtype=SKINNING_INPUT_DTYPE)
CASE_IDS = [f"{s}{n}" for s, n in cases.SHAPES]


def run(backend, library, jobs, targets, buf, inputs=NO_SKELETONS):
    backend.set_animations(*library.arrays())
    backend.set_skeletons(inputs, buf)
    backend.set_pose_jobs(jobs, targets)
    backend.pose_skeletons()
    return backend.readback_joint_matrices(0, len(buf))


# ------------------------------------------------------------------ CPU: the oracle against the restatements
@pytest.mark.parametrize("shape,n", cases.SHAPES, ids=CASE_IDS)
def test_oracle_equals_float32_restatement_bit_for_bit(shape, n):
    library, jobs, targets, buf = cases.case(shape, n, seed=n)
    want = pose_f32(library, jobs, targets, buf)
    orc = load_anim_oracle_backend()
    got = run(orc, library, jobs, targets, buf)
    orc.close()
    assert same_bits(got, want), f"{shape}{n}: {np.count_nonzero(got.view(np.uint32) != want.view(np.uint32))} words differ"
    assert np.array_equal(got[-3:], buf[-3:]), "matrices no job targets are kept"
    assert np.isnan(got).any() and np.isfinite(got).any(), "the NaN time must reach the matrices, the others must not"


LAYOUT_CASES = {
    "shared_joint_range": lambda: cases.overlap_case(seed=1),
    "shared_joint_range_smaller_skin_only": lambda: cases.overlap_case(seed=2, small_only=True),
    "shared_memory_and_spill_in_one_launch": lambda: cases.mixed_case(seed=3),
}


@pytest.mark.parametrize("name", list(LAYOUT_CASES))
def test_oracle_equals_float32_restatement_on_shared_and_mixed_skins(name):
    """Skins that share joint records, and one launch mixing skins of <= 512 joints with a larger one."""
    library, jobs, targets, buf = LAYOUT_CASES[name]()
    want = pose_f32(library, jobs, targets, buf)
    orc = load_anim_oracle_backend()
    got = run(orc, library, jobs, targets, buf)
    orc.close()
    assert same_bits(got, want)
    assert np.isfinite(got[:-1]).any() and np.array_equal(got[-1], buf[-1])


@pytest.mark.parametrize("shape,n", [("chain", 200), ("humanoid", 65), ("random", 33)])
def test_float32_restatement_is_close_to_float64(shape, n):
    """On finite times and moderately deep skins the f32 path is within rounding of the f64 one: 2e-4 relative to the matrix scale
    per level of depth (200-level chains of scales in [0.5, 1.5] multiply the error; their entries stay bounded only relatively)."""
    library, jobs, targets, buf = cases.case(shape, n, seed=n)
    keep = np.isfinite(jobs["time"])
    jobs = jobs[keep]
    a, b = pose_f32(library, jobs, targets, buf), pose_f64(library, jobs, targets, buf)
    ok = np.isfinite(b).all(axis=1)
    depth = n if shape == "chain" else 12
    scale = np.maximum(1.0, np.abs(b[ok]).max(axis=1, keepdims=True))
    assert np.max(np.abs(a[ok] - b[ok]) / scale) <= 2e-4 * depth


def _one_joint(parent_not_joint, translation=(0.0, 0.0, 0.0), animated=True, inv_bind=None, track=None):
    nodes = [Node(None), Node(0 if parent_not_joint else None, translation, (0.0, 0.0, 0.0, 1.0), (1.0, 1.0, 1.0))]
    ib = glam.identity().reshape(1, 16) if inv_bind is None else inv_bind.reshape(1, 16)
    ch = {1: track or NodeChannels(Track(np.array([0.0, 1.0], f32), np.array([translation, translation], f32)))} if animated else {}
    data = AnimationData(nodes, [Skin([1], ib)], [Animation(ch, 1.0)])
    return data


def _pose_one(data, t=0.5):
    jobs, targets = data.pose_jobs([(0, t, {0: [(0, 1)]})])
    buf = np.zeros((1, 16), f32)
    orc = load_anim_oracle_backend()
    got = run(orc, data.library, jobs, targets, buf)
    orc.close()
    assert same_bits(got, pose_f32(data.library, jobs, targets, buf))
    return got[0]


def test_quirk_unanimated_joint_is_identity_not_bind_pose():
    data = _one_joint(False, translation=(3.0, 4.0, 5.0), animated=False)
    assert np.array_equal(_pose_one(data), glam.identity().reshape(16)), "a joint without a channel gets IDENTITY (lib.rs:219)"


def test_quirk_identity_times_local_turns_negative_zero_positive():
    """global = IDENTITY * local for a joint whose parent node is not a joint: the -0.0 x entry of the translation column becomes +0.0
    (1 * -0.0 + 0 * 1 + ...), where a root joint keeps local's -0.0.  The translation is the bind pose's (a lerp would already give +0.0:
    -0.0 + (+0.0 * s)); an inverse bind with -0.0 in its last column carries the sign out."""
    ib = glam.identity()
    ib[3, :3] = -0.0
    rot = NodeChannels(None, Track(np.array([0.0, 1.0], f32), np.array([[0, 0, 0, 1], [0, 0, 0, 1]], f32)))
    root = _pose_one(_one_joint(False, (-0.0, 1.0, 2.0), inv_bind=ib, track=rot))
    under = _pose_one(_one_joint(True, (-0.0, 1.0, 2.0), inv_bind=ib, track=rot))
    assert np.signbit(root[12]) and not np.signbit(under[12])
    assert np.array_equal(root[13:], under[13:])


def test_quirk_single_key_at_its_time_is_nan():
    one = NodeChannels(Track(np.array([0.25], f32), np.array([[1.0, 2.0, 3.0]], f32)))
    data = _one_joint(False, track=one)
    assert np.isnan(_pose_one(data, 0.25)[12:15]).all(), "0 / 0 factor (lib.rs:169-173)"
    assert np.array_equal(_pose_one(data, 0.5)[12:15], [1.0, 2.0, 3.0]), "after the key: factor clamps to 1"


def test_quirk_negative_zero_dot_flips():
    """Keys (1, 0, 0, 0) and (-0, -1, -0, -0) have a dot of exactly -0.0: its sign bit flips the second key, so halfway is a rotation
    about +(x + y), not -(x - y)."""
    rot = NodeChannels(None, Track(np.array([0.0, 1.0], f32), np.array([[1, 0, 0, 0], [-0.0, -1, -0.0, -0.0]], f32)))
    m = _pose_one(_one_joint(False, track=rot), 0.5)
    q = np.array([np.sqrt(0.5), np.sqrt(0.5), 0, 0])
    want = np.array(glam.from_scale_rotation_translation((1, 1, 1), q.astype(f32), (0, 0, 0))).reshape(16)
    assert np.allclose(m, want, atol=1e-6)


def _valid(n_joints=4):
    return cases.case("random", n_joints, seed=3)


def _invalid_libraries(library):
    """(what, arrays) of libraries that break one rule each"""
    s, j, o, c, ch, k = [x.copy() for x in library.arrays()]
    animated = int(np.flatnonzero(ch["animated"] & (ch["translation"]["times"] != 0xFFFFFFFF))[0])
    out = []

    def variant(what, **kw):
        arrays = dict(skins=s, joints=j, order=o, clips=c, channels=ch, keys=k)
        for name, fn in kw.items():
            arrays[name] = fn(arrays[name].copy())
        out.append((what, [arrays[x] for x in ("skins", "joints", "order", "clips", "channels", "keys")]))

    def chan(fn):
        def f(a):
            fn(a[animated])
            return a
        return f

    variant("empty key channel", channels=chan(lambda r: r["translation"].__setitem__("count", 0)))
    variant("fewer values than times", channels=chan(lambda r: r["translation"].__setitem__("value_count", r["translation"]["count"] - 1)))
    variant("key range outside the blob", channels=chan(lambda r: r["translation"].__setitem__("times", len(k))))
    variant("NaN duration", clips=lambda a: (a.__setitem__("duration", np.nan), a)[1])
    variant("negative duration", clips=lambda a: (a.__setitem__("duration", -1.0), a)[1])
    variant("clip skin out of range", clips=lambda a: (a.__setitem__("skin", 7), a)[1])
    variant("clip channels out of range", clips=lambda a: (a.__setitem__("first_channel", len(ch)), a)[1])
    variant("skin joints out of range", skins=lambda a: (a.__setitem__("joint_count", len(j) + 1), a)[1])
    variant("parent out of range", joints=lambda a: (a["parent"].__setitem__(1, 1000), a)[1])
    variant("order not a permutation", order=lambda a: (a.__setitem__(1, a[0]), a)[1])
    variant("order lists a child first", order=lambda a: a[::-1].copy())
    kk = k.copy()
    t0 = int(ch[animated]["translation"]["times"])
    for what, bad in (("non-increasing key times", lambda x: x.__setitem__(t0, x[t0 + 1]) if ch[animated]["translation"]["count"] > 1 else x.__setitem__(t0, -1.0)),
                      ("NaN key time", lambda x: x.__setitem__(t0, np.nan)), ("negative key time", lambda x: x.__setitem__(t0, -1.0))):
        x = kk.copy()
        bad(x)
        out.append((what, [s, j, o, c, ch, x]))
    return out


def _check_rejections(b):
    """Every invalid call is rejected; afterwards, with nothing uploaded again, the joint buffer still holds what r3_set_skeletons gave
    it and the first pose runs the jobs of the last accepted r3_set_pose_jobs against the last accepted library."""
    library, jobs, targets, buf = _valid()
    want = pose_f32(library, jobs, targets, buf)
    assert not same_bits(want, buf)
    b.set_animations(*library.arrays())
    b.set_skeletons(NO_SKELETONS, buf)
    b.set_pose_jobs(jobs, targets)
    for what, arrays in _invalid_libraries(library):
        with pytest.raises(R3Error) as e:
            b.set_animations(*arrays)
        assert e.value.code == E_INVALID, what
    n = len(buf)
    bad_jobs = []
    j = jobs.copy(); j["clip"][0] = 99; bad_jobs.append(("clip out of range", j, targets))
    j = jobs.copy(); j["first_target"][0] = len(targets); bad_jobs.append(("targets out of range", j, targets))
    t = targets.copy(); t["joint_count"][0] = 5; bad_jobs.append(("target above the skin's joint count", jobs, t))
    t = targets.copy(); t["joint_matrix_base_offset"][0] = n - 1; bad_jobs.append(("target outside the joint buffer", jobs, t))
    t = targets.copy(); t["joint_matrix_base_offset"][1] = t["joint_matrix_base_offset"][0]; bad_jobs.append(("overlapping targets", jobs, t))
    for what, jb, tg in bad_jobs:
        with pytest.raises(R3Error) as e:
            b.set_pose_jobs(jb, tg)
        assert e.value.code == E_INVALID, what
    with pytest.raises(R3Error) as e:
        b.readback_joint_matrices(n - 1, 2)
    assert e.value.code == E_INVALID
    # nothing changed, and nothing is uploaded again
    assert np.array_equal(b.readback_joint_matrices(0, n), buf), "rejected calls must not touch the joint buffer"
    b.pose_skeletons()
    assert same_bits(b.readback_joint_matrices(0, n), want), "the accepted library and jobs must survive the rejected calls"


def _check_state_errors(b):
    library, jobs, targets, buf = _valid()
    for call in (b.pose_skeletons, b.skin_posed, lambda: b.readback_joint_matrices(0, 1), lambda: b.set_pose_jobs(jobs, targets)):
        with pytest.raises(R3Error) as e:
            call()
        assert e.value.code == E_STATE
    b.set_animations(*library.arrays())
    with pytest.raises(R3Error) as e:
        b.set_pose_jobs(jobs, targets)
    assert e.value.code == E_STATE, "jobs need the joint buffer"
    b.set_skeletons(NO_SKELETONS, buf)
    with pytest.raises(R3Error) as e:
        b.pose_skeletons()
    assert e.value.code == E_STATE, "no jobs yet"
    b.set_pose_jobs(jobs, targets)
    b.set_animations(*library.arrays())
    with pytest.raises(R3Error) as e:
        b.pose_skeletons()
    assert e.value.code == E_STATE, "a new library drops the jobs"


def test_oracle_rejects_every_invalid_input_and_keeps_its_state():
    b = load_anim_oracle_backend()
    _check_rejections(b)
    b.close()
    b = load_anim_oracle_backend()
    _check_state_errors(b)
    b.close()


def test_animation_layouts_match_c_header():
    import os
    import subprocess
    import tempfile

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    probes = {"r3_anim_skin": ANIM_SKIN_DTYPE, "r3_anim_joint": ANIM_JOINT_DTYPE, "r3_anim_channel": ANIM_CHANNEL_DTYPE, "r3_anim_clip": ANIM_CLIP_DTYPE,
              "r3_pose_job": POSE_JOB_DTYPE, "r3_pose_target": POSE_TARGET_DTYPE, "r3_anim_track": ANIM_CHANNEL_DTYPE["translation"]}
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{root}/include/r3_layouts.h"', "int main(void){"]
    for name, dt in probes.items():
        lines.append(f'printf("{name} %zu\\n", sizeof({name}));')
        lines += [f'printf("{name}.{f} %zu\\n", offsetof({name}, {f}));' for f in dt.names]
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


# ------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def cuda_backend():
    from rend3_b200.backend import load_cuda_backend

    return lambda: load_cuda_backend(0)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,n", cases.SHAPES, ids=CASE_IDS)
def test_gpu_pose_equals_oracle_bit_for_bit(cuda_backend, shape, n):
    library, jobs, targets, buf = cases.case(shape, n, seed=n)
    orc = load_anim_oracle_backend()
    want = run(orc, library, jobs, targets, buf)
    orc.close()
    b = cuda_backend()
    got = run(b, library, jobs, targets, buf)
    b.close()
    assert same_bits(got, want), f"{shape}{n}: {np.count_nonzero(got.view(np.uint32) != want.view(np.uint32))} words differ"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(LAYOUT_CASES))
def test_gpu_pose_equals_oracle_on_shared_and_mixed_skins(cuda_backend, name):
    library, jobs, targets, buf = LAYOUT_CASES[name]()
    orc = load_anim_oracle_backend()
    want = run(orc, library, jobs, targets, buf)
    orc.close()
    b = cuda_backend()
    got = run(b, library, jobs, targets, buf)
    b.close()
    assert same_bits(got, want), f"{name}: {np.count_nonzero(got.view(np.uint32) != want.view(np.uint32))} words differ"


@pytest.mark.gpu
def test_gpu_crowd_equals_oracle(cuda_backend):
    data, jobs, targets, buf = cases.crowd(4096)
    orc = load_anim_oracle_backend()
    want = run(orc, data.library, jobs, targets, buf)
    orc.close()
    b = cuda_backend()
    got = run(b, data.library, jobs, targets, buf)
    b.close()
    assert same_bits(got, want)


@pytest.mark.gpu
def test_gpu_rejects_every_invalid_input_and_keeps_its_state(cuda_backend):
    b = cuda_backend()
    _check_rejections(b)
    b.close()
    b = cuda_backend()
    _check_state_errors(b)
    b.close()


def _skinned_world(library_case, seed=5):
    """skinning_case's mesh buffer and records, with their joint ranges covered by the case's targets"""
    import skinning_case

    library, jobs, targets, buf = library_case
    words, inputs, _, _ = skinning_case.build(seed=seed, vertex_counts=(257, 3000), joints_per_skeleton=(30, 30))
    # the targets of the job at a time off every key (the last of animation_case.times_for): finite matrices, so that the mesh buffers
    # compare word for word (a NaN's payload is not part of either rule)
    job = jobs[len(jobs) // 2 - 1]
    first = int(job["first_target"])
    inputs["joint_matrix_base_offset"] = [int(targets["joint_matrix_base_offset"][first]), int(targets["joint_matrix_base_offset"][first + 1])]
    return words, inputs


@pytest.mark.gpu
def test_gpu_skin_posed_equals_skin_of_the_posed_matrices(cuda_backend):
    """r3_skin_posed over the resident data == r3_skin(records, readback_joint_matrices()) == the oracle's r3o_skin_posed.  A range no
    job targets keeps the matrices r3_set_skeletons gave it."""
    c = cases.case("humanoid", 65, seed=4)
    library, jobs, targets, buf = c
    words, inputs = _skinned_world(c)
    outs = []
    for b in (cuda_backend(), load_anim_oracle_backend()):
        b.set_mesh_buffer(words)
        run(b, library, jobs, targets, buf, inputs)
        b.skin_posed()
        outs.append((b.readback_mesh_buffer(len(words)), b.readback_joint_matrices(0, len(buf))))
        b.close()
    (mesh_c, jm_c), (mesh_o, jm_o) = outs
    assert same_bits(jm_c, jm_o)
    skinned = np.concatenate([jm_c[int(o):int(o) + 30] for o in inputs["joint_matrix_base_offset"]])
    assert np.isfinite(skinned).all()
    assert np.array_equal(jm_c[-3:], buf[-3:]), "skeletons without a job keep their matrices"
    ref = cuda_backend()
    ref.set_mesh_buffer(words)
    ref.skin(inputs, jm_c)
    assert np.array_equal(ref.readback_mesh_buffer(len(words)), mesh_c)
    ref.close()
    assert np.array_equal(mesh_c, mesh_o)
    assert not np.array_equal(mesh_c, words)


@pytest.mark.gpu
def test_gpu_posed_frames_stay_one_graph(cuda_backend):
    """Six frames through add_to_graph(posed_skinning=True) with the frame graph on and the time changing per frame: no early flush,
    the same bits as the same frames run eagerly, the oracle's shading within 1e-4; a mesh-buffer growth between frames 3 and 4 keeps
    the posed path right.  r3_skin in the same place flushes once per frame."""
    from rend3_b200.backend import load_cuda_backend
    from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings

    ev, rec, data = cases._posed_cube_world()
    settings = BaseRenderGraphSettings(clear_color=(0.1, 0.05, 0.1, 1.0))
    graph_b, eager_b, orc = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True), load_anim_oracle_backend()
    runs = [(graph_b, True), (eager_b, False), (orc, False)]
    graphs = {id(b): BaseRenderGraph(b) for b, _ in runs}
    growth = np.random.default_rng(2).integers(0, 2 ** 32, 2 * len(ev.mesh_buffer), dtype=np.uint32)
    n_words = len(ev.mesh_buffer)
    for b, _ in runs:   # a first, eager frame allocates the render targets and culling buffers (a graphed first frame flushes there)
        graphs[id(b)].upload_world(ev)
        b.set_animations(*data.library.arrays())
        b.set_skeletons(rec, np.zeros((4, 16), f32))
        b.set_pose_jobs(*data.pose_jobs([(0, 0.0, {0: [(0, 4)]})]))
        graphs[id(b)].add_to_graph(ev, (256, 144), 1, settings, upload=False, posed_skinning=True, frame_graph=False)
    for frame, t in enumerate([0.0, 0.3, 0.7, 1.1, 1.6, 2.5]):
        jobs, targets = data.pose_jobs([(0, t, {0: [(0, 4)]})])
        if frame == 3:
            n_words = len(ev.mesh_buffer) + 8 + len(growth)
        out = []
        flushed = graph_b.frame_graph_stats()["flushed"]
        for b, fg in runs:
            if frame == 3 and b is orc:   # the oracle has no range writes: the full upload they equal
                b.set_mesh_buffer(np.concatenate([b.readback_mesh_buffer(len(ev.mesh_buffer)), np.zeros(8, np.uint32), growth]))
            elif frame == 3:
                b.update_mesh_buffer(4 * (len(ev.mesh_buffer) + 8), growth)
            b.set_pose_jobs(jobs, targets)
            graphs[id(b)].add_to_graph(ev, (256, 144), 1, settings, upload=False, posed_skinning=True, frame_graph=fg)
            out.append((b.readback_hdr_f32().copy(), b.readback_mesh_buffer(n_words), b.readback_joint_matrices(0, 4)))
        assert graph_b.frame_graph_stats()["flushed"] == flushed, f"frame {frame} flushed early"
        (hg, mg, jg), (he, me, je), (ho, mo, jo) = out
        assert np.array_equal(hg.view(np.uint32), he.view(np.uint32)) and np.array_equal(mg, me) and same_bits(jg, je), f"frame {frame}: graph != eager"
        assert same_bits(jg, jo) and np.array_equal(mg, mo), f"frame {frame}: joint matrices / skinned mesh differ from the oracle"
        err = np.abs(hg - ho) / np.maximum(1.0, np.abs(ho))
        assert err.max() <= 1e-4, f"frame {frame}: shading differs from the oracle by {err.max()}"
    stats = graph_b.frame_graph_stats()
    assert stats["graphed"] == 6 and stats["flushed"] == 0, stats
    # the host-matrix path in the same place drains the stream inside the frame
    graphs[id(graph_b)].add_to_graph(ev, (256, 144), 1, settings, upload=False, skinning=(rec, jg), frame_graph=True)
    assert graph_b.frame_graph_stats()["flushed"] == 1
    for b, _ in runs:
        b.close()
