"""PointLightManager on the device (rule R14, DESIGN.md §2): the handle table set and updated from host or device memory and evaluated by
a kernel into the buffer the shading reads.  The oracle (oracle/r3_oracle_points.c) and the kernels must produce world.py's point_buffer
bit for bit, any NaN equal to any NaN; graphed frames whose lights a CUDA producer moves equal eager frames and the host
r3_set_point_lights path bit for bit, and the oracle within the HDR tolerance, with no early flush."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

from harness import same_bytes
from oracle.points import load_points_oracle_backend
from point_light_case import apply_to_world, as_update, records, same_buffer, sequence
from rend3_b200 import glam
from rend3_b200.backend import ENTRY_POINTS, R3Error, load_cuda_backend
from rend3_b200.layouts import POINT_LIGHT_SOURCE_DTYPE
from rend3_b200.world import BLEND, LEFT, RIGHT, Camera, DirectionalLight, MeshBuilder, Object, PbrMaterial, PointLight, Renderer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R3_E_INVALID, R3_E_STATE = -1, -5
NEW_ENTRY_POINTS = {
    "set_point_light_sources": "int r3_set_point_light_sources(r3_ctx*, const r3_point_light_source* lights, const uint8_t* live_or_null, uint32_t n_handles);",
    "update_point_light_sources": "int r3_update_point_light_sources(r3_ctx*, const uint32_t* handles, const r3_point_light_source* lights, const uint8_t* live, uint32_t n);",
    "update_point_light_sources_device": "int r3_update_point_light_sources_device(r3_ctx*, const uint32_t* d_handles, const r3_point_light_source* d_lights,\n                                         const uint8_t* d_live_or_null, uint32_t n);",
    "evaluate_point_lights": "int r3_evaluate_point_lights(r3_ctx*);",
    "readback_point_lights": "int r3_readback_point_lights(r3_ctx*, void* bytes, uint64_t capacity_bytes);",
}


# ------------------------------------------------------------------ CPU
def test_point_light_source_layout_matches_c_header():
    fields = POINT_LIGHT_SOURCE_DTYPE.names
    prog = '#include <stdio.h>\n#include <stddef.h>\n#include "r3_layouts.h"\nint main(void){printf("%zu\\n", sizeof(r3_point_light_source));'
    prog += "".join(f'printf("%zu\\n", offsetof(r3_point_light_source, {f}));' for f in fields) + "return 0;}\n"
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "l.c"), os.path.join(d, "l")
        open(src, "w").write(prog)
        subprocess.run(["/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe], check=True)
        out = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    assert out[0] == POINT_LIGHT_SOURCE_DTYPE.itemsize == 32
    assert out[1:] == [POINT_LIGHT_SOURCE_DTYPE.fields[f][1] for f in fields] == [0, 12, 24, 28]


def test_new_symbols_are_exported_and_declared():
    from rend3_b200.backend import CUDA_LIB_PATH

    lib = ctypes.CDLL(CUDA_LIB_PATH)
    header = open(os.path.join(ROOT, "include", "rend3_b200.h")).read()
    for name, decl in NEW_ENTRY_POINTS.items():
        assert hasattr(lib, "r3_" + name), f"r3_{name} not exported"
        assert decl in header, f"r3_{name}: declaration differs"
    assert "set_point_lights" in ENTRY_POINTS


def world_buffer(renderer):
    return renderer.evaluate().point_buffer


def drive_host_form(b, seed):
    """Apply a seeded sequence through r3_update_point_light_sources; after each step the evaluated buffer equals world.py's."""
    r = Renderer(LEFT)
    for k, ops in enumerate(sequence(seed)):
        apply_to_world(r, ops)
        b.update_point_light_sources(*as_update(ops))
        b.evaluate_point_lights()
        got, want = b.readback_point_lights(), world_buffer(r)
        assert same_buffer(got, want), f"seed {seed} step {k}: {np.frombuffer(got[:4], np.uint32)} vs {np.frombuffer(want[:4], np.uint32)} lights"
    return r


def check_sequences(b):
    b.evaluate_point_lights()   # an empty table: count 0
    assert same_buffer(b.readback_point_lights(), np.zeros(4, np.uint32).tobytes())
    for seed in range(6):
        b.set_point_light_sources(np.zeros(0, dtype=POINT_LIGHT_SOURCE_DTYPE))
        r = drive_host_form(b, seed)
        # the whole table in one call gives the same buffer
        src, live = r.evaluate().point_sources
        b.set_point_light_sources(src, live)
        b.evaluate_point_lights()
        assert same_buffer(b.readback_point_lights(), world_buffer(r))
    b.set_point_light_sources(records([PointLight((1, 2, 3), (1, 1, 1), 4.0, 2.0)] * 3))   # live == NULL: all live
    b.evaluate_point_lights()
    assert np.frombuffer(b.readback_point_lights()[:4], np.uint32)[0] == 3


def test_oracle_evaluate_equals_world_point_buffer():
    b = load_points_oracle_backend()
    check_sequences(b)
    b.close()


def check_rejections(b):
    """A repeated handle, a null pointer and the handle 0xFFFFFFFF are R3_E_INVALID and leave the table as it was."""
    r = drive_host_form(b, 11)
    before = b.readback_point_lights()
    light = PointLight((0.5, 0.5, 0.5), (1, 0, 0), 3.0, 1.0)
    bad = [([4, 9, 4], [light] * 3, [1, 1, 1]), ([300, 301, 300], [light] * 3, [1, 0, 1]), ([0, 0xFFFFFFFF], [light] * 2, [1, 1])]
    for handles, lights, live in bad:
        with pytest.raises(R3Error) as e:
            b.update_point_light_sources(np.array(handles, np.uint32), records(lights), np.array(live, np.uint8))
        assert e.value.code == R3_E_INVALID
    h, s, l = as_update([(2, light)])
    fn = getattr(b.lib, b.prefix + "update_point_light_sources")
    for args in ((None, s.ctypes.data, l.ctypes.data), (h.ctypes.data, None, l.ctypes.data), (h.ctypes.data, s.ctypes.data, None)):
        rc = fn(b.ctx, *[ctypes.c_void_p(a) for a in args], ctypes.c_uint32(1))
        assert rc == R3_E_INVALID
    rc = getattr(b.lib, b.prefix + "set_point_light_sources")(b.ctx, None, None, ctypes.c_uint32(2))
    assert rc == R3_E_INVALID
    rc = getattr(b.lib, b.prefix + "readback_point_lights")(b.ctx, ctypes.c_void_p(None), ctypes.c_uint64(8))
    assert rc == R3_E_INVALID
    assert b.readback_point_lights() == before, "a rejected call changed the evaluated buffer"
    b.evaluate_point_lights()
    assert same_buffer(b.readback_point_lights(), world_buffer(r)), "a rejected call changed the handle table"


def test_oracle_rejects_invalid_calls_and_keeps_its_state():
    b = load_points_oracle_backend()
    check_rejections(b)
    b.close()


def test_set_point_lights_and_the_sources_replace_each_other_in_the_oracle():
    b = load_points_oracle_backend()
    check_switching(b)
    b.close()


def check_switching(b):
    r = drive_host_form(b, 3)
    other = Renderer(LEFT)
    apply_to_world(other, sequence(4)[0])
    host = world_buffer(other)
    b.set_point_lights(host)                     # replaces the evaluated table and empties it
    assert same_buffer(b.readback_point_lights(), host)
    b.evaluate_point_lights()                    # an empty table now
    assert same_buffer(b.readback_point_lights(), np.zeros(4, np.uint32).tobytes())
    b.set_point_lights(host)
    src, live = r.evaluate().point_sources
    b.set_point_light_sources(src, live)         # and back
    b.evaluate_point_lights()
    assert same_buffer(b.readback_point_lights(), world_buffer(r))


# ------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_gpu_evaluated_buffer_equals_world_host_form():
    b = load_cuda_backend(0, parity_target=False)
    check_sequences(b)
    b.close()


def device_update(b, ops, extra_handles=()):
    """The step through r3_update_point_light_sources_device, with CUDA tensors produced on the context's stream."""
    import torch

    h, s, l = as_update(ops)
    h = np.concatenate([h, np.asarray(extra_handles, np.uint32)])
    s = np.concatenate([s, records([PointLight((9, 9, 9), (1, 1, 1), 1.0, 1.0)] * len(extra_handles))])
    l = np.concatenate([l, np.ones(len(extra_handles), np.uint8)])
    with torch.cuda.stream(torch.cuda.ExternalStream(b.stream())):
        th = torch.from_numpy(h.view(np.int32).copy()).cuda(non_blocking=True)
        ts = torch.from_numpy(s.view(np.float32).reshape(-1, 8).copy()).cuda(non_blocking=True)
        tl = torch.from_numpy(l.copy()).cuda(non_blocking=True)
        b.update_point_light_sources_device(th, ts, tl)
    return th, ts, tl


@pytest.mark.gpu
def test_gpu_evaluated_buffer_equals_world_device_form():
    """The same sequences through the device form over a table sized up front; out-of-range handles are dropped, the others written."""
    b = load_cuda_backend(0, parity_target=False)
    for seed in range(6):
        steps = sequence(seed)
        size = max(h for ops in steps for h, _ in ops) + 1
        r = Renderer(LEFT)
        r.remove_point_light(size - 1)            # world.py's table at that size, every handle dead
        src, live = r.evaluate().point_sources
        b.set_point_light_sources(src, live)
        keep = []
        for k, ops in enumerate(steps):
            apply_to_world(r, ops)
            keep.append(device_update(b, ops, extra_handles=(size, size + 7, 0xFFFFFFFF)))
            b.evaluate_point_lights()
            assert same_buffer(b.readback_point_lights(), world_buffer(r)), f"seed {seed} step {k}"
        keep.append(device_update(b, [], extra_handles=(size + 1,)))   # only out-of-range handles: nothing changes
        b.evaluate_point_lights()
        assert same_buffer(b.readback_point_lights(), world_buffer(r))
    b.close()


@pytest.mark.gpu
def test_gpu_rejects_invalid_calls_and_keeps_its_state():
    b = load_cuda_backend(0, parity_target=False)
    check_rejections(b)
    b.close()


@pytest.mark.gpu
def test_gpu_set_point_lights_and_the_sources_replace_each_other():
    b = load_cuda_backend(0, parity_target=False)
    check_switching(b)
    b.close()


def walk_world(left):
    """A ground plane, a field of cubes, a translucent (blend) pane, two shadowed directional lights and a table of 160 point-light
    handles over the cubes."""
    from rend3_b200.runner import cube_mesh

    r = Renderer(LEFT if left else RIGHT, aspect_ratio=192 / 108)
    lit = r.add_material(PbrMaterial(albedo_value=(0.6, 0.5, 0.4, 1.0), roughness_factor=0.6))
    glass = r.add_material(PbrMaterial(albedo_value=(0.2, 0.4, 0.9, 0.45), roughness_factor=0.3, transparency=BLEND))
    plane = MeshBuilder.new([(-1, 0, -1), (-1, 0, 1), (1, 0, 1), (1, 0, -1)], LEFT).with_indices([0, 1, 2, 0, 2, 3] if left else [0, 2, 1, 0, 3, 2]).build()
    r.add_object(Object(r.add_mesh(plane), lit, glam.from_scale((12.0, 1.0, 12.0))))
    cube = r.add_mesh(cube_mesh())
    rng = np.random.default_rng(7)
    for k in range(40):
        p = (float(rng.uniform(-8, 8)), 0.4, float(rng.uniform(-8, 8)))
        r.add_object(Object(cube, lit, glam.from_scale_rotation_translation((0.4, 0.4, 0.4), glam.QUAT_IDENTITY, p)))
    assert r.add_object(Object(cube, glass, glam.from_scale_rotation_translation((2.0, 1.2, 0.05), glam.QUAT_IDENTITY, (0.0, 1.0, -2.0)))) == PANE
    r.add_directional_light(DirectionalLight(color=(1.0, 1.0, 1.0), intensity=0.3, direction=(-1.0, -2.0, 0.5), distance=30.0, resolution=256))
    r.add_directional_light(DirectionalLight(color=(0.3, 0.3, 0.5), intensity=0.2, direction=(0.5, -1.5, -1.0), distance=30.0, resolution=128))
    return r


N_HANDLES = 160
PANE = 41   # the blend pane's object slot
LIVE_COUNTS = [32, 0, 128, 129, 100, 129]   # the last frame is SampleCount Four
BASE = np.random.default_rng(9).uniform((-9.0, 0.3, -9.0), (9.0, 2.5, 9.0), (N_HANDLES, 3)).astype(np.float32)


def produce(stream, frame):
    """The CUDA producer: every handle's light moved for this frame, and which handles are live, computed by torch on `stream`."""
    import torch

    with torch.cuda.stream(stream):
        base = torch.from_numpy(BASE).cuda(non_blocking=True)
        k = torch.arange(N_HANDLES, device="cuda", dtype=torch.float32)
        phase = k * 0.37 + frame * 0.9
        src = torch.zeros((N_HANDLES, 8), device="cuda", dtype=torch.float32)
        src[:, 0] = base[:, 0] + 0.8 * torch.cos(phase)
        src[:, 1] = base[:, 1]
        src[:, 2] = base[:, 2] + 0.8 * torch.sin(phase)
        src[:, 3] = 0.5 + 0.5 * torch.cos(k * 1.3)
        src[:, 4] = 0.5 + 0.5 * torch.cos(k * 0.7 + 1.0)
        src[:, 5] = 0.5 + 0.5 * torch.sin(k * 0.4)
        src[:, 6] = 1.5 + (k % 7) * 0.5                  # radius
        src[:, 7] = 0.25 + 0.25 * (k % 3)                 # intensity: 100+ overlapping lights keep the sum inside the 1e-4 tolerance
        order = torch.from_numpy(np.random.default_rng(frame).permutation(N_HANDLES)).cuda(non_blocking=True)
        live = torch.zeros(N_HANDLES, device="cuda", dtype=torch.uint8)
        live[order[:LIVE_COUNTS[frame]]] = 1
        handles = torch.arange(N_HANDLES, device="cuda", dtype=torch.int32)
    return handles, src, live


def walk_camera(frame, left):
    eye = (0.5 + 0.04 * frame, 6.0 - 0.02 * frame, -11.0 + 0.05 * frame)
    return Camera(("perspective", 60.0, 0.1), (glam.look_at_lh if left else glam.look_at_rh)(eye, (0.0, 0.5, 0.0), (0.0, 1.0, 0.0)))


def frame_outputs(b):
    return b.readback_hdr_f16().copy(), b.readback_hdr_f32().copy(), b.readback_depth().copy()


ENQUEUE_ONLY = {"frame_begin", "frame_end", "clear_shadow_atlas", "set_frame_uniforms", "evaluate_shadow_cameras", "shadow_uniform_upload",
                "object_uniform_upload", "batch_objects", "cull", "shadow_pass", "forward_begin", "forward_pass", "hiz_build", "forward_resolve",
                "forward_blend", "tonemap", "update_point_light_sources_device", "evaluate_point_lights"}


class CallLog:
    def __init__(self, b):
        self.b, self.calls = b, []

    def __getattr__(self, name):
        attr = getattr(self.b, name)
        if callable(attr):
            def wrapped(*a, **k):
                self.calls.append(name)
                return attr(*a, **k)
            return wrapped
        return attr


@pytest.mark.gpu
@pytest.mark.parametrize("left", [True, False])
def test_gpu_graphed_walkthrough_with_moving_point_lights(left):
    """Six frames, camera moving, every light moved by a torch producer on the context's stream, the live count crossing 0, 32, 128 and
    129 (one light outside the shared-memory window and its tile mask), a blend pane in the first frame and a SampleCount Four frame last.
    Graphed device-form frames equal eager ones and the host r3_set_point_lights path fed world.py's bytes bit for bit (rgba16f, f32
    parity target, depth) and match the oracle within 1e-4.  Walked a second time, no frame flushes early and every call of a frame only
    enqueues work, frames 2-4 (128, 129 and 100 lights) held to it: frame 0 has transparent objects, whose blend routine waits for the stream
    by design, frame 1 uploads the world without them and frame 5 sets a new render target."""
    import torch

    from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings

    r = walk_world(left)
    settings = BaseRenderGraphSettings(clear_color=(0.1, 0.05, 0.1, 1.0), ambient_color=(0.02, 0.02, 0.02, 0.0))
    graph_b, eager_b, host_b = (load_cuda_backend(0, parity_target=True) for _ in range(3))
    orc = load_points_oracle_backend()
    log = CallLog(graph_b)
    g_graph, g_eager, g_host, g_orc = BaseRenderGraph(log), BaseRenderGraph(eager_b), BaseRenderGraph(host_b), BaseRenderGraph(orc)
    res = (192, 108)
    samples_prev, transparent_prev = None, None
    # the walk runs twice: the first pass lets every buffer that depends on the camera's view grow to its size, the second must not flush
    for walk, frame in [(w, f) for w in range(2) for f in range(len(LIVE_COUNTS))]:
        count = LIVE_COUNTS[frame]
        samples = 4 if frame == len(LIVE_COUNTS) - 1 else 1
        r.set_camera_data(walk_camera(frame, left))
        transparent = frame == 0
        # the pane is live in frame 0 only: the blend routine's pool check waits for the stream, so a frame with transparent objects
        # flushes by design; the world is uploaded again (outside the frame bracket) when the pane comes or goes
        up = (walk == 0 and frame == 0) or transparent != transparent_prev
        transparent_prev = transparent
        if up:
            for h in range(N_HANDLES):
                r.remove_point_light(h)           # the table's size, every handle dead until the first update
        pg = produce(torch.cuda.ExternalStream(graph_b.stream()), frame)
        pe = produce(torch.cuda.ExternalStream(eager_b.stream()), frame)
        # world.py follows the producer: the same records, read back once the producer has run
        hs, src, live = (t.cpu().numpy() for t in pg)
        recs = np.ascontiguousarray(src).view(POINT_LIGHT_SOURCE_DTYPE).reshape(-1)
        for h in range(N_HANDLES):
            if live[h]:
                s = recs[h]
                r.update_point_light(h, PointLight(tuple(s["position"]), tuple(s["color"]), float(s["radius"]), float(s["intensity"])))
            else:
                r.remove_point_light(h)
        ev = r.evaluate()
        if not transparent:
            ev.object_live[PANE] = 0
            ev.object_buffer[PANE]["enabled"] = 0
        assert np.frombuffer(ev.point_buffer[:4], np.uint32)[0] == count
        flushed = graph_b.frame_graph_stats()["flushed"]
        log.calls = []
        g_graph.add_to_graph(ev, res, samples, settings, upload=up, frame_graph=True, device_shadow_cameras=True, device_point_lights=True,
                             point_light_updates=pg)
        if walk == 1 and samples == samples_prev and not transparent and not up:
            assert graph_b.frame_graph_stats()["flushed"] == flushed, f"frame {frame} flushed early"
            assert set(log.calls) <= ENQUEUE_ONLY, sorted(set(log.calls) - ENQUEUE_ONLY)
        samples_prev = samples
        g_eager.add_to_graph(ev, res, samples, settings, upload=up, frame_graph=False, device_shadow_cameras=True, device_point_lights=True,
                             point_light_updates=pe)
        g_orc.add_to_graph(ev, res, samples, settings, upload=up, device_shadow_cameras=True, device_point_lights=True,
                           point_light_updates=(hs.view(np.uint32), recs, live))
        if not up:
            host_b.set_point_lights(ev.point_buffer)
        g_host.add_to_graph(ev, res, samples, settings, upload=up, device_shadow_cameras=True)
        assert same_buffer(graph_b.readback_point_lights(), ev.point_buffer), f"frame {frame}: evaluated buffer"
        assert same_buffer(eager_b.readback_point_lights(), ev.point_buffer), f"frame {frame}: evaluated buffer (eager)"
        og, oe, oh = frame_outputs(graph_b), frame_outputs(eager_b), frame_outputs(host_b)
        for what, x, y in (("eager", og, oe), ("host r3_set_point_lights", og, oh)):
            for name, a, c in zip(("rgba16f", "f32", "depth"), x, y):
                assert same_bytes(a, c), f"frame {frame}: graph vs {what}: {name} differs"
        ho = orc.readback_hdr_f32()
        ok = np.isfinite(ho)
        err = np.abs(og[1][ok] - ho[ok]) / np.maximum(1.0, np.abs(ho[ok]))
        assert err.max() <= 1e-4, f"frame {frame}: {err.max()} from the oracle"
        assert np.array_equal(og[2], orc.readback_depth()), f"frame {frame}: depth differs from the oracle"
        assert (graph_b.forward_stats()[3] > 0) == transparent, f"frame {frame}: the blend routine shades the pane in frame 0 only"
        del pg, pe
    stats = graph_b.frame_graph_stats()
    # the only flushes are the blend routine's, in the pane's frame of each walk
    assert stats["frames"] == 2 * len(LIVE_COUNTS) and stats["flushed"] == 2 and stats["graphed"] == 2 * len(LIVE_COUNTS) - 2, stats
    for b in (graph_b, eager_b, host_b, orc):
        b.close()


@pytest.mark.gpu
def test_gpu_resolve_after_an_update_without_evaluation_is_a_state_error():
    """r3_forward_resolve and r3_forward_blend refuse a stale light buffer; an evaluation makes the frame legal again."""
    from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings

    r = walk_world(True)
    r.set_camera_data(walk_camera(0, True))
    for h in range(8):
        r.update_point_light(h, PointLight((float(h), 1.0, 0.0), (1.0, 0.5, 0.2), 4.0, 2.0))
    ev = r.evaluate()
    b = load_cuda_backend(0, parity_target=True)
    g = BaseRenderGraph(b)
    g.add_to_graph(ev, (192, 108), 1, BaseRenderGraphSettings(), device_point_lights=True)
    g.add_to_graph(ev, (192, 108), 1, BaseRenderGraphSettings(), upload=False, device_point_lights=True)   # last frame's lists predict
    want = frame_outputs(b)
    before = b.readback_point_lights()
    b.update_point_light_sources(*as_update([(3, PointLight((0.0, 2.0, 0.0), (0.0, 1.0, 0.0), 5.0, 3.0))]))
    for call in (b.forward_resolve, b.forward_blend):
        with pytest.raises(R3Error) as e:
            call()
        assert e.value.code == R3_E_STATE
    assert b.readback_point_lights() == before
    assert all(same_bytes(x, y) for x, y in zip(frame_outputs(b), want)), "a rejected resolve changed the frame"
    b.set_point_light_sources(*ev.point_sources)
    with pytest.raises(R3Error) as e:
        b.forward_resolve()
    assert e.value.code == R3_E_STATE
    b.evaluate_point_lights()
    g.add_to_graph(ev, (192, 108), 1, BaseRenderGraphSettings(), upload=False, device_point_lights=True)
    assert all(same_bytes(x, y) for x, y in zip(frame_outputs(b), want))
    b.close()
