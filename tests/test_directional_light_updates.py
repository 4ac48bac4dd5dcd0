"""DirectionalLightManager::update on the device (r3_update_directional_light_sources[_device]): DirectionalLightChanges applied to the
lights of the current set, from host records passed as kernel parameters or from device memory, both enqueue only.  Frames whose lights
change through either form equal, bit for bit (any NaN equal to any NaN), frames that re-set the changed list with
r3_set_directional_light_sources; they stay one graph launch; they match the oracle fed the updated lights; and the calls keep their
documented checks and state rules."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

from directional_change_case import NAN_FRAMES, RES, STEPS, C, camera, same_bits, world
from harness import ROOT, check_declared_and_exported, unbound_backend
from rend3_b200 import layouts
from rend3_b200.backend import R3Error, load_cuda_backend
from rend3_b200.layouts import DIRECTIONAL_LIGHT_CHANGE_DTYPE, LIGHT_SOURCE_DTYPE
from rend3_b200.world import LEFT, DirectionalLight, Renderer

R3_E_INVALID, R3_E_STATE = -1, -5
DECLS = ("int r3_update_directional_light_sources(r3_ctx*, const r3_directional_light_change* changes, uint32_t n);",
         "int r3_update_directional_light_sources_device(r3_ctx*, const r3_directional_light_change* d_changes, uint32_t n);")


# ------------------------------------------------------------------ CPU
def test_new_symbols_are_exported_and_declared():
    check_declared_and_exported(DECLS, (None, None, 1))


def test_change_record_layout_matches_c_header():
    fields = DIRECTIONAL_LIGHT_CHANGE_DTYPE.names
    prog = '#include <stdio.h>\n#include <stddef.h>\n#include "r3_layouts.h"\nint main(void){printf("%zu\\n", sizeof(r3_directional_light_change));'
    prog += "".join(f'printf("%zu\\n", offsetof(r3_directional_light_change, {f}));' for f in fields)
    prog += 'printf("%u %u %u %u\\n", R3_DIR_CHANGE_COLOR, R3_DIR_CHANGE_INTENSITY, R3_DIR_CHANGE_DIRECTION, R3_DIR_CHANGE_DISTANCE);return 0;}\n'
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "l.c"), os.path.join(d, "l")
        open(src, "w").write(prog)
        subprocess.run(["/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe], check=True)
        out = [int(v) for v in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    assert out[0] == DIRECTIONAL_LIGHT_CHANGE_DTYPE.itemsize == 48
    assert out[1:1 + len(fields)] == [DIRECTIONAL_LIGHT_CHANGE_DTYPE.fields[f][1] for f in fields] == [0, 4, 8, 20, 24, 36]
    assert out[1 + len(fields):] == [layouts.DIR_CHANGE_COLOR, layouts.DIR_CHANGE_INTENSITY, layouts.DIR_CHANGE_DIRECTION,
                                     layouts.DIR_CHANGE_DISTANCE] == [1, 2, 4, 8]


def test_wrappers_reject_wrong_dtype_shape_and_stride():
    b = unbound_backend()
    good = np.zeros(4, dtype=DIRECTIONAL_LIGHT_CHANGE_DTYPE)
    for bad in (np.zeros(4, dtype=LIGHT_SOURCE_DTYPE), good.view(np.uint8).reshape(4, 48), good.reshape(2, 2), good[::2], [good[0]]):
        with pytest.raises(AssertionError):
            b.update_directional_light_sources(bad)


def test_device_wrapper_rejects_host_and_misshapen_tensors():
    torch = pytest.importorskip("torch")
    b = unbound_backend()
    for bad in (torch.zeros((2, 48), dtype=torch.uint8),                        # a CPU tensor
                np.zeros(2, dtype=DIRECTIONAL_LIGHT_CHANGE_DTYPE)):             # host memory
        with pytest.raises(AssertionError):
            b.update_directional_light_sources_device(bad)
    with pytest.raises(AssertionError):
        b.update_directional_light_sources_device(0x1000)                     # a raw pointer without its count


def test_world_changes_merge_field_by_field_later_wins():
    r = Renderer(LEFT)
    h = r.add_directional_light(DirectionalLight(color=(1.0, 1.0, 1.0), intensity=1.0, direction=(0.0, -1.0, 1.0), distance=10.0, resolution=64))
    r.update_directional_light(h, C(color=(0.5, 0.5, 0.5)))
    r.update_directional_light(h, C(intensity=2.0))
    r.update_directional_light(h, C(color=(0.1, 0.2, 0.3), distance=5.0))
    r.update_directional_light(h, C())
    assert r.dir_lights[h] == DirectionalLight(color=(0.1, 0.2, 0.3), intensity=2.0, direction=(0.0, -1.0, 1.0), distance=5.0, resolution=64)


def test_world_after_changes_equals_world_built_with_the_final_lights():
    for left in (True, False):
        r = world(left)
        for frame, step in enumerate(STEPS):
            r.set_camera_data(camera(frame, left))
            for h, c in step:
                r.update_directional_light(h, c)
        final = Renderer(r.handedness, r.aspect_ratio)
        for light in r.dir_lights:
            final.add_directional_light(light)
        final.set_camera_data(camera(len(STEPS) - 1, left))
        got, want = r.evaluate(), final.evaluate()
        assert same_bits(got.directional_sources, want.directional_sources)
        assert same_bits(np.frombuffer(got.directional_buffer, np.uint32), np.frombuffer(want.directional_buffer, np.uint32))
        assert [s.offset for s in got.shadows] == [s.offset for s in want.shadows]


def test_shadow_index_follows_the_atlas_order_and_skips_removed_handles():
    r = Renderer(LEFT)
    for res in (128, 256, 128, 64):
        r.add_directional_light(DirectionalLight((1.0, 1.0, 1.0), 1.0, (0.0, -1.0, 0.5), 20.0, res))
    assert [r.directional_shadow_index(h) for h in range(4)] == [1, 0, 2, 3]
    r.remove_directional_light(1)
    assert [r.directional_shadow_index(h) for h in (0, 2, 3)] == [0, 1, 2]
    with pytest.raises(KeyError):
        r.directional_shadow_index(1)
    # the index is the position in evaluate()'s sources
    src = r.evaluate().directional_sources
    assert [int(s["resolution"]) for s in src] == [128, 128, 64]


def test_change_records_name_shadow_indices_and_refuse_resolution():
    r = world(True)
    recs = r.directional_change_records([(0, C(color=(0.5, 0.5, 0.5), distance=3.0)), (1, C()), (2, C(intensity=0.25, direction=(1.0, -1.0, 0.0)))])
    assert list(recs["index"]) == [1, 0, 2] and list(recs["mask"]) == [1 | 8, 0, 2 | 4]
    assert recs[0]["distance"] == np.float32(3.0) and tuple(recs[2]["direction"]) == (1.0, -1.0, 0.0)
    with pytest.raises(ValueError):
        r.directional_change_records([(0, C(resolution=512))])


# ------------------------------------------------------------------ GPU
def device_records(b, recs):
    """The records as a CUDA tensor produced on the context's stream."""
    import torch

    with torch.cuda.stream(torch.cuda.ExternalStream(b.stream())):
        return torch.from_numpy(np.ascontiguousarray(recs).view(np.uint8).reshape(-1, 48).copy()).cuda(non_blocking=True)


class SetInFrame:
    """Today's path: the changed list re-set with r3_set_directional_light_sources inside the frame, before the evaluation."""

    def __init__(self, b):
        self.b, self.ev = b, None

    def __getattr__(self, name):
        return getattr(self.b, name)

    def evaluate_shadow_cameras(self, loc):
        ev = self.ev
        self.b.set_directional_light_sources(ev.directional_sources, ev.shadow_target_size[0], ev.shadow_target_size[1],
                                             ev.camera.handedness == LEFT)
        self.b.evaluate_shadow_cameras(loc)


def products(b, ev):
    n = len(ev.directional_sources)
    heads, lights = b.readback_shadow_cameras(n)
    out = dict(heads=heads.copy(), lights=lights.copy(), atlas=b.readback_shadow_atlas(*ev.shadow_target_size).copy(),
               depth=b.readback_depth().copy(), hdr_f32=b.readback_hdr_f32().copy(), ldr=b.readback_ldr().copy())
    for i in range(n):
        out[f"visible{i}"] = b.readback_visible(i).copy()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("left", [True, False])
def test_gpu_updates_equal_re_setting_the_lights(left, graph):
    """Three contexts walk the sequence twice: A re-sets the changed list each frame, B applies the changes with the host form, C with
    the device form.  Light records, camera headers, atlas, each shadow camera's visible list, depth, f32 parity target and LDR are
    identical.  As frame graphs, B's and C's frames of the second walk are submitted with no early flush; A flushes at its set."""
    from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings

    r = world(left)
    settings = BaseRenderGraphSettings(clear_color=(0.1, 0.05, 0.1, 1.0), ambient_color=(0.02, 0.02, 0.02, 0.0))
    a, hb, db = load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True), load_cuda_backend(0, parity_target=True)
    set_a = SetInFrame(a)
    ga, gh, gd = BaseRenderGraph(set_a), BaseRenderGraph(hb), BaseRenderGraph(db)
    keep = []
    for walk in range(2):
        for frame, step in enumerate(STEPS):
            r.set_camera_data(camera(frame, left))
            recs = r.directional_change_records(step)
            for h, c in step:
                r.update_directional_light(h, c)
            ev = r.evaluate()
            up = walk == 0 and frame == 0
            flushed = [x.frame_graph_stats()["flushed"] for x in (a, hb, db)]
            set_a.ev = ev
            ga.add_to_graph(ev, RES, 1, settings, upload=up, frame_graph=graph, device_shadow_cameras=True)
            gh.add_to_graph(ev, RES, 1, settings, upload=up, frame_graph=graph, device_shadow_cameras=True, directional_changes=recs)
            keep.append(device_records(db, recs))
            gd.add_to_graph(ev, RES, 1, settings, upload=up, frame_graph=graph, device_shadow_cameras=True, directional_changes=keep[-1])
            if graph and walk == 1:
                after = [x.frame_graph_stats()["flushed"] for x in (a, hb, db)]
                assert after[1] == flushed[1] and after[2] == flushed[2], f"frame {frame}: an update flushed the frame early"
                assert after[0] > flushed[0], f"frame {frame}: re-setting the lights inside the frame flushes it"
            pa, ph, pd = products(a, ev), products(hb, ev), products(db, ev)
            for what, p in (("host form", ph), ("device form", pd)):
                for k in pa:
                    assert same_bits(pa[k], p[k]), f"walk {walk} frame {frame}: {what}: {k} differs from re-setting the lights"
            if frame == 6:
                assert np.isnan(pa["heads"][0]["view_proj"]).any() and np.isnan(pa["heads"][2]["view_proj"]).any(), "the +-Y cameras are NaN"
            if frame in NAN_FRAMES:
                assert np.isnan(pa["lights"][0]["color"]).all(), "NaN intensity reaches the light record"
    if graph:
        for x in (hb, db):
            s = x.frame_graph_stats()
            assert s["frames"] == 2 * len(STEPS) and s["flushed"] <= 1, s   # only the first frame may flush (its buffers are allocated)
    for x in (a, hb, db):
        x.close()


@pytest.mark.gpu
def test_gpu_device_form_matches_the_oracle():
    """The device form's frames 4 and 9 match the oracle rendering the updated lights: visible lists, atlas and depth bit for bit,
    the f32 shading within 1e-4."""
    from oracle.lights import load_lights_oracle_backend
    from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings

    r = world(True)
    settings = BaseRenderGraphSettings(clear_color=(0.1, 0.05, 0.1, 1.0), ambient_color=(0.02, 0.02, 0.02, 0.0))
    db, orc = load_cuda_backend(0, parity_target=True), load_lights_oracle_backend()
    gd, go = BaseRenderGraph(db), BaseRenderGraph(orc)
    keep = []
    compared = 0
    for frame, step in enumerate(STEPS):
        r.set_camera_data(camera(frame, True))
        recs = r.directional_change_records(step)
        for h, c in step:
            r.update_directional_light(h, c)
        ev = r.evaluate()
        keep.append(device_records(db, recs))
        gd.add_to_graph(ev, RES, 1, settings, upload=frame == 0, frame_graph=True, device_shadow_cameras=True, directional_changes=keep[-1])
        go.add_to_graph(ev, RES, 1, settings, device_shadow_cameras=True)
        if frame not in (4, 9):
            continue
        n = len(ev.directional_sources)
        for i in range(n):
            assert np.array_equal(db.readback_visible(i), orc.readback_visible(i)), f"frame {frame}: shadow camera {i}'s visible list"
        assert same_bits(db.readback_shadow_atlas(*ev.shadow_target_size), orc.readback_shadow_atlas(*ev.shadow_target_size)), f"frame {frame}: atlas"
        assert np.array_equal(db.readback_depth(), orc.readback_depth()), f"frame {frame}: depth"
        hc, ho = db.readback_hdr_f32(), orc.readback_hdr_f32()
        ok = np.isfinite(ho)
        err = np.abs(hc[ok] - ho[ok]) / np.maximum(1.0, np.abs(ho[ok]))
        assert ok.all() and err.max() <= 1e-4, f"frame {frame}: {err.max()} from the oracle"
        compared += 1
    assert compared == 2
    db.close()
    orc.close()


def cat(*parts):
    """Change records end to end (np.concatenate would not keep the record dtype's padding)."""
    out = np.zeros(sum(len(p) for p in parts), dtype=DIRECTIONAL_LIGHT_CHANGE_DTYPE)
    k = 0
    for p in parts:
        out[k:k + len(p)] = p
        k += len(p)
    return out


def set_world(b, r):
    ev = r.evaluate()
    b.set_directional_light_sources(ev.directional_sources, ev.shadow_target_size[0], ev.shadow_target_size[1], True)
    return ev


def raw(b, name, ptr, n):
    return getattr(b.lib, "r3_" + name)(b.ctx, ctypes.c_void_p(ptr), ctypes.c_uint32(n))


@pytest.mark.gpu
def test_gpu_calls_and_state():
    import torch

    from rend3_b200.routines import BaseRenderGraph, BaseRenderGraphSettings

    r = world(True)
    r.set_camera_data(camera(0, True))
    ev = r.evaluate()
    one = r.directional_change_records([(0, C(intensity=0.2))])
    b = load_cuda_backend(0, parity_target=False)
    # no sources yet, and the host-evaluated path: R3_E_STATE from both forms
    for set_first in (False, True):
        if set_first:
            b.set_directional_lights(ev.directional_buffer, *ev.shadow_target_size)
        with pytest.raises(R3Error) as e:
            b.update_directional_light_sources(one)
        assert e.value.code == R3_E_STATE
        with pytest.raises(R3Error) as e:
            b.update_directional_light_sources_device(device_records(b, one))
        assert e.value.code == R3_E_STATE
    # a frame through the sources, then rejected host calls leave every readback as it was
    g = BaseRenderGraph(b)
    g.add_to_graph(ev, RES, 1, BaseRenderGraphSettings(), device_shadow_cameras=True)
    n = len(ev.directional_sources)
    before = b.readback_shadow_cameras(n)
    launches = b.launch_count()
    bad_index, bad_mask = one.copy(), one.copy()
    bad_index[0]["index"] = n
    bad_mask[0]["mask"] = 16
    for bad in (cat(one, bad_index), bad_mask):
        with pytest.raises(R3Error) as e:
            b.update_directional_light_sources(bad)
        assert e.value.code == R3_E_INVALID
    assert raw(b, "update_directional_light_sources", None, 2) == R3_E_INVALID
    assert raw(b, "update_directional_light_sources_device", None, 2) == R3_E_INVALID
    # n == 0 launches nothing, in both forms
    b.update_directional_light_sources(np.zeros(0, dtype=DIRECTIONAL_LIGHT_CHANGE_DTYPE))
    assert raw(b, "update_directional_light_sources_device", None, 0) == 0
    assert b.launch_count() == launches, "a rejected call or n == 0 launched a kernel"
    after = b.readback_shadow_cameras(n)
    assert same_bits(before[0], after[0]) and same_bits(before[1], after[1]), "a rejected call changed the cameras or the lights"
    # the device form drops exactly its bad entries: index n, index 0xFFFFFFFF, an unknown bit (with known ones); the rest apply
    good = [(0, C(color=(0.2, 0.4, 0.6))), (1, C(direction=(0.3, -1.0, 0.2))), (2, C(distance=12.0, intensity=0.9))]
    recs = r.directional_change_records(good)
    junk = r.directional_change_records([(0, C(intensity=5.0)), (1, C(intensity=6.0)), (2, C(intensity=7.0, distance=1.0))])
    junk[0]["index"], junk[1]["index"] = n, 0xFFFFFFFF
    junk[2]["mask"] |= 32
    mixed = cat(recs[:1], junk[:1], recs[1:2], junk[1:2], junk[2:], recs[2:])
    keep = device_records(b, mixed)
    b.update_directional_light_sources_device(keep)
    b.evaluate_shadow_cameras(ev.camera.location())
    want_b = load_cuda_backend(0, parity_target=False)
    want_b.set_directional_light_sources(ev.directional_sources, *ev.shadow_target_size, True)
    want_b.update_directional_light_sources(recs)
    want_b.evaluate_shadow_cameras(ev.camera.location())
    got, want = b.readback_shadow_cameras(n), want_b.readback_shadow_cameras(n)
    assert same_bits(got[0], want[0]) and same_bits(got[1], want[1]), "the device form did not drop exactly its bad entries"
    for h, c in good:
        r.update_directional_light(h, c)
    fresh = load_cuda_backend(0, parity_target=False)
    set_world(fresh, r)
    fresh.evaluate_shadow_cameras(ev.camera.location())
    ref = fresh.readback_shadow_cameras(n)
    assert same_bits(got[0], ref[0]) and same_bits(got[1], ref[1]), "the updates differ from setting the updated lights"
    # after an update: uploads, readbacks and shading are R3_E_STATE until the evaluation, then they succeed
    b.update_directional_light_sources(one)
    for call in (lambda: b.shadow_uniform_upload(0, len(ev.object_buffer)), lambda: b.readback_shadow_cameras(n), b.forward_resolve,
                 b.forward_blend):
        with pytest.raises(R3Error) as e:
            call()
        assert e.value.code == R3_E_STATE
    b.evaluate_shadow_cameras(ev.camera.location())
    b.shadow_uniform_upload(0, len(ev.object_buffer))
    b.readback_shadow_cameras(n)
    b.forward_resolve()
    b.forward_blend()
    # a later set replaces everything, the pending evaluation included
    b.update_directional_light_sources_device(device_records(b, one))
    ev2 = set_world(b, r)
    b.forward_resolve()
    b.evaluate_shadow_cameras(ev2.camera.location())
    got = b.readback_shadow_cameras(n)
    assert same_bits(got[0], ref[0]) and same_bits(got[1], ref[1]), "a set after an update did not replace the lights"
    torch.cuda.synchronize()
    for x in (b, want_b, fresh):
        x.close()
