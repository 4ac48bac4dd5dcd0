"""Helpers the test modules share: error and export checks, a fake library for the wrappers' argument checks, staging data on a
context's stream, whole-frame and cull + batch comparisons between two backends, and bit comparisons of arrays."""
import ctypes
import os
import re

import numpy as np
import pytest

from rend3_b200.backend import CAMERA_VIEWPORT, CB_BAKE, CB_CULL, CUDA_LIB_PATH, ENTRY_POINTS, Backend, R3Error

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E_INVALID = -1
TOL = 1e-4


def expect_error(code, fn, *args, **kw):
    with pytest.raises(R3Error) as e:
        fn(*args, **kw)
    assert e.value.code == code, str(e.value)


def check_declared_and_exported(decls, no_context_args):
    """Each declaration is in include/rend3_b200.h (comments dropped, whitespace folded), the library exports its symbol, ENTRY_POINTS
    lists it, and a call without a context returns R3_E_INVALID before it touches anything.  `no_context_args` is that call's argument
    tuple, or a function giving it for a declaration."""
    lib = ctypes.CDLL(CUDA_LIB_PATH)
    header = re.sub(r"\s+", " ", re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "rend3_b200.h")).read(), flags=re.S))
    for decl in decls:
        assert decl in header, decl
        name = decl.split("(")[0].split()[-1]
        assert hasattr(lib, name) and name[3:] in ENTRY_POINTS
        args = no_context_args(decl) if callable(no_context_args) else no_context_args
        assert getattr(lib, name)(*args) == E_INVALID, name


class _NoCalls:
    """Stands in for the library: any call through it fails the test."""

    def __getattr__(self, name):
        def call(*args):
            pytest.fail(f"{name} was called")
        return call


def unbound_backend():
    """A Backend whose library is _NoCalls: a wrapper that rejects its arguments never reaches the C call."""
    b = Backend.__new__(Backend)
    b.lib, b.prefix, b.ctx = _NoCalls(), "r3_", None
    return b


def on_stream(b, fn):
    """Run torch work on the context's stream, so that it is ordered before the library's next kernel."""
    import torch

    with torch.cuda.stream(torch.cuda.ExternalStream(b.stream())):
        return fn()


def to_device(b, array, dtype=None):
    import torch

    host = torch.from_numpy(np.ascontiguousarray(array).copy())
    return on_stream(b, lambda: host.to("cuda", dtype=dtype, non_blocking=False))


def settings():
    from rend3_b200.routines import BaseRenderGraphSettings

    return BaseRenderGraphSettings(clear_color=(0.1, 0.05, 0.1, 1.0), ambient_color=(0.02, 0.02, 0.02, 1.0))


def assert_same_frame(a, b, ev, what):
    """Every artefact of the last frame, bit for bit."""
    n = len(ev.object_buffer)
    for cam in [CAMERA_VIEWPORT] + list(range(len(ev.shadows))):
        w = f"{what} camera {cam}"
        assert np.array_equal(a.readback_visible(cam), b.readback_visible(cam)), f"{w}: visible lists differ"
        assert a.readback_object_matrices(cam, 0, n).tobytes() == b.readback_object_matrices(cam, 0, n).tobytes(), f"{w}: MV/MVP differ"
        assert a.batching_info(cam) == b.batching_info(cam), f"{w}: batching path"
        ba, ra = a.readback_batches(cam)
        bb, rb = b.readback_batches(cam)
        assert ba.tobytes() == bb.tobytes() and ra.tobytes() == rb.tobytes(), f"{w}: batches / regions differ"
        for part in (0, 1):
            da, db = a.readback_draw_calls(cam, part), b.readback_draw_calls(cam, part)
            assert da.tobytes() == db.tobytes(), f"{w}: draw calls (partition {part}) differ"
            ia, ib = a.readback_indices(cam, part), b.readback_indices(cam, part)
            assert len(ia) == len(ib), f"{w}: index list lengths (partition {part})"
            for r in da:
                b0, cnt = int(r["base_index"]), int(r["vertex_count"])
                assert np.array_equal(ia[b0:b0 + cnt], ib[b0:b0 + cnt]), f"{w}: index list (partition {part})"
            assert a.readback_culling_results(cam, part).tobytes() == b.readback_culling_results(cam, part).tobytes(), f"{w}: culling results ({part})"
    assert a.readback_depth().tobytes() == b.readback_depth().tobytes(), f"{what}: depth differs"
    assert a.readback_hdr_f16().tobytes() == b.readback_hdr_f16().tobytes(), f"{what}: rgba16f differs"
    assert a.readback_hdr_f32().tobytes() == b.readback_hdr_f32().tobytes(), f"{what}: f32 parity target differs"
    sw, sh = ev.shadow_target_size
    assert a.readback_shadow_atlas(sw, sh).tobytes() == b.readback_shadow_atlas(sw, sh).tobytes(), f"{what}: shadow atlas differs"
    assert a.forward_stats() == b.forward_stats(), f"{what}: forward_stats"
    assert a.forward_light_evaluations() == b.forward_light_evaluations(), f"{what}: light evaluations"


def assert_same_ldr(a, b, what):
    assert a.readback_ldr().tobytes() == b.readback_ldr().tobytes(), f"{what}: LDR differs"


def _cull_cloud(b, n):
    from rend3_b200.routines import per_camera_header
    from rend3_b200.scenes import cloud_camera

    header = per_camera_header(cloud_camera(pull_back=12.0), CAMERA_VIEWPORT, (640, 360), 1, n)
    b.object_uniform_upload(CAMERA_VIEWPORT, header, CB_BAKE | CB_CULL)


def cull_and_batch(b, n, batch=True):
    """Cull + bake of n objects seen by the cloud camera, then batch_objects from (1, 2, 3): the visible list, MV / MVP, and with `batch`
    the batches and regions, as bytes."""
    _cull_cloud(b, n)
    out = [b.readback_visible(CAMERA_VIEWPORT).tobytes(), b.readback_object_matrices(CAMERA_VIEWPORT, 0, n).tobytes()]
    if batch:
        b.batch_objects(CAMERA_VIEWPORT, np.array([1.0, 2.0, 3.0], dtype=np.float32))
        bt, rg = b.readback_batches(CAMERA_VIEWPORT)
        out += [bt.tobytes(), rg.tobytes()]
    return out


def cull_and_batch_defined(b, n, vp=(1.0, 2.0, 3.0)):
    """cull_and_batch from `vp`, keeping only the batch bytes batching defines, so that the device and the oracle compare."""
    _cull_cloud(b, n)
    b.batch_objects(CAMERA_VIEWPORT, np.array(vp, dtype=np.float32))
    bt, rg = b.readback_batches(CAMERA_VIEWPORT)
    info = bt["object_culling_information"].copy()
    for k in range(len(bt)):   # the entries past total_objects are not part of a batch (the device and the oracle leave different bytes)
        info[k, int(bt[k]["total_objects"]):] = 0
    # field by field: the batch records end in padding, which numpy's structured copies do not carry
    batches = b"".join(bt[f].tobytes() for f in ("total_objects", "total_invocations", "batch_base_invocation")) + info.tobytes()
    regions = b"".join(rg[f].tobytes() for f in rg.dtype.names)
    return (b.readback_visible(CAMERA_VIEWPORT).tobytes(), b.readback_object_matrices(CAMERA_VIEWPORT, 0, n).tobytes(), batches, regions)


def assert_same_bake(cuda, orc, rec, what, culled=True):
    """The cull + bake of `rec` on the device against the oracle: the visible list, and every MV / MVP word of the enabled slots."""
    n = len(rec)
    if culled:
        assert np.array_equal(cuda.readback_visible(CAMERA_VIEWPORT), orc.readback_visible(CAMERA_VIEWPORT)), f"{what}: visible list"
    en = rec["enabled"] != 0
    a = cuda.readback_object_matrices(CAMERA_VIEWPORT, 0, n).view(np.uint32).reshape(n, 32)[en]
    o = orc.readback_object_matrices(CAMERA_VIEWPORT, 0, n).view(np.uint32).reshape(n, 32)[en]
    # NaN payloads may differ between x86 and the GPU: NaN == NaN, every other word bit for bit
    an, on = np.isnan(a.view(np.float32)), np.isnan(o.view(np.float32))
    assert np.array_equal(an, on), f"{what}: NaN positions differ"
    bad = (a != o) & ~an
    assert not bad.any(), f"{what}: MV/MVP words differ in slots {np.nonzero(en)[0][bad.any(axis=1)][:16]}"


def hdr_close(a, b, what="", f16_samples=False):
    """TOL = 1e-4 (north_star), relative above 1.0.  With SampleCount::Four the samples live in an rgba16f target BEFORE the
    box filter (base.rs:245-255), so a 1e-6 difference in a shaded colour can land on the other side of a half-precision
    rounding boundary: there the bound is TOL plus one f16 ulp of the value."""
    ref = np.abs(b.astype(np.float64))
    err = np.abs(a.astype(np.float64) - b.astype(np.float64)) / np.maximum(1.0, ref)
    bound = TOL + (np.maximum(ref * 2.0 ** -10, 2.0 ** -24) / np.maximum(1.0, ref) if f16_samples else 0.0)
    bad = np.nan_to_num(err, nan=np.inf) > bound
    both_nan = np.isnan(a) & np.isnan(b)
    bad &= ~both_nan
    assert not bad.any(), f"{what}: {bad.sum()} channel values differ by more than {TOL} (max {np.nanmax(err):.3e})"


def compare_frame_state(cuda, orc, ev, cameras, check_pixels=True, what="", f16_samples=False):
    for cam in cameras:
        bc, rc = cuda.readback_batches(cam)
        bo, ro = orc.readback_batches(cam)
        assert len(bc) == len(bo) and rc.tobytes() == ro.tobytes(), f"{what} camera {cam}: batch / region tables differ"
        for k in range(len(bo)):   # slots past total_objects are unspecified (the reference reuses its scratch array, batching.rs:186)
            n_obj = int(bo[k]["total_objects"])
            for f in ("total_objects", "total_invocations", "batch_base_invocation"):
                assert bc[k][f] == bo[k][f], f"{what} camera {cam}: batch {k} {f}"
            assert bc[k]["object_culling_information"][:n_obj].tobytes() == bo[k]["object_culling_information"][:n_obj].tobytes(), \
                f"{what} camera {cam}: batch {k} object table differs"
        for part in (0, 1):
            # the CUDA path sizes its buffers with device-side upper bounds: compare what the oracle defines, the rest stays cleared
            dc, do = cuda.readback_draw_calls(cam, part), orc.readback_draw_calls(cam, part)
            assert dc[:len(do)].tobytes() == do.tobytes(), f"{what} camera {cam}: draw calls (partition {part}) differ"
            assert not dc[len(do):].view(np.uint8).any(), f"{what} camera {cam}: stray draw calls"
            ic, io = cuda.readback_indices(cam, part), orc.readback_indices(cam, part)
            for r in range(len(do)):   # only the listed part of each region is defined
                b0, cnt = int(do[r]["base_index"]), int(do[r]["vertex_count"])
                if part == 1 and cam != CAMERA_VIEWPORT:
                    continue
                assert np.array_equal(ic[b0:b0 + cnt], io[b0:b0 + cnt]), f"{what} camera {cam}: index list of region {r} differs"
        ro_bits = orc.readback_culling_results(cam, 0)
        assert np.array_equal(cuda.readback_culling_results(cam, 0)[:len(ro_bits)], ro_bits), f"{what}: visibility bits differ"
    if check_pixels:
        assert np.array_equal(cuda.readback_depth().view(np.uint32), orc.readback_depth().view(np.uint32)), f"{what}: depth differs"
        hdr_close(cuda.readback_hdr_f32(), orc.readback_hdr_f32(), what + " hdr f32", f16_samples)
        h16c, h16o = cuda.readback_hdr_f16().astype(np.float32), orc.readback_hdr_f16().astype(np.float32)
        ulp = np.maximum(np.abs(h16o) * 2.0 ** -10, 2.0 ** -24)
        assert np.all(np.abs(h16c - h16o) <= ulp + TOL * np.maximum(1.0, np.abs(h16o))), f"{what}: rgba16f target differs by more than 1 ulp"
        lc, lo = cuda.readback_ldr().astype(int), orc.readback_ldr().astype(int)
        assert np.abs(lc - lo).max() <= 1, f"{what}: 8-bit output differs by more than 1 LSB"
        assert np.count_nonzero(lc != lo) <= 1e-3 * lc.size
        if ev.shadows:
            w, h = ev.shadow_target_size
            assert np.array_equal(cuda.readback_shadow_atlas(w, h).view(np.uint32), orc.readback_shadow_atlas(w, h).view(np.uint32)), f"{what}: shadow atlas differs"


def same_words_nan_equal(a, b):
    """Bit-identical float32 words, any NaN equal to any NaN."""
    a, b = np.ascontiguousarray(a).view(np.uint32).ravel(), np.ascontiguousarray(b).view(np.uint32).ravel()
    fa, fb = a.view(np.float32), b.view(np.float32)
    return bool(np.all((a == b) | (np.isnan(fa) & np.isnan(fb))))


def same_bytes(a, b):
    """The same shape and the same bytes."""
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))
